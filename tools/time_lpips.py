"""Time per-frame LPIPS (mcvd_b200.lpips.LPIPS) on the GPU against a batched torchvision AlexNet-LPIPS.

    python tools/time_lpips.py [--reps 5]

Three evaluation batches shaped like the outputs of the benchmark workloads, with synthetic weights
(``oracle.lpips_oracle.synthetic_weights``) and random frames:
  * cfg2: 64 clips x 20 frames, 64x64, 1 channel;
  * cfg4: 64 clips x 28 frames, 64x64, 3 channels;
  * cfg5: 32 clips x 28 frames, 128x128, 3 channels (the resize is an identity).
``native`` is the whole ``LPIPS`` call (quantise, resize, AlexNet, heads) with the default chunk of 256 pairs;
``native_tf32`` is the same call with ``LPIPS(..., tf32=True)`` (the convolutions on the TF32 tensor cores).
``torchvision`` is ``alexnet().features[0:12]`` with the same weights plus the LPIPS head in torch, batched over all
pairs of the batch (chunks of 256, like the native path), on the network input the native prep computed; its own
input preparation is not timed, so it is a lower bound on that path.  It runs with TF32 off and on.
All are timed with CUDA events after a warm-up, alternated ``--reps`` times; the median is reported.  Each case
also reports the largest relative difference of the native fp32 and TF32 distances from torchvision's fp32 ones, of
the TF32 distances from the native fp32 ones, and of torchvision's TF32 distances from its fp32 ones.  Prints the
GPU's name and power limit, then one JSON line per case.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as Fn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import lib, lpips as LP  # noqa: E402
from oracle import lpips_oracle as LO  # noqa: E402

CASES = {"cfg2": (64, 20, 64, 1), "cfg4": (64, 28, 64, 3), "cfg5": (32, 28, 128, 3)}


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def timed_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def torchvision_lpips(features, lins, x0, x1):
    """LPIPS of NCHW network inputs with torchvision's AlexNet features and the net-lin head."""
    d = 0.0
    h0, h1, k = x0, x1, 0
    for i, layer in enumerate(features):
        h0, h1 = layer(h0), layer(h1)
        if isinstance(layer, torch.nn.ReLU):
            n0 = h0 / (h0.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            n1 = h1 / (h1.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            d = d + Fn.conv2d((n0 - n1) ** 2, lins[k]).mean((2, 3))
            k += 1
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_lpips.py measures on a CUDA device"
    import torchvision
    dev = torch.device("cuda", torch.cuda.current_device())
    print(f"# {torch.cuda.get_device_name(dev)}, power limit {power_limit_w()} W")
    sd = LO.synthetic_weights()
    net = LP.LPIPS(sd, device=dev)
    net_tf32 = LP.LPIPS(sd, device=dev, tf32=True)
    tv, lin = LO.torchvision_format(sd)
    alex = torchvision.models.alexnet(weights=None)
    alex.features.load_state_dict({k[len("features."):]: v for k, v in tv.items()})
    features = alex.features[:12].to(dev).eval()
    lins = [lin[f"lin{k}.model.1.weight"].to(dev) for k in range(5)]
    g = torch.Generator(device=dev).manual_seed(0)
    for name, (B, F, S, C) in CASES.items():
        real = torch.rand(B, C * F, S, S, device=dev, generator=g)
        pred = (real + 0.1 * torch.randn(real.shape, device=dev, generator=g)).clamp(0, 1)
        N = B * F
        # the network inputs of all pairs, made by the native prep, for the torchvision path
        inputs = []
        p, r = pred.reshape(N, C, S, S), real.reshape(N, C, S, S)
        for lo in range(0, N, 256):
            n = min(256, N - lo)
            ws = torch.empty(2 * n * (LP._WS_A + LP._WS_B), device=dev)
            out = torch.empty(n, dtype=torch.float64, device=dev)
            ops = net.program(p[lo:lo + n], r[lo:lo + n], C, out, ws)[:1]
            lib.run_program(lib.make_ops(ops), 1, torch.cuda.current_stream(dev).cuda_stream)
            x = ws[:2 * n * LP._WS_A].reshape(2 * n, 128, 128, 4)[..., :3].permute(0, 3, 1, 2).contiguous()
            inputs.append((x[:n], x[n:]))

        def tv_run():
            with torch.no_grad():
                return torch.cat([torchvision_lpips(features, lins, a, b) for a, b in inputs])

        res = {"case": name, "clips": B, "frames": F, "side": S, "channels": C, "pairs": N}
        runs = {"native": lambda: net(pred, real, C), "native_tf32": lambda: net_tf32(pred, real, C)}
        for tf32 in (False, True):
            runs[f"torchvision_tf32_{'on' if tf32 else 'off'}"] = (lambda t=tf32: (
                setattr(torch.backends.cudnn, "allow_tf32", t), setattr(torch.backends.cuda.matmul, "allow_tf32", t),
                tv_run()))
        times = {k: [] for k in runs}
        for fn in runs.values():
            fn()                                                     # warm-up
        for _ in range(args.reps):
            for k, fn in runs.items():
                times[k].append(timed_ms(fn))
        for k, ts in times.items():
            ms = statistics.median(ts)
            res[f"{k}_ms"] = round(ms, 3)
            res[f"{k}_pairs_per_s"] = round(N / ms * 1e3, 1)
        d_native = net(pred, real, C).reshape(-1).double()
        d_tf32 = net_tf32(pred, real, C).reshape(-1).double()
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
        d_tv_tf32 = tv_run().reshape(-1).double()
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        d_tv = tv_run().reshape(-1).double()

        def max_rel(a, b):
            return float(((a - b).abs() / b.abs()).max())
        res["max_rel_diff_vs_torchvision_fp32"] = max_rel(d_native, d_tv)
        res["tf32_max_rel_diff_vs_torchvision_fp32"] = max_rel(d_tf32, d_tv)
        res["tf32_max_rel_diff_vs_native_fp32"] = max_rel(d_tf32, d_native)
        res["torchvision_tf32_max_rel_diff_vs_torchvision_fp32"] = max_rel(d_tv_tf32, d_tv)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
