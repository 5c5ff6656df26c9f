"""Time FVD's I3D features (mcvd_b200.fvd.I3D) on the GPU against the same network in cuDNN.

    python tools/time_fvd.py [--reps 5] [--cases cfg2,cfg4,cfg5] [--profile DIR]

The video sets of the benchmark workloads' FVD (real plus fake videos, one prediction per test clip), with synthetic
weights (``oracle.i3d_oracle.synthetic_weights``) and synthetic videos:
  * cfg2: 64 + 64 videos of 25 frames (5 conditioning + 20 predicted), 64x64, 1 channel;
  * cfg4: 64 + 64 videos of 30 frames (2 + 28), 64x64, 3 channels;
  * cfg5: 32 + 32 videos of 30 frames (2 + 28), 128x128, 3 channels.
``native`` is the whole ``I3D`` call (prep, 57 convolutions, 13 pools, head) with the default chunk of 16 videos, fp32
FFMA convolutions; ``native_tf32`` the same with ``tf32=True`` (TF32 wgmma convolutions).
``cudnn`` is ``F.interpolate`` + ``F.conv3d`` / ``F.max_pool3d`` / ``F.avg_pool3d`` with the same folded weights, in
chunks of 16 videos, with TF32 off and on.  Each is timed with CUDA events after a warm-up, alternated ``--reps``
times; the median is reported.  FLOPs are counted from the shapes (2 per multiply-add of the convolutions and the
logits).  Prints the GPU's name and power limit, then one JSON line per case.  ``--profile DIR``: afterwards, one
``native_tf32`` call per case under ``torch.profiler`` (a run of its own), with the summed CUDA time per kernel name
printed and the trace written to DIR.
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
from mcvd_b200 import fvd as FV  # noqa: E402
from oracle import i3d_oracle as IO  # noqa: E402
from tools.time_fid import profile_kernels  # noqa: E402

CASES = {"cfg2": (64, 25, 64, 1), "cfg4": (64, 30, 64, 3), "cfg5": (32, 30, 128, 3)}


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


def flops_per_video(T: int) -> float:
    steps, _ = FV.plan(T)
    total = 0.0
    for st in steps:
        if st["kind"] == "conv":
            to, so = FV.same_out(st["t"], st["kt"], st["st"]), FV.same_out(st["s"], st["ks"], st["ss"])
            cin = 3 if st["key"] == "Conv3d_1a_7x7" else st["c"]
            total += 2.0 * to * so * so * st["cout"] * cin * st["kt"] * st["ks"] ** 2
        elif st["kind"] == "head":
            total += 2.0 * (st["t"] - 1) * FV.HEAD_CHANNELS * FV.NUM_CLASSES
    return total


class CudnnI3D:
    """The same network from torch ops, batch norm folded exactly as the native path folds it."""

    def __init__(self, sd, dev):
        packed = FV.pack_weights(sd)
        self.w = {}
        for key, cin, cout, k in FV.units():
            w, b = packed[key]
            cin4 = -(-cin // 4) * 4
            wt = w.reshape(k, k, k, cin4, cout)[..., :cin, :].permute(4, 3, 0, 1, 2).contiguous()
            self.w[key] = (wt.to(dev), b.to(dev))
        lw, lb = packed["logits"]
        self.logits = (lw.t().reshape(400, 1024, 1, 1, 1).contiguous().to(dev), lb.to(dev))

    def unit(self, x, key, k, s=1):
        w, b = self.w[key]
        return torch.relu(Fn.conv3d(IO.same_pad(x, (k,) * 3, (s,) * 3), w, b, stride=s))

    def __call__(self, videos, channels):
        B, CT, S, _ = videos.shape
        x = IO.to_i3d(videos, channels)
        Ht, Wt = FV.resize_target(S)
        x = Fn.interpolate(x.reshape(B, 3 * (CT // channels), S, S), size=(Ht, Wt), mode="bilinear",
                           align_corners=False)
        h0 = (Ht - 224) // 2
        x = ((x[:, :, h0:h0 + 224] - 0.5) * 2).reshape(B, 3, CT // channels, 224, 224)
        x = self.unit(x, "Conv3d_1a_7x7", 7, 2)
        x = IO.max_pool(x, (1, 3, 3), (1, 2, 2))
        x = self.unit(x, "Conv3d_2b_1x1", 1)
        x = self.unit(x, "Conv3d_2c_3x3", 3)
        x = IO.max_pool(x, (1, 3, 3), (1, 2, 2))
        for key, _, _ in IO.MIXED:
            b0 = self.unit(x, f"{key}.b0", 1)
            b1 = self.unit(self.unit(x, f"{key}.b1a", 1), f"{key}.b1b", 3)
            b2 = self.unit(self.unit(x, f"{key}.b2a", 1), f"{key}.b2b", 3)
            b3 = self.unit(IO.max_pool(x, (3, 3, 3), (1, 1, 1)), f"{key}.b3b", 1)
            x = torch.cat([b0, b1, b2, b3], 1)
            if key == "Mixed_3c":
                x = IO.max_pool(x, (3, 3, 3), (2, 2, 2))
            elif key == "Mixed_4f":
                x = IO.max_pool(x, (2, 2, 2), (2, 2, 2))
        x = Fn.conv3d(Fn.avg_pool3d(x, (2, 7, 7), 1), *self.logits)
        return x.squeeze(3).squeeze(3).mean(2).double()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--profile", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_fvd.py measures on a CUDA device"
    dev = torch.device("cuda", torch.cuda.current_device())
    print(f"# {torch.cuda.get_device_name(dev)}, power limit {power_limit_w()} W", flush=True)
    sd = IO.synthetic_weights()
    net = FV.I3D(sd, device=dev)
    net_tf32 = FV.I3D(sd, device=dev, tf32=True)
    ref = CudnnI3D(sd, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for name in args.cases.split(","):
        B, T, S, C = CASES[name]
        real = torch.rand(B, C * T, S, S, device=dev, generator=g)
        fake = (real + 0.1 * torch.randn(real.shape, device=dev, generator=g)).clamp(0, 1)
        videos = torch.cat([real, fake])
        N = videos.shape[0]

        def cudnn_run():
            with torch.no_grad():
                return torch.cat([ref(videos[lo:lo + 16], C) for lo in range(0, N, 16)])

        runs = {"native": lambda: net(videos, C), "native_tf32": lambda: net_tf32(videos, C)}
        for tf32 in (False, True):
            runs[f"cudnn_tf32_{'on' if tf32 else 'off'}"] = (lambda t=tf32: (
                setattr(torch.backends.cudnn, "allow_tf32", t), setattr(torch.backends.cuda.matmul, "allow_tf32", t),
                cudnn_run()))
        times = {k: [] for k in runs}
        for fn in runs.values():
            fn()                                                     # warm-up
        for _ in range(args.reps):
            for k, fn in runs.items():
                times[k].append(timed_ms(fn))
        flops = N * flops_per_video(T)
        res = {"case": name, "videos": N, "frames": T, "side": S, "channels": C, "tflop": round(flops / 1e12, 2)}
        for k, ts in times.items():
            ms = statistics.median(ts)
            res[f"{k}_ms"] = round(ms, 2)
            res[f"{k}_tflops"] = round(flops / ms / 1e9, 2)
        f_native, f_tf32 = net(videos, C), net_tf32(videos, C)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
        f_ref_tf32 = cudnn_run()
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        f_ref = cudnn_run()
        res["max_abs_diff_vs_cudnn_fp32_over_scale"] = float((f_native - f_ref).abs().max() / f_ref.abs().max())
        res["native_tf32_vs_native_over_scale"] = float((f_tf32 - f_native).abs().max() / f_native.abs().max())
        res["cudnn_tf32_vs_cudnn_fp32_over_scale"] = float((f_ref_tf32 - f_ref).abs().max() / f_ref.abs().max())
        res["fvd_native"] = FV.frechet_distance(f_native[B:], f_native[:B])
        res["fvd_native_tf32"] = FV.frechet_distance(f_tf32[B:], f_tf32[:B])
        res["fvd_cudnn_fp32"] = FV.frechet_distance(f_ref[B:], f_ref[:B])
        res["fvd_cudnn_tf32"] = FV.frechet_distance(f_ref_tf32[B:], f_ref_tf32[:B])
        print(json.dumps(res), flush=True)
        if args.profile:
            profile_kernels(lambda: net_tf32(videos, C), args.profile, name)


if __name__ == "__main__":
    main()
