"""Time FID's Inception features and k-NN precision / recall (mcvd_b200.fid) on the GPU against torch baselines.

    python tools/time_fid.py [--reps 5] [--frames 2000] [--cases cfg2,cfg4,cfg5] [--pr 10000,50000] [--profile DIR]

Features: frame sets shaped like the benchmark workloads' ``fast_fid`` output, with synthetic weights
(``oracle.inception_oracle.synthetic_weights``) and random frames:
  * cfg2: 64x64, 1 channel;  cfg4: 64x64, 3 channels;  cfg5: 128x128, 3 channels.
``native`` is the whole ``InceptionV3`` call (prep, 94 convolutions, 4 pools, head) with the default chunk, fp32 FFMA
convolutions; ``native_tf32`` the same with ``tf32=True`` (TF32 wgmma convolutions).
``cudnn`` is ``F.interpolate`` + ``F.conv2d`` / pools with the same folded weights, in chunks of the same size, with
TF32 off and on.  FLOPs are counted from the shapes (2 per multiply-add of the convolutions).

Precision / recall at N rows per side of 2048-d features (ReLU of a normal, like pool features): ``native`` is
``fid.precision_recall`` (two radius and two cover launches); ``torch_full`` restates the reference's
``calculate_precision_recall_full`` on the GPU -- ``torch.cdist`` in 10000-column blocks copied to the host, the
(k+1)-th value per row, the comparisons on the host -- and runs only where its three N x N fp32 host matrices fit in
half of the host's free memory.

Each measurement is timed with CUDA events around work that ends in a synchronise, after a warm-up, alternated
``--reps`` times; the median is reported.  Prints the GPU's name and power limit, then one JSON line per case.
``--profile DIR``: afterwards, one ``native_tf32`` call per case under ``torch.profiler`` (a run of its own), with the
summed CUDA time per kernel name printed and the trace written to DIR.
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
from mcvd_b200 import fid as FD  # noqa: E402
from oracle import inception_oracle as NO  # noqa: E402

CASES = {"cfg2": (64, 1), "cfg4": (64, 3), "cfg5": (128, 3)}


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


def flops_per_frame() -> float:
    total = 0.0
    for st in FD.plan()[0]:
        if st["kind"] == "conv":
            (kh, kw), (ph, pw) = st["k"], st["pad"]
            ho, wo = FD.conv_out(st["s"], kh, st["stride"], ph), FD.conv_out(st["s"], kw, st["stride"], pw)
            total += 2.0 * ho * wo * st["cout"] * st["cin"] * kh * kw
    return total


class TorchInception:
    """The same network from torch ops, batch norm folded exactly as the native path folds it."""

    def __init__(self, sd, dev):
        packed = FD.pack_weights(sd)
        self.w = {}
        for key, cin, cout, (kh, kw) in FD.units():
            w, b = packed[key]
            cin4 = -(-cin // 4) * 4
            wt = w.reshape(kh, kw, cin4, cout)[:, :, :cin].permute(3, 2, 0, 1).contiguous()
            self.w[key] = (wt.to(dev), b.to(dev))

    def basic(self, x, key, stride=1, padding=0):
        return torch.relu(Fn.conv2d(x, *self.w[key], stride=stride, padding=padding))

    def __call__(self, frames):
        x = frames.repeat(1, 3 // frames.shape[1], 1, 1)
        x = 2 * Fn.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False) - 1
        return NO.network(x, None, unit=self.basic).double()


def reference_pr(feat_r, feat_g, k=3, bs=10000):
    """calculate_precision_recall_full restated: GPU cdist blocks, host matrices, kthvalue, comparisons."""
    def full(a, b):
        rows = [torch.cat([torch.cdist(ab, bb).cpu() for bb in b.split(bs)], 1) for ab in a.split(bs)]
        return torch.cat(rows, 0)
    nn_r = full(feat_r, feat_r).kthvalue(k + 1).values
    nn_g = full(feat_g, feat_g).kthvalue(k + 1).values
    d_gr = full(feat_g, feat_r)
    return ((d_gr <= nn_r).any(1).float().mean().item(), (d_gr.T <= nn_g).any(1).float().mean().item())


def host_free_bytes():
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        pass
    return 0


def median_times(runs, reps):
    times = {k: [] for k in runs}
    for fn in runs.values():
        fn()                                                        # warm-up
    for _ in range(reps):
        for k, fn in runs.items():
            times[k].append(timed_ms(fn))
    return {k: statistics.median(v) for k, v in times.items()}


def profile_kernels(fn, out_dir, tag):
    """One call of ``fn`` under torch.profiler: prints the summed CUDA time per kernel and writes the trace."""
    from torch.profiler import ProfilerActivity, profile
    os.makedirs(out_dir, exist_ok=True)
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, f"{tag}.pt.trace.json"))
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = e.name.split("(")[0][:90]
            n, t = per.get(k, (0, 0.0))
            per[k] = (n + 1, t + e.device_time_total / 1e3)
    total = sum(t for _, t in per.values())
    rows = sorted(per.items(), key=lambda kv: -kv[1][1])[:12]
    print(json.dumps({"profile": tag, "kernel_ms_total": round(total, 2),
                      "top": [[k, n, round(t, 2)] for k, (n, t) in rows]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--pr", default="10000,50000")
    ap.add_argument("--profile", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_fid.py measures on a CUDA device"
    dev = torch.device("cuda", torch.cuda.current_device())
    print(f"# {torch.cuda.get_device_name(dev)}, power limit {power_limit_w()} W", flush=True)
    sd = NO.synthetic_weights()
    net = FD.InceptionV3(sd, device=dev)
    net_tf32 = FD.InceptionV3(sd, device=dev, tf32=True)
    ref = TorchInception(sd, dev)
    chunk = net.max_chunk_frames
    g = torch.Generator(device=dev).manual_seed(0)
    for name in [c for c in args.cases.split(",") if c]:
        S, C = CASES[name]
        frames = torch.rand(args.frames, C, S, S, device=dev, generator=g)
        N = frames.shape[0]

        def torch_run():
            with torch.no_grad():
                return torch.cat([ref(frames[lo:lo + chunk]) for lo in range(0, N, chunk)])

        runs = {"native": lambda: net(frames, C), "native_tf32": lambda: net_tf32(frames, C)}
        for tf32 in (False, True):
            runs[f"cudnn_tf32_{'on' if tf32 else 'off'}"] = (lambda t=tf32: (
                setattr(torch.backends.cudnn, "allow_tf32", t), setattr(torch.backends.cuda.matmul, "allow_tf32", t),
                torch_run()))
        med = median_times(runs, args.reps)
        flops = N * flops_per_frame()
        res = {"case": name, "frames": N, "side": S, "channels": C, "tflop": round(flops / 1e12, 2)}
        for k, ms in med.items():
            res[f"{k}_ms"] = round(ms, 1)
            res[f"{k}_tflops"] = round(flops / ms / 1e9, 2)
        f_native, f_tf32 = net(frames, C), net_tf32(frames, C)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
        f_ref_tf32 = torch_run()
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        f_ref = torch_run()
        res["max_abs_diff_vs_cudnn_fp32_over_scale"] = float((f_native - f_ref).abs().max() / f_ref.abs().max())
        res["native_tf32_vs_native_over_scale"] = float((f_tf32 - f_native).abs().max() / f_native.abs().max())
        res["cudnn_tf32_vs_cudnn_fp32_over_scale"] = float((f_ref_tf32 - f_ref).abs().max() / f_ref.abs().max())
        half = N // 2
        res["fid_native"] = FD.fid(f_native[half:], f_native[:half])
        res["fid_native_tf32"] = FD.fid(f_tf32[half:], f_tf32[:half])
        res["fid_cudnn_fp32"] = FD.fid(f_ref[half:], f_ref[:half])
        res["fid_cudnn_tf32"] = FD.fid(f_ref_tf32[half:], f_ref_tf32[:half])
        print(json.dumps(res), flush=True)
        if args.profile:
            profile_kernels(lambda: net_tf32(frames, C), args.profile, name)
        del frames, f_native, f_tf32, f_ref, f_ref_tf32
        torch.cuda.empty_cache()
    for n in [int(v) for v in args.pr.split(",") if v]:
        real = torch.relu(torch.randn(n, 2048, device=dev, generator=g))
        fake = torch.relu(torch.randn(n, 2048, device=dev, generator=g) + 0.05)
        runs = {"native": lambda: FD.precision_recall(real, fake, 3, dev)}
        fits = 3 * n * n * 4 <= host_free_bytes() // 2
        if fits:
            runs["torch_full"] = lambda: reference_pr(real, fake)
        med = median_times(runs, max(1, args.reps if n <= 10000 else 1))
        res = {"case": f"pr_{n}", "rows_per_side": n, "dims": 2048,
               "pair_terms_per_pass": float(n) * n * 2048}
        for k, ms in med.items():
            res[f"{k}_ms"] = round(ms, 1)
        res["native"] = FD.precision_recall(real, fake, 3, dev)
        if fits:
            res["torch_full"] = reference_pr(real, fake)
        else:
            res["torch_full"] = f"not run: 3 x {n * n * 4 / 2**30:.1f} GiB host matrices"
        print(json.dumps(res), flush=True)
        del real, fake
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
