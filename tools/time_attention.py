"""Time the attention op at every attention shape of the wide-head recipes (cfg6 UCF-101, head dim 288; cfg7
Cityscapes SPADE, head dim 256): the tensor-core kernel (OP_ATTENTION_UMMA, pre-split + attention) and, where it
exists (head dim 256), the CUDA-core kernel (OP_ATTENTION).  FLOPs are 4*B*T^2*C (S = QK^T and O = PV); each time is
the median of alternated rounds of CUDA-event-timed launches.

    python tools/time_attention.py [workload ...] [--rounds N] [--iters N]
"""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from mcvd_b200 import arch, configs, lib


def shapes(name):
    """(B, T, heads, d) of every distinct attention layer of the workload, at its benchmark batch"""
    cfg = configs.workload(name)
    spec = arch.build_spec(cfg)
    seen = []
    for ms in spec.mods:
        if ms.kind == "attn":
            s = (cfg.bench_batch, ms.res * ms.res, ms.heads, ms.in_ch // ms.heads)
            if s not in seen:
                seen.append(s)
    return seen


def op_of(kind, B, T, heads, d, qkv, out, scratch):
    o = lib.McvdOp()
    side = int(round(T ** 0.5))
    o.kind, o.B, o.H, o.W, o.C0, o.i0, o.i1, o.f0 = kind, B, side, side, heads * d, heads, d, float(d) ** -0.5
    o.src0, o.dst = qkv.data_ptr(), out.data_ptr()
    if scratch is not None:
        o.dst2 = scratch.data_ptr()
    return lib.make_ops([o])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workloads", nargs="*", default=["cfg6", "cfg7"])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    stream = torch.cuda.current_stream().cuda_stream
    for name in args.workloads:
        for B, T, heads, d in shapes(name):
            C = heads * d
            qkv = torch.randn(B, T, 3 * C, device="cuda")
            out = torch.empty(B, T, C, device="cuda")
            scratch = torch.empty(lib.attention_scratch_bytes(B, T, C), dtype=torch.uint8, device="cuda")
            arms = {"tensor-core": op_of(lib.OP_ATTENTION_UMMA, B, T, heads, d, qkv, out, scratch)}
            if lib.attention_kind(T, d, "simt") == lib.OP_ATTENTION:
                arms["cuda-core"] = op_of(lib.OP_ATTENTION, B, T, heads, d, qkv, out, None)
            times = {k: [] for k in arms}
            for arr in arms.values():                    # warm-up: module load, function attributes
                for _ in range(3):
                    lib.run_program(arr, 1, stream)
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for k, arr in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        lib.run_program(arr, 1, stream)
                    e1.record()
                    e1.synchronize()
                    times[k].append(e0.elapsed_time(e1) * 1e3 / args.iters)
            flop = 4.0 * B * T * T * C
            for k, ts in times.items():
                us = statistics.median(ts)
                print(f"{name} B={B} T={T} heads={heads} d={d} {k:11s} {us:9.1f} us {flop / us * 1e-6:7.1f} TFLOP/s "
                      f"(spread {min(ts):.1f}..{max(ts):.1f})")


if __name__ == "__main__":
    main()
