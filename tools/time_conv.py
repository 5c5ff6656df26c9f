"""Time every tensor-core conv launch of one forward of a workload (default cfg2, B = 64) with CUDA events, grouped by
(ks, H, Cin | Csc, Cout, NT): microseconds per forward, algorithmic and executed TFLOP/s, and share of the forward.
Algorithmic work counts 2 * pixels * Cout * (Cin * ks^2 + Csc); executed work counts every padded-flat position row
(padding positions included) rounded up to whole 128-position tiles, and the three fp16 products of the hi/lo split
(one product for the half-mode convs of --precision fp16).
Convs the launcher runs in 192-position tiles execute up to 191 rather than 127 rows past the last position, which
this count leaves out (under 0.4 % of the rows at 16x16 and above for the default batch).  The GPU name and power
limit are read (not set) in the same run.

    python tools/time_conv.py [--workload cfg2] [--batch 64] [--reps 20] [--precision fp32|fp16]
"""
import argparse
import collections
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, lib  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402


def time_ops(ops, reps):
    arr = lib.make_ops(ops)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        lib.run_program(arr, len(ops), stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        lib.run_program(arr, len(ops), stream)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "fp16"], help="model.conv_precision")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_conv.py measures on a CUDA device"
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    cfg = configs.workload(args.workload)
    B = args.batch or cfg.bench_batch
    cfg.model.conv_precision = args.precision
    _, net, _ = make_module(cfg, "cuda:0")
    P = net.engine().program(B)
    ops = list(P.step_ops)
    fwd = time_ops(ops, args.reps)
    groups = collections.OrderedDict()
    for op in ops:
        if op.kind not in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
            continue
        ks, cin, csc = op.i0, op.C0 + op.C1, (op.C2 if op.src2 else 0) + (op.C3 if op.src3 else 0)
        us = time_ops([op], args.reps)
        pimg = (op.H + 1) * (op.W + 1) if ks == 3 else op.H * op.W
        rows = -(-op.B * pimg // 128) * 128
        alg = 2.0 * op.B * op.H * op.W * op.Cout * (cin * ks * ks + csc)
        exe = (1 if op.flags & lib.F_HALF else 3) * 2.0 * rows * op.Cout * (cin * ks * ks + csc)
        key = (ks, op.H, cin, csc, op.Cout, op.i1)
        g = groups.setdefault(key, [0, 0.0, 0.0, 0.0])
        g[0] += 1; g[1] += us; g[2] += alg; g[3] += exe
    print(f"GPU: {q}")
    print(f"{args.workload} B={B} conv_precision={args.precision}: forward {fwd:.0f} us ({len(ops)} ops)")
    print(f"{'ks':>2} {'H':>4} {'Cin|Csc':>9} {'Cout':>5} {'NT':>4} {'n':>3} {'us':>9} {'alg_TF/s':>9} {'exe_TF/s':>9} {'share':>6}")
    tot = 0.0
    for (ks, H, cin, csc, cout, nt), (n, us, alg, exe) in groups.items():
        tot += us
        print(f"{ks:>2} {H:>4} {f'{cin}|{csc}':>9} {cout:>5} {nt:>4} {n:>3} {us:>9.1f} {alg / us / 1e6:>9.1f} "
              f"{exe / us / 1e6:>9.1f} {us / fwd:>6.1%}")
    print(f"convs total {tot:.0f} us = {tot / fwd:.1%} of the forward")


if __name__ == "__main__":
    main()
