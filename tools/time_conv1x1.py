"""Time every 1x1 convolution of a workload's lowered forward on the GPU in both work organisations of
OP_CONV_UMMA (i2 = 1 streaming, i2 = 2 input-stationary) and print what the launcher picks (i2 = 0).

    python tools/time_conv1x1.py [--workload cfg2] [--batch 64] [--reps 50]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, lib  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402


def time_op(op, reps):
    arr = lib.make_ops([op])
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        lib.run_program(arr, 1, stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        lib.run_program(arr, 1, stream)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    cfg = configs.workload(args.workload)
    B = args.batch or cfg.bench_batch
    _, net, _ = make_module(args.workload, "cuda:0")
    P = net.engine().program(B)
    print(torch.cuda.get_device_name(0))
    print("B  HxW  Cin  Cout  NT | streaming_us  stationary_us  auto_us")
    tot = [0.0, 0.0, 0.0]
    for op in P.step_ops:
        if op.kind != lib.OP_CONV_UMMA or op.i0 != 1:
            continue
        t = []
        for mode in (1, 2, 0):
            op.i2 = mode
            t.append(time_op(op, args.reps))
        op.i2 = 0
        tot = [a + b for a, b in zip(tot, t)]
        print(f"{op.B} {op.H}x{op.W} {op.C0 + op.C1} {op.Cout} {op.i1} | {t[0]:.1f}  {t[1]:.1f}  {t[2]:.1f}")
    print(f"total per forward | {tot[0]:.1f}  {tot[1]:.1f}  {tot[2]:.1f}")


if __name__ == "__main__":
    main()
