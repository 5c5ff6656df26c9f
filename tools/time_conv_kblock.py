"""Time single launches of the 64x64 3x3 wgmma convs of a workload's forward (default cfg2, B = 64: 192->96, 288->96
and 192->192) in variants that take parts of the per-K-block work away, and report microseconds per K-block per SM:

    base     the launch as the forward runs it
    notab    without the norm table and the input SiLU (the producers only split the raw input into hi/lo)
    hh       i3 = 4: the hi*hi product only (a third of the MMA work)
    notab+hh both
    ntN      another n tile where Cout allows (the packed weights are read in the wrong order: timing only)
    mtM      a forced tile height (CONV_UMMA i4)
    saS      a forced number of slab stages (CONV_UMMA i5)

A K-block is KB input channels of one work item (all nine taps); a launch runs ceil(items * nKB / SMs) of them per SM.
The GPU name and power limit are read (not set) in the same run.

    python tools/time_conv_kblock.py [--workload cfg2] [--batch 64] [--reps 50]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, lib  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402

SHAPES = [(192, 96), (288, 96), (192, 192)]      # (Cin, Cout) of the 64x64 3x3 convs without a shortcut segment


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


def variants(op):
    v = [("base", {})]
    if op.aux1:
        v += [("notab", {"aux1": 0, "flags": op.flags & ~lib.F_ACT_IN})]
    v += [("hh", {"i3": 4})]
    if op.aux1:
        v += [("notab+hh", {"aux1": 0, "flags": op.flags & ~lib.F_ACT_IN, "i3": 4})]
    for nt in (96, 192):
        if nt != op.i1 and op.Cout % nt == 0:
            v += [(f"nt{nt}", {"i1": nt}), (f"nt{nt}+hh", {"i1": nt, "i3": 4})]
    for mt in (128, 192):
        v += [(f"mt{mt}", {"i4": mt})]
        for sa in (2, 3):
            v += [(f"mt{mt}+sa{sa}", {"i4": mt, "i5": sa})]
    return v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg2")
    ap.add_argument("--batch", type=int, default=0)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_conv_kblock.py measures on a CUDA device"
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = configs.workload(args.workload)
    B = args.batch or cfg.bench_batch
    _, net, _ = make_module(args.workload, "cuda:0")
    P = net.engine().program(B)
    picked = {}
    for op in P.step_ops:
        if op.kind not in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2) or op.i0 != 3 or op.H != 64 or op.src2:
            continue
        key = (op.C0 + op.C1, op.Cout)
        if key in SHAPES and key not in picked:
            picked[key] = op
    print(f"GPU: {q}")
    print(f"{args.workload} B={B}, 64x64 3x3, {sms} SMs; us per launch and per K-block per SM")
    print(f"{'Cin->Cout':>10} {'kind':>5} {'tab':>3} {'variant':>12} {'NT':>4} {'MT':>4} {'us':>8} {'us/KB/SM':>9}")
    for key in SHAPES:
        if key not in picked:
            print(f"{key[0]}->{key[1]}: not in this forward")
            continue
        base = picked[key]
        for name, kw in variants(base):
            op = type(base).from_buffer_copy(base)
            for k, val in kw.items():
                setattr(op, k, val)
            if op.kind == lib.OP_CONV_UMMA2 and ("i4" in kw or "i5" in kw):
                continue                      # the planar variant takes no tile-height or stage override
            try:
                us = time_op(op, args.reps)
            except RuntimeError as e:         # a forced setting the plan cannot run
                print(f"{key[0]:>4}->{key[1]:<5} {name:>12}: {e}")
                continue
            kb = lib.umma_kblock(op.C0, op.C1)
            mt = op.i4 or 128
            pimg = (op.H + 1) * (op.W + 1)
            items = -(-op.B * pimg // mt) * (op.Cout // op.i1)
            per_sm = items * ((op.C0 + op.C1) // kb) / min(sms, items)
            print(f"{key[0]:>4}->{key[1]:<5} {op.kind:>5} {int(bool(op.aux1)):>3} {name:>12} {op.i1:>4} "
                  f"{op.i4 or 'auto':>4} {us:>8.1f} {us / per_sm:>9.2f}")


if __name__ == "__main__":
    main()
