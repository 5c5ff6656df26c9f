"""Time the score network in both conv precisions (model.conv_precision = "fp32" / "fp16") in one session: one forward
and one AR block (one DDPM sampler call of the workload's step count, final frames only) at the workload's batch,
for cfg2 .. cfg5.  The two modes share weights and inputs and alternate run by run; each figure is the median of
--runs runs (CUDA events around work that ends in a device synchronise).  The GPU's name and power limit are read
(not set) in the same run.

    python tools/time_precision.py [--workloads cfg2,cfg3,cfg4,cfg5] [--runs 3] [--forwards 20] [--steps 0]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, detfill, samplers  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402

MODES = ("fp32", "fp16")


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3,cfg4,cfg5")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--forwards", type=int, default=20)
    ap.add_argument("--steps", type=int, default=0, help="DDPM steps of a block (default: the workload's)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_precision.py measures on a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(f"GPU: {gpu}")
    rows = []
    for name in args.workloads.split(","):
        nets = {}
        for mode in MODES:
            cfg = configs.workload(name)
            cfg.model.conv_precision = mode
            cfg, nets[mode], _ = make_module(cfg, "cuda:0")
        B, L = cfg.bench_batch, args.steps or cfg.sampling.subsample
        x, cond = detfill.synthetic_inputs(cfg, B)
        x, cond = x.cuda(), cond.cuda()
        t = torch.full((B,), 500, dtype=torch.long, device="cuda:0")
        kw = dict(cond=cond, final_only=True, denoise=True, subsample_steps=L, clip_before=True, log=False,
                  philox_seed=1234)
        fwd = {m: (lambda n=nets[m]: n(x, t, cond=cond)) for m in MODES}
        blk = {m: (lambda n=nets[m]: samplers.ddpm_sampler(x, n, **kw)) for m in MODES}
        for m in MODES:                                            # build, pack, capture the graphs
            fwd[m]()
            blk[m]()
        res = {m: {"fwd": [], "blk": []} for m in MODES}
        for _ in range(args.runs):
            for m in MODES:
                res[m]["fwd"].append(timed(fwd[m], args.forwards))
                res[m]["blk"].append(timed(blk[m], 1))
        med = {m: {k: statistics.median(v) for k, v in res[m].items()} for m in MODES}
        row = dict(workload=name, B=B, steps=L, **{f"{m}_{k}_ms": med[m][k] for m in MODES for k in ("fwd", "blk")})
        row["fwd_speedup"] = med["fp32"]["fwd"] / med["fp16"]["fwd"]
        row["blk_speedup"] = med["fp32"]["blk"] / med["fp16"]["blk"]
        rows.append(row)
        print(f"{name} B={B}: forward fp32 {med['fp32']['fwd']:.2f} ms, fp16 {med['fp16']['fwd']:.2f} ms "
              f"(x{row['fwd_speedup']:.3f}); {L}-step block fp32 {med['fp32']['blk']:.0f} ms, fp16 "
              f"{med['fp16']['blk']:.0f} ms (x{row['blk_speedup']:.3f}); runs fp32 {res['fp32']['blk']}, "
              f"fp16 {res['fp16']['blk']}", flush=True)
        del nets, fwd, blk
        gc.collect()
        torch.cuda.empty_cache()
    print(json.dumps(dict(gpu=gpu, rows=rows)))


if __name__ == "__main__":
    main()
