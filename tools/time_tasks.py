"""Time the three video_gen tasks of a "general" MCVD model on the GPU: interpolation, prediction with the future
block zeroed and unconditional generation.

    python tools/time_tasks.py [--clips 64] [--steps 100]

The model is cfg2 (SMMNIST, ngf 96, 5 past frames, 5 generated) with 5 future frames and past and future masked
with probability 0.5 in training: the reference's ``smmnist_64_5c5f5_unetm_b2_pmask50_futurepast`` recipe at ngf 96,
with synthetic weights and data.  Each task's whole AR loop runs through ``runner.video_gen_sharded(task=...)``
and is timed with CUDA events after one warm-up block of every task.  For comparison the same run times cfg2
(no future frames) predicting as many frames.  Prints the GPU's name and power limit, then one JSON line per task.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, detfill, runner, samplers  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402


def general_cfg2():
    cfg = configs.workload("cfg2")
    cfg.workload = "cfg2_5c5f5_pmask50_futurepast"
    cfg.data.num_frames_future, cfg.data.prob_mask_cond, cfg.data.prob_mask_future = 5, 0.5, 0.5
    return cfg


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def run(cfg, net, data, task, steps, num_frames_pred=None):
    """One task's whole AR loop over the clips of ``data`` (the test batch X, or for ``task=None`` the conditioning
    of a plain prediction)."""
    kw = dict(sampler=samplers.ddpm_sampler, sampler_kwargs=dict(subsample_steps=steps))
    if num_frames_pred is not None:
        kw["num_frames_pred"] = num_frames_pred
    return runner.video_gen_sharded(cfg, net, data, 0, 1, task=task, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--steps", type=int, default=100, help="DDPM steps per block")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_tasks.py measures on a CUDA device; none is present")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu, watts = torch.cuda.get_device_name(dev), power_limit_w()
    print(json.dumps({"gpu": gpu, "power_limit_w": watts}))

    cfg, net, _ = make_module(general_cfg2(), dev)
    base_cfg, base_net, _ = make_module("cfg2", dev)
    d = cfg.data
    T = d.num_frames_cond + max(d.num_frames + d.num_frames_future, cfg.sampling.num_frames_pred)
    X = detfill.uniform("task_clips", (args.clips, T, d.channels, d.image_size, d.image_size), 0.0, 1.0).to(dev)
    base_cond = detfill.synthetic_inputs(base_cfg, args.clips)[1].to(dev)
    runs = [(cfg, net, X, t) for t in runner.tasks_for(cfg)] + [(base_cfg, base_net, base_cond, None)]
    for c, n, data, task in runs:     # warm-up: one short block of every task builds and captures every program
        run(c, n, data, task, 2, num_frames_pred=0 if task == "gen" else c.data.num_frames)
    for c, n, data, task in runs:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        out = run(c, n, data, task, args.steps)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        nfp = out.shape[1] // c.data.channels
        blocks = -(-nfp // c.data.num_frames)
        print(json.dumps({
            "workload": c.workload, "task": task or "pred", "clips": args.clips, "ddpm_steps": args.steps,
            "frames_per_clip": nfp, "blocks": blocks, "ms": round(ms, 1), "ms_per_block": round(ms / blocks, 1),
            "frames_per_s": round(args.clips * nfp / (ms / 1e3), 2),
            "launches_per_block": samplers.ddpm_sampler.last_launches, "gpu": gpu, "power_limit_w": watts}))


if __name__ == "__main__":
    main()
