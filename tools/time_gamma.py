"""Time Gamma-noise sampling (model.gamma=True) against normal noise on the GPU.

    python tools/time_gamma.py [--clips 64] [--steps 100] [--reps 2] [--launches 200]

The model is workload cfg2 (SMMNIST, ngf 96, 5 past frames, 5 generated) with synthetic weights, once with
``model.gamma=True`` and once without.  Two measurements, both with CUDA events after a warm-up:
  * one AR block (``--steps`` DDPM steps, ``--clips`` clips) through ``runner.video_gen_sharded``, the two models
    alternated ``--reps`` times: frames/s and launches per block;
  * the fused update launch alone on the same [clips, 5, 64, 64] state, ``--launches`` times each: normal Philox
    noise, and Gamma noise with the shape of the noisiest level (k_cum[0] = 2.5e10) and of the middle one.
Prints the GPU's name and power limit, then one JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, detfill, lib, runner, samplers  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def gamma_cfg2():
    cfg = configs.workload("cfg2")
    cfg.workload = "cfg2_gamma"
    cfg.model.gamma = True
    return cfg


def block(cfg, net, cond, steps):
    return runner.video_gen_sharded(cfg, net, cond, 0, 1, sampler=samplers.ddpm_sampler,
                                    sampler_kwargs=dict(subsample_steps=steps), num_frames_pred=cfg.data.num_frames)


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def update_launch_us(net, B, n, gamma):
    """mean time of one fused update launch (sigma != 0, in-kernel noise) on the engine's state buffer"""
    eng = net.engine()
    with eng._devctx():
        P = eng.program(B)
        u = P.update_arr[0]
        u.f0, u.f1, u.f2, u.f3, u.f4, u.f5 = 1.0, 0.0, 0.5, 0.5, 0.0, 0.01
        u.flags = lib.F_CLIP | lib.F_PHILOX | (lib.F_GAMMA if gamma else 0)
        u.i0, u.i1, u.i2, u.i3 = 5, 0, 0, 0
        if gamma:
            u.f6, u.f7 = gamma
        for _ in range(10):
            eng._run(P.update_arr, 1)

        def loop():
            for i in range(n):
                u.i3 = i
                eng._run(P.update_arr, 1)
        return timed(loop) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--steps", type=int, default=100, help="DDPM steps per block")
    ap.add_argument("--reps", type=int, default=2, help="alternations of the two models")
    ap.add_argument("--launches", type=int, default=200, help="update launches timed per variant")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_gamma.py measures on a CUDA device; none is present")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu, watts = torch.cuda.get_device_name(dev), power_limit_w()
    print(json.dumps({"gpu": gpu, "power_limit_w": watts}))

    models = {"cfg2": make_module("cfg2", dev)[:2], "cfg2_gamma": make_module(gamma_cfg2(), dev)[:2]}
    cond = detfill.synthetic_inputs(models["cfg2"][0], args.clips)[1].to(dev)
    for cfg, net in models.values():                   # warm-up: builds and captures the programs
        block(cfg, net, cond, 2)
    for rep in range(args.reps):
        for name, (cfg, net) in models.items():
            ms = timed(lambda: block(cfg, net, cond, args.steps))
            nfp = cfg.data.num_frames
            print(json.dumps({
                "workload": name, "rep": rep, "clips": args.clips, "ddpm_steps": args.steps, "frames_per_clip": nfp,
                "ms_per_block": round(ms, 1), "frames_per_s": round(args.clips * nfp / (ms / 1e3), 2),
                "launches_per_block": samplers.ddpm_sampler.last_launches, "gpu": gpu, "power_limit_w": watts}))

    net = models["cfg2_gamma"][1]
    kc, th, al = net.k_cum.cpu(), net.theta_t.cpu(), net.alphas.cpu()
    variants = [("normal", None)] + [(f"gamma k={float(kc[i]):.3g}", samplers._gamma_params(kc, th, al, i))
                                     for i in (0, len(kc) // 2)]
    for name, gp in variants:
        us = update_launch_us(net, args.clips, args.launches, gp)
        print(json.dumps({"update_launch": name, "state": [args.clips, 5, 64, 64], "us_per_launch": round(us, 2),
                          "gpu": gpu, "power_limit_w": watts}))


if __name__ == "__main__":
    main()
