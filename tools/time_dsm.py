"""Time the native denoising score-matching test loss against the reference's formula around the same forward.

    python tools/time_dsm.py [--workloads cfg2 cfg5] [--batch 100] [--reps 5] [--launches 50]

For each workload (synthetic weights, one test batch of ``--batch`` clips, the reference configs'
``test.batch_size`` = 100), with CUDA events after a warm-up of each:
  * ``native``: ``runner.test_loss`` -- perturbation, network with per-clip timesteps and per-clip loss as CUDA ops;
  * ``torch``: the reference's ``anneal_dsm_score_estimation`` written out in torch (``randn_like``, the fp32
    perturbation, ``(z - eps)^2`` summed per clip) around the same native forward, which is what ``patch.install()``
    gave the reference's ``--test`` before the loss was native;
the two alternated ``--reps`` times, median reported; and each of the two DSM ops alone (``--launches`` launches,
mean), with in-kernel normal noise.  Prints the GPU's name and power limit, then one JSON line per workload.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mcvd_b200 import configs, detfill, runner  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--id=%d" % torch.cuda.current_device(), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip())
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


@torch.no_grad()
def torch_formula(cfg, net, X, labels):
    """losses/dsm.py's DDPM branch in torch around the native forward (one test batch, as NCSNRunner.test runs it)"""
    X = runner.data_transform(cfg, X)
    x, cond, _ = runner.conditioning_fn(cfg, X, num_frames_pred=cfg.data.num_frames)
    used = net.alphas[labels].reshape(x.shape[0], 1, 1, 1)
    z = torch.randn_like(x)
    x_t = used.sqrt() * x + (1 - used).sqrt() * z
    loss = (0.5 * (z - net(x_t, labels, cond)).square()).reshape(len(x), -1).sum(dim=-1)
    return loss.mean(dim=0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", nargs="+", default=["cfg2", "cfg5"])
    ap.add_argument("--batch", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    print(f"GPU: {torch.cuda.get_device_name(dev)}, power limit {power_limit_w()} W", flush=True)
    for name in a.workloads:
        cfg = configs.workload(name)
        cfg, net, _ = make_module(cfg, dev)
        C, S = cfg.data.channels, cfg.data.image_size
        T = cfg.data.num_frames_cond + cfg.data.num_frames
        B = a.batch
        X = detfill.uniform("time_dsm_X", (B, T, C, S, S), 0.0, 1.0).to(dev)
        labels = torch.randint(0, len(net.alphas), (B,), device=dev)
        native = lambda: runner.test_loss(cfg, net, X, labels=labels, philox_seed=1)  # noqa: E731
        ref = lambda: torch_formula(cfg, net, X, labels)  # noqa: E731
        native()
        ref()
        t_native, t_torch = [], []
        for _ in range(a.reps):
            t_native.append(timed(native))
            t_torch.append(timed(ref))
        eng = net.engine()
        D = eng.programs[B].dsm

        op_us = {}
        for op, arr in (("perturb", D.perturb_arr), ("loss", D.loss_arr)):
            def launches():
                for _ in range(a.launches):
                    eng._run(arr, 1)
            launches()
            op_us[op] = round(timed(launches) * 1000.0 / a.launches, 1)
        print(json.dumps(dict(workload=name, clips=B, native_ms=round(statistics.median(t_native), 2),
                              torch_ms=round(statistics.median(t_torch), 2),
                              native_runs_ms=[round(t, 2) for t in t_native],
                              torch_runs_ms=[round(t, 2) for t in t_torch],
                              perturb_us=op_us["perturb"], loss_us=op_us["loss"],
                              launches=eng.launches_last_dsm)), flush=True)
        del net, eng, D
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
