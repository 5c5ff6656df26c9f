"""Activation memory of the lowered score-network program, per workload.

For each workload: MiB per clip with one allocation per buffer (how programs were allocated before liveness
planning), persistent buffers (inputs and outputs included) and planned temporaries (mcvd_b200/memplan.py), and the
planner's overhead over the liveness lower bound of the temporaries.  Host arithmetic from ``Engine.plan``: nothing
is allocated or run.  With ``--fit`` on a GPU it also finds the largest batch whose program build plus one DDPM
sampler call fits on the card.

    python tools/memory_plan.py [--workloads cfg2,cfg7] [--batch B] [--fit]
"""
import argparse
import gc
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from mcvd_b200 import configs, detfill, samplers  # noqa: E402
from mcvd_b200.program import Engine  # noqa: E402
from mcvd_b200.synthetic import make_module  # noqa: E402

MiB = 2.0 ** 20


class HostPacking:
    """Engine backend for planning on a host without a GPU: weight images stay fp32 taps (their size does not enter
    the activation plan); no op ever runs"""

    def pack_umma(self, taps, nt, kb):
        return taps.contiguous().float(), 1.0


def fits(net, cfg, B):
    """True when the batch-B program builds and one 2-step DDPM call runs without running out of memory"""
    eng = net.engine()
    eng.programs.clear()
    gc.collect()
    torch.cuda.empty_cache()
    try:
        x, cond = detfill.synthetic_inputs(cfg, B)
        samplers.ddpm_sampler(x.cuda(), net, cond=cond.cuda(), final_only=True, subsample_steps=2, philox_seed=1)
        torch.cuda.synchronize()
        return True
    except torch.cuda.OutOfMemoryError:
        return False
    finally:
        eng.programs.clear()
        gc.collect()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--workloads", default=",".join(configs.ALL_WORKLOADS))
    ap.add_argument("--batch", type=int, default=0, help="clips to plan (default: the workload's bench batch)")
    ap.add_argument("--fit", action="store_true", help="on a GPU: find the largest batch that fits")
    args = ap.parse_args()
    gpu = torch.cuda.is_available()
    if args.fit and not gpu:
        raise SystemExit("--fit needs a CUDA device")
    if gpu:
        p = torch.cuda.get_device_properties(0)
        print(f"# {p.name}, {p.total_memory / 2 ** 30:.1f} GiB")
    print(f"{'workload':<9} {'B':>4} {'one per buffer':>15} {'persistent':>11} {'temporaries':>12} {'planned':>9} "
          f"{'overhead':>9}" + ("  largest batch" if args.fit else ""))
    for name in args.workloads.split(","):
        cfg, net, _ = make_module(name, "cuda:0" if gpu else "cpu")
        eng = Engine(net, _test_backend=None if gpu else HostPacking())
        B = args.batch or cfg.bench_batch
        P = eng.plan(B)
        per = lambda n: n / MiB / B
        line = (f"{name:<9} {B:>4} {per(P.unplanned_bytes):>11.1f} MiB {per(P.io_bytes + P.persistent_bytes):>7.1f} MiB "
                f"{per(P.arena_bytes):>8.1f} MiB {per(P.io_bytes + P.persistent_bytes + P.arena_bytes):>5.1f} MiB "
                f"{P.arena_bytes / max(1, P.lower_bound_bytes) - 1:>8.2%}")
        del eng, P
        if args.fit:
            lo, hi = 1, 2
            while fits(net, cfg, hi):
                lo, hi = hi, hi * 2
            while hi - lo > 1:
                mid = (lo + hi) // 2
                lo, hi = (mid, hi) if fits(net, cfg, mid) else (lo, mid)
            line += f"  {lo}"
        print(line, flush=True)
        del net
        gc.collect()
        if gpu:
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
