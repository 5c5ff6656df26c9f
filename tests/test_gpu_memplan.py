"""Liveness-planned activation memory on the H100: NaN-poisoned temporaries change no bit of eps, and the Cityscapes
SPADE recipe samples its 45 clips in one call, bit-identical to the same clips split over two calls."""
import gc

import pytest
import torch

from common import make_module
from mcvd_b200 import configs, detfill, samplers
from mcvd_b200.program import Engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

MODES = {"umma": dict(conv_mode="umma"), "umma2": dict(conv_mode="umma2", epilogue_stats=True),
         "simt": dict(conv_mode="simt", attn_mode="simt"), "fp16": dict(conv_mode="umma", conv_precision="fp16")}
ROWS = [("tiny", None), ("tiny_spade", None), ("cfg2", 64), ("cfg7", 2)]


def poison(P):
    P.arena[P.persistent_bytes:].view(torch.float32).fill_(float("nan"))


def run(eng, B, x, cond, t, graph, poisoned):
    """cond program, then two network evaluations (the second from the CUDA graph when ``graph``); with
    ``poisoned`` every temporary is NaN before the cond program, between it and the steps and before each step"""
    P = eng.program(B)
    eng.set_inputs(P, x=x, t=t, cond=cond)
    if poisoned:
        poison(P)
    eng.run_cond(P)
    outs = []
    for _ in range(2):
        if poisoned:
            poison(P)
        (eng.run_step_graphed if graph else eng.run_step)(P)
        outs.append(P.eps_nhwc.clone())
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name,B", ROWS, ids=[r[0] for r in ROWS])
def test_poisoned_temporaries_change_no_bit(name, B, mode):
    cfg, net, _ = make_module(name, DEV)
    eng = Engine(net)
    for k, v in MODES[mode].items():
        setattr(eng, k, v)
    B = B or cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    x, cond = x.to(DEV), cond.to(DEV)
    for t, graph in ((437.0, True), (torch.linspace(10, 990, B, device=DEV), False)):      # uniform t, per-clip t
        clean = run(eng, B, x, cond, t, graph, False)
        dirty = run(eng, B, x, cond, t, graph, True)
        assert all(bool(torch.isfinite(e).all()) for e in clean)
        for a, b in zip(clean, dirty):
            assert torch.equal(a, b), (name, mode, t if graph else "per-clip t")
    del eng, net
    gc.collect()
    torch.cuda.empty_cache()


def test_cityscapes_recipe_batch_in_one_call():
    """cfg7 at the recipe's 45 clips: one DDPM call (subsample 5, Philox noise) equals a 32-clip call and a 13-clip
    call at clip offset 32, bit for bit"""
    cfg, net, _ = make_module("cfg7", DEV)
    x, cond = detfill.synthetic_inputs(cfg, 45)
    x, cond = x.to(DEV), cond.to(DEV)
    kw = dict(final_only=True, denoise=True, subsample_steps=5, philox_seed=1234)
    torch.cuda.reset_peak_memory_stats()
    whole = samplers.ddpm_sampler(x.clone(), net, cond=cond, **kw)[0]
    peak = torch.cuda.max_memory_allocated()
    P = net.engine().program(45)
    print(f"\ncfg7 B=45: persistent {P.persistent_bytes / 2 ** 30:.2f} GiB + temporaries {P.arena_bytes / 2 ** 30:.2f} "
          f"GiB; max_memory_allocated {peak / 2 ** 30:.2f} GiB on {torch.cuda.get_device_name()}")
    del P
    net.engine().programs.clear()                  # 45 + 32 + 13 clips' programs at once would not fit
    gc.collect()
    torch.cuda.empty_cache()
    print(f"after dropping the 45-clip program: {torch.cuda.memory_allocated() / 2 ** 30:.2f} GiB allocated")
    a = samplers.ddpm_sampler(x[:32].clone(), net, cond=cond[:32], **kw)[0]
    b = samplers.ddpm_sampler(x[32:].clone(), net, cond=cond[32:], clip_offset=32, **kw)[0]
    assert torch.isfinite(whole).all()
    assert torch.equal(whole, torch.cat([a, b]))
