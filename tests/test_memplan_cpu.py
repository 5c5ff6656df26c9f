"""Liveness planning of the lowered program's activation memory (mcvd_b200/memplan.py, Engine.plan) on the CPU: the
packer's invariants, the plan of every workload in every lowering mode, and a poison test -- the temporaries' region
filled with NaN before the cond program and before every network evaluation -- on the op interpreter."""
import random

import pytest
import torch

from common import golden, make_module, max_err, step_noise
from mcvd_b200 import configs, detfill, dsm, lib, memplan, samplers
from mcvd_b200.program import Engine
from op_interpreter import Interpreter
from oracle import gen_golden_dsm as GD
from oracle import mcvd_oracle as O
from test_dsm_cpu import DsmInterpreter

MODES = {"umma": dict(conv_mode="umma"), "umma2_stats": dict(conv_mode="umma2", epilogue_stats=True),
         "simt": dict(conv_mode="simt"), "fp16": dict(conv_mode="umma", conv_precision="fp16")}


def test_packer_places_random_intervals_without_sharing_live_bytes():
    rng = random.Random(7)
    for _ in range(50):
        n = rng.randint(1, 60)
        sizes = [rng.choice([0, 4, 300, 4096, 70000]) * rng.randint(1, 9) for _ in range(n)]
        ivs = []
        for _ in range(n):
            a = rng.randint(0, 40)
            ivs.append(None if rng.random() < 0.1 else (a, a + rng.randint(0, 10)))
        offs, pers, top = memplan.place(sizes, ivs)
        memplan.check(sizes, ivs, offs)
        assert pers == sum(memplan.align(s) for s, iv in zip(sizes, ivs) if iv is None)
        assert all(o + s <= pers + top for o, s in zip(offs, sizes))
        assert memplan.lower_bound(sizes, ivs) <= top


def test_buffers_of_different_kinds_never_share_a_start():
    rng = random.Random(11)
    for _ in range(50):
        n = rng.randint(2, 60)
        sizes = [rng.choice([256, 512, 4096]) for _ in range(n)]
        ivs = [(a, a + rng.randint(0, 3)) for a in (rng.randint(0, 30) for _ in range(n))]
        kinds = [(rng.choice("fi"), s) for s in sizes]
        offs, _, _ = memplan.place(sizes, ivs, kinds)
        memplan.check(sizes, ivs, offs, kinds)
    with pytest.raises(AssertionError, match="start at"):
        memplan.check([512, 512], [(0, 1), (2, 3)], [0, 0], [("f", 512), ("i", 512)])


def test_check_rejects_live_buffers_that_share_bytes():
    memplan.check([512, 512], [(0, 3), (4, 5)], [0, 0])                    # disjoint lifetimes may share
    with pytest.raises(AssertionError, match="share bytes"):
        memplan.check([512, 512], [(0, 3), (3, 5)], [0, 256])
    with pytest.raises(AssertionError, match="share bytes"):
        memplan.check([512, 512], [None, (3, 5)], [0, 0])                  # persistent overlaps every interval
    with pytest.raises(AssertionError, match="aligned"):
        memplan.check([512], [(0, 1)], [16])


_modules = {}


def engine(name, mode):
    if name not in _modules:
        _modules.clear()                        # one workload's module at a time
        _modules[name] = make_module(name, "cpu")
    cfg, net, _ = _modules[name]
    eng = Engine(net, _test_backend=Interpreter())
    for k, v in MODES[mode].items():
        setattr(eng, k, v)
    return cfg, eng


@pytest.mark.parametrize("name", configs.ALL_WORKLOADS + configs.TEST_WORKLOADS)
def test_plan_of_every_workload(name):
    """Engine.plan runs the planner's own checks (first use of a temporary is a write, no live buffers share a byte,
    every op's extent fits its buffer); the temporaries come within 1.25x of the liveness lower bound and the whole
    plan below one allocation per buffer"""
    for mode in MODES:
        cfg, eng = engine(name, mode)
        for B in sorted({1, cfg.bench_batch}):
            P = eng.plan(B)
            assert P.arena_bytes <= 1.25 * P.lower_bound_bytes, (mode, B, P.arena_bytes, P.lower_bound_bytes)
            assert P.io_bytes + P.persistent_bytes + P.arena_bytes < P.unplanned_bytes, (mode, B)
            assert P.arena is None                                 # planned, nothing allocated


def test_spade_gamma_beta_persist_and_temporaries_share_bytes():
    cfg, eng = engine("tiny_spade", "umma")
    P = eng.program(cfg.bench_batch)
    base = P.arena.data_ptr()
    step_reads = {getattr(o, f) for o in P.step_ops if o.kind == lib.OP_APPLY for f in ("aux1", "aux2") if getattr(o, f)}
    cond_writes = {o.dst for o in P.cond_ops}
    assert step_reads and step_reads <= cond_writes
    assert all(p - base < P.persistent_bytes for p in step_reads)
    dsts = [o.dst for o in P.step_ops]
    assert len(set(dsts)) < len(dsts)                          # outputs of different ops reuse one address
    assert all(P.persistent_bytes <= p - base < P.persistent_bytes + P.arena_bytes
               for p in dsts if p not in (P.eps_nhwc.data_ptr(), P.film.data_ptr()))


# ---------------------------------------------------------------------------------------------------------------
# poison: NaN in every temporary before the cond program and before every network evaluation
# ---------------------------------------------------------------------------------------------------------------
def poison(P):
    P.arena[P.persistent_bytes:].view(torch.float32).fill_(float("nan"))


def poisoned(eng):
    run_cond, run_step = eng.run_cond, eng.run_step

    def cond(P):
        poison(P)
        run_cond(P)
        poison(P)

    def step(P):
        poison(P)
        run_step(P)

    eng.run_cond, eng.run_step = cond, step
    return eng


POISON_NAMES = ["tiny", "tiny_spade", "tiny_general", "tiny_gamma", "tiny128"]


@pytest.mark.parametrize("name", POISON_NAMES)
def test_poisoned_temporaries_forward_and_ddpm(name):
    cfg, net, sd = make_module(name, "cpu")
    net._engine = poisoned(Engine(net, _test_backend=Interpreter()))
    B = 1 if name == "tiny128" else cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    tt = torch.full((B,), 37, dtype=torch.long)
    eps = net(x, tt, cond=cond)
    assert max_err(eps, O.unet_forward(cfg, sd, x, tt, cond)) < 5e-5
    if name in ("tiny", "tiny_spade"):
        assert max_err(eps, torch.from_numpy(golden(name)["eps_t37"])) < 5e-5
    L = 4
    zs = step_noise(x.shape, L)
    out = samplers.ddpm_sampler(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, noise_list=zs)[0]
    fn = lambda xx, t_, cc: O.unet_forward(cfg, sd, xx, t_, cc)
    ref = O.ddpm_sample(fn, O.make_schedule(cfg), x.clone(), cond, L, True, True, noise=zs)[0]
    assert max_err(out, ref) < 2e-3


@pytest.mark.parametrize("key,name,l1", GD.CASES)
def test_poisoned_temporaries_dsm(key, name, l1):
    g = golden("dsm")
    cfg, net, _ = make_module(name, "cpu")
    net._engine = poisoned(Engine(net, _test_backend=DsmInterpreter()))
    labels = torch.from_numpy(g["labels"])
    x, cond = GD.clean(cfg, len(labels))
    gamma = bool(cfg.model.gamma)
    z = GD.reference_noise(net, labels, x.shape, gamma)
    mean = dsm.anneal_dsm_score_estimation(net, x, labels=labels, cond=cond, gamma=gamma, L1=l1, noise=z)
    assert abs(float(mean) / float(g[f"{key}_mean"]) - 1) < 1e-4
