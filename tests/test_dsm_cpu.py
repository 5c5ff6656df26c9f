"""Denoising score-matching test loss on the CPU: host checks and launch counts of MCVD_OP_DSM_PERTURB / DSM_LOSS, the
native loss with the reference's noise injected against tests/golden/dsm.npz (oracle/gen_golden_dsm.py) with the
lowered program executed by tests/op_interpreter.py, the plumbing of runner.test_loss, loss_per_level, and the
patch.install dispatch against a stub with the reference's module layout."""
import ctypes
import os
import re
import sys

import pytest
import torch

from common import golden, make_module
from mcvd_b200 import dsm, lib, runner, samplers
from mcvd_b200.program import Engine
from op_interpreter import Interpreter
from oracle import gen_golden_dsm as GD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class DsmInterpreter(Interpreter):
    """The op interpreter plus the two DSM kinds: the perturbation as the two rounded fp32 products and rounded add
    the op is defined as (injected noise only: no Philox on the CPU), the loss summed in fp64."""

    def exec(self, op, magnitude=False):
        B, C, HW = op.B, op.C0, op.H * op.W
        if op.kind == lib.OP_DSM_PERTURB:
            assert not op.flags & lib.F_PHILOX, "interpreter has no Philox"
            n = B * C * HW
            x, z = self.get(op.src0, n).view(B, -1), self.get(op.src1, n).view(B, -1)
            tab = self.get(op.aux0, B * 4).view(B, 4)
            xt = tab[:, 0:1] * x + tab[:, 1:2] * z
            self.get(op.dst, n).copy_(xt.reshape(-1))
            if op.dst2:
                self.get(op.dst2, n).copy_(z.reshape(-1))
        elif op.kind == lib.OP_DSM_LOSS:
            pitch = op.Cout if op.Cout > 0 else C
            eps = self.get(op.src0, B * HW * pitch).view(B, HW, pitch)[..., :C].transpose(1, 2)
            d = (self.get(op.src1, B * C * HW).view(B, C, HW) - eps).double()       # fp32 difference
            per = d.abs() if op.flags & lib.F_L1 else 0.5 * d * d
            self.get(op.dst, B, torch.float64).copy_(per.sum(dim=(1, 2)))
        else:
            super().exec(op, magnitude)


def cpu_module(name):
    cfg, net, _ = make_module(name, "cpu")
    net._engine = Engine(net, _test_backend=DsmInterpreter())
    return cfg, net


# ---------------------------------------------------------------------------------------------------------------
# host checks
# ---------------------------------------------------------------------------------------------------------------
def dsm_op(kind, **kw):
    o = lib.McvdOp()
    o.kind, o.B, o.H, o.W, o.C0 = kind, 2, 4, 4, 3
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_validate_program_accepts_and_rejects_dsm_ops():
    buf = torch.zeros(4096)
    ptr = buf.data_ptr()
    P = lib.OP_DSM_PERTURB
    good = [dsm_op(P, src0=ptr, src1=ptr, aux0=ptr, dst=ptr),                                   # injected z
            dsm_op(P, src0=ptr, aux0=ptr, dst=ptr, dst2=ptr, flags=lib.F_PHILOX),
            dsm_op(P, src0=ptr, aux0=ptr, dst=ptr, dst2=ptr, flags=lib.F_PHILOX | lib.F_GAMMA),
            dsm_op(lib.OP_DSM_LOSS, src0=ptr, src1=ptr, dst=ptr, Cout=16),
            dsm_op(lib.OP_DSM_LOSS, src0=ptr, src1=ptr, dst=ptr, flags=lib.F_L1)]
    for o in good:
        lib.validate_program(lib.make_ops([o]), 1)
        assert lib.load().mcvd_count_launches(ctypes.byref(o), 1) == 1
    assert lib.load().mcvd_count_launches(lib.make_ops(good), len(good)) == len(good)
    bad = [
        (dsm_op(P, src1=ptr, aux0=ptr, dst=ptr), "null src0/dst"),
        (dsm_op(P, src0=ptr, src1=ptr, aux0=ptr), "null src0/dst"),
        (dsm_op(P, src0=ptr, src1=ptr, dst=ptr), "null coefficient table"),
        (dsm_op(P, src0=ptr, aux0=ptr, dst=ptr), "null injected noise"),
        (dsm_op(P, src0=ptr, aux0=ptr, dst=ptr, flags=lib.F_PHILOX), "null noise output"),
        (dsm_op(P, src0=ptr, src1=ptr, aux0=ptr, dst=ptr, dst2=ptr, flags=lib.F_GAMMA), "needs MCVD_F_PHILOX"),
        (dsm_op(P, src0=ptr, src1=ptr, aux0=ptr, dst=ptr, flags=lib.F_L1), "flags other than"),
        (dsm_op(P, src0=ptr, aux0=ptr, dst=ptr, dst2=ptr, flags=lib.F_PHILOX | lib.F_CLIP), "flags other than"),
        (dsm_op(lib.OP_DSM_LOSS, src0=ptr, dst=ptr), "null noise src1"),
        (dsm_op(lib.OP_DSM_LOSS, src0=ptr, src1=ptr), "null src0/dst"),
        (dsm_op(lib.OP_DSM_LOSS, src0=ptr, src1=ptr, dst=ptr, flags=lib.F_PHILOX), "flags other than MCVD_F_L1"),
        (dsm_op(lib.OP_DSM_LOSS, src0=ptr, src1=ptr, dst=ptr, Cout=2), "pitch"),
    ]
    for o, why in bad:
        with pytest.raises(RuntimeError, match=why):
            lib.validate_program(lib.make_ops([o]), 1)


def test_header_and_binding_agree_on_dsm_surface():
    hdr = open(os.path.join(ROOT, "include", "mcvd_b200.h")).read()
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.ABI_VERSION == 5 == lib.load().mcvd_abi_version()
    assert int(re.search(r"MCVD_OP_DSM_PERTURB\s*=\s*(\d+)", hdr).group(1)) == lib.OP_DSM_PERTURB == 26
    assert int(re.search(r"MCVD_OP_DSM_LOSS\s*=\s*(\d+)", hdr).group(1)) == lib.OP_DSM_LOSS == 27
    assert int(re.search(r"#define MCVD_F_L1\s+\(1 << (\d+)\)", hdr).group(1)) == 10 and lib.F_L1 == 1 << 10
    assert dsm.DSM_STEP not in (samplers.GAMMA_WARM_STEP, samplers.GAMMA_INIT_STEP) and dsm.DSM_STEP > 1000


# ---------------------------------------------------------------------------------------------------------------
# golden parity with the reference's noise injected
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key,name,l1", GD.CASES)
def test_injected_dsm_matches_reference_golden(key, name, l1):
    g = golden("dsm")
    cfg, net = cpu_module(name)
    labels = torch.from_numpy(g["labels"])
    x, cond = GD.clean(cfg, len(labels))
    gamma = bool(cfg.model.gamma)
    z = GD.reference_noise(net, labels, x.shape, gamma)
    hooked = {}
    mean = dsm.anneal_dsm_score_estimation(net, x, labels=labels, cond=cond, gamma=gamma, L1=l1, noise=z,
                                           hook=lambda loss, lab: hooked.update(loss=loss, labels=lab))
    eng = net.engine()
    P = eng.programs[len(labels)]
    x_t = P.x_in
    assert torch.equal(x_t, torch.from_numpy(g[f"{'tiny' if key == 'tiny_l1' else key}_xt"]))
    want = torch.from_numpy(g[f"{key}_loss"]).double()
    assert hooked["loss"].dtype == torch.float32 and hooked["labels"] is labels
    assert torch.allclose(hooked["loss"].double(), want, rtol=1e-4, atol=0), (hooked["loss"], want)
    assert mean.dtype == torch.float32 and mean.shape == ()
    assert abs(float(mean) / float(g[f"{key}_mean"]) - 1) < 1e-4
    assert eng.launches_last_dsm == P.cond_launches + P.step_launches + 2


def test_dsm_refuses_what_it_does_not_cover():
    cfg, net = cpu_module("tiny")
    x, cond = GD.clean(cfg, 2)
    with pytest.raises(NotImplementedError, match="all frames"):
        dsm.anneal_dsm_score_estimation(net, x, cond=cond, all_frames=True)
    with pytest.raises(TypeError, match="UNetMore_DDPM"):
        dsm.anneal_dsm_score_estimation(torch.nn.Linear(2, 2), x, cond=cond)
    with pytest.raises(ValueError, match="exactly one"):
        net.engine().dsm(x, torch.zeros(2), cond)
    with pytest.raises(ValueError, match="model.gamma"):
        net.engine().dsm(x, torch.zeros(2), cond, philox=(1, 0, dsm.DSM_STEP), gamma=True)


# ---------------------------------------------------------------------------------------------------------------
# runner
# ---------------------------------------------------------------------------------------------------------------
def test_test_loss_draws_masks_labels_and_seed_as_the_reference(monkeypatch):
    """test_loss = data_transform, conditioning_fn with the training masks, labels, Philox seed, in that order of
    draws from torch's generator; model.gamma and training.L1 come from the config."""
    cfg, net = cpu_module("tiny_general")
    import argparse
    cfg.training = argparse.Namespace(L1=True)
    seen = {}

    def fake_dsm(x, labels, cond, *, z=None, philox=None, gamma=False, l1=False):
        seen.update(x=x.clone(), labels=labels.clone(), cond=cond.clone(), philox=philox, gamma=gamma, l1=l1)
        return torch.arange(x.shape[0], dtype=torch.float64)

    monkeypatch.setattr(net.engine(), "dsm", fake_dsm)
    B, T = 8, cfg.data.num_frames_cond + cfg.data.num_frames + cfg.data.num_frames_future
    X = torch.rand(B, T, cfg.data.channels, cfg.data.image_size, cfg.data.image_size)
    torch.manual_seed(5)
    out = runner.test_loss(cfg, net, X, clip_offset=3)
    torch.manual_seed(5)
    x, cond, _ = runner.conditioning_fn(cfg, runner.data_transform(cfg, X), num_frames_pred=cfg.data.num_frames,
                                        prob_mask_cond=0.5, prob_mask_future=0.5)
    labels = torch.randint(0, 1000, (B,))
    seed = samplers.draw_seed()
    assert torch.equal(seen["x"], x) and torch.equal(seen["cond"], cond) and torch.equal(seen["labels"], labels)
    assert seen["philox"] == (seed, 3, dsm.DSM_STEP) and seen["l1"] is True and seen["gamma"] is False
    assert bool((cond.flatten(1).abs().sum(1) < cond.flatten(1).abs().sum(1).max()).any())    # some clip masked
    assert torch.equal(out["labels"], labels) and out["loss"].dtype == torch.float64
    assert float(out["mean"]) == 3.5
    # fixed labels and seed are passed through; model.gamma reaches the loss
    cfg, net = cpu_module("tiny_gamma")
    monkeypatch.setattr(net.engine(), "dsm", fake_dsm)
    X = torch.rand(2, 5, 1, 32, 32)
    runner.test_loss(cfg, net, X, labels=torch.tensor([4, 9]), philox_seed=77)
    assert seen["gamma"] is True and seen["l1"] is False and seen["philox"] == (77, 0, dsm.DSM_STEP)
    assert seen["labels"].tolist() == [4, 9]


def test_loss_per_level():
    loss = torch.tensor([1.0, 2.0, 3.0, 4.0], dtype=torch.float64)
    per = runner.loss_per_level(loss, torch.tensor([0, 2, 2, 5]), 6)
    assert per.dtype == torch.float64 and per.shape == (6,)
    assert per[0] == 1.0 and per[2] == 2.5 and per[5] == 4.0
    assert torch.isnan(per[[1, 3, 4]]).all()


# ---------------------------------------------------------------------------------------------------------------
# drop-in
# ---------------------------------------------------------------------------------------------------------------
def test_patch_install_dispatches_the_dsm_loss(tmp_path, monkeypatch):
    """A stub with the reference's layout (losses/dsm.py; runners/ncsn_runner.py importing it and the samplers) stands
    in for the reference tree: native networks without grad and without all_frames get the native loss, everything
    else the reference function, under both names."""
    for d in ("runners", "models", "losses"):
        (tmp_path / d).mkdir()
        (tmp_path / d / "__init__.py").write_text("")
    (tmp_path / "models" / "__init__.py").write_text(
        "def ddpm_sampler(x_mod, scorenet, **kw):\n    return 'reference ddpm'\n"
        "def ddim_sampler(x_mod, scorenet, **kw):\n    return 'reference ddim'\n"
        "def FPNDM_sampler(x_mod, scorenet, **kw):\n    return 'reference fpndm'\n")
    (tmp_path / "losses" / "dsm.py").write_text(
        "def anneal_dsm_score_estimation(scorenet, x, labels=None, loss_type='a', hook=None, cond=None,\n"
        "                                cond_mask=None, gamma=False, L1=False, all_frames=False, **kw):\n"
        "    return 'reference dsm'\n")
    (tmp_path / "runners" / "ncsn_runner.py").write_text(
        "from losses.dsm import anneal_dsm_score_estimation\n"
        "from models import ddpm_sampler, ddim_sampler, FPNDM_sampler\n"
        "def get_model(config):\n    return 'reference model'\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    mods = ("runners", "runners.ncsn_runner", "models", "losses", "losses.dsm")
    for m in mods:
        sys.modules.pop(m, None)
    try:
        from mcvd_b200 import patch
        patch.install(verbose=False)
        import importlib
        R = importlib.import_module("runners.ncsn_runner")
        LD = importlib.import_module("losses.dsm")
        assert R.anneal_dsm_score_estimation is LD.anneal_dsm_score_estimation
        g = golden("dsm")
        cfg, net = cpu_module("tiny")
        labels = torch.from_numpy(g["labels"])
        x, cond = GD.clean(cfg, len(labels))
        z = GD.reference_noise(net, labels, x.shape, False)
        want = dsm.anneal_dsm_score_estimation(net, x, labels=labels, cond=cond, noise=z)
        wrapped = torch.nn.Module()
        wrapped.module = net                                        # DataParallel-style wrapper
        with torch.no_grad():
            for f in (R.anneal_dsm_score_estimation, LD.anneal_dsm_score_estimation):
                assert torch.equal(f(net, x, labels=labels, cond=cond, noise=z), want)
                assert torch.equal(f(wrapped, x, labels, "a", None, cond, noise=z), want)
            assert R.anneal_dsm_score_estimation(net, x, labels, "a", None, cond, None, False, False, True) == \
                "reference dsm"                                     # all_frames, positional
            assert R.anneal_dsm_score_estimation(net, x, cond=cond, all_frames=True) == "reference dsm"
            assert R.anneal_dsm_score_estimation(torch.nn.Linear(2, 2), x, cond=cond) == "reference dsm"
        with torch.enable_grad():                                    # training: gradients need the reference
            assert R.anneal_dsm_score_estimation(net, x, labels=labels, cond=cond, noise=z) == "reference dsm"
    finally:
        for m in mods:
            sys.modules.pop(m, None)
