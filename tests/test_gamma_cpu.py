"""Gamma-noise models (model.gamma=True) on the CPU: what the fast path accepts, the reference's k / k_cum / theta_t
buffers, the DDPM / DDIM Gamma samplers and the AR loop with the reference's recorded draws injected, against
tests/golden/tiny_gamma.npz (oracle/gen_golden_gamma.py) with the lowered program executed by
tests/op_interpreter.py, and the host checks of the Gamma ops."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from common import golden, make_module
from mcvd_b200 import arch, configs, detfill, lib, runner, samplers
from mcvd_b200.program import Engine
from op_interpreter import Interpreter
from oracle import gamma_oracle as GO, gen_golden_gamma as GG, mcvd_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_check_supported_accepts_gamma_but_not_the_other_options():
    cfg = configs.workload("tiny_gamma")
    assert cfg.model.gamma is True and arch.check_supported(cfg) is None
    for flag in ("noise_in_cond", "cond_emb", "output_all_frames"):
        cfg = configs.workload("tiny_gamma")
        setattr(cfg.model, flag, True)
        assert arch.check_supported(cfg) == f"model.{flag}=True is not accelerated"
    assert configs.workload("tiny").model.gamma is False


def test_gamma_buffers_and_keys_equal_the_reference():
    """Names, order and values of the reference's buffers (ncsnpp_more.py:743-748): a reference gamma checkpoint
    loads with strict=True."""
    g = golden("tiny_gamma")
    cfg, net, sd = make_module("tiny_gamma", "cpu")
    assert list(net.state_dict().keys()) == list(g["keys"])
    for name in ("k", "k_cum", "theta_t"):
        assert np.array_equal(getattr(net, name).numpy(), g[name]), name
    assert net.gamma and net.k_cum[0] > 2e10 and net.k_cum[-1] < 2e3
    net.load_state_dict(sd, strict=True)
    # a plain model has none of them, as in the reference
    _, plain, _ = make_module("tiny", "cpu")
    assert not {"k", "k_cum", "theta_t"} & set(plain.state_dict())


def cpu_module():
    cfg, net, sd = make_module("tiny_gamma", "cpu")
    net._engine = Engine(net, _test_backend=Interpreter())
    return cfg, net


def to01(a):
    return ((a + 1) / 2).clamp(0, 1)


def sampler_inputs(cfg, net, prefix, t_min=-1, per_step=True):
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    warm, noise = GG.reference_noise(net.k_cum, net.theta_t, net.alphas, x.shape, cfg.sampling.subsample, prefix,
                                     t_min, per_step)
    return x, cond, warm, noise


@pytest.mark.parametrize("key,prefix,t_min", [("ddpm", "ddpm_g", -1), ("ddpm_tmin", "tmin_g", GG.T_MIN)])
def test_ddpm_gamma_with_injected_draws_matches_reference_golden(key, prefix, t_min):
    cfg, net = cpu_module()
    x, cond, warm, noise = sampler_inputs(cfg, net, prefix, t_min)
    assert (warm is None) == (t_min < 0) and noise[-1] is not None
    out = samplers.ddpm_sampler(x, net, cond=cond, final_only=True, denoise=True, subsample_steps=cfg.sampling.subsample,
                                clip_before=True, gamma=True, t_min=t_min, noise_list=noise, warm_noise=warm)[0]
    assert O.psnr01(to01(out), to01(torch.from_numpy(golden("tiny_gamma")[key]))) > 50.0


def test_ddim_gamma_warm_start_matches_reference_golden():
    cfg, net = cpu_module()
    x, cond, warm, _ = sampler_inputs(cfg, net, "ddim_g", GG.T_MIN, per_step=False)
    out = samplers.ddim_sampler(x, net, cond=cond, final_only=True, denoise=True, subsample_steps=cfg.sampling.subsample,
                                clip_before=True, gamma=True, t_min=GG.T_MIN, warm_noise=warm, log=False)[0]
    assert O.psnr01(to01(out), to01(torch.from_numpy(golden("tiny_gamma")["ddim_tmin"]))) > 50.0


def test_ar_loop_gamma_matches_reference_golden():
    cfg, net = cpu_module()
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    L = cfg.sampling.subsample
    vid = runner.video_gen_clips(
        cfg, net, cond, GG.NUM_FRAMES_PRED, init_fn=lambda i, shape: GG.reference_init(net.k_cum, net.theta_t, shape, i),
        noise_fn=lambda i: GG.reference_noise(net.k_cum, net.theta_t, net.alphas, x.shape, L, f"ar{i}_g")[1])
    assert O.psnr01(vid, torch.from_numpy(golden("tiny_gamma")["video"])) > 50.0


def test_gamma_log_lines_are_tagged(caplog):
    cfg, net = cpu_module()
    x, cond, _, noise = sampler_inputs(cfg, net, "ddpm_g")
    import logging
    with caplog.at_level(logging.INFO):
        samplers.ddpm_sampler(x, net, cond=cond, final_only=True, subsample_steps=10, gamma=True, noise_list=noise,
                              log=True)
        samplers.ddim_sampler(x, net, cond=cond, final_only=True, subsample_steps=10, gamma=True, log=True)
    assert "DDPM gamma: 1/10" in caplog.text and "DDIM gamma: 1/10" in caplog.text


def noise_op(**kw):
    o = lib.McvdOp()
    o.kind, o.B, o.H, o.W, o.C0 = lib.OP_NOISE, 2, 4, 4, 3
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_validate_program_rejects_bad_gamma_and_noise_ops():
    buf = torch.zeros(4096)
    ptr = buf.data_ptr()
    good = noise_op(dst=ptr, flags=lib.F_GAMMA, f5=1.0, f6=2.5, f7=0.1)
    lib.validate_program(lib.make_ops([good]), 1)                          # src0 is not read
    lib.validate_program(lib.make_ops([noise_op(dst=ptr, f5=1.0)]), 1)     # normal draw
    with pytest.raises(RuntimeError, match="null src0/dst"):
        lib.validate_program(lib.make_ops([noise_op(flags=lib.F_GAMMA, f6=2.5, f7=0.1)]), 1)
    for f6, f7, what in ((0.0, 1.0, "shape"), (-1.0, 1.0, "shape"), (float("inf"), 1.0, "shape"),
                         (float("nan"), 1.0, "shape"), (2.5, float("inf"), "scale"), (2.5, float("nan"), "scale")):
        with pytest.raises(RuntimeError, match=f"Gamma {what}"):
            lib.validate_program(lib.make_ops([noise_op(dst=ptr, flags=lib.F_GAMMA, f6=f6, f7=f7)]), 1)
        u = lib.McvdOp()
        u.kind, u.B, u.H, u.W, u.C0, u.f5 = lib.OP_DIFFUSION_UPDATE, 2, 4, 4, 3, 1.0
        u.src0 = u.dst = ptr
        u.flags, u.f6, u.f7 = lib.F_PHILOX | lib.F_GAMMA, f6, f7
        with pytest.raises(RuntimeError, match=f"Gamma {what}"):
            lib.validate_program(lib.make_ops([u]), 1)
    u = lib.McvdOp()
    u.kind, u.B, u.H, u.W, u.C0, u.f5, u.f6, u.f7 = lib.OP_DIFFUSION_UPDATE, 2, 4, 4, 3, 1.0, 2.5, 0.1
    u.src0 = u.src1 = u.dst = ptr
    u.flags = lib.F_GAMMA                                                  # Gamma noise is drawn in-kernel only
    with pytest.raises(RuntimeError, match="needs MCVD_F_PHILOX"):
        lib.validate_program(lib.make_ops([u]), 1)
    u.flags = lib.F_GAMMA | lib.F_PHILOX
    lib.validate_program(lib.make_ops([u]), 1)
    # one launch each: the Gamma draw is fused, not a separate kernel
    assert lib.load().mcvd_count_launches(ctypes.byref(u), 1) == 1
    assert lib.load().mcvd_count_launches(lib.make_ops([good, good]), 2) == 2


def test_header_and_binding_agree_on_gamma_surface():
    hdr = open(os.path.join(ROOT, "include", "mcvd_b200.h")).read()
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.ABI_VERSION == 5
    assert int(re.search(r"MCVD_OP_NOISE\s*=\s*(\d+)", hdr).group(1)) == lib.OP_NOISE == 18
    assert int(re.search(r"#define MCVD_F_GAMMA\s+\(1 << (\d+)\)", hdr).group(1)) == 8 and lib.F_GAMMA == 1 << 8
    assert lib.load().mcvd_abi_version() == 5


def test_gamma_oracle_philox_matches_the_normal_stream_and_is_exact_for_large_k():
    """The oracle's Philox4x32-10 is the kernel's (the Random123 known-answer vector), and its centred draw for
    k = 2.5e10 is free of cancellation: it does not collapse to the ~1.6e5 / 2^24 grid of k * theta in fp32."""
    r = GO.philox4x32_10(np.array([0xFFFFFFFF], np.uint32), 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF)
    assert [int(v[0]) for v in r] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    g, att, _ = GO.gamma_centred(2.48e10, 5, 0, 0, 20000)
    assert (att == 0).mean() > 0.99 and len(np.unique(np.float32(g / np.sqrt(2.48e10)))) > 19000
    # k < 1 (boost) draws are positive Gamma variates
    g, _, _ = GO.gamma_centred(0.5, 5, 0, 0, 20000)
    assert (g + 0.5 > 0).all()


def test_runner_gamma_init_params():
    cfg, net, _ = make_module("tiny_gamma", "cpu")
    k, th = runner.gamma_init_params(cfg, net)
    assert k == float(net.k_cum[0]) and th == float(net.theta_t[0])
    assert runner.gamma_init_params(configs.workload("tiny"), net) is None
    with pytest.raises(RuntimeError, match="CUDA"):
        samplers.gamma_noise((1, 1, 2, 2), k, th, 1, device="cpu")
