"""Gamma-noise models (model.gamma=True) on the H100: the in-kernel Gamma draw of MCVD_F_GAMMA / MCVD_OP_NOISE element
by element against oracle/gamma_oracle.py and in distribution against scipy.stats.gamma, golden parity of the Gamma
samplers and AR loop with the reference's recorded draws injected (tests/golden/tiny_gamma.npz), bit-exact clip
sharding, equal launch counts and the drop-in shim.

Tolerances: a draw is compared as the centred value G - k, which can be near zero, so the bound is absolute,
1e-5 of the draw's standard deviation sqrt(k) (the kernel rounds to fp32 once; everything before is fp64).  An
acceptance test within 1e-12 of its threshold could flip between the kernel's and numpy's libm; such draws are
counted and none is expected.  Sampler and AR-loop parity: PSNR >= 50 dB on [0, 1] frames."""
import math

import numpy as np
import pytest
import scipy.stats
import torch

from common import golden, make_module
from mcvd_b200 import configs, detfill, lib, runner, samplers
from mcvd_b200.lib import McvdOp
from oracle import gamma_oracle as GO, gen_golden_gamma as GG, mcvd_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KS = (0.5, 1.0, 2.5, 1898.0, 1.17e7, 2.48e10)


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def noise(B, C, H, W, k, scale, seed, clip0=0, step=0):
    out = torch.empty(B, C, H, W, device=DEV)
    o = McvdOp()
    o.kind, o.flags, o.B, o.H, o.W, o.C0 = lib.OP_NOISE, lib.F_GAMMA, B, H, W, C
    lo, hi = GO.seed_words(seed)
    o.i0, o.i1, o.i2, o.i3, o.f5, o.f6, o.f7 = lo, hi, clip0, step, 1.0, k, scale
    o.dst = out.data_ptr()
    run([o])
    return out


@pytest.mark.parametrize("k", KS)
def test_kernel_draws_equal_oracle_per_element(k):
    B, C, S, seed, step = 2, 3, 64, 20261015, 7
    n = C * S * S
    kf = float(np.float32(k))
    for scale in (1.0, 1.0 / math.sqrt(kf)):
        z = noise(B, C, S, S, k, scale, seed, clip0=5, step=step).cpu().double().reshape(B, n)
        sf = float(np.float32(scale))
        for b in range(B):
            g, att, margin = GO.gamma_centred(k, seed, 5 + b, step, n)
            near = int((margin < 1e-12).sum())
            assert near == 0, f"{near} acceptance tests within 1e-12 of the threshold"
            assert (att >= 0).all()
            err = np.abs(z[b].numpy() - sf * g).max()
            assert err <= 1e-5 * sf * math.sqrt(kf), (k, b, err)
    # the update's fused draw is the same draw: x = 0 * x0 + 1 * x + sigma * z with x = 0
    x = torch.zeros(B, C, S, S, device=DEV)
    eps = torch.zeros(B, S, S, C, device=DEV)
    u = McvdOp()
    u.kind, u.B, u.H, u.W, u.C0 = lib.OP_DIFFUSION_UPDATE, B, S, S, C
    u.flags = lib.F_PHILOX | lib.F_GAMMA
    lo, hi = GO.seed_words(seed)
    u.i0, u.i1, u.i2, u.i3, u.f3, u.f5, u.f6, u.f7 = lo, hi, 5, step, 1.0, 1.0, k, 1.0
    u.src0, u.dst = eps.data_ptr(), x.data_ptr()
    run([u])
    assert torch.equal(x, noise(B, C, S, S, k, 1.0, seed, clip0=5, step=step))


@pytest.mark.parametrize("k", KS)
def test_kernel_draws_follow_scipy_gamma(k):
    kf = float(np.float32(k))
    scale = float(np.float32(1.0 / math.sqrt(kf)))
    z = noise(4, 1, 500, 500, k, scale, seed=4242 + KS.index(k)).cpu().double().numpy().reshape(-1)
    s = z / (scale * math.sqrt(kf))                           # (G - k) / sqrt(k): mean 0, variance 1
    n = s.size
    assert n == 1_000_000
    p = scipy.stats.kstest(s, lambda t: scipy.stats.gamma.cdf(kf + t * math.sqrt(kf), kf)).pvalue
    assert p > 1e-3, p
    assert abs(s.mean()) < 4 / math.sqrt(n)
    assert abs(s.var() - 1.0) < 4 * math.sqrt((2 + 6 / kf) / n)
    assert np.isfinite(s).all() and (s * math.sqrt(kf) + kf > -1e-6 * kf).all()     # G >= 0 up to fp32 rounding


def gpu_module():
    return make_module("tiny_gamma", DEV)


def to01(a):
    return ((a + 1) / 2).clamp(0, 1)


@pytest.mark.parametrize("key,prefix,t_min,ddim", [("ddpm", "ddpm_g", -1, False), ("ddpm_tmin", "tmin_g", GG.T_MIN, False),
                                                   ("ddim_tmin", "ddim_g", GG.T_MIN, True)])
def test_gamma_samplers_vs_reference_golden(key, prefix, t_min, ddim):
    cfg, net, _ = gpu_module()
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    L = cfg.sampling.subsample
    warm, zs = GG.reference_noise(net.k_cum.cpu(), net.theta_t.cpu(), net.alphas.cpu(), x.shape, L, prefix, t_min,
                                  per_step=not ddim)
    kw = dict(cond=cond.to(DEV), final_only=True, denoise=True, subsample_steps=L, clip_before=True, gamma=True,
              t_min=t_min, warm_noise=None if warm is None else warm.to(DEV), log=False)
    if ddim:
        out = samplers.ddim_sampler(x.to(DEV), net, **kw)
    else:
        out = samplers.ddpm_sampler(x.to(DEV), net, noise_list=[None if z is None else z.to(DEV) for z in zs], **kw)
    assert out.is_cuda
    assert O.psnr01(to01(out[0].cpu()), to01(torch.from_numpy(golden("tiny_gamma")[key]))) >= 50.0


def test_gamma_ar_loop_vs_reference_golden():
    cfg, net, _ = gpu_module()
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    L = cfg.sampling.subsample
    kc, th, al = net.k_cum.cpu(), net.theta_t.cpu(), net.alphas.cpu()
    vid = runner.video_gen_clips(
        cfg, net, cond.to(DEV), GG.NUM_FRAMES_PRED, init_fn=lambda i, sh: GG.reference_init(kc, th, sh, i).to(DEV),
        noise_fn=lambda i: [z.to(DEV) for z in GG.reference_noise(kc, th, al, x.shape, L, f"ar{i}_g")[1]])
    assert O.psnr01(vid.cpu(), torch.from_numpy(golden("tiny_gamma")["video"])) >= 50.0


def test_gamma_video_gen_sharded_split_batches_bit_exact():
    """x_T keyed by (init seed, global clip, AR iteration) and per-step Gamma noise keyed by global clip: clips [0, 2)
    and [2, 5) generated apart equal one batch of 5 bit for bit."""
    cfg, net, _ = gpu_module()
    cfg.sampling.num_frames_pred = 4
    cond = detfill.synthetic_inputs(cfg, 5)[1].to(DEV)
    full = runner.video_gen_sharded(cfg, net, cond, 0, 1, philox_seed=99, init_seed=7)
    gp = runner.gamma_init_params(cfg, net)
    parts = [runner.video_gen_clips(cfg, net, cond[lo:hi], clip_offset=lo, philox_seed=99,
                                    init_fn=runner.clip_init_fn(7, lo, hi, DEV, gamma=gp))
             for lo, hi in ((0, 2), (2, 5))]
    assert full.shape == (5, 4, 32, 32)
    assert torch.equal(torch.cat(parts), full), float((torch.cat(parts) - full).abs().max())
    # x_T is the centred Gamma draw G - k theta: mean ~ 0, std ~ sqrt(k) theta, not the normal init
    x_T = runner.clip_init_fn(7, 0, 5, DEV, gamma=gp)(0, (5, 2, 32, 32))
    want = math.sqrt(gp[0]) * gp[1]
    assert abs(float(x_T.std()) / want - 1) < 0.05 and abs(float(x_T.mean())) < 0.05 * want
    assert not torch.equal(x_T, runner.clip_init_fn(7, 0, 5, DEV)(0, (5, 2, 32, 32)).to(DEV))


def test_gamma_without_seed_follows_torch_manual_seed():
    cfg, net, _ = gpu_module()
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    kw = dict(cond=cond.to(DEV), final_only=True, subsample_steps=cfg.sampling.subsample, gamma=True)
    outs = []
    for seed in (3, 3, 4):
        torch.manual_seed(seed)
        outs.append(samplers.ddpm_sampler(x.to(DEV), net, **kw))
    assert torch.equal(outs[0], outs[1]) and not torch.equal(outs[0], outs[2])
    assert bool(torch.isfinite(outs[0]).all())


def test_gamma_costs_no_extra_launch():
    launches = {}
    for name in ("tiny", "tiny_gamma"):
        cfg, net, _ = make_module(name, DEV)
        x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
        for t_min in (-1, GG.T_MIN):
            samplers.ddpm_sampler(x.to(DEV), net, cond=cond.to(DEV), final_only=True, subsample_steps=10,
                                  philox_seed=11, t_min=t_min, gamma=cfg.model.gamma)
            launches[name, t_min] = samplers.ddpm_sampler.last_launches
    assert launches["tiny", -1] == launches["tiny_gamma", -1]
    assert launches["tiny", GG.T_MIN] == launches["tiny_gamma", GG.T_MIN]


def test_patch_install_routes_gamma_config_to_the_cuda_path(tmp_path, monkeypatch):
    """A stub with the reference's module layout (runners.ncsn_runner.get_model, models.{ddpm,ddim,FPNDM}_sampler)
    stands in for the reference tree, which the GPU machines do not have."""
    import importlib
    import sys
    (tmp_path / "runners").mkdir()
    (tmp_path / "models").mkdir()
    (tmp_path / "runners" / "__init__.py").write_text("")
    (tmp_path / "models" / "__init__.py").write_text(
        "def ddpm_sampler(x_mod, scorenet, **kw):\n    return 'reference ddpm'\n"
        "def ddim_sampler(x_mod, scorenet, **kw):\n    return 'reference ddim'\n"
        "def FPNDM_sampler(x_mod, scorenet, **kw):\n    return 'reference fpndm'\n")
    (tmp_path / "runners" / "ncsn_runner.py").write_text(
        "from models import ddpm_sampler, ddim_sampler, FPNDM_sampler\n"
        "def get_model(config):\n    return 'reference model'\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    for m in ("runners", "runners.ncsn_runner", "models"):
        sys.modules.pop(m, None)
    try:
        from mcvd_b200 import patch, model as fast_model
        patch.install(verbose=False)
        R = importlib.import_module("runners.ncsn_runner")
        M = importlib.import_module("models")
        cfg = configs.workload("tiny_gamma")
        cfg.device = torch.device(DEV)
        net = R.get_model(cfg)
        assert isinstance(net, fast_model.UNetMore_DDPM) and net.gamma and net.k_cum.is_cuda
        _, twin, sd = make_module("tiny_gamma", DEV)
        net.load_state_dict(sd, strict=True)
        x, cond = detfill.synthetic_inputs(cfg, 2)
        kw = dict(cond=cond.to(DEV), final_only=True, subsample_steps=10, philox_seed=1, gamma=True)
        out = M.ddpm_sampler(x.to(DEV), net, n_steps_each=0, step_lr=0.0, config=cfg, **kw)
        assert torch.is_tensor(out) and out.is_cuda
        assert torch.equal(out, samplers.ddpm_sampler(x.to(DEV), twin, **kw))
        assert torch.is_tensor(M.ddim_sampler(x.to(DEV), net, **kw))
    finally:
        for m in ("runners", "runners.ncsn_runner", "models"):
            sys.modules.pop(m, None)
