"""Host-side lowering (mcvd_b200/program.py, samplers.py, runner.py) checked on the CPU: the op program
is executed by tests/op_interpreter.py and compared with the oracle and the golden fixtures."""
import numpy as np
import pytest
import torch

from common import golden, make_module, max_err, step_noise
from mcvd_b200 import detfill, samplers, runner
from mcvd_b200.program import Engine
from op_interpreter import Interpreter
from oracle import mcvd_oracle as O


def cpu_module(name, conv_mode):
    cfg, net, sd = make_module(name, "cpu")
    eng = Engine(net, _test_backend=Interpreter())
    eng.conv_mode = conv_mode
    net._engine = eng
    return cfg, net, sd


@pytest.mark.parametrize("name", ["tiny", "tiny_spade", "tiny_rgb"])
@pytest.mark.parametrize("conv_mode", ["umma", "simt"])
def test_forward_lowering_matches_oracle_and_golden(name, conv_mode):
    cfg, net, sd = cpu_module(name, conv_mode)
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    g = golden(name)
    for t in (0, 37, 990):
        tt = torch.full((B,), t, dtype=torch.long)
        mine = net(x, tt, cond=cond)
        ref = O.unet_forward(cfg, sd, x, tt, cond)
        assert max_err(mine, ref) < 5e-5, (name, t, max_err(mine, ref))
        assert max_err(mine, torch.from_numpy(g[f"eps_t{t}"])) < 5e-5
    P = net.engine().program(B)
    if conv_mode == "umma":
        assert P.n_umma > 0
    # the lowered program is valid for the C ABI, and host and library agree on its kernel-launch count
    from mcvd_b200 import lib
    for arr, ops, n in ((P.step_arr, P.step_ops, P.step_launches), (P.cond_arr, P.cond_ops, P.cond_launches)):
        if ops:
            lib.validate_program(arr, len(ops))
            assert lib.load().mcvd_count_launches(arr, len(ops)) == n >= len(ops)


@pytest.mark.parametrize("mode", ["auto", "0", "1"])
def test_skip_projection_lowering_modes(mode):
    """Conv_2 (the 1x1 skip projection) either rides along Conv_1 as a second K-segment ('auto', the default, and '1')
    or is its own 1x1 convolution whose output enters Conv_1 as the residual ('0').  Same network function either
    way; the unfused program has one more op per ResBlock with a channel change."""
    from mcvd_b200 import lib
    cfg, net, sd = make_module("tiny", "cpu")
    eng = Engine(net, _test_backend=Interpreter())
    eng.conv_mode, eng.fuse_shortcut = "umma", mode
    net._engine = eng
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    tt = torch.full((B,), 37, dtype=torch.long)
    assert max_err(net(x, tt, cond=cond), O.unet_forward(cfg, sd, x, tt, cond)) < 5e-5
    P = eng.program(B)
    fused = sum(1 for op in P.step_ops if op.kind == lib.OP_CONV_UMMA and op.src2)
    plain_1x1 = sum(1 for op in P.step_ops if op.kind == lib.OP_CONV_UMMA and op.i0 == 1)
    assert (fused > 0) == (mode != "0")
    if mode == "0":
        assert plain_1x1 > sum(1 for op in P.step_ops if op.kind in (lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA)) * 2
    lib.validate_program(P.step_arr, len(P.step_ops))


def test_forward_lowering_128px_five_levels():
    """cityscapes-like topology (128 px, ch_mult of length 5, attention at 8/16/32): no reference golden at this
    size, the oracle (itself pinned to the reference on the small configs) is the checker."""
    cfg, net, sd = cpu_module("tiny128", "umma")
    x, cond = detfill.synthetic_inputs(cfg, 1)
    tt = torch.full((1,), 37, dtype=torch.long)
    assert max_err(net(x, tt, cond=cond), O.unet_forward(cfg, sd, x, tt, cond)) < 5e-5


@pytest.mark.parametrize("name", ["tiny", "tiny_spade"])
def test_samplers_lowering(name):
    cfg, net, sd = cpu_module(name, "umma")
    B = cfg.bench_batch
    L = cfg.sampling.subsample
    x, cond = detfill.synthetic_inputs(cfg, B)
    g = golden(name)
    zs = step_noise(x.shape, L)
    out = samplers.ddpm_sampler(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, noise_list=zs)
    assert out.shape == (1,) + tuple(x.shape)
    assert max_err(out[0], torch.from_numpy(g["ddpm"])) < 2e-3
    out = samplers.ddim_sampler(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, log=False)
    assert max_err(out[0], torch.from_numpy(g["ddim"])) < 2e-3
    out = samplers.FPNDM_sampler(x.clone(), net, cond=cond, final_only=True, subsample_steps=L, clip_before=True,
                                 log=False)
    assert max_err(out[0], torch.from_numpy(g["fpndm"])) < 2e-3
    # non-final_only returns the trajectory, same length as the reference (L steps + denoise)
    traj = samplers.ddpm_sampler(x.clone(), net, cond=cond, final_only=False, denoise=True, subsample_steps=L,
                                 noise_list=zs)
    assert traj.shape[0] == L + 1
    assert max_err(traj[-1], torch.from_numpy(g["ddpm"])) < 2e-3


def test_video_gen_loop_lowering():
    name = "tiny"
    cfg, net, sd = cpu_module(name, "umma")
    B = cfg.bench_batch
    L = cfg.sampling.subsample
    x, cond = detfill.synthetic_inputs(cfg, B)
    g = golden(name)
    nfp = cfg.sampling.num_frames_pred
    vid = runner.video_gen_clips(cfg, net, cond, nfp,
                                 init_fn=lambda i, shape: detfill.normal(f"ar_init{i}", shape),
                                 noise_fn=lambda i: step_noise(x.shape, L, tag=f"ar{i}_z"))
    ref = torch.from_numpy(g["video"])
    assert vid.shape == ref.shape
    assert O.psnr01(vid, ref) > 50.0


def test_evaluate_clips_preds_per_test_plumbing(monkeypatch):
    """The test-batch driver of the reference's video_gen (runners/ncsn_runner.py:1392-1395, 1463-1470, 1580-1609):
    repeat_interleave by preds_per_test, conditioning split, AR generation, per-frame metrics, best repeat per clip.  The
    GPU metric kernel is replaced by its oracle here (it has its own GPU parity test); everything else is the product
    code on the CPU interpreter."""
    from oracle import metrics_oracle as M
    cfg, net, sd = cpu_module("tiny", "umma")
    C, S = cfg.data.channels, cfg.data.image_size
    nfp, p, nclips = 2, 3, 2
    T = cfg.data.num_frames_cond + nfp
    X = detfill.uniform("clips", (nclips, T, C, S, S), 0.0, 1.0)

    def cpu_metrics(config, pred, real):
        return torch.from_numpy(M.frame_metrics(pred.numpy(), real.numpy(), C))

    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    frames, m = runner.evaluate_clips(cfg, net, X, preds_per_test=p, num_frames_pred=nfp,
                                      sampler=samplers.ddpm_sampler, sampler_kwargs=dict(subsample_steps=3),
                                      philox_seed=None)
    assert frames.shape == (nclips * p, C * nfp, S, S) and float(frames.min()) >= 0.0 and float(frames.max()) <= 1.0
    assert m["per_frame"].shape == (nclips * p, nfp, 2)
    assert m["mse"].shape == m["psnr"].shape == m["ssim"].shape == (nclips,)
    # best-of-repeats: the product function against the oracle restatement on the same per-frame numbers
    mse, psnr, ssim = M.best_of_repeats(m["per_frame"].numpy(), p)
    assert np.allclose(m["mse"].numpy(), mse) and np.allclose(m["psnr"].numpy(), psnr) and np.allclose(m["ssim"].numpy(), ssim)
    # repeats of one clip share the conditioning frames but are sampled with their own noise: they differ
    assert not torch.equal(frames[0], frames[1])


def test_warm_start_t_min_matches_reference_golden_and_oracle():
    """init_prev_t warm start (t_min > 0), replicated as the reference writes it (models/__init__.py:269-280)."""
    name = "tiny"
    cfg, net, sd = cpu_module(name, "umma")
    B, L = cfg.bench_batch, cfg.sampling.subsample
    x, cond = detfill.synthetic_inputs(cfg, B)
    zs = step_noise(x.shape, L)
    warm = detfill.normal("warm", x.shape)
    out = samplers.ddpm_sampler(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, noise_list=zs, t_min=0.35, warm_noise=warm)
    g = golden(name)
    # the reference's randn_like sequence is [warm, z0, z1, ...] consumed in order, so step i draws zs[k] with k
    # counting only the steps that were not skipped
    sched = O.make_schedule(cfg)
    fn = lambda xx, tt, cc: O.unet_forward(cfg, sd, xx, tt, cc)
    steps = list(range(0, 1000, 1000 // L))
    kept = [i for i, s_ in enumerate(steps) if not (s_ < 0.35 * L)]
    # our sampler indexes noise_list by step index i; build the list the reference's consumption order implies
    aligned = [None] * (L - 1)
    for k, i in enumerate(kept[:-1]):
        aligned[i] = zs[k]
    out = samplers.ddpm_sampler(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, noise_list=aligned, t_min=0.35, warm_noise=warm)
    assert max_err(out[0], torch.from_numpy(g["ddpm_tmin"])) < 2e-3
    ref = O.ddpm_sample(fn, sched, x.clone(), cond, L, True, True, noise=aligned, t_min=0.35, warm_noise=warm)
    assert max_err(out[0], ref[0]) < 2e-3
