"""The three tasks of the reference's video_gen on the H100: interpolation, prediction with the future block
zeroed and unconditional generation of a "general" model (past and future frames masked in training), against
goldens written from the unmodified reference (tests/golden/tiny_general.npz, tiny_spade_general.npz).

Tolerance: generated frames PSNR >= 50 dB on [0,1] images, as for the prediction AR loop.  A task changes only
the conditioning window between blocks, so each block runs the same program: the same launches per block for
every task."""
import pytest
import torch

from common import golden, make_module
from mcvd_b200 import runner, samplers
from oracle import gen_golden_tasks as GT, mcvd_oracle as O, tasks_oracle as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("name", ["tiny_general", "tiny_spade_general"])
def test_tasks_vs_reference_golden(name):
    cfg, net, sd = make_module(name, DEV)
    X = T.golden_clips(cfg)
    g = golden(name)
    launches = {}
    for task in runner.tasks_for(cfg):
        _, cond, nfp = runner.task_inputs(cfg, X, task)
        init_fn, noise_fn = GT.task_noise(cfg, task, len(X))
        vid = runner.video_gen_clips(cfg, net, cond.to(DEV), nfp, init_fn=lambda i, sh: init_fn(i).to(DEV),
                                     noise_fn=lambda i: [z.to(DEV) for z in noise_fn(i)])
        launches[task] = samplers.ddpm_sampler.last_launches
        ref = torch.from_numpy(g[f"video_{task}"])
        assert vid.shape == ref.shape and vid.is_cuda
        assert O.psnr01(vid.cpu(), ref) >= 50.0, task
    assert list(launches) == ["interp", "pred", "gen"]
    assert len(set(launches.values())) == 1, launches


@pytest.mark.parametrize("task", ["interp", "pred", "gen"])
def test_task_split_batches_bit_exact(task):
    """Clips [0, k) and [k, B) generated apart, each with its global clip offset, equal one full batch bit for bit:
    what sharding the clips over GPUs relies on."""
    cfg, net, sd = make_module("tiny_general", DEV)
    X = T.golden_clips(cfg, batch=5).to(DEV)
    full = runner.video_gen_sharded(cfg, net, X, 0, 1, philox_seed=99, init_seed=7, task=task)
    k = runner.task_index(cfg, task)
    _, cond, nfp = runner.task_inputs(cfg, X, task)
    parts = [runner.video_gen_clips(cfg, net, cond[lo:hi], nfp, clip_offset=lo,
                                    philox_seed=runner.task_seed(99, k),
                                    init_fn=runner.clip_init_fn(runner.task_seed(7, k), lo, hi, DEV))
             for lo, hi in ((0, 2), (2, 5))]
    assert full.shape == (5, cfg.data.channels * nfp, 32, 32)
    assert torch.equal(torch.cat(parts), full), float((torch.cat(parts) - full).abs().max())


def test_evaluate_tasks_metrics_on_gpu():
    cfg, net, sd = make_module("tiny_spade_general", DEV)
    X = T.golden_clips(cfg, batch=2).to(DEV)
    out = runner.evaluate_tasks(cfg, net, X, preds_per_test=2, philox_seed=5, init_seed=6)
    assert list(out) == ["interp", "pred", "gen"]
    C = cfg.data.channels
    for task, nfp in (("interp", 2), ("pred", 5), ("gen", 8)):
        frames, m = out[task]
        assert frames.shape == (4, C * nfp, 32, 32) and frames.is_cuda
        assert float(frames.min()) >= 0.0 and float(frames.max()) <= 1.0
        if task == "gen":
            assert m is None
            continue
        assert m["per_frame"].shape == (4, nfp, 2) and m["per_frame"].dtype == torch.float64
        assert m["mse"].shape == m["psnr"].shape == m["ssim"].shape == (2,)
        assert bool(torch.isfinite(m["psnr"]).all())
    # evaluate_clips is task (1) of the same run
    frames, m = runner.evaluate_clips(cfg, net, X, preds_per_test=2, philox_seed=5, init_seed=6)
    assert torch.equal(frames, out["interp"][0]) and torch.equal(m["psnr"], out["interp"][1]["psnr"])
