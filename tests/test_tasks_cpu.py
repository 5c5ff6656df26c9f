"""The three tasks of the reference's video_gen -- interpolation, prediction with a future-frame model and
unconditional generation -- on the CPU: the task table, the conditioning each task samples with, the AR window
with a future block, and the frames of each task against goldens written from the unmodified reference
(tests/golden/tiny_general.npz, tiny_spade_general.npz by oracle/gen_golden_tasks.py), with the lowered program
executed by tests/op_interpreter.py."""
import itertools
import logging
import types

import pytest
import torch

from common import golden, make_module
from mcvd_b200 import configs, runner
from mcvd_b200.program import Engine
from op_interpreter import Interpreter
from oracle import gen_golden_tasks as GT, mcvd_oracle as O, ref_import, tasks_oracle as T

GENERAL = ("tiny_general", "tiny_spade_general")


def general_cfg(condp=0.5, futrf=2, futrp=0.5, sync=False):
    cfg = configs.workload("tiny")
    d = cfg.data
    d.prob_mask_cond, d.num_frames_future, d.prob_mask_future, d.prob_mask_sync = condp, futrf, futrp, sync
    return cfg


@pytest.mark.parametrize("condp,futrf,futrp,sync", list(itertools.product((0.0, 0.5), (0, 2), (0.0, 0.5),
                                                                          (False, True))))
def test_tasks_for_matches_reference_mode_table(condp, futrf, futrp, sync):
    cfg = general_cfg(condp, futrf, futrp, sync)
    assert runner.tasks_for(cfg) == T.tasks_in_order(cfg)
    if ref_import.available():
        R = ref_import.ref_runner()
        me = types.SimpleNamespace(config=cfg)
        cfg.sampling.ssim = True
        R.NCSNRunner.get_mode(me)                    # sets no mode at all where no row matches
        modes = tuple(getattr(me, m, None) for m in ("mode_pred", "mode_interp", "mode_gen"))
        assert modes == T.mode_table(condp, futrf, futrp, sync)


def test_tasks_for_rows():
    assert runner.tasks_for(configs.workload("tiny")) == ["pred"]
    assert runner.tasks_for(general_cfg(0.0, 2, 0.0)) == ["interp"]
    assert runner.tasks_for(general_cfg(0.0, 2, 0.5)) == ["interp", "pred"]
    assert runner.tasks_for(general_cfg(0.5, 0, 0.0)) == ["pred", "gen"]
    assert runner.tasks_for(general_cfg(0.5, 2, 0.5)) == ["interp", "pred", "gen"]
    assert runner.tasks_for(general_cfg(0.5, 2, 0.5, True)) == ["interp", "gen"]
    assert runner.tasks_for(general_cfg(0.5, 2, 0.0)) == []


@pytest.mark.parametrize("name", GENERAL)
def test_task_inputs_match_oracle_split(name):
    cfg = configs.workload(name)
    X = T.golden_clips(cfg)
    for task in runner.tasks_for(cfg):
        real, cond, nfp = runner.task_inputs(cfg, X, task)
        want_nfp, pc, pf = T.task_setup(cfg, task)
        want_real, want_cond = T.conditioning_split(cfg, 2 * X - 1, want_nfp, pc, pf)
        assert nfp == want_nfp
        assert torch.equal(cond, want_cond), task
        assert (real is None) == (task == "gen")
        if real is not None:
            assert torch.equal(real, runner.inverse_data_transform(cfg, want_real))
    # prediction without future frames: the old split, unmasked
    cfg = configs.workload("tiny")
    X = T.golden_clips(cfg)
    real, cond, nfp = runner.task_inputs(cfg, X, "pred")
    r0, c0, _ = runner.conditioning_fn(cfg, runner.data_transform(cfg, X), num_frames_pred=5)
    assert nfp == 5 and torch.equal(cond, c0) and torch.equal(real, runner.inverse_data_transform(cfg, r0))


def recording_sampler(log):
    """Stands in for the sampler: records each block's window and returns frames that differ per block."""
    def sampler(x_T, scorenet, cond=None, **kw):
        out = torch.tanh(x_T + cond.mean(dim=1, keepdim=True) + 0.1 * len(log))
        log.append(dict(cond=cond.clone(), gen=out.clone(), **kw))
        return out.unsqueeze(0)
    return sampler


@pytest.mark.parametrize("name,task", [("tiny_general", "pred"), ("tiny_general", "gen"), ("tiny", "pred"),
                                       ("tiny_rgb", "pred")])
def test_window_keeps_width_and_future_block(name, task):
    cfg = configs.workload(name)
    C, F, Fc, Ff = cfg.data.channels, cfg.data.num_frames, cfg.data.num_frames_cond, cfg.data.num_frames_future
    _, cond, nfp = runner.task_inputs(cfg, T.golden_clips(cfg), task)
    log = []
    runner.video_gen_clips(cfg, torch.nn.Identity(), cond, nfp, sampler=recording_sampler(log),
                           init_fn=lambda i, shape: torch.full(shape, 0.01 * i))
    assert len(log) == -(-nfp // F) >= 3
    for prev, cur in zip(log, log[1:]):
        assert cur["cond"].shape[1] == C * (Fc + Ff)
        assert torch.equal(cur["cond"][:, C * Fc:], cond[:, C * Fc:])                    # future block held
        if Ff == 0:                                                                      # the rule without future frames
            want = torch.cat([prev["cond"][:, C * F:], prev["gen"][:, C * max(0, F - Fc):]], dim=1)
        else:
            want = torch.cat([prev["cond"][:, C * F:-C * Ff], prev["gen"][:, C * max(0, F - Fc):],
                              prev["cond"][:, -C * Ff:]], dim=1)
        assert torch.equal(cur["cond"], want)


def cpu_module(name):
    cfg, net, sd = make_module(name, "cpu")
    net._engine = Engine(net, _test_backend=Interpreter())
    return cfg, net


@pytest.mark.parametrize("name", GENERAL)
def test_task_frames_match_reference_golden(name):
    cfg, net = cpu_module(name)
    X = T.golden_clips(cfg)
    g = golden(name)
    assert sorted(g.files) == sorted(f"video_{t}" for t in runner.tasks_for(cfg))
    for task in runner.tasks_for(cfg):
        _, cond, nfp = runner.task_inputs(cfg, X, task)
        init_fn, noise_fn = GT.task_noise(cfg, task, len(X))
        vid = runner.video_gen_clips(cfg, net, cond, nfp, init_fn=init_fn, noise_fn=noise_fn)
        ref = torch.from_numpy(g[f"video_{task}"])
        assert vid.shape == ref.shape == (len(X), cfg.data.channels * nfp, 32, 32)
        assert O.psnr01(vid, ref) > 50.0, task


def cpu_metrics(config, pred, real):
    from oracle import metrics_oracle as M
    return torch.from_numpy(M.frame_metrics(pred.numpy(), real.numpy(), config.data.channels))


def test_evaluate_clips_masks_no_clip_on_general_model(monkeypatch):
    """A general model (prob_mask_cond 0.5) is evaluated on task (1), interpolation, with every past and future
    frame given, as the reference does (runners/ncsn_runner.py:1458-1459)."""
    cfg = configs.workload("tiny_general")
    C = cfg.data.channels
    X = T.golden_clips(cfg, batch=8)
    _, full = T.conditioning_split(cfg, 2 * X - 1, cfg.data.num_frames)
    torch.manual_seed(3)
    _, _, keep = runner.conditioning_fn(cfg, 2 * X - 1, cfg.data.num_frames, cfg.data.prob_mask_cond)
    assert not bool(keep.all())                    # drawing the training mask would blank some clips
    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    log = []
    torch.manual_seed(3)
    frames, m = runner.evaluate_clips(cfg, torch.nn.Linear(1, 1), X, preds_per_test=1,
                                      sampler=recording_sampler(log))
    assert len(log) == 1 and torch.equal(log[0]["cond"], full)
    assert frames.shape == (8, C * cfg.data.num_frames, 32, 32) and m["psnr"].shape == (8,)


def test_evaluate_tasks_seeds_metrics_and_short_data(monkeypatch, caplog):
    cfg = configs.workload("tiny_general")
    C, F = cfg.data.channels, cfg.data.num_frames
    X = T.golden_clips(cfg, batch=3)
    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    log = []
    out = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, preds_per_test=2, sampler=recording_sampler(log),
                                philox_seed=99, init_seed=7, clip_offset=4)
    assert list(out) == ["interp", "pred", "gen"]
    nfp = {"interp": F, "pred": 5, "gen": 8}
    for task, (frames, m) in out.items():
        assert frames.shape == (6, C * nfp[task], 32, 32)
        if task == "gen":
            assert m is None
        else:
            assert m["per_frame"].shape == (6, nfp[task], 2) and m["mse"].shape == m["psnr"].shape == (3,)
    # one block for interp, 3 for pred, 4 for gen; task (1) keeps the caller's Philox seed, (2) and (3) get their own
    seeds = [e["philox_seed"] for e in log]
    assert seeds[0] == 99 + 7919 and all(e["clip_offset"] == 4 for e in log)
    assert len(set(seeds)) == len(seeds) == 8
    assert [runner.task_seed(99, k) for k in range(3)] == [99, 99 + 2 ** 40, 99 + 2 ** 41]
    # x_T per global clip from the task's init seed: clip 4 of task (1) is what video_gen_sharded would draw
    x0 = runner.clip_init_fn(7, 4, 10, "cpu")(0, (6, C * F, 32, 32))
    first = [e for e in log if e["philox_seed"] == 99 + 7919][0]
    assert torch.equal(first["gen"], torch.tanh(x0 + first["cond"].mean(dim=1, keepdim=True)))
    # predicting past the real frames of X: no metrics, and a warning
    log.clear()
    with caplog.at_level(logging.WARNING):
        out = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, preds_per_test=1, tasks=["pred"],
                                    num_frames_pred=9, sampler=recording_sampler(log))
    assert out["pred"][1] is None and out["pred"][0].shape[1] == C * 9 and "no metrics" in caplog.text


def test_task_misuse_raises():
    cfg = configs.workload("tiny_general")
    X = T.golden_clips(cfg)
    cfg.sampling.one_frame_at_a_time = True
    _, cond, _ = runner.task_inputs(cfg, X, "pred")
    with pytest.raises(ValueError, match="1699-1703"):
        runner.video_gen_clips(cfg, torch.nn.Identity(), cond, 3, sampler=recording_sampler([]))
    with pytest.raises(ValueError, match="num_frames_future"):
        runner.task_inputs(configs.workload("tiny"), X, "interp")
    with pytest.raises(ValueError, match="num_frames_pred=3"):
        runner.task_inputs(cfg, X, "interp", num_frames_pred=3)
    with pytest.raises(ValueError, match="unknown task"):
        runner.task_inputs(cfg, X, "predict")
    with pytest.raises(ValueError, match="too few"):
        runner.task_inputs(cfg, X[:, :6], "interp")
