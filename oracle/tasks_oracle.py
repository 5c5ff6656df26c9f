"""CPU oracle for the three tasks of the reference's ``video_gen``.  TEST INFRASTRUCTURE ONLY.

A restatement (not a copy) of ``runners/ncsn_runner.py`` @ 451da2e, paths relative to the reference root:
the mode table of ``NCSNRunner.get_mode`` (:208-227), the frame counts and masking probabilities each task
samples with (:1446-1459, :1618-1623, :1795-1799), the conditioning split with future frames
(``conditioning_fn``, :104-147, for masking probabilities of 0 or 1) and the AR block loop whose window keeps
the future block in place (:1537-1539, :1702-1708, :1872-1882).  ``oracle/gen_golden_tasks.py`` drives the
unmodified reference sampler through this loop to write ``tests/golden/tiny_general.npz`` and
``tiny_spade_general.npz``.  The product package ``mcvd_b200`` never imports this module.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch

from mcvd_b200 import detfill

Tensor = torch.Tensor


def mode_table(condp: float, futrf: int, futrp: float, sync: bool) -> Tuple[Optional[str], Optional[str], Optional[str]]:
    """(mode_pred, mode_interp, mode_gen) of ``get_mode`` for a run that computes metrics (:213-227).  The value
    names the task number the mode runs as: "one" = (1), "two" = (2), "three" = (3); None = not run."""
    if condp == 0.0 and futrf == 0:                                         # (1) Prediction
        return "one", None, None
    if condp == 0.0 and futrf > 0 and futrp == 0.0:                        # (1) Interpolation
        return None, "one", None
    if condp == 0.0 and futrf > 0 and futrp > 0.0:                         # (1) Interp + (2) Pred
        return "two", "one", None
    if condp > 0.0 and futrf == 0:                                         # (1) Pred + (3) Gen
        return "one", None, "three"
    if condp > 0.0 and futrf > 0 and futrp > 0.0 and not sync:             # (1) Interp + (2) Pred + (3) Gen
        return "two", "one", "three"
    if condp > 0.0 and futrf > 0 and futrp > 0.0 and sync:                 # (1) Interp + (3) Gen
        return None, "one", "three"
    return None, None, None


def tasks_in_order(config) -> List[str]:
    """The task names of ``mode_table`` for ``config``, ordered by task number."""
    d = config.data
    modes = mode_table(d.prob_mask_cond, d.num_frames_future, d.prob_mask_future, d.prob_mask_sync)
    num = {"one": 1, "two": 2, "three": 3}
    return [t for _, t in sorted((num[m], t) for m, t in zip(modes, ("pred", "interp", "gen")) if m is not None)]


def task_setup(config, task: str) -> Tuple[int, float, float]:
    """(frames to generate, prob_mask_cond, prob_mask_future) the reference samples ``task`` with:
    interpolation ``num_frames`` frames, nothing masked (:1446-1459); prediction ``num_frames_pred`` frames with
    the future block masked when the model has one (:1618-1623); generation ``num_frames_cond + num_frames_pred``
    frames with everything masked (:1795-1799)."""
    if task == "interp":
        return config.data.num_frames, 0.0, 0.0
    if task == "pred":
        return config.sampling.num_frames_pred, 0.0, (1.0 if config.data.num_frames_future > 0 else 0.0)
    if task == "gen":
        return config.data.num_frames_cond + config.sampling.num_frames_pred, 1.0, 1.0
    raise KeyError(task)


def conditioning_split(config, X: Tensor, num_frames_pred: int, prob_mask_cond: float = 0.0,
                       prob_mask_future: float = 0.0):
    """conditioning_fn (:104-147) with future frames, for masking probabilities of 0 (kept) or 1 (zeroed).

    X [B, T, C, S, S]: frames [0, Fc) are the past, [Fc, Fc + nfp) the frames to predict and
    [Fc + F, Fc + F + Ff) the future block, which follows the model's F generated frames.
    """
    assert prob_mask_cond in (0.0, 1.0) and prob_mask_future in (0.0, 1.0)
    B, S = len(X), config.data.image_size
    Fc, F, Ff = config.data.num_frames_cond, config.data.num_frames, config.data.num_frames_future
    pred = X[:, Fc:Fc + num_frames_pred].reshape(B, -1, S, S)
    cond = X[:, :Fc].reshape(B, -1, S, S) * (1.0 - prob_mask_cond)
    if Ff > 0:
        fut = X[:, Fc + F:Fc + F + Ff].reshape(B, -1, S, S) * (1.0 - prob_mask_future)
        cond = torch.cat([cond, fut], dim=1)
    return pred, cond


def golden_clips(config, batch: Optional[int] = None) -> Tensor:
    """The test batch of the task goldens: [B, Fc + max(F + Ff, nfp), C, S, S] ~ U[0, 1), long enough for the
    interpolation's future block and the prediction's real frames."""
    d = config.data
    T = d.num_frames_cond + max(d.num_frames + d.num_frames_future, config.sampling.num_frames_pred)
    B = batch or config.bench_batch
    return detfill.uniform("task_clips", (B, T, d.channels, d.image_size, d.image_size), 0.0, 1.0)


@torch.no_grad()
def video_gen_loop(config, sampler, cond: Tensor, init_noise: List[Tensor], num_frames_pred: int) -> Tensor:
    """AR block loop of ``video_gen`` for every task (:1501-1570, :1684-1720, :1847-1894), block by block.

    ``sampler(x_T, cond, i_iter) -> [1, B, C*F, S, S]``.  After a block the past part of the window slides:
    ``cat(cond[:, C*F : C*Fc], gen[:, C*max(0, F - Fc):])``; a future block of ``C*Ff`` channels stays at the end.
    Returns ``clamp((pred + 1) / 2, 0, 1)`` of the first ``num_frames_pred`` frames.
    """
    C, Fr, Fc = config.data.channels, config.data.num_frames, config.data.num_frames_cond
    Ff = config.data.num_frames_future
    n_iter = math.ceil(num_frames_pred / Fr)
    preds = []
    for i in range(n_iter):
        gen = sampler(init_noise[i], cond, i)[-1]
        gen = gen.reshape(gen.shape[0], C * Fr, config.data.image_size, config.data.image_size)
        preds.append(gen)
        if i == n_iter - 1:
            continue
        past = torch.cat([cond[:, C * Fr:C * Fc], gen[:, C * max(0, Fr - Fc):]], dim=1)
        cond = torch.cat([past, cond[:, C * Fc:C * (Fc + Ff)]], dim=1)
    pred = torch.cat(preds, dim=1)[:, :C * num_frames_pred]
    return torch.clamp((pred + 1.0) / 2.0, 0.0, 1.0)
