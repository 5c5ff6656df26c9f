"""Sampling slice of the reference runner: conditioning, the autoregressive block loop, clip sharding.

Restates (does not copy) ``runners/ncsn_runner.py``: ``conditioning_fn`` (:104-147), the AR loop of
``NCSNRunner.video_gen`` (:1501-1570), its three tasks -- prediction or interpolation, prediction with a
future-frame model, unconditional generation -- chosen by the mode table of ``get_mode`` (:208-227), and
``get_sampler`` (:2702-2714); the dataset, gif and checkpoint-sweep code around them is out of scope.  The
per-clip metrics (MSE, PSNR, SSIM, and LPIPS with ``mcvd_b200.lpips``) and FVD's I3D features (with
``mcvd_b200.fvd``) of each task are computed on the GPU by ``evaluate_tasks``.

Multi-GPU: the reference wraps the network in ``torch.nn.DataParallel`` (:1377) and re-broadcasts all
weights on every one of the 101 x n_iter network calls.  Here every clip (batch element) is
independent through the whole AR x diffusion loop, so rank r owns clips [r*B/G, (r+1)*B/G), runs with
its own weight copy and ZERO communication, and the ranks meet in exactly one NCCL all-gather of the
finished frames (``gather_clips``).
"""
from __future__ import annotations

import logging
import math
from typing import Callable, Dict, List, Optional, Tuple

import torch

from . import samplers
from .samplers import get_sampler


def data_transform(config, X):
    """x -> 2x - 1 for ``rescaled`` data (reference datasets/__init__.py:235-249, sampling-relevant part)."""
    if getattr(config.data, "rescaled", True):
        return 2 * X - 1.0
    return X


def inverse_data_transform(config, X):
    """clamp((x + 1) / 2, 0, 1) (reference datasets/__init__.py:252-261)."""
    if getattr(config.data, "rescaled", True):
        X = (X + 1.0) / 2.0
    return torch.clamp(X, 0.0, 1.0)


def conditioning_fn(config, X, num_frames_pred=0, prob_mask_cond=0.0, prob_mask_future=0.0, conditional=True):
    """Split ``X [B, T, C, S, S]`` into (frames to predict, conditioning frames, cond_mask).

    Same contract as reference ``runners/ncsn_runner.py:104-147`` including the Bernoulli masking of
    past / future frames used by the paper's "general" models.
    """
    S = config.data.image_size
    if not conditional:
        return X.reshape(len(X), -1, S, S), None, None
    n_cond = config.data.num_frames_cond
    n_train = config.data.num_frames
    n_future = getattr(config.data, "num_frames_future", 0)
    pred_frames = X[:, n_cond:n_cond + num_frames_pred].reshape(len(X), -1, S, S)
    cond_frames = X[:, :n_cond].reshape(len(X), -1, S, S)
    cond_mask = None
    if prob_mask_cond > 0.0:
        keep = torch.rand(X.shape[0], device=X.device) > prob_mask_cond
        cond_frames = keep.reshape(-1, 1, 1, 1) * cond_frames
        cond_mask = keep.to(torch.int32)
    if n_future > 0:
        if prob_mask_future == 1.0:
            fut = torch.zeros(len(X), config.data.channels * n_future, S, S)
        else:
            fut = X[:, n_cond + n_train:n_cond + n_train + n_future].reshape(len(X), -1, S, S)
            if prob_mask_future > 0.0:
                if getattr(config.data, "prob_mask_sync", False):
                    fmask = cond_mask
                else:
                    fmask = torch.rand(X.shape[0], device=X.device) > prob_mask_future
                fut = fmask.reshape(-1, 1, 1, 1) * fut
        cond_frames = torch.cat([cond_frames, fut.to(cond_frames.device)], dim=1)
    return pred_frames, cond_frames, cond_mask


def shard_range(n_clips: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous clip range owned by ``rank`` (first ranks take the remainder)."""
    base, rem = divmod(n_clips, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


@torch.no_grad()
def video_gen_clips(config, scorenet, cond: torch.Tensor, num_frames_pred: Optional[int] = None,
                    init_fn: Optional[Callable[[int, Tuple[int, ...]], torch.Tensor]] = None,
                    sampler=None, sampler_kwargs=None, clip_offset: int = 0, philox_seed: Optional[int] = None,
                    noise_fn: Optional[Callable[[int], List[torch.Tensor]]] = None) -> torch.Tensor:
    """Autoregressive block generation for the clips in ``cond`` (reference runner:1501-1570).

    Each iteration samples ``num_frames`` frames, appends them, slides the conditioning window
    ``cond <- cat(cond[:, C*F:], gen[:, C*max(0, F - Fc):])`` (:1537-1539) and draws a fresh init.  With
    ``num_frames_future = Ff > 0`` the last ``C*Ff`` channels of ``cond`` (the future block) stay where they are
    and only the past part slides, ``cat(cond[:, C*F:-C*Ff], gen[:, C*max(0, F - Fc):], cond[:, -C*Ff:])``
    (:1702-1708, :1872-1882), so the window keeps its width ``C*(Fc + Ff)``.
    Returns ``inverse_data_transform(pred)[:, :C*num_frames_pred]`` on the input device.
    ``init_fn(i, shape)`` supplies x_T of AR iteration i (default ``torch.randn``, :1476/:1551; for a Gamma-noise
    model ``Gamma(k_cum[0], scale theta_t[0]) - k_cum[0] theta_t[0]``, :1471-1474/:1546-1549, drawn on the GPU with
    one torch-drawn seed per call, keyed by global clip and AR iteration);
    ``noise_fn(i)`` optionally supplies the per-step noise list (parity tests).
    """
    C, F, Fc = config.data.channels, config.data.num_frames, config.data.num_frames_cond
    S = config.data.image_size
    nfp = num_frames_pred if num_frames_pred is not None else config.sampling.num_frames_pred
    one_at_a_time = getattr(config.sampling, "one_frame_at_a_time", False)
    if one_at_a_time and getattr(config.data, "num_frames_future", 0) > 0:
        raise ValueError("one_frame_at_a_time with num_frames_future > 0 is not supported: the reference's window "
                         "grows by C*num_frames_future channels per block there (runners/ncsn_runner.py:1699-1703)")
    past = C * Fc                                        # channels of the window that slide; the rest is the future block
    n_iter = nfp if one_at_a_time else math.ceil(nfp / F)
    sampler = sampler or get_sampler(config)
    kw = dict(final_only=True, denoise=config.sampling.denoise,
              subsample_steps=getattr(config.sampling, "subsample", None),
              clip_before=getattr(config.sampling, "clip_before", True), verbose=False, log=False,
              t_min=getattr(config.sampling, "init_prev_t", -1), gamma=getattr(config.model, "gamma", False))
    kw.update(sampler_kwargs or {})
    B = cond.shape[0]
    shape = (B, C * F, S, S)
    preds = []
    warm = (getattr(config.sampling, "init_prev_t", -1) or -1) > 0
    if init_fn is None and getattr(config.model, "gamma", False):
        init_fn = clip_init_fn(samplers.draw_seed(), clip_offset, clip_offset + B, cond.device,
                               gamma=gamma_init_params(config, scorenet))
    gen = None
    for i in range(n_iter):
        if warm and i > 0:
            x_T = gen                                    # init_prev_t > 0: restart from the previous block (:1513)
        else:
            x_T = init_fn(i, shape) if init_fn is not None else torch.randn(shape, device=cond.device)
        extra = {}
        if noise_fn is not None:
            extra["noise_list"] = noise_fn(i)
        elif philox_seed is not None:
            # one Philox stream per (clip, AR iteration, step): fold the AR iteration into the seed
            extra.update(philox_seed=philox_seed + 7919 * (i + 1), clip_offset=clip_offset)
        gen = sampler(x_T.to(cond.device), scorenet, cond=cond, **kw, **extra)[-1].reshape(shape)
        preds.append(gen)
        if i == n_iter - 1:
            continue
        if one_at_a_time:
            cond = torch.cat([cond[:, C:], gen[:, :C]], dim=1)
        else:
            cond = torch.cat([cond[:, C * F:past], gen[:, C * max(0, F - Fc):], cond[:, past:]], dim=1)
    pred = torch.cat(preds, dim=1)[:, :C * nfp]
    return inverse_data_transform(config, pred)


def gather_clips(local: torch.Tensor, n_clips: int, rank: int, world: int, group=None) -> torch.Tensor:
    """The one collective of the path: all-gather every rank's finished frames (NCCL over NVLink).

    Shards may differ by one clip, so each rank pads to the largest shard, all-gathers into one flat
    buffer and the padding is dropped on reassembly.
    """
    import torch.distributed as dist
    if world == 1:
        return local
    sizes = [shard_range(n_clips, r, world) for r in range(world)]
    mx = max(hi - lo for lo, hi in sizes)
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
    pad[:local.shape[0]] = local
    out = torch.empty((world * mx,) + tuple(local.shape[1:]), device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(out, pad.contiguous(), group=group)
    parts = [out[r * mx:r * mx + (hi - lo)] for r, (lo, hi) in enumerate(sizes)]
    return torch.cat(parts, dim=0)


# ---------------------------------------------------------------------------------------------------------------
# the reference's video_gen tasks
# ---------------------------------------------------------------------------------------------------------------
TASKS = ("interp", "pred", "gen")


def tasks_for(config) -> List[str]:
    """Tasks ``video_gen`` evaluates a model on, in the reference's order (1), (2), (3).

    The mode table of ``NCSNRunner.get_mode`` (runners/ncsn_runner.py:208-227) for runs that compute metrics.
    (1) is prediction for a model without future frames and interpolation for one with them; (2) is prediction
    with the future block zeroed; (3) is unconditional generation.  A model trained without past masking but
    with future frames it never masks does interpolation only; one that masks both gets all three, or (1) and
    (3) when the masks are drawn together (``prob_mask_sync``).  A model that masks the past but never its
    future frames has no row in the table: no tasks.
    """
    condp = getattr(config.data, "prob_mask_cond", 0.0)
    futrf = getattr(config.data, "num_frames_future", 0)
    futrp = getattr(config.data, "prob_mask_future", 0.0)
    if condp == 0.0:
        if futrf == 0:
            return ["pred"]
        return ["interp"] if futrp == 0.0 else ["interp", "pred"]
    if futrf == 0:
        return ["pred", "gen"]
    if futrp == 0.0:
        return []
    return ["interp", "gen"] if getattr(config.data, "prob_mask_sync", False) else ["interp", "pred", "gen"]


def task_index(config, task: str) -> int:
    """0, 1 or 2 for the reference's task (1), (2) or (3): interpolation, and prediction without future frames,
    are (1); prediction with them is (2); generation is (3)."""
    if task == "interp":
        return 0
    if task == "pred":
        return 1 if getattr(config.data, "num_frames_future", 0) > 0 else 0
    if task == "gen":
        return 2
    raise ValueError(f"unknown task {task!r}; expected one of {TASKS}")


def task_seed(seed: Optional[int], index: int) -> Optional[int]:
    """The seed task ``index`` runs with, derived from the caller's.  Task (1) keeps it, so prediction runs
    exactly as before tasks existed; (2) and (3) move 2**40 apart, far beyond the ``7919 * n_iter`` the AR
    loop adds to a Philox seed and the ``1009 * clip`` a per-clip x_T seed adds, so no two tasks share a noise
    stream."""
    return seed if seed is None or index == 0 else seed + (index << 40)


def task_inputs(config, X: torch.Tensor, task: str, num_frames_pred: Optional[int] = None):
    """(real frames, conditioning, frames to generate) of one task for the test batch ``X`` [B, T, C, S, S] in [0, 1].

    ``conditioning_fn`` runs with the masking probabilities the reference evaluates the task with
    (runners/ncsn_runner.py:1458-1459, 1622-1623, 1798-1799):
      * ``interp``: past and future frames given, ``(0, 0)``.  It fills the ``num_frames`` frames between
        them, so ``num_frames_pred`` may not exceed ``num_frames``.  Needs ``num_frames_future > 0``.
      * ``pred``: ``(0, 0)``; with future frames ``(0, 1)``, the future block zeroed.
        ``num_frames_pred`` defaults to ``sampling.num_frames_pred``.
      * ``gen``: ``(1, 1)``, all conditioning zeroed.  Generates ``num_frames_cond + num_frames_pred`` frames
        and has no real frames (``None``).
    Real frames are in [0, 1] (``inverse_data_transform``); the conditioning is in the model's range.
    """
    C, F, Fc = config.data.channels, config.data.num_frames, config.data.num_frames_cond
    Ff = getattr(config.data, "num_frames_future", 0)
    nfp = num_frames_pred if num_frames_pred is not None else config.sampling.num_frames_pred
    if task == "interp":
        if Ff == 0:
            raise ValueError("task 'interp' needs a model with data.num_frames_future > 0")
        nfp = num_frames_pred if num_frames_pred is not None else F
        if nfp > F:
            raise ValueError(f"task 'interp' fills the {F} frames between past and future; "
                             f"num_frames_pred={nfp} is more")
        probs = (0.0, 0.0)
    elif task == "pred":
        probs = (0.0, 1.0 if Ff > 0 else 0.0)
    elif task == "gen":
        nfp = Fc + nfp
        probs = (1.0, 1.0)
    else:
        raise ValueError(f"unknown task {task!r}; expected one of {TASKS}")
    real, cond, _ = conditioning_fn(config, data_transform(config, X), num_frames_pred=nfp,
                                    prob_mask_cond=probs[0], prob_mask_future=probs[1])
    if cond.shape[1] != C * (Fc + Ff):
        raise ValueError(f"X has {X.shape[1]} frames, too few for the {Fc} past + {F} generated + {Ff} future "
                         "frames of the conditioning window")
    return (None if task == "gen" else inverse_data_transform(config, real)), cond, nfp


def gamma_init_params(config, scorenet) -> Optional[Tuple[float, float]]:
    """(k_cum[0], theta_t[0]) of a Gamma-noise model, whose x_T is Gamma(k_cum[0], scale theta_t[0]) - k_cum[0] theta_t[0]
    (runners/ncsn_runner.py:1471-1474); None for a model with normal noise."""
    if not getattr(config.model, "gamma", False):
        return None
    net = scorenet.module if hasattr(scorenet, "module") else scorenet
    return float(net.k_cum[0]), float(net.theta_t[0])


def clip_init_fn(init_seed: int, lo: int, hi: int, dev,
                 gamma: Optional[Tuple[float, float]] = None) -> Callable[[int, Tuple[int, ...]], torch.Tensor]:
    """``init_fn`` for ``video_gen_clips`` over the global clips [lo, hi): one CPU generator per clip and AR
    iteration, so clip g of AR iteration i sees the same x_T in any batch and on any GPU.

    ``gamma = (k, theta)`` (``gamma_init_params``): x_T is the centred Gamma draw ``G - k theta``, G ~ Gamma(k, scale
    theta), made on the GPU by ``MCVD_OP_NOISE`` from the Philox stream keyed by (init_seed, global clip, AR
    iteration): the same per-clip guarantee without a host tensor."""
    if gamma is not None:
        def gamma_fn(i, shape):
            return samplers.gamma_noise((hi - lo,) + tuple(shape[1:]), gamma[0], gamma[1], init_seed, clip0=lo,
                                        step=samplers.GAMMA_INIT_STEP + i, device=dev)
        return gamma_fn

    def init_fn(i, shape):
        outs = []
        for g in range(lo, hi):
            gen = torch.Generator(device="cpu")
            gen.manual_seed(init_seed * 1000003 + g * 1009 + i)
            outs.append(torch.randn(shape[1:], generator=gen))
        return torch.stack(outs).to(dev) if outs else torch.empty((0,) + tuple(shape[1:]), device=dev)
    return init_fn


@torch.no_grad()
def video_gen_sharded(config, scorenet, cond_all: torch.Tensor, rank: int, world: int, philox_seed: int = 1234,
                      init_seed: int = 1234, task: Optional[str] = None, **kw) -> torch.Tensor:
    """Clip-sharded ``video_gen``: this rank generates its clips, then one all-gather.

    Initial noise and per-step noise are keyed by the GLOBAL clip index so the result is independent of
    the sharding (world size 1 == world size G, bit for bit).

    With a ``task`` ("interp", "pred" or "gen"), ``cond_all`` is the test batch ``X`` [B, T, C, S, S] in [0, 1]
    instead: each rank builds the task's conditioning for its clips (``task_inputs``; ``num_frames_pred`` in
    ``kw`` is passed on to it) and runs with the task's seeds (``task_seed``), so the guarantee holds per task.
    """
    n = cond_all.shape[0]
    lo, hi = shard_range(n, rank, world)
    dev = cond_all.device if cond_all.is_cuda else torch.device("cuda", torch.cuda.current_device())
    if task is None:
        cond = cond_all[lo:hi].to(dev)
    else:
        _, cond, kw["num_frames_pred"] = task_inputs(config, cond_all[lo:hi], task, kw.get("num_frames_pred"))
        cond = cond.to(dev)
        k = task_index(config, task)
        philox_seed, init_seed = task_seed(philox_seed, k), task_seed(init_seed, k)
    init_fn = clip_init_fn(init_seed, lo, hi, dev, gamma=gamma_init_params(config, scorenet))
    local = video_gen_clips(config, scorenet, cond, init_fn=init_fn, clip_offset=lo, philox_seed=philox_seed, **kw)
    return gather_clips(local, n, rank, world)


# ---------------------------------------------------------------------------------------------------------------
# evaluation of generated clips on the GPU
# ---------------------------------------------------------------------------------------------------------------
def frame_metrics(config, pred: torch.Tensor, real: torch.Tensor) -> torch.Tensor:
    """Per-frame MSE and SSIM of generated clips, on the GPU: float64 [B, frames, 2].

    Replaces the reference's per-frame CPU loop over PIL images (runners/ncsn_runner.py:1581-1600).  ``pred`` and
    ``real`` are [B, C*frames, S, S] in [0, 1] (``inverse_data_transform`` output).  MovingMNIST-style datasets get the
    reference's rounding before the grey conversion (:1596-1599)."""
    from . import lib
    C, S = config.data.channels, config.data.image_size
    B, CF = pred.shape[0], pred.shape[1]
    dev = pred.device
    if dev.type != "cuda":
        raise RuntimeError("mcvd_b200.runner.frame_metrics runs on CUDA tensors only (no CPU fallback)")
    p = pred.contiguous().float()
    r = real.to(dev).contiguous().float()
    out = torch.empty(B, CF // C, 2, dtype=torch.float64, device=dev)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i0 = lib.OP_FRAME_METRICS, B, S, S, C, CF // C
    name = str(getattr(config.data, "dataset", "")).upper()
    op.flags = lib.F_ROUND if name in ("STOCHASTICMOVINGMNIST", "MOVINGMNIST") else 0
    op.src0, op.src1, op.dst = p.data_ptr(), r.data_ptr(), out.data_ptr()
    with torch.cuda.device(dev):
        lib.run_program(lib.make_ops([op]), 1, torch.cuda.current_stream(dev).cuda_stream)
    return out


def best_of_repeats(per_frame: torch.Tensor, preds_per_test: int):
    """(mse, psnr, ssim) per test clip: video metric = mean over frames, then the best of the clip's
    ``preds_per_test`` samples (reference runners/ncsn_runner.py:1602-1604, 2194-2196)."""
    vid_mse = per_frame[..., 0].mean(1)
    vid_ssim = per_frame[..., 1].mean(1)
    mse = vid_mse.reshape(-1, preds_per_test).min(-1).values
    psnr = (10 * torch.log10(1 / vid_mse)).reshape(-1, preds_per_test).max(-1).values
    ssim = vid_ssim.reshape(-1, preds_per_test).max(-1).values
    return mse, psnr, ssim


@torch.no_grad()
def evaluate_tasks(config, scorenet, X: torch.Tensor, preds_per_test: Optional[int] = None,
                   tasks: Optional[List[str]] = None, num_frames_pred: Optional[int] = None,
                   lpips: Optional[Callable] = None, i3d: Optional[Callable] = None,
                   **gen_kw) -> Dict[str, Tuple[torch.Tensor, Optional[dict]]]:
    """One test batch of the reference's ``video_gen`` (runners/ncsn_runner.py:1392-1395, 1444-1915), every task.

    ``X`` is [B, T, C, S, S] in [0, 1].  Every test clip is repeated ``preds_per_test`` times (``repeat_interleave``,
    the reference's collate function), and each repeat is sampled with its own noise.  ``tasks`` defaults to
    ``tasks_for(config)``; ``num_frames_pred`` applies to ``pred`` and ``gen`` (``interp`` always fills
    ``num_frames``).  Returns ``{task: (frames [B*p, C*nfp, S, S] in [0, 1], metrics)}``.  ``metrics`` holds
    per-clip ``mse`` / ``psnr`` / ``ssim`` of the best repeat and the ``per_frame`` values, or is ``None`` for
    ``gen``, which has no ground truth, and for a task that predicts past the real frames of ``X`` (:1573-1579).
    With an ``lpips`` (a ``mcvd_b200.lpips.LPIPS``), ``metrics`` also holds ``per_frame_lpips`` [B*p, nfp] and per-clip
    ``lpips``: the mean over frames of the best (lowest) repeat (:1606-1609, 2199).

    With an ``i3d`` (a ``mcvd_b200.fvd.I3D``), every task whose video has at least 10 frames (``fvd_videos``: the
    reference's gate, :1311-1332) and whose real frames cover the prediction also gets ``i3d_fake`` [B*p, 400] and
    ``i3d_real`` [B, 400] float64 features and the ``fvd_summary`` keys ``fvd``, ``fvd_traj_mean``, ``fvd_traj_std``
    and ``fvd_traj_conf95`` of this batch (:1918-1982, 2217-2229).  ``gen`` then gets a dict of only those keys,
    scored against the real videos of task (2) when the model runs it and of task (1) otherwise (:1975-1977).  The
    reference computes FVD over its whole test set: concatenate the features of every batch and call
    ``fvd.fvd_summary`` once.

    ``gen_kw`` go to ``video_gen_clips``.  A ``philox_seed`` among them is replaced by the task's
    (``task_seed``).  An ``init_seed`` draws x_T per global clip (``clip_init_fn``, clips numbered from
    ``clip_offset``) from the task's seed.  ``init_fn`` and ``noise_fn`` reach every task unchanged.
    """
    p = preds_per_test if preds_per_test is not None else getattr(config.sampling, "preds_per_test", 1)
    X = X.repeat_interleave(p, dim=0)
    dev = next(scorenet.parameters()).device
    init_seed = gen_kw.pop("init_seed", None)
    out = {}
    C = config.data.channels
    for task in (tasks_for(config) if tasks is None else tasks):
        real, cond, nfp = task_inputs(config, X, task, None if task == "interp" else num_frames_pred)
        k = task_index(config, task)
        kw = dict(gen_kw)
        if kw.get("philox_seed") is not None:
            kw["philox_seed"] = task_seed(kw["philox_seed"], k)
        if init_seed is not None:
            lo = kw.get("clip_offset", 0)
            kw["init_fn"] = clip_init_fn(task_seed(init_seed, k), lo, lo + X.shape[0], dev,
                                         gamma=gamma_init_params(config, scorenet))
        frames = video_gen_clips(config, scorenet, cond.to(dev), nfp, **kw)
        metrics = None
        if real is not None and real.shape[1] < frames.shape[1]:
            logging.warning("evaluate_tasks: task %r generates %d frames but X holds only %d after the conditioning "
                            "frames; no metrics", task, nfp, real.shape[1] // config.data.channels)
        elif real is not None:
            per_frame = frame_metrics(config, frames, real.to(dev))
            mse, psnr, ssim = best_of_repeats(per_frame, p)
            metrics = {"mse": mse, "psnr": psnr, "ssim": ssim, "per_frame": per_frame}
            if lpips is not None:
                per_frame_lpips = lpips(frames, real.to(dev), config.data.channels)
                metrics["lpips"] = per_frame_lpips.mean(1).reshape(-1, p).min(-1).values
                metrics["per_frame_lpips"] = per_frame_lpips
            if i3d is not None:
                fake_v, real_v = fvd_videos(config, task, cond, frames, real)
                if fake_v.shape[1] // C >= FVD_MIN_FRAMES:
                    metrics.update(_fvd_metrics(i3d, fake_v, real_v[::p], C, p))
        if task == "gen" and i3d is not None and frames.shape[1] // C >= FVD_MIN_FRAMES:
            future = getattr(config.data, "num_frames_future", 0) > 0
            src = "pred" if future and "pred" in tasks_for(config) else ("interp" if future else "pred")
            real_s, cond_s, nfp_s = task_inputs(config, X, src, None if src == "interp" else num_frames_pred)
            if real_s.shape[1] < C * nfp_s:
                logging.warning("evaluate_tasks: X is too short for the real videos of task %r; no FVD for 'gen'", src)
            else:
                _, real_v = fvd_videos(config, src, cond_s, real_s, real_s)
                if real_v.shape[1] // C < MIN_I3D_FRAMES:
                    logging.warning("evaluate_tasks: the real videos of task %r have %d frames, too few for I3D; no "
                                    "FVD for 'gen'", src, real_v.shape[1] // C)
                else:
                    metrics = _fvd_metrics(i3d, frames, real_v[::p], C, p)
        out[task] = (frames, metrics)
    return out


FVD_MIN_FRAMES = 10          # video_gen scores a task's FVD only when its videos have at least 10 frames
MIN_I3D_FRAMES = 9           # InceptionI3d's shortest input


def fvd_videos(config, task: str, cond: torch.Tensor, frames: torch.Tensor, real: torch.Tensor):
    """(fake, real) videos [N, C*L, S, S] in [0, 1] the reference scores with I3D for ``task``
    (runners/ncsn_runner.py:1925-1972): the past conditioning frames, then the generated (or real) frames, then for
    interpolation the future frames.  ``cond`` is the task's conditioning in the model's range (``task_inputs``);
    for ``gen`` the fake video is ``frames`` alone (:1980)."""
    if task == "gen":
        return frames, None
    C, Fc = config.data.channels, config.data.num_frames_cond
    c01 = inverse_data_transform(config, cond).to(frames.device)
    past, future = c01[:, :C * Fc], (c01[:, C * Fc:] if task == "interp" else c01[:, :0])
    return (torch.cat([past, frames, future], dim=1),
            torch.cat([past, real.to(frames.device), future], dim=1))


def _fvd_metrics(i3d, fake: torch.Tensor, real: torch.Tensor, channels: int, p: int) -> dict:
    from .fvd import fvd_summary
    f, r = i3d(fake, channels), i3d(real, channels)
    return dict(i3d_fake=f, i3d_real=r, **fvd_summary(f, r, p))


@torch.no_grad()
def evaluate_clips(config, scorenet, X: torch.Tensor, preds_per_test: Optional[int] = None,
                   num_frames_pred: Optional[int] = None, lpips: Optional[Callable] = None,
                   i3d: Optional[Callable] = None, **gen_kw):
    """Task (1) of ``evaluate_tasks``: prediction, or interpolation for a model with future frames, with no
    conditioning masked (runners/ncsn_runner.py:1458-1459).  ``X`` is [B, T, C, S, S] in [0, 1].  Returns
    (frames [B*p, C*nfp, S, S] in [0, 1], dict of per-clip mse / psnr / ssim tensors and ``per_frame``, plus
    ``lpips`` and ``per_frame_lpips`` with an ``lpips``, and the FVD keys with an ``i3d``)."""
    task = "interp" if getattr(config.data, "num_frames_future", 0) > 0 else "pred"
    return evaluate_tasks(config, scorenet, X, preds_per_test, tasks=[task], num_frames_pred=num_frames_pred,
                          lpips=lpips, i3d=i3d, **gen_kw)[task]


# ---------------------------------------------------------------------------------------------------------------
# the reference's test loss (main.py --test)
# ---------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def test_loss(config, scorenet, X: torch.Tensor, labels: Optional[torch.Tensor] = None,
              philox_seed: Optional[int] = None, clip_offset: int = 0) -> Dict[str, torch.Tensor]:
    """Denoising score-matching loss of one test batch, as ``NCSNRunner.test`` scores it (runners/ncsn_runner.py:
    2402-2418): ``data_transform``, then ``conditioning_fn`` with the training masks ``data.prob_mask_cond`` /
    ``data.prob_mask_future`` (drawn from torch's generator, as the reference does), then the loss with ``model.gamma``
    and ``training.L1`` from the config (``mcvd_b200.dsm``).

    ``X`` is [B, T, C, S, S] in [0, 1].  ``labels`` default to ``randint(0, num levels)``; the noise of global clip
    ``clip_offset + b`` is drawn from ``philox_seed`` (from torch's default generator when None), so with fixed labels
    and seed a batch split into shards gives the same bits per clip.  Returns ``{"loss": per-clip float64 [B],
    "labels": [B], "mean": float64 scalar}``; the reference logs ``mean``."""
    from . import dsm
    from .model import UNetMore_DDPM
    net = scorenet.module if hasattr(scorenet, "module") else scorenet
    if not isinstance(net, UNetMore_DDPM):
        raise TypeError(f"mcvd_b200.runner.test_loss drives mcvd_b200.UNetMore_DDPM modules (got {type(net).__name__})")
    dev = next(net.parameters()).device
    X = data_transform(config, X.to(dev))
    x, cond, _ = conditioning_fn(config, X, num_frames_pred=config.data.num_frames,
                                 prob_mask_cond=getattr(config.data, "prob_mask_cond", 0.0),
                                 prob_mask_future=getattr(config.data, "prob_mask_future", 0.0),
                                 conditional=config.data.num_frames_cond > 0)
    if labels is None:
        labels = torch.randint(0, len(net.alphas), (x.shape[0],), device=dev)
    if philox_seed is None:
        philox_seed = samplers.draw_seed()
    l1 = getattr(getattr(config, "training", None), "L1", False)
    loss = net.engine().dsm(x, labels, cond, philox=(philox_seed, clip_offset, dsm.DSM_STEP),
                            gamma=getattr(config.model, "gamma", False), l1=l1)
    return {"loss": loss, "labels": labels, "mean": loss.mean()}


def loss_per_level(loss: torch.Tensor, labels: torch.Tensor, num_classes: int) -> torch.Tensor:
    """Mean loss per noise level, float64 [num_classes], NaN where no clip has that level: the breakdown of the
    reference's ``test_hook`` (runners/ncsn_runner.py:317-320), with one scatter of (loss, 1) pairs."""
    pairs = torch.stack([loss.double(), torch.ones_like(loss, dtype=torch.float64)], dim=1)
    acc = torch.zeros(num_classes, 2, dtype=torch.float64, device=loss.device)
    acc.index_add_(0, labels.to(loss.device).long(), pairs)
    return acc[:, 0] / acc[:, 1]
