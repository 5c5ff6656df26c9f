"""Denoising score-matching (DSM) test loss with the reference's signature.

Drop-in for ``anneal_dsm_score_estimation`` of the reference ``losses/dsm.py``, which ``NCSNRunner.test``
(``main.py --test``, runners/ncsn_runner.py:2370-2430) uses to score every checkpoint of a sweep.  The perturbation
``x_t = sqrt(a) x + sqrt(1 - a) z`` and the per-clip loss run as two CUDA ops around the lowered network
(``Engine.dsm``); the network evaluates every clip at its own level.

The noise is drawn in-kernel from a Philox stream keyed by (seed, global clip, element) under one step tag,
``DSM_STEP``, whatever the label.  With the same ``philox_seed`` every checkpoint of a sweep, and every noise level,
therefore sees the same perturbations, so the comparison between checkpoints is a paired one.  Gamma-noise models
(``gamma=True``) draw the centred Gamma noise ``(G - k theta) / sqrt(1 - a)`` in-kernel without the cancellation of
the reference's fp32 difference.
"""
from __future__ import annotations

import torch

from . import samplers
from .model import UNetMore_DDPM

# Philox step tag of the DSM noise: distinct from the sampler's per-step tags (< number of levels) and from
# samplers.GAMMA_WARM_STEP / GAMMA_INIT_STEP (+ small offsets)
DSM_STEP = 1 << 28


@torch.no_grad()
def anneal_dsm_score_estimation(scorenet, x, labels=None, loss_type="a", hook=None, cond=None, cond_mask=None,
                                gamma=False, L1=False, all_frames=False, *, philox_seed=None, clip_offset=0,
                                noise=None):
    """Reference ``anneal_dsm_score_estimation`` (losses/dsm.py) for ``mcvd_b200.UNetMore_DDPM`` networks.

    ``x`` [B, C*F, S, S] are the clean, data-transformed frames.  ``labels=None`` draws
    ``torch.randint(0, len(alphas), (B,))`` on ``x.device`` as the reference does.  Returns the fp32 batch mean on
    ``x.device`` and calls ``hook(per_clip_loss_fp32, labels)``; the per-clip sums are accumulated in fp64.
    ``loss_type`` is accepted and unused, as in the reference.

    ``cond_mask`` is accepted and ignored: only ``cond_emb`` networks read it, and those are not native.
    ``all_frames=True`` raises ``NotImplementedError``: native networks have no ``output_all_frames``.

    Keyword-only extensions: ``noise`` injects ``z`` (the reference's standardised noise, for parity tests); otherwise
    z is the in-kernel draw of clip ``clip_offset + b`` from ``philox_seed``, drawn from torch's default generator
    when None (so ``torch.manual_seed`` reproduces a run).
    """
    if all_frames:
        raise NotImplementedError("mcvd_b200 networks do not output all frames (model.output_all_frames); "
                                  "use the reference anneal_dsm_score_estimation")
    net = scorenet.module if hasattr(scorenet, "module") else scorenet
    if not isinstance(net, UNetMore_DDPM):
        raise TypeError("mcvd_b200.dsm drives mcvd_b200.UNetMore_DDPM modules "
                        f"(got {type(net).__name__}); use the reference losses.dsm for reference modules")
    if labels is None:
        labels = torch.randint(0, len(net.alphas), (x.shape[0],), device=x.device)
    philox = None
    if noise is None:
        if philox_seed is None:
            philox_seed = samplers.draw_seed()
        philox = (philox_seed, clip_offset, DSM_STEP)
    loss = net.engine().dsm(x, labels, cond, z=noise, philox=philox, gamma=gamma, l1=L1).to(x.device)
    if hook is not None:
        hook(loss.float(), labels)
    return loss.mean(dim=0).float()
