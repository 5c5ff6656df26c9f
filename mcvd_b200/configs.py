"""Workload configurations for the MCVD DDPM-sampling hot path.

The reference drives everything from YAML files turned into nested ``argparse.Namespace``
objects (reference ``main.py:359-367`` ``dict2namespace``) and read with
``getattr(config.model, name, default)`` all over the model code.  The GPU box has no copy of
the reference, so the five benchmark workloads are restated here programmatically with the
same field names (values after the ``--config_mod`` overrides the workloads imply).  ``namespace_from_dict`` is the equivalent of ``dict2namespace`` so a
YAML loaded by the caller works as well.
"""
from __future__ import annotations

import argparse
import copy
from typing import Any, Dict


def namespace_from_dict(d: Dict[str, Any]) -> argparse.Namespace:
    """dict -> nested Namespace (same contract as reference ``main.py:359-367``)."""
    ns = argparse.Namespace()
    for k, v in d.items():
        setattr(ns, k, namespace_from_dict(v) if isinstance(v, dict) else v)
    return ns


def namespace_to_dict(ns: argparse.Namespace) -> Dict[str, Any]:
    out = {}
    for k, v in vars(ns).items():
        out[k] = namespace_to_dict(v) if isinstance(v, argparse.Namespace) else v
    return out


_COMMON_SAMPLING = dict(
    batch_size=100, data_init=False, final_only=True, denoise=True, subsample=100,
    consistent=True, step_lr=0.0, n_steps_each=0, num_frames_pred=20, clip_before=True,
    init_prev_t=-1.0, one_frame_at_a_time=False, preds_per_test=1,
)

_COMMON_DATA = dict(
    image_size=64, channels=1, logit_transform=False, uniform_dequantization=False,
    gaussian_dequantization=False, rescaled=True, num_workers=0, num_frames=5, num_frames_cond=5,
    num_frames_future=0, prob_mask_cond=0.0, prob_mask_future=0.0, prob_mask_sync=False,
)

_COMMON_MODEL = dict(
    depth="deep", version="DDPM", gamma=False, arch="unetmore", type="v1", time_conditional=True,
    dropout=0.1, sigma_dist="linear", sigma_begin=0.02, sigma_end=0.0001, num_classes=1000,
    ema=True, ema_rate=0.999, spec_norm=False, normalization="InstanceNorm++",
    nonlinearity="swish", ngf=64, ch_mult=[1, 2, 3, 4], num_res_blocks=2,
    attn_resolutions=[8, 16, 32], n_head_channels=64, conditional=True, noise_in_cond=False,
    output_all_frames=False, cond_emb=False, spade=False, spade_dim=128,
)


def _mk(name, batch, data=None, model=None, sampling=None):
    d = dict(
        data={**_COMMON_DATA, **(data or {})},
        model={**_COMMON_MODEL, **(model or {})},
        sampling={**_COMMON_SAMPLING, **(sampling or {})},
    )
    d = copy.deepcopy(d)
    ns = namespace_from_dict(d)
    ns.workload = name
    ns.bench_batch = batch
    return ns


def workload(name: str) -> argparse.Namespace:
    """Return one of the benchmark workloads (``cfg1`` .. ``cfg7``) or a small test config.

    cfg1  smmnist_DDPM_small5.yml + model.arch=unetmore, subsample=10, B=2
    cfg2  smmnist_DDPM_big5.yml   + ngf=96 n_head_channels=96, subsample=100, B=64   (the headline)
    cfg3  kth64_big_spade.yml     + ngf=128 n_head_channels=128 spade_dim=128, B=32
    cfg4  bair_big.yml            + ngf=192 n_head_channels=192, B=64, num_frames_pred=28
    cfg5  cityscapes_big.yml      + ch_mult=[1,2,3,4,4], subsample=1000, B=32, num_frames_pred=28
    cfg6  ucf101.yml              + ngf=288 n_head_channels=288, subsample=100, B=60, num_frames_pred=16
                                    (ucf10132_big288_4c4_unetm: head dim 288)
    cfg7  cityscapes_big.yml      + spade=True spade_dim=128 ngf=256 n_head_channels=256, subsample=100, B=32,
                                    num_frames_pred=28 (city16_big128_256_5c2_unetm_long_spade: head dim 256; the
                                    recipe samples 45 clips, but the lowered program keeps ~1.7 GiB of activation
                                    buffers per clip, so 45 do not fit in 80 GB)
    """
    if name == "cfg1":
        return _mk(name, 2, data=dict(num_frames=2),
                   model=dict(ngf=32, ch_mult=[1, 2, 2, 2], num_res_blocks=1),
                   sampling=dict(subsample=10))
    if name == "cfg2":
        return _mk(name, 64, model=dict(ngf=96, n_head_channels=96))
    if name == "cfg3":
        return _mk(name, 32, data=dict(num_frames_cond=10),
                   model=dict(depth="deeper", ngf=128, n_head_channels=128, spade=True, spade_dim=128))
    if name == "cfg4":
        return _mk(name, 64, data=dict(channels=3, num_frames_cond=2),
                   model=dict(depth="deeper", ngf=192, n_head_channels=192),
                   sampling=dict(num_frames_pred=28))
    if name == "cfg5":
        return _mk(name, 32, data=dict(image_size=128, channels=3, num_frames_cond=2),
                   model=dict(depth="deeper", dropout=0.0, ngf=128, n_head_channels=128,
                              ch_mult=[1, 2, 3, 4, 4]),
                   sampling=dict(num_frames_pred=28, subsample=1000))
    if name == "cfg6":
        return _mk(name, 60, data=dict(channels=3, num_frames=4, num_frames_cond=4),
                   model=dict(depth="deeper", ngf=288, n_head_channels=288),
                   sampling=dict(num_frames_pred=16))
    if name == "cfg7":
        return _mk(name, 32, data=dict(image_size=128, channels=3, num_frames=5, num_frames_cond=2),
                   model=dict(depth="deeper", dropout=0.0, ngf=256, n_head_channels=256, ch_mult=[1, 1, 2, 3, 4],
                              spade=True, spade_dim=128),
                   sampling=dict(num_frames_pred=28))
    # --- small configurations used by the parity tests (oracle finishes in seconds) ---
    if name == "tiny":      # concat conditioning, every block type, 32x32
        return _mk(name, 2, data=dict(image_size=32, num_frames=2, num_frames_cond=3),
                   model=dict(ngf=32, ch_mult=[1, 2, 2], num_res_blocks=1, n_head_channels=32,
                              attn_resolutions=[8, 16]),
                   sampling=dict(subsample=10, num_frames_pred=5))
    if name == "tiny_spade":
        return _mk(name, 2, data=dict(image_size=32, num_frames=2, num_frames_cond=3),
                   model=dict(ngf=32, ch_mult=[1, 2, 2], num_res_blocks=1, n_head_channels=32,
                              attn_resolutions=[8, 16], spade=True, spade_dim=32),
                   sampling=dict(subsample=10, num_frames_pred=5))
    if name in ("tiny_general", "tiny_spade_general"):
        # a "general" model (past and future masked in training, reference recipes *_pmask50_futurepast):
        # interpolation, prediction with the future block zeroed and unconditional generation
        cfg = workload(name[:-len("_general")])
        cfg.workload = name
        cfg.data.num_frames_future, cfg.data.prob_mask_cond, cfg.data.prob_mask_future = 2, 0.5, 0.5
        return cfg
    if name == "tiny_gamma":  # tiny trained with Gamma noise (model.gamma=True, Nachmani et al. 2021)
        cfg = workload("tiny")
        cfg.workload = name
        cfg.model.gamma = True
        return cfg
    if name == "tiny_rgb":  # 3 channels, 2 res blocks, heads > 1, odd group sizes
        return _mk(name, 3, data=dict(image_size=32, channels=3, num_frames=2, num_frames_cond=2),
                   model=dict(ngf=48, ch_mult=[1, 2, 3], num_res_blocks=2, n_head_channels=48,
                              attn_resolutions=[8, 16]),
                   sampling=dict(subsample=20, num_frames_pred=5))
    if name == "tiny128":   # 128-px, 5 levels (cityscapes-like topology): wide slabs, 3 slab rows per producer thread
        return _mk(name, 2, data=dict(image_size=128, channels=3, num_frames=2, num_frames_cond=2),
                   model=dict(ngf=32, ch_mult=[1, 1, 2, 2, 4], num_res_blocks=1, n_head_channels=32,
                              attn_resolutions=[8, 16, 32]),
                   sampling=dict(subsample=5, num_frames_pred=4))
    raise KeyError(f"unknown workload {name!r}")


ALL_WORKLOADS = ("cfg1", "cfg2", "cfg3", "cfg4", "cfg5", "cfg6", "cfg7")
TEST_WORKLOADS = ("tiny", "tiny_spade", "tiny_rgb", "tiny128", "tiny_general", "tiny_spade_general", "tiny_gamma")
