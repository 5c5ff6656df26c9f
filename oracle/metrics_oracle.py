"""CPU restatement of the per-frame quality metrics of the reference's ``video_gen``.  TEST INFRASTRUCTURE ONLY
(checker of MCVD_OP_FRAME_METRICS; nothing in the product imports it).

Follows reference ``runners/ncsn_runner.py:1581-1600`` (MSE via ``F.mse_loss``; SSIM via
``skimage.metrics.structural_similarity(pred_grey, real_grey, data_range=255, gaussian_weights=True,
use_sample_covariance=False)`` on the 8-bit grey images made by ``ToPILImage()(x).convert("RGB").convert("L")``)
and ``:2194-2196`` (best of ``preds_per_test`` repeats).  scikit-image is not a dependency,
so its SSIM is restated from its published algorithm (skimage/metrics/_structural_similarity.py,
v0.19-0.24: Gaussian weights sigma = 1.5, truncate = 3.5 -> 11x11 window, ``scipy.ndimage.gaussian_filter`` with
mode='reflect', K1 = 0.01, K2 = 0.03, population covariances, mean over the image cropped by (win - 1) // 2 = 5);
the grey conversion is checked against PIL itself in tests/test_host_cpu.py.
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import gaussian_filter


def to_grey_u8(frame: np.ndarray, round_first: bool = False) -> np.ndarray:
    """frame [C, H, W] float in [0,1] -> uint8 [H, W] as ToPILImage()(frame).convert('RGB').convert('L') gives.
    torchvision: pic.mul(255).byte() (truncation); PIL rgb2l: (R*19595 + G*38470 + B*7471 + 0x8000) >> 16."""
    f = np.asarray(frame, dtype=np.float32)
    if round_first:                                   # torch.round: half to even (ncsn_runner.py:1598-1599)
        f = np.rint(f)
    b = (f * np.float32(255.0)).astype(np.int64).astype(np.uint8).astype(np.int64)
    if b.shape[0] == 1:
        return b[0].astype(np.uint8)
    return ((b[0] * 19595 + b[1] * 38470 + b[2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def ssim_u8(x: np.ndarray, y: np.ndarray) -> float:
    """structural_similarity(x, y, data_range=255, gaussian_weights=True, use_sample_covariance=False) of two uint8
    grey images."""
    x = x.astype(np.float64)
    y = y.astype(np.float64)
    filt = lambda a: gaussian_filter(a, sigma=1.5, truncate=3.5, mode="reflect")
    ux, uy = filt(x), filt(y)
    uxx, uyy, uxy = filt(x * x), filt(y * y), filt(x * y)
    vx, vy, vxy = uxx - ux * ux, uyy - uy * uy, uxy - ux * uy
    C1, C2 = (0.01 * 255.0) ** 2, (0.03 * 255.0) ** 2
    S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux * ux + uy * uy + C1) * (vx + vy + C2))
    pad = 5
    return float(S[pad:-pad, pad:-pad].mean(dtype=np.float64))


def frame_metrics(pred: np.ndarray, real: np.ndarray, channels: int, round_first: bool = False) -> np.ndarray:
    """pred, real [B, channels*F, H, W] in [0,1] -> float64 [B, F, 2] = (MSE, SSIM) per frame."""
    B, CF, H, W = pred.shape
    F = CF // channels
    out = np.zeros((B, F, 2), dtype=np.float64)
    for b in range(B):
        for f in range(F):
            p = pred[b, f * channels:(f + 1) * channels].astype(np.float64)
            r = real[b, f * channels:(f + 1) * channels].astype(np.float64)
            out[b, f, 0] = ((r - p) ** 2).mean()
            out[b, f, 1] = ssim_u8(to_grey_u8(pred[b, f * channels:(f + 1) * channels], round_first),
                                   to_grey_u8(real[b, f * channels:(f + 1) * channels], round_first))
    return out


def best_of_repeats(per_frame: np.ndarray, preds_per_test: int):
    """per-clip video metrics and the best of every clip's ``preds_per_test`` repeats (ncsn_runner.py:1602-1604,
    2194-2196): vid_mse = mean over frames; mse = min, psnr = max of 10 log10(1 / vid_mse), ssim = max."""
    vid_mse = per_frame[..., 0].mean(1)
    vid_ssim = per_frame[..., 1].mean(1)
    mse = vid_mse.reshape(-1, preds_per_test).min(-1)
    psnr = (10 * np.log10(1 / vid_mse)).reshape(-1, preds_per_test).max(-1)
    ssim = vid_ssim.reshape(-1, preds_per_test).max(-1)
    return mse, psnr, ssim
