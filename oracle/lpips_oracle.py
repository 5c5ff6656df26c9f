"""numpy / fp64 restatement of the reference's per-frame LPIPS (checker of mcvd_b200/lpips.py; nothing in the product
imports it).  TEST INFRASTRUCTURE.

Per frame pair, as runners/ncsn_runner.py:1427-1431, 1590-1609 computes it with
``PerceptualLoss(model='net-lin', net='alex')`` (models/eval_models.py, dist_model.py:60-72, networks_basic.py:25-97,
pretrained_networks.py:56-94):
  1. ``ToPILImage()(x).convert("RGB")``: u8 = trunc(x * 255) in fp32, one channel replicated to RGB;
  2. ``Resize((128, 128))``: Pillow's two-pass 8-bit bilinear resampling (Resample.c), restated below;
  3. ``ToTensor``, ``Normalize(0.5, 0.5)``, ``ScalingLayer`` in fp32 (so the network input is bit-exact);
  4. torchvision ``alexnet().features[0:12]`` in fp64, taps relu1..relu5;
  5. per tap: unit-normalise over channels (eps 1e-10), squared difference, 1x1 ``lin{k}``, spatial mean; summed;
  6. per clip: mean over frames, then the min over the ``preds_per_test`` repeats (:2199).
"""
from __future__ import annotations

import math

import numpy as np
import torch

from mcvd_b200 import detfill

SHIFT = np.array([-.030, -.088, -.188], dtype=np.float32)
SCALE = np.array([.458, .448, .450], dtype=np.float32)
# PNetLin state_dict keys of the backbone convolutions: (key prefix, Cout, Cin, kernel, stride, padding, pool before)
CONVS = [("net.slice1.0", 64, 3, 11, 4, 2, False), ("net.slice2.3", 192, 64, 5, 1, 2, True),
         ("net.slice3.6", 384, 192, 3, 1, 1, True), ("net.slice4.8", 256, 384, 3, 1, 1, False),
         ("net.slice5.10", 256, 256, 3, 1, 1, False)]


def pil_coefficients(in_size: int, out_size: int = 128) -> np.ndarray:
    """Dense int64 [out_size, in_size] matrix of Pillow's 8-bit bilinear coefficients (precompute_coeffs +
    normalize_coeffs_8bpc): triangle filter of half-width max(1, scale), weights of each output normalised to 1 and
    rounded to 22 fractional bits."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    M = np.zeros((out_size, in_size), dtype=np.int64)
    for o in range(out_size):
        c = (o + 0.5) * scale
        lo = max(int(c - fs + 0.5), 0)
        hi = min(int(c + fs + 0.5), in_size)
        w = np.array([max(0.0, 1.0 - abs((x - c + 0.5) * (1.0 / fs))) for x in range(lo, hi)])
        if w.sum() != 0.0:
            w = w / w.sum()
        M[o, lo:hi] = [int(v * (1 << 22) + (0.5 if v >= 0 else -0.5)) for v in w]
    return M


def _clip8(v: np.ndarray) -> np.ndarray:
    return np.where(v >= 1 << 30, 255, np.where(v <= 0, 0, v >> 22)).astype(np.int64)


def pil_resize(u8: np.ndarray, out_size: int = 128) -> np.ndarray:
    """[H, W] (or [H, W, C]) uint8 -> [out, out(, C)] uint8 as ``Image.resize((out, out), BILINEAR)``: a horizontal
    pass, then a vertical pass, each rounded and clipped to 8 bits."""
    if u8.ndim == 3:
        return np.stack([pil_resize(u8[..., c], out_size) for c in range(u8.shape[2])], -1)
    Mx, My = pil_coefficients(u8.shape[1], out_size), pil_coefficients(u8.shape[0], out_size)
    h = _clip8(u8.astype(np.int64) @ Mx.T + (1 << 21))
    return _clip8(My @ h + (1 << 21)).astype(np.uint8)


def network_input(frame: np.ndarray) -> np.ndarray:
    """[C, S, S] float32 frame (C = 1|3) -> the float32 [3, 128, 128] input of the AlexNet (steps 1-3)."""
    x = np.clip(frame.astype(np.float32), np.float32(0), np.float32(1))
    u8 = (x * np.float32(255)).astype(np.uint8)                        # ToPILImage: mul(255).byte()
    if u8.shape[0] == 1:
        u8 = np.repeat(u8, 3, axis=0)                                 # convert("RGB")
    r = pil_resize(u8.transpose(1, 2, 0)).transpose(2, 0, 1)
    v = r.astype(np.float32) / np.float32(255)                         # ToTensor
    v = (v - np.float32(0.5)) / np.float32(0.5)                        # Normalize
    return (v - SHIFT[:, None, None]) / SCALE[:, None, None]           # ScalingLayer


def _conv_relu(x: np.ndarray, w: np.ndarray, b: np.ndarray, stride: int, pad: int) -> np.ndarray:
    C, H, W = x.shape
    k = w.shape[-1]
    xp = np.pad(x, ((0, 0), (pad, pad), (pad, pad)))
    oh, ow = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    s = xp.strides
    cols = np.lib.stride_tricks.as_strided(xp, (C, k, k, oh, ow), (s[0], s[1], s[2], s[1] * stride, s[2] * stride))
    y = np.tensordot(w.reshape(w.shape[0], -1), cols.reshape(C * k * k, oh * ow), axes=1).reshape(-1, oh, ow)
    return np.maximum(y + b[:, None, None], 0.0)


def _maxpool(x: np.ndarray) -> np.ndarray:
    C, H, W = x.shape
    oh, ow = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    return np.max([x[:, dy:dy + 2 * oh - 1:2, dx:dx + 2 * ow - 1:2] for dy in range(3) for dx in range(3)], axis=0)


def taps(x: np.ndarray, sd) -> list:
    """relu1..relu5 of the fp64 AlexNet for one [3, 128, 128] input."""
    out, h = [], x.astype(np.float64)
    for key, _, _, _, stride, pad, pool in CONVS:
        if pool:
            h = _maxpool(h)
        h = _conv_relu(h, sd[key + ".weight"].double().numpy(), sd[key + ".bias"].double().numpy(), stride, pad)
        out.append(h)
    return out


def distance(xa: np.ndarray, xb: np.ndarray, sd) -> float:
    """LPIPS between two network inputs (steps 4-5)."""
    d = 0.0
    for k, (fa, fb) in enumerate(zip(taps(xa, sd), taps(xb, sd))):
        na = fa / (np.sqrt((fa ** 2).sum(0, keepdims=True)) + 1e-10)
        nb = fb / (np.sqrt((fb ** 2).sum(0, keepdims=True)) + 1e-10)
        lin = sd[f"lin{k}.model.1.weight"].double().numpy().reshape(-1, 1, 1)
        d += float((lin * (na - nb) ** 2).sum(0).mean())
    return d


def lpips(pred: np.ndarray, real: np.ndarray, channels: int, sd) -> np.ndarray:
    """float64 [B, F] per-frame LPIPS of [B, channels*F, S, S] frames."""
    B, CF = pred.shape[:2]
    out = np.zeros((B, CF // channels))
    for b in range(B):
        for f in range(CF // channels):
            sl = slice(f * channels, (f + 1) * channels)
            out[b, f] = distance(network_input(pred[b, sl]), network_input(real[b, sl]), sd)
    return out


def clip_lpips(per_frame: np.ndarray, preds_per_test: int) -> np.ndarray:
    """Per test clip: mean over frames, then the best (lowest) of the clip's repeats (step 6)."""
    return per_frame.mean(1).reshape(-1, preds_per_test).min(-1)


def synthetic_weights(seed: int = 1234) -> dict:
    """A PNetLin (net='alex') state_dict from ``detfill.uniform`` keyed by parameter name: conv weights
    U(+-sqrt(3 / fan_in)), biases U(+-0.1), lin weights U(0, 0.1) (non-negative, as trained ones are)."""
    sd = {}
    for key, cout, cin, k, _, _, _ in CONVS:
        a = math.sqrt(3.0 / (cin * k * k))
        sd[key + ".weight"] = detfill.uniform(key + ".weight", (cout, cin, k, k), -a, a, seed)
        sd[key + ".bias"] = detfill.uniform(key + ".bias", (cout,), -0.1, 0.1, seed)
    for k, (_, cout, *_rest) in enumerate(CONVS):
        sd[f"lin{k}.model.1.weight"] = detfill.uniform(f"lin{k}.model.1.weight", (1, cout, 1, 1), 0.0, 0.1, seed)
    return sd


def torchvision_format(sd) -> tuple:
    """(torchvision AlexNet state_dict, LPIPS lin state_dict) holding the same weights as the PNetLin ``sd``."""
    tv = {}
    for key, *_ in CONVS:
        idx = key.split(".")[-1]
        tv[f"features.{idx}.weight"], tv[f"features.{idx}.bias"] = sd[key + ".weight"], sd[key + ".bias"]
    return tv, {k: v for k, v in sd.items() if k.startswith("lin")}


def golden_cases(seed: int = 1234) -> dict:
    """{name: (pred, real, channels)} of the LPIPS fixture: [B, C*F, S, S] float32 in [0, 1] for S in {32, 64, 128},
    C in {1, 3}, binary MovingMNIST-like digits, smooth content, and near-identical pairs (a fifth of the pixels moved by
    three 8-bit levels), so the distances span about 1e-4 to 0.5."""
    def smooth(tag, shape):
        S = shape[-1]
        yy, xx = np.meshgrid(np.arange(S) / S, np.arange(S) / S, indexing="ij")
        ph = detfill.uniform(tag, shape[:-2] + (4,), 0.0, 2 * math.pi, seed).numpy()[..., None, None]
        v = 0.5 + 0.25 * np.sin(3 * xx + ph[..., 0, :, :]) * np.cos(2 * yy + ph[..., 1, :, :]) \
            + 0.2 * np.sin(7 * (xx + yy) + ph[..., 2, :, :]) + 0.05 * np.cos(11 * xx * yy + ph[..., 3, :, :])
        return v.astype(np.float32)

    def digits(tag, shape):
        u = detfill.uniform(tag, shape, 0.0, 1.0, seed).numpy()
        blob = smooth(tag + "_b", shape)
        return ((blob > 0.62) | (u > 0.995)).astype(np.float32)

    def nudge(tag, x):
        u = detfill.uniform(tag, x.shape, 0.0, 1.0, seed).numpy()
        step = np.where(u < 0.1, 3.0 / 255, np.where(u > 0.9, -3.0 / 255, 0.0)).astype(np.float32)
        return np.clip(x + step, 0, 1).astype(np.float32)

    cases = {}
    real = digits("mnist32_r", (2, 3, 32, 32))
    cases["mnist32"] = (np.concatenate([np.roll(real[:1], 1, axis=-1) * 0.98 + 0.01,
                                        detfill.uniform("mnist32_p", real[1:].shape, 0.0, 1.0, seed).numpy()]), real, 1)
    real = smooth("rgb64_r", (1, 6, 64, 64))
    cases["rgb64"] = (smooth("rgb64_p", (1, 6, 64, 64)), real, 3)
    real = smooth("grey128_r", (1, 1, 128, 128))
    cases["grey128"] = (np.clip(real + 0.1 * detfill.normal("grey128_n", real.shape, 1.0, seed).numpy(), 0, 1)
                        .astype(np.float32), real, 1)
    real = smooth("near64_r", (1, 3, 64, 64))
    cases["near64"] = (nudge("near64_n", real), real, 1)
    real = smooth("near128_r", (1, 3, 128, 128))[:, :3]
    cases["near128rgb"] = (nudge("near128_n", real), real, 3)
    return cases
