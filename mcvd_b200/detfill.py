"""Deterministic, machine-independent synthetic tensors (weights, inputs, noise).

There is no network for checkpoints or datasets, and the reference's default initialisation
zeroes half of the network (``init_scale=0`` on every ``Conv_1``, attention ``NIN_3`` and the last
conv: reference ``models/better/layers.py:79``, ``layerspp.py:219,586``, ``ncsnpp_more.py:247``),
which would make parity on fresh weights vacuous.  Everything synthetic in this repo therefore
comes from a counter-based integer hash (splitmix64) keyed by a string, so the oracle, the golden
fixtures, the tests and the benchmark regenerate bit-identical arrays anywhere without shipping
hundreds of MB of tensors.
"""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _key(name: str, seed: int) -> np.uint64:
    h = hashlib.sha256(f"{seed}:{name}".encode()).digest()
    return np.uint64(int.from_bytes(h[:8], "little"))


def _splitmix64(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        x = (x + np.uint64(0x9E3779B97F4A7C15)) & _M64
        z = x
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _M64
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _M64
        return z ^ (z >> np.uint64(31))


def _bits(name: str, n: int, seed: int, stream: int = 0) -> np.ndarray:
    k = _key(name, seed)
    with np.errstate(over="ignore"):
        idx = np.arange(n, dtype=np.uint64) * np.uint64(2) + np.uint64(stream)
        return _splitmix64(idx ^ k)


def uniform(name: str, shape, lo: float = -1.0, hi: float = 1.0, seed: int = 1234) -> torch.Tensor:
    """U[lo, hi) float32 tensor; 24 random mantissa bits per element."""
    n = int(np.prod(shape)) if len(shape) else 1
    u = (_bits(name, n, seed) >> np.uint64(40)).astype(np.float64) / float(1 << 24)
    out = (lo + (hi - lo) * u).astype(np.float32).reshape(shape)
    return torch.from_numpy(out)


def normal(name: str, shape, std: float = 1.0, seed: int = 1234) -> torch.Tensor:
    """N(0, std^2) float32 tensor (Box-Muller in float64 on two hash streams)."""
    n = int(np.prod(shape)) if len(shape) else 1
    u1 = ((_bits(name, n, seed, 0) >> np.uint64(11)).astype(np.float64) + 0.5) / float(1 << 53)
    u2 = ((_bits(name, n, seed, 1) >> np.uint64(11)).astype(np.float64) + 0.5) / float(1 << 53)
    z = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * math.pi * u2)
    return torch.from_numpy((std * z).astype(np.float32).reshape(shape))


def randomize_state_dict(sd, seed: int = 1234):
    """Re-randomise every parameter of a (reference-format) ``state_dict`` in place.

    * conv / linear / NIN weights: U(-a, a) with a = sqrt(3 / fan_in)  (unit-variance preserving)
    * biases, NIN ``b``: U(-0.1, 0.1)
    * GroupNorm affine weight: 1 + U(-0.2, 0.2); GroupNorm bias: U(-0.1, 0.1)
    * registered buffers (betas/alphas/alphas_prev/sigmas) are left untouched.
    """
    for k, v in sd.items():
        if not torch.is_floating_point(v):
            continue
        leaf = k.split(".")[-1]
        if leaf in ("betas", "alphas", "alphas_prev", "sigmas", "k", "k_cum", "theta_t"):
            continue
        shape = tuple(v.shape)
        if leaf == "W":                       # NIN: W[in, out]
            a = math.sqrt(3.0 / shape[0])
            new = uniform(k, shape, -a, a, seed)
        elif leaf == "weight" and v.dim() >= 2:   # conv OIHW / linear [out, in]
            fan_in = int(np.prod(shape[1:]))
            a = math.sqrt(3.0 / fan_in)
            new = uniform(k, shape, -a, a, seed)
        elif leaf == "weight":                # GroupNorm affine scale
            new = 1.0 + uniform(k, shape, -0.2, 0.2, seed)
        else:                                 # biases
            new = uniform(k, shape, -0.1, 0.1, seed)
        v.copy_(new.to(v.dtype))
    return sd


def synthetic_inputs(config, batch: int, seed: int = 1234):
    """x_T ~ N(0,1) [B, C*F, S, S] and cond ~ U(-1,1) [B, C*Fc, S, S]."""
    C, F = config.data.channels, config.data.num_frames
    Fc = config.data.num_frames_cond + getattr(config.data, "num_frames_future", 0)
    S = config.data.image_size
    x = normal("x_T", (batch, C * F, S, S), 1.0, seed)
    cond = uniform("cond", (batch, C * Fc, S, S), -1.0, 1.0, seed)
    return x, cond
