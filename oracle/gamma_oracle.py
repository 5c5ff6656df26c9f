"""numpy restatement of the in-kernel Gamma draw of ``MCVD_F_GAMMA`` / ``MCVD_OP_NOISE``.  TEST INFRASTRUCTURE ONLY.

``philox_gamma_centred`` in ``mcvd_b200/csrc/elementwise.cu``, element by element: Philox4x32-10 on uint32 words,
Box-Muller and the Marsaglia-Tsang acceptance test in float64.  For one key (seed, clip, step tag) it returns the
centred draws ``G - k`` (G ~ Gamma(k, 1)) of every element, and for each element the accepted attempt and the
distance of its acceptance test from the threshold, so a test can tell a real disagreement from a rounding tie.
"""
from __future__ import annotations

import numpy as np

GAMMA_TAG = 0x47414D00          # 'GAM\0' | attempt
ATTEMPTS = 16
_M0, _M1, _W0, _W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_INV32 = 2.3283064365386963e-10


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 arrays (broadcast); returns the four output words."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in (c0, c1, c2, c3))
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = np.uint32(k0), np.uint32(k1)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = _M0 * c0.astype(np.uint64)
            p1 = _M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0, k1 = np.uint32(k0 + _W0), np.uint32(k1 + _W1)
    return c0, c1, c2, c3


def seed_words(seed: int):
    """the two 31-bit key words the samplers put in i0 / i1"""
    return seed & 0x7FFFFFFF, (seed >> 31) & 0x7FFFFFFF


def gamma_centred(k: float, seed: int, clip: int, step: int, n: int):
    """(G - k for elements 0..n-1 as float64, accepted attempt per element (-1: bound reached), margin of the accepted
    attempt's test ``rhs - log u``) for shape ``k`` (the fp32 value the kernel receives) and one (seed, clip, step)."""
    k = float(np.float32(k))
    boost = k < 1.0
    kk = k + 1.0 if boost else k
    d = kk - 1.0 / 3.0
    c = 1.0 / np.sqrt(9.0 * d)
    lo, hi = seed_words(seed)
    elem = np.arange(n, dtype=np.uint32)
    w = np.zeros(n)
    ub = np.full(n, 0.5)
    attempt = np.full(n, -1)
    margin = np.full(n, np.inf)
    open_ = np.ones(n, dtype=bool)
    for a in range(ATTEMPTS):
        if not open_.any():
            break
        r0, r1, r2, r3 = philox4x32_10(elem, clip, step, GAMMA_TAG | a, lo, hi)
        u1 = (r0.astype(np.float64) + 1.0) * _INV32
        u2 = (r1.astype(np.float64) + 0.5) * _INV32
        x = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
        cx = c * x
        ub = np.where(open_, (r3.astype(np.float64) + 0.5) * _INV32, ub)
        pos = cx > -1.0
        cxs = np.where(pos, cx, 0.0)
        wc = cxs * (3.0 + cxs * (3.0 + cxs))
        u = (r2.astype(np.float64) + 0.5) * _INV32
        m = 0.5 * x * x + d * (np.log1p(wc) - wc) - np.log(u)
        acc = open_ & pos & (m > 0)
        w = np.where(acc, wc, w)
        attempt = np.where(acc, a, attempt)
        margin = np.where(open_ & pos, np.minimum(margin, np.abs(m)), margin)
        open_ &= ~acc
    if boost:
        g = d * (1.0 + w) * np.exp(np.log(ub) / k) - k
    else:
        g = d * w - 1.0 / 3.0
    return g, attempt, margin
