"""torch fp64 restatement of the reference's FVD pipeline (checker of mcvd_b200/fvd.py; nothing in the product
imports it).  TEST INFRASTRUCTURE.

Per video, as runners/ncsn_runner.py:1918-1982 and models/fvd/fvd.py:41-49, 160-186, 275-287 compute it:
  1. ``to_i3d``: [C*T, S, S] frame-major -> [3, T, S, S], a grey frame repeated to RGB;
  2. ``preprocess_single``: bilinear resize (align_corners=False) so the shorter side is 224, centre crop,
     ``(x - 0.5) * 2``; the resize is restated below as two dense interpolation matrices;
  3. ``InceptionI3d`` (models/fvd/pytorch_i3d.py) in eval mode: every Unit3D pads TF-"SAME" from its input size
     (front = pad // 2), convolves, applies BatchNorm3d (running statistics, eps 1e-5; not folded here) and ReLU;
     pools pad with zeros; Inception blocks concatenate [b0, b1, b2, b3]; the head is AvgPool3d([2, 7, 7], 1),
     the 1x1x1 logits conv with bias and the mean over time;
  4. Fréchet distance of the feature sets, here via the eigenvalues of sigma_fake @ sigma_real (whose square roots
     sum to the trace of its square root) rather than scipy's ``sqrtm``.
"""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as Fn

from mcvd_b200 import detfill

SIDE = 224
EPS = 1e-5
# (key, Cin, Cout, kernel, stride) of the stem; Inception blocks (key, Cin, [b0, b1a, b1b, b2a, b2b, b3b])
STEM = [("Conv3d_1a_7x7", 3, 64, 7, 2), ("Conv3d_2b_1x1", 64, 64, 1, 1), ("Conv3d_2c_3x3", 64, 192, 3, 1)]
MIXED = [("Mixed_3b", 192, [64, 96, 128, 16, 32, 32]), ("Mixed_3c", 256, [128, 128, 192, 32, 96, 64]),
         ("Mixed_4b", 480, [192, 96, 208, 16, 48, 64]), ("Mixed_4c", 512, [160, 112, 224, 24, 64, 64]),
         ("Mixed_4d", 512, [128, 128, 256, 24, 64, 64]), ("Mixed_4e", 512, [112, 144, 288, 32, 64, 64]),
         ("Mixed_4f", 528, [256, 160, 320, 32, 128, 128]), ("Mixed_5b", 832, [256, 160, 320, 32, 128, 128]),
         ("Mixed_5c", 832, [384, 192, 384, 48, 128, 128])]


def units():
    """(key, Cin, Cout, kernel) of the 57 Unit3D with batch norm."""
    out = [(k, ci, co, ks) for k, ci, co, ks, _ in STEM]
    for key, cin, o in MIXED:
        out += [(f"{key}.b0", cin, o[0], 1), (f"{key}.b1a", cin, o[1], 1), (f"{key}.b1b", o[1], o[2], 3),
                (f"{key}.b2a", cin, o[3], 1), (f"{key}.b2b", o[3], o[4], 3), (f"{key}.b3b", cin, o[5], 1)]
    return out


# ---- step 2 ------------------------------------------------------------------------------------------------------
def interp_matrix(n_in: int, n_out: int) -> np.ndarray:
    """fp64 [n_out, n_in]: bilinear weights of ``F.interpolate(align_corners=False)`` along one axis
    (source = (dst + 0.5) * n_in / n_out - 0.5, clamped at 0; the right neighbour clamped at the edge)."""
    M = np.zeros((n_out, n_in))
    scale = n_in / n_out
    for o in range(n_out):
        src = max((o + 0.5) * scale - 0.5, 0.0)
        i0 = int(math.floor(src))
        i1 = min(i0 + 1, n_in - 1)
        l1 = src - i0
        M[o, i0] += 1.0 - l1
        M[o, i1] += l1
    return M


def preprocess(video: torch.Tensor) -> torch.Tensor:
    """[3, T, S, S] in [0, 1] -> fp64 [3, T, 224, 224] (step 2)."""
    S = video.shape[-1]
    Ht = math.ceil(S * (SIDE / S))                  # the shorter-side rule of preprocess_single for a square frame
    My = torch.from_numpy(interp_matrix(S, Ht))
    Mx = torch.from_numpy(interp_matrix(S, SIDE))
    x = My @ video.double() @ Mx.T
    h0 = (Ht - SIDE) // 2
    return (x[:, :, h0:h0 + SIDE] - 0.5) * 2


def to_i3d(videos: torch.Tensor, channels: int) -> torch.Tensor:
    """[B, C*T, S, S] -> [B, 3, T, S, S] (step 1)."""
    B, CT, S, _ = videos.shape
    x = videos.reshape(B, CT // channels, channels, S, S)
    if channels == 1:
        x = x.repeat(1, 1, 3, 1, 1)
    return x.permute(0, 2, 1, 3, 4)


# ---- step 3 ------------------------------------------------------------------------------------------------------
def same_pad(x: torch.Tensor, k, s) -> torch.Tensor:
    """TF-"SAME" padding of the last three axes with zeros: total max(k - (n % s or s), 0), front half."""
    pads = []
    for n, kk, ss in reversed(list(zip(x.shape[-3:], k, s))):
        p = max(kk - (ss if n % ss == 0 else n % ss), 0)
        pads += [p // 2, p - p // 2]
    return Fn.pad(x, pads)


def unit(x: torch.Tensor, sd, key: str, k: int, s: int = 1, bn: bool = True) -> torch.Tensor:
    w = sd[key + ".conv3d.weight"].double()
    y = Fn.conv3d(same_pad(x, (k,) * 3, (s,) * 3), w, stride=s)
    g, b = sd[key + ".bn.weight"].double(), sd[key + ".bn.bias"].double()
    m, v = sd[key + ".bn.running_mean"].double(), sd[key + ".bn.running_var"].double()
    sh = (1, -1, 1, 1, 1)
    return torch.relu((y - m.view(sh)) / torch.sqrt(v.view(sh) + EPS) * g.view(sh) + b.view(sh))


def max_pool(x: torch.Tensor, k, s) -> torch.Tensor:
    return Fn.max_pool3d(same_pad(x, k, s), k, s)


def mixed(x: torch.Tensor, sd, key: str) -> torch.Tensor:
    b0 = unit(x, sd, f"{key}.b0", 1)
    b1 = unit(unit(x, sd, f"{key}.b1a", 1), sd, f"{key}.b1b", 3)
    b2 = unit(unit(x, sd, f"{key}.b2a", 1), sd, f"{key}.b2b", 3)
    b3 = unit(max_pool(x, (3, 3, 3), (1, 1, 1)), sd, f"{key}.b3b", 1)
    return torch.cat([b0, b1, b2, b3], 1)


def network(x: torch.Tensor, sd) -> torch.Tensor:
    """fp64 [N, 3, T, 224, 224] -> [N, 400]."""
    x = unit(x, sd, "Conv3d_1a_7x7", 7, 2)
    x = max_pool(x, (1, 3, 3), (1, 2, 2))
    x = unit(x, sd, "Conv3d_2b_1x1", 1)
    x = unit(x, sd, "Conv3d_2c_3x3", 3)
    x = max_pool(x, (1, 3, 3), (1, 2, 2))
    for key, _, _ in MIXED:
        x = mixed(x, sd, key)
        if key == "Mixed_3c":
            x = max_pool(x, (3, 3, 3), (2, 2, 2))
        elif key == "Mixed_4f":
            x = max_pool(x, (2, 2, 2), (2, 2, 2))
    x = Fn.avg_pool3d(x, (2, 7, 7), 1)
    x = Fn.conv3d(x, sd["logits.conv3d.weight"].double(), sd["logits.conv3d.bias"].double())
    return x.squeeze(3).squeeze(3).mean(2)


@torch.no_grad()
def features(videos, channels: int, sd, batch: int = 2) -> np.ndarray:
    """fp64 [B, 400] I3D features of [B, channels*T, S, S] videos in [0, 1] (steps 1-3)."""
    v = to_i3d(torch.as_tensor(videos), channels)
    out = []
    for lo in range(0, v.shape[0], batch):
        x = torch.stack([preprocess(video) for video in v[lo:lo + batch]])
        out.append(network(x, sd))
    return torch.cat(out).numpy()


# ---- step 4 ------------------------------------------------------------------------------------------------------
def frechet_distance(fake: np.ndarray, real: np.ndarray) -> float:
    f, r = np.asarray(fake, np.float64), np.asarray(real, np.float64)
    df, dr = f - f.mean(0), r - r.mean(0)
    sf, sr = df.T @ df / (len(f) - 1), dr.T @ dr / (len(r) - 1)
    ev = np.linalg.eigvals(sf @ sr)
    tr_sqrt = np.sqrt(ev.astype(np.complex128)).real.sum()
    return float(((f.mean(0) - r.mean(0)) ** 2).sum() + np.trace(sf) + np.trace(sr) - 2 * tr_sqrt)


# ---- synthetic weights and videos ---------------------------------------------------------------------------------
def synthetic_weights(seed: int = 1234) -> dict:
    """An ``InceptionI3d`` state_dict from ``detfill.uniform`` keyed by parameter name: conv weights He-scaled,
    U(+-sqrt(6 / fan_in)), so the second moment survives each ReLU; batch norm near the identity (gamma 1 +- 0.1,
    beta +- 0.05, running mean +- 0.05, running variance 1 +- 0.1); logits U(+-sqrt(3 / 1024)), bias U(+-0.1)."""
    sd = {}
    for key, cin, cout, k in units():
        a = math.sqrt(6.0 / (cin * k ** 3))
        sd[key + ".conv3d.weight"] = detfill.uniform(key + ".conv3d.weight", (cout, cin, k, k, k), -a, a, seed)
        sd[key + ".bn.weight"] = detfill.uniform(key + ".bn.weight", (cout,), 0.9, 1.1, seed)
        sd[key + ".bn.bias"] = detfill.uniform(key + ".bn.bias", (cout,), -0.05, 0.05, seed)
        sd[key + ".bn.running_mean"] = detfill.uniform(key + ".bn.running_mean", (cout,), -0.05, 0.05, seed)
        sd[key + ".bn.running_var"] = detfill.uniform(key + ".bn.running_var", (cout,), 0.9, 1.1, seed)
        sd[key + ".bn.num_batches_tracked"] = torch.tensor(0)
    a = math.sqrt(3.0 / 1024)
    sd["logits.conv3d.weight"] = detfill.uniform("logits.conv3d.weight", (400, 1024, 1, 1, 1), -a, a, seed)
    sd["logits.conv3d.bias"] = detfill.uniform("logits.conv3d.bias", (400,), -0.1, 0.1, seed)
    return sd


def blob_videos(tag: str, B: int, T: int, S: int, C: int, seed: int = 1234) -> np.ndarray:
    """[B, C*T, S, S] float32 in [0, 1]: two Gaussian blobs moving in straight lines over low-amplitude noise."""
    u = detfill.uniform(tag + "_traj", (B, 2, 5), 0.0, 1.0, seed).numpy().astype(np.float64)
    noise = detfill.uniform(tag + "_noise", (B, T, C, S, S), 0.0, 0.25, seed).numpy()
    tint = detfill.uniform(tag + "_tint", (B, 2, C), 0.5, 1.0, seed).numpy()
    yy, xx = np.meshgrid(np.arange(S) / S, np.arange(S) / S, indexing="ij")
    out = noise.astype(np.float64)
    for t in range(T):
        for j in range(2):
            y = u[:, j, 0] + (u[:, j, 2] - 0.5) * 0.04 * t
            x = u[:, j, 1] + (u[:, j, 3] - 0.5) * 0.04 * t
            r = 0.06 + 0.08 * u[:, j, 4]
            g = np.exp(-((yy - y[:, None, None]) ** 2 + (xx - x[:, None, None]) ** 2) / (2 * r[:, None, None] ** 2))
            out[:, t] += g[:, None] * tint[:, j, :, None, None]
    return np.clip(out, 0, 1).astype(np.float32).reshape(B, T * C, S, S)


def perturbed(tag: str, real: np.ndarray, p: int, seed: int = 1234) -> np.ndarray:
    """[B*p, ...] "generated" videos: each real video repeated p times (repeat_interleave), each repeat shifted by
    a pixel or two and given its own noise, so fake and real feature sets differ (FVD > 0)."""
    out = np.repeat(real, p, axis=0).astype(np.float64)
    for i in range(out.shape[0]):
        out[i] = np.roll(out[i], (i % 3) + 1, axis=-1)
    out += detfill.normal(tag, out.shape, 0.08, seed).numpy()
    return np.clip(out, 0, 1).astype(np.float32)


def golden_cases(seed: int = 1234) -> dict:
    """{name: (real [B, C*T, S, S], fake [B*p, C*T, S, S], channels, p)} of the FVD fixture."""
    cases = {}
    for name, B, T, S, C, p in (("grey32_t10", 3, 10, 32, 1, 1), ("rgb64_t11", 3, 11, 64, 3, 1),
                                ("grey64_t25_p2", 3, 25, 64, 1, 2)):
        real = blob_videos(name, B, T, S, C, seed)
        cases[name] = (real, perturbed(name + "_fake", real, p, seed), C, p)
    return cases


def checksum(x: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes()).hexdigest()
