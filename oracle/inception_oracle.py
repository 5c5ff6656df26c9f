"""torch fp64 restatement of the reference's FID / precision / recall pipeline (checker of mcvd_b200/fid.py; nothing in
the product imports it).  TEST INFRASTRUCTURE.

Per frame, as evaluation/inception.py and evaluation/fid_PR.py compute it with ``InceptionV3([3])``:
  1. ``F.interpolate(size=(299, 299), mode='bilinear', align_corners=False)`` and ``2x - 1``; the resize is restated
     below as two dense interpolation matrices (``i3d_oracle.interp_matrix``); a grey frame is repeated to RGB
     first (the reference itself only takes RGB);
  2. torchvision's Inception3 in eval mode up to Mixed_7c with the FID patches: every BasicConv2d is a conv without
     bias, BatchNorm2d (running statistics, eps 1e-3; not folded here) and ReLU; FIDInceptionA / C / E_1 average
     their branch_pool input with count_include_pad=False, FIDInceptionE_2 max-pools it; the stride-2 max-pools
     have no padding; blocks concatenate their branches in torchvision's order;
  3. the global average pool to [2048];
  4. precision / recall (``calculate_precision_recall_full``) from exact fp64 distances ``sqrt(sum (a - b)^2)``.
"""
from __future__ import annotations

import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as Fn

from mcvd_b200 import detfill
from oracle import i3d_oracle as IO

SIDE = 299
EPS = 1e-3


# ---- the network, written out by block type -------------------------------------------------------------------------
def conv_specs():
    """(key, Cin, Cout, (kh, kw)) of the 94 BasicConv2d in forward order (torchvision's Inception3 __init__ and the
    FID blocks' constructors, evaluation/inception.py:170-196)."""
    out = [("Conv2d_1a_3x3", 3, 32, (3, 3)), ("Conv2d_2a_3x3", 32, 32, (3, 3)), ("Conv2d_2b_3x3", 32, 64, (3, 3)),
           ("Conv2d_3b_1x1", 64, 80, (1, 1)), ("Conv2d_4a_3x3", 80, 192, (3, 3))]
    for key, cin, pf in (("Mixed_5b", 192, 32), ("Mixed_5c", 256, 64), ("Mixed_5d", 288, 64)):
        out += [(f"{key}.branch1x1", cin, 64, (1, 1)), (f"{key}.branch5x5_1", cin, 48, (1, 1)),
                (f"{key}.branch5x5_2", 48, 64, (5, 5)), (f"{key}.branch3x3dbl_1", cin, 64, (1, 1)),
                (f"{key}.branch3x3dbl_2", 64, 96, (3, 3)), (f"{key}.branch3x3dbl_3", 96, 96, (3, 3)),
                (f"{key}.branch_pool", cin, pf, (1, 1))]
    out += [("Mixed_6a.branch3x3", 288, 384, (3, 3)), ("Mixed_6a.branch3x3dbl_1", 288, 64, (1, 1)),
            ("Mixed_6a.branch3x3dbl_2", 64, 96, (3, 3)), ("Mixed_6a.branch3x3dbl_3", 96, 96, (3, 3))]
    for key, c7 in (("Mixed_6b", 128), ("Mixed_6c", 160), ("Mixed_6d", 160), ("Mixed_6e", 192)):
        out += [(f"{key}.branch1x1", 768, 192, (1, 1)), (f"{key}.branch7x7_1", 768, c7, (1, 1)),
                (f"{key}.branch7x7_2", c7, c7, (1, 7)), (f"{key}.branch7x7_3", c7, 192, (7, 1)),
                (f"{key}.branch7x7dbl_1", 768, c7, (1, 1)), (f"{key}.branch7x7dbl_2", c7, c7, (7, 1)),
                (f"{key}.branch7x7dbl_3", c7, c7, (1, 7)), (f"{key}.branch7x7dbl_4", c7, c7, (7, 1)),
                (f"{key}.branch7x7dbl_5", c7, 192, (1, 7)), (f"{key}.branch_pool", 768, 192, (1, 1))]
    out += [("Mixed_7a.branch3x3_1", 768, 192, (1, 1)), ("Mixed_7a.branch3x3_2", 192, 320, (3, 3)),
            ("Mixed_7a.branch7x7x3_1", 768, 192, (1, 1)), ("Mixed_7a.branch7x7x3_2", 192, 192, (1, 7)),
            ("Mixed_7a.branch7x7x3_3", 192, 192, (7, 1)), ("Mixed_7a.branch7x7x3_4", 192, 192, (3, 3))]
    for key, cin in (("Mixed_7b", 1280), ("Mixed_7c", 2048)):
        out += [(f"{key}.branch1x1", cin, 320, (1, 1)), (f"{key}.branch3x3_1", cin, 384, (1, 1)),
                (f"{key}.branch3x3_2a", 384, 384, (1, 3)), (f"{key}.branch3x3_2b", 384, 384, (3, 1)),
                (f"{key}.branch3x3dbl_1", cin, 448, (1, 1)), (f"{key}.branch3x3dbl_2", 448, 384, (3, 3)),
                (f"{key}.branch3x3dbl_3a", 384, 384, (1, 3)), (f"{key}.branch3x3dbl_3b", 384, 384, (3, 1)),
                (f"{key}.branch_pool", cin, 192, (1, 1))]
    return out


def basic(x, sd, key, stride=1, padding=0):
    w = sd[key + ".conv.weight"].double()
    y = Fn.conv2d(x, w, stride=stride, padding=padding)
    g, b = sd[key + ".bn.weight"].double(), sd[key + ".bn.bias"].double()
    m, v = sd[key + ".bn.running_mean"].double(), sd[key + ".bn.running_var"].double()
    sh = (1, -1, 1, 1)
    return torch.relu((y - m.view(sh)) / torch.sqrt(v.view(sh) + EPS) * g.view(sh) + b.view(sh))


def avg3(x):
    return Fn.avg_pool2d(x, 3, 1, 1, count_include_pad=False)


def block_a(x, u, k):
    b1 = u(x, f"{k}.branch1x1")
    b5 = u(u(x, f"{k}.branch5x5_1"), f"{k}.branch5x5_2", padding=2)
    b3 = u(u(u(x, f"{k}.branch3x3dbl_1"), f"{k}.branch3x3dbl_2", padding=1), f"{k}.branch3x3dbl_3", padding=1)
    return torch.cat([b1, b5, b3, u(avg3(x), f"{k}.branch_pool")], 1)


def block_b(x, u, k):
    b3 = u(x, f"{k}.branch3x3", stride=2)
    bd = u(u(u(x, f"{k}.branch3x3dbl_1"), f"{k}.branch3x3dbl_2", padding=1), f"{k}.branch3x3dbl_3", stride=2)
    return torch.cat([b3, bd, Fn.max_pool2d(x, 3, 2)], 1)


def block_c(x, u, k):
    row, col = (0, 3), (3, 0)
    b1 = u(x, f"{k}.branch1x1")
    b7 = u(u(u(x, f"{k}.branch7x7_1"), f"{k}.branch7x7_2", padding=row), f"{k}.branch7x7_3", padding=col)
    bd = u(x, f"{k}.branch7x7dbl_1")
    for i, p in ((2, col), (3, row), (4, col), (5, row)):
        bd = u(bd, f"{k}.branch7x7dbl_{i}", padding=p)
    return torch.cat([b1, b7, bd, u(avg3(x), f"{k}.branch_pool")], 1)


def block_d(x, u, k):
    b3 = u(u(x, f"{k}.branch3x3_1"), f"{k}.branch3x3_2", stride=2)
    b7 = u(x, f"{k}.branch7x7x3_1")
    b7 = u(b7, f"{k}.branch7x7x3_2", padding=(0, 3))
    b7 = u(b7, f"{k}.branch7x7x3_3", padding=(3, 0))
    b7 = u(b7, f"{k}.branch7x7x3_4", stride=2)
    return torch.cat([b3, b7, Fn.max_pool2d(x, 3, 2)], 1)


def block_e(x, u, k, pool):
    b1 = u(x, f"{k}.branch1x1")
    b3 = u(x, f"{k}.branch3x3_1")
    b3 = torch.cat([u(b3, f"{k}.branch3x3_2a", padding=(0, 1)), u(b3, f"{k}.branch3x3_2b", padding=(1, 0))], 1)
    bd = u(u(x, f"{k}.branch3x3dbl_1"), f"{k}.branch3x3dbl_2", padding=1)
    bd = torch.cat([u(bd, f"{k}.branch3x3dbl_3a", padding=(0, 1)), u(bd, f"{k}.branch3x3dbl_3b", padding=(1, 0))], 1)
    bp = avg3(x) if pool == "avg" else Fn.max_pool2d(x, 3, 1, 1)
    return torch.cat([b1, b3, bd, u(bp, f"{k}.branch_pool")], 1)


def network(x, sd, unit=None):
    """fp64 [N, 3, 299, 299] (already 2x - 1) -> [N, 2048] (steps 2-3).  ``unit(x, key, stride, padding)`` replaces
    the BasicConv2d (default: ``basic`` on ``sd``), so a timing baseline can run the same graph on folded weights."""
    u = unit or (lambda x, key, stride=1, padding=0: basic(x, sd, key, stride, padding))
    x = u(x, "Conv2d_1a_3x3", stride=2)
    x = u(x, "Conv2d_2a_3x3")
    x = u(x, "Conv2d_2b_3x3", padding=1)
    x = Fn.max_pool2d(x, 3, 2)
    x = u(x, "Conv2d_3b_1x1")
    x = u(x, "Conv2d_4a_3x3")
    x = Fn.max_pool2d(x, 3, 2)
    for k in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        x = block_a(x, u, k)
    x = block_b(x, u, "Mixed_6a")
    for k in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        x = block_c(x, u, k)
    x = block_d(x, u, "Mixed_7a")
    x = block_e(x, u, "Mixed_7b", "avg")
    x = block_e(x, u, "Mixed_7c", "max")
    return x.mean((2, 3))


def preprocess(frames: torch.Tensor) -> torch.Tensor:
    """[N, C, S, S] in [0, 1] -> fp64 [N, 3, 299, 299] (step 1)."""
    S = frames.shape[-1]
    M = torch.from_numpy(IO.interp_matrix(S, SIDE))
    x = M @ frames.double() @ M.T
    if x.shape[1] == 1:
        x = x.repeat(1, 3, 1, 1)
    return 2 * x - 1


@torch.no_grad()
def features(frames, sd, batch: int = 4) -> np.ndarray:
    """fp64 [N, 2048] pool features of frames [N, C, S, S] in [0, 1] (steps 1-3)."""
    f = torch.as_tensor(frames)
    return torch.cat([network(preprocess(f[lo:lo + batch]), sd) for lo in range(0, len(f), batch)]).numpy()


# ---- step 4 ------------------------------------------------------------------------------------------------------
def distances(a, b) -> np.ndarray:
    """fp64 [Na, Nb] exact Euclidean distances (difference form: a row's distance to itself is 0)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.sqrt(((a[:, None, :] - b[None, :, :]) ** 2).sum(-1))


def precision_recall(real, fake, k: int = 3) -> tuple:
    """``calculate_precision_recall_full`` restated: radii = (k+1)-th smallest distance within a set, itself
    included (``kthvalue(k + 1)``); precision = share of fake rows within some real row's radius, recall the
    converse; the shares rounded to fp32 as the reference's ``.float().mean().item()``."""
    rr, gg, gr = distances(real, real), distances(fake, fake), distances(fake, real)
    nn_r, nn_g = np.sort(rr, 1)[:, k], np.sort(gg, 1)[:, k]
    prec = (gr <= nn_r[None, :]).any(1).mean()
    rec = (gr.T <= nn_g[None, :]).any(1).mean()
    return float(np.float32(prec)), float(np.float32(rec))


def cover_margin(real, fake, k: int = 3) -> float:
    """The smallest |d - radius| / radius over every pair the precision / recall tests compare: how far the
    features are from a decision that fp32 rounding could flip."""
    rr, gg, gr = distances(real, real), distances(fake, fake), distances(fake, real)
    nn_r, nn_g = np.sort(rr, 1)[:, k], np.sort(gg, 1)[:, k]
    return float(min((np.abs(gr - nn_r[None, :]) / nn_r[None, :]).min(),
                     (np.abs(gr.T - nn_g[None, :]) / nn_g[None, :]).min()))


# ---- synthetic weights and frames ---------------------------------------------------------------------------------
def synthetic_weights(seed: int = 1234) -> dict:
    """A torchvision-``Inception3`` state_dict (the FID variant's keys, as ``fid_inception_v3`` loads them strictly)
    from ``detfill.uniform`` keyed by parameter name: conv weights He-scaled, U(+-sqrt(6 / fan_in)), so the second
    moment survives each ReLU; batch norm near the identity (gamma 1 +- 0.1, beta +- 0.05, running mean +- 0.05,
    running variance 1 +- 0.1); ``fc`` (1008 classes, unused by the features) U(+-0.01)."""
    sd = {}
    for key, cin, cout, (kh, kw) in conv_specs():
        a = math.sqrt(6.0 / (cin * kh * kw))
        sd[key + ".conv.weight"] = detfill.uniform(key + ".conv.weight", (cout, cin, kh, kw), -a, a, seed)
        sd[key + ".bn.weight"] = detfill.uniform(key + ".bn.weight", (cout,), 0.9, 1.1, seed)
        sd[key + ".bn.bias"] = detfill.uniform(key + ".bn.bias", (cout,), -0.05, 0.05, seed)
        sd[key + ".bn.running_mean"] = detfill.uniform(key + ".bn.running_mean", (cout,), -0.05, 0.05, seed)
        sd[key + ".bn.running_var"] = detfill.uniform(key + ".bn.running_var", (cout,), 0.9, 1.1, seed)
        sd[key + ".bn.num_batches_tracked"] = torch.tensor(0)
    sd["fc.weight"] = detfill.uniform("fc.weight", (1008, 2048), -0.01, 0.01, seed)
    sd["fc.bias"] = detfill.uniform("fc.bias", (1008,), -0.01, 0.01, seed)
    return sd


def wrapper_state_dict(sd: dict) -> dict:
    """The same weights under the reference wrapper's ``blocks.*`` names (``InceptionV3([3]).state_dict()``)."""
    from mcvd_b200.fid import BLOCK_PREFIX
    out = {}
    for k, v in sd.items():
        top, _, rest = k.partition(".")
        if top in BLOCK_PREFIX:
            out[f"{BLOCK_PREFIX[top]}.{rest}"] = v
    return out


def blob_frames(tag: str, N: int, S: int, C: int, seed: int = 1234) -> np.ndarray:
    """[N, C, S, S] float32 in [0, 1]: two Gaussian blobs over low-amplitude noise per frame."""
    return IO.blob_videos(tag, N, 1, S, C, seed)


def perturbed(tag: str, real: np.ndarray, seed: int = 1234) -> np.ndarray:
    """"Generated" frames: each real frame shifted by a pixel or two with its own noise (FID > 0)."""
    out = real.astype(np.float64).copy()
    for i in range(out.shape[0]):
        out[i] = np.roll(out[i], (i % 3) + 1, axis=-1)
    out += detfill.normal(tag, out.shape, 0.08, seed).numpy()
    return np.clip(out, 0, 1).astype(np.float32)


def golden_cases(seed: int = 1234) -> dict:
    """{name: (real [N, C, S, S], fake [M, C, S, S])} of the FID fixture; ``dup_grey64`` repeats each of its real
    frames twice, so the k-NN radii meet exact ties."""
    cases = {}
    for name, N, S, C in (("grey64", 8, 64, 1), ("rgb64", 8, 64, 3), ("rgb128", 6, 128, 3)):
        real = blob_frames(name, N, S, C, seed)
        cases[name] = (real, perturbed(name + "_fake", real, seed))
    base = blob_frames("dup_grey64", 4, 64, 1, seed)
    cases["dup_grey64"] = (np.repeat(base, 2, axis=0), perturbed("dup_grey64_fake", base, seed))
    return cases


def frechet_cases(seed: int = 1234) -> dict:
    """{name: (mu1, sigma1, mu2, sigma2)} for the Fréchet distance: two full-rank 8-d Gaussians, and a 3-d pair
    whose covariances are zero, for which SciPy's sqrtm of the product is not finite, so the eps retry runs."""
    def gauss(tag, n, d):
        f = detfill.normal(tag, (n, d), 1.0, seed).numpy().astype(np.float64)
        return f.mean(0), np.cov(f, rowvar=False)
    m1, s1 = gauss("fd_a", 40, 8)
    m2, s2 = gauss("fd_b", 40, 8)
    z = np.zeros((3, 3))
    return {"full": (m1, s1, m2, s2), "singular": (m1[:3], z, m2[:3], z.copy())}


def checksum(x: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(x, dtype=np.float32).tobytes()).hexdigest()
