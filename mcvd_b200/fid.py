"""FID, precision and recall of generated frames, with Inception-v3 pool features and the k-NN tests on the GPU.

MCVD scores checkpoints with FID and k-NN precision / recall (reference ``main.py --fast_fid``,
runners/ncsn_runner.py:2432-2586, and ``--sample`` with ``sampling.fid``, :1190-1290) through evaluation/fid_PR.py:
the 2048-d pool features of the FID Inception-v3 (evaluation/inception.py ``InceptionV3([3])``: bilinear resize to
299x299, ``2x - 1``, torchvision's Inception3 up to ``Mixed_7c`` with the four FID-patched blocks, global average
pool), the Fréchet distance of Gaussians fitted to the feature sets, and precision / recall as the share of each
set that falls inside the k-NN balls (k = 3) of the other.

``InceptionV3`` computes the features for whole chunks of frames with the library's own kernels
(``MCVD_OP_FID_PREP``, ``MCVD_OP_CONV2D``, ``MCVD_OP_MAXPOOL2D``, ``MCVD_OP_FID_HEAD``): ``LAUNCHES_PER_CHUNK``
launches per chunk, whatever its size; a frame's features do not depend on the batch or chunk it is computed in.
``InceptionV3(..., tf32=True)`` runs the convolutions on the TF32 tensor cores instead (``MCVD_OP_CONV2D_TF32``):
both operands rounded once to TF32, fp32 accumulation, the numerics class of cuDNN with ``allow_tf32``.  The drop-ins
use it when the environment sets ``MCVD_EVAL_TF32=1``; by default they keep the fp32 path.
Grey frames are accepted (replicated to RGB); the reference raises on them.  ``precision_recall`` runs
``MCVD_OP_KNN_RADIUS`` and ``MCVD_OP_KNN_COVER`` (four launches) and never forms the N x N distance matrix the
reference moves to the host; its distances are exact differences, so a point's distance to itself is 0.

Weights are never downloaded.  ``InceptionV3`` takes either the torchvision-``Inception3`` state_dict of
``pt_inception-2015-12-05-6726825d.pth`` (``Conv2d_1a_3x3.conv.weight``, ``Conv2d_1a_3x3.bn.*``,
``Mixed_5b.branch1x1.conv.weight``, ...; ``fc.*`` is ignored) or the ``blocks.*`` state_dict of the reference's
``InceptionV3`` wrapper, as a dict of tensors or a path for ``torch.load``.  The drop-ins ``get_fid``,
``get_fid_PR`` and ``get_PR`` read the weights file from the torch hub cache, where the reference's
``load_state_dict_from_url`` stores it, and raise ``FileNotFoundError`` when it is not there.
"""
from __future__ import annotations

import functools
import os
from typing import List, Optional, Union

import numpy as np
import torch

from . import eval_weights as EW

SIDE = 299                         # InceptionV3.forward resizes to 299x299 (evaluation/inception.py:146-150)
DIMS = 2048
BN_EPS = 1e-3                      # torchvision BasicConv2d: BatchNorm2d(eps=0.001)
WEIGHTS_FILE = "pt_inception-2015-12-05-6726825d.pth"     # evaluation/inception.py:13 FID_WEIGHTS_URL
WORKSPACE_BUDGET = 2 << 30         # bytes of fp32 workspace the default chunk stays under

# The FID Inception-v3 up to Mixed_7c (evaluation/inception.py:83-128, 170-196 and torchvision's Inception3), in
# forward order:
#   ("conv", key, Cin, Cout, (kh, kw), stride, (ph, pw))    BasicConv2d
#   ("pool",)                                               nn.MaxPool2d(3, stride=2)
#   ("A", key, Cin, pool_features)                          FIDInceptionA (avg pool, count_include_pad=False)
#   ("B", key, Cin)                                         torchvision InceptionB (Mixed_6a)
#   ("C", key, Cin, channels_7x7)                           FIDInceptionC
#   ("D", key, Cin)                                         torchvision InceptionD (Mixed_7a)
#   ("E", key, Cin, "avg" | "max")                          FIDInceptionE_1 / FIDInceptionE_2 (branch_pool's pool)
ARCH = [
    ("conv", "Conv2d_1a_3x3", 3, 32, (3, 3), 2, (0, 0)),
    ("conv", "Conv2d_2a_3x3", 32, 32, (3, 3), 1, (0, 0)),
    ("conv", "Conv2d_2b_3x3", 32, 64, (3, 3), 1, (1, 1)),
    ("pool",),
    ("conv", "Conv2d_3b_1x1", 64, 80, (1, 1), 1, (0, 0)),
    ("conv", "Conv2d_4a_3x3", 80, 192, (3, 3), 1, (0, 0)),
    ("pool",),
    ("A", "Mixed_5b", 192, 32),
    ("A", "Mixed_5c", 256, 64),
    ("A", "Mixed_5d", 288, 64),
    ("B", "Mixed_6a", 288),
    ("C", "Mixed_6b", 768, 128),
    ("C", "Mixed_6c", 768, 160),
    ("C", "Mixed_6d", 768, 160),
    ("C", "Mixed_6e", 768, 192),
    ("D", "Mixed_7a", 768),
    ("E", "Mixed_7b", 1280, "avg"),
    ("E", "Mixed_7c", 2048, "max"),
]

# the reference wrapper's module list (evaluation/inception.py:83-124): torchvision name -> ``blocks.*`` prefix
BLOCK_PREFIX = {"Conv2d_1a_3x3": "blocks.0.0", "Conv2d_2a_3x3": "blocks.0.1", "Conv2d_2b_3x3": "blocks.0.2",
                "Conv2d_3b_1x1": "blocks.1.0", "Conv2d_4a_3x3": "blocks.1.1",
                **{k: f"blocks.2.{i}" for i, k in enumerate(["Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b",
                                                              "Mixed_6c", "Mixed_6d", "Mixed_6e"])},
                "Mixed_7a": "blocks.3.0", "Mixed_7b": "blocks.3.1", "Mixed_7c": "blocks.3.2"}


def _block(layer) -> tuple:
    """(output width, [branch op]) of one Inception block.  A branch op is ("conv", name, Cin, Cout, (kh, kw),
    stride, (ph, pw), src, dst, off, pool) or ("pool", src, dst, off) for the stride-2 max-pool branch; src / dst
    are "x" (block input), "t1", "t2" (temporaries) or "out" (the concat, written at channel offset off)."""
    kind, key, cin = layer[:3]
    one, s1 = (1, 1), (0, 0)
    if kind == "A":
        pf = layer[3]
        return 224 + pf, [
            ("conv", "branch1x1", cin, 64, one, 1, s1, "x", "out", 0, None),
            ("conv", "branch5x5_1", cin, 48, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch5x5_2", 48, 64, (5, 5), 1, (2, 2), "t1", "out", 64, None),
            ("conv", "branch3x3dbl_1", cin, 64, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch3x3dbl_2", 64, 96, (3, 3), 1, (1, 1), "t1", "t2", 0, None),
            ("conv", "branch3x3dbl_3", 96, 96, (3, 3), 1, (1, 1), "t2", "out", 128, None),
            ("conv", "branch_pool", cin, pf, one, 1, s1, "x", "out", 224, "avg")]
    if kind == "B":
        return 480 + cin, [
            ("conv", "branch3x3", cin, 384, (3, 3), 2, s1, "x", "out", 0, None),
            ("conv", "branch3x3dbl_1", cin, 64, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch3x3dbl_2", 64, 96, (3, 3), 1, (1, 1), "t1", "t2", 0, None),
            ("conv", "branch3x3dbl_3", 96, 96, (3, 3), 2, s1, "t2", "out", 384, None),
            ("pool", "x", "out", 480)]
    if kind == "C":
        c7 = layer[3]
        r, c = ((1, 7), (0, 3)), ((7, 1), (3, 0))           # a 1x7 row and a 7x1 column kernel with their padding
        return 768, [
            ("conv", "branch1x1", cin, 192, one, 1, s1, "x", "out", 0, None),
            ("conv", "branch7x7_1", cin, c7, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch7x7_2", c7, c7, r[0], 1, r[1], "t1", "t2", 0, None),
            ("conv", "branch7x7_3", c7, 192, c[0], 1, c[1], "t2", "out", 192, None),
            ("conv", "branch7x7dbl_1", cin, c7, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch7x7dbl_2", c7, c7, c[0], 1, c[1], "t1", "t2", 0, None),
            ("conv", "branch7x7dbl_3", c7, c7, r[0], 1, r[1], "t2", "t1", 0, None),
            ("conv", "branch7x7dbl_4", c7, c7, c[0], 1, c[1], "t1", "t2", 0, None),
            ("conv", "branch7x7dbl_5", c7, 192, r[0], 1, r[1], "t2", "out", 384, None),
            ("conv", "branch_pool", cin, 192, one, 1, s1, "x", "out", 576, "avg")]
    if kind == "D":
        return 512 + cin, [
            ("conv", "branch3x3_1", cin, 192, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch3x3_2", 192, 320, (3, 3), 2, s1, "t1", "out", 0, None),
            ("conv", "branch7x7x3_1", cin, 192, one, 1, s1, "x", "t1", 0, None),
            ("conv", "branch7x7x3_2", 192, 192, (1, 7), 1, (0, 3), "t1", "t2", 0, None),
            ("conv", "branch7x7x3_3", 192, 192, (7, 1), 1, (3, 0), "t2", "t1", 0, None),
            ("conv", "branch7x7x3_4", 192, 192, (3, 3), 2, s1, "t1", "out", 320, None),
            ("pool", "x", "out", 512)]
    assert kind == "E", kind
    return 2048, [
        ("conv", "branch1x1", cin, 320, one, 1, s1, "x", "out", 0, None),
        ("conv", "branch3x3_1", cin, 384, one, 1, s1, "x", "t1", 0, None),
        ("conv", "branch3x3_2a", 384, 384, (1, 3), 1, (0, 1), "t1", "out", 320, None),
        ("conv", "branch3x3_2b", 384, 384, (3, 1), 1, (1, 0), "t1", "out", 704, None),
        ("conv", "branch3x3dbl_1", cin, 448, one, 1, s1, "x", "t1", 0, None),
        ("conv", "branch3x3dbl_2", 448, 384, (3, 3), 1, (1, 1), "t1", "t2", 0, None),
        ("conv", "branch3x3dbl_3a", 384, 384, (1, 3), 1, (0, 1), "t2", "out", 1088, None),
        ("conv", "branch3x3dbl_3b", 384, 384, (3, 1), 1, (1, 0), "t2", "out", 1472, None),
        ("conv", "branch_pool", cin, 192, one, 1, s1, "x", "out", 1856, layer[3])]


def conv_out(s: int, k: int, stride: int, pad: int) -> int:
    return (s + 2 * pad - k) // stride + 1


def pool_out(s: int) -> int:
    return (s - 3) // 2 + 1


@functools.lru_cache(maxsize=None)
def plan() -> tuple:
    """(steps, floats per frame of each workspace buffer).

    A step is a dict: ``kind`` (prep | conv | pool | head), ``src`` / ``dst`` buffer names, the input side ``s``
    and channels ``c``; for conv ``key`` (torchvision name), ``cin`` (unpadded), ``cout``, ``k`` = (kh, kw),
    ``stride``, ``pad`` = (ph, pw), ``pitch``, ``off``, ``pool`` (None | "avg" | "max"); for pool ``pitch``, ``off``.
    The main chain ping-pongs between buffers A and B; a block keeps its intermediate branch outputs in t1 and t2
    and writes its branches into channel slices of its output."""
    steps = []
    size = {"A": 0, "B": 0, "t1": 0, "t2": 0}

    def need(buf, n):
        size[buf] = max(size[buf], n)

    def conv(key, cin, cout, k, stride, pad, src, dst, s, c, pitch=None, off=0, pool=None):
        so_h, so_w = conv_out(s, k[0], stride, pad[0]), conv_out(s, k[1], stride, pad[1])
        assert so_h == so_w, key
        steps.append(dict(kind="conv", key=key, cin=cin, cout=cout, k=k, stride=stride, pad=pad, src=src, dst=dst,
                          s=s, c=c, pitch=pitch or cout, off=off, pool=pool))
        need(dst, so_h * so_h * (pitch or cout))
        return so_h

    s, c = SIDE, 4
    need("A", s * s * c)
    steps.append(dict(kind="prep", src=None, dst="A", s=SIDE, c=c))
    cur, oth = "A", "B"
    for layer in ARCH:
        if layer[0] == "conv":
            _, key, cin, cout, k, stride, pad = layer
            s = conv(key, cin, cout, k, stride, pad, cur, oth, s, c)
            c = cout
        elif layer[0] == "pool":
            steps.append(dict(kind="pool", src=cur, dst=oth, s=s, c=c, pitch=c, off=0))
            s = pool_out(s)
            need(oth, s * s * c)
        else:
            width, ops = _block(layer)
            key = layer[1]
            names = {"x": cur, "out": oth, "t1": "t1", "t2": "t2"}
            geom = {"x": (c, s)}                    # (channels, side) of the block input and of each temporary
            so = s
            for op in ops:
                if op[0] == "pool":
                    _, src, dst, off = op
                    steps.append(dict(kind="pool", src=names[src], dst=names[dst], s=s, c=c, pitch=width, off=off))
                    need(names[dst], pool_out(s) ** 2 * width)
                    continue
                _, name, cin, cout, k, stride, pad, src, dst, off, pool = op
                ci, si = geom[src]
                pitch = width if dst == "out" else None
                o = conv(f"{key}.{name}", cin, cout, k, stride, pad, names[src], names[dst], si, ci, pitch, off, pool)
                if dst == "out":
                    so = o
                else:
                    geom[dst] = (cout, o)
            s, c = so, width
        cur, oth = oth, cur
    steps.append(dict(kind="head", src=cur, dst=None, s=s, c=c))
    return steps, size


def units() -> List[tuple]:
    """(torchvision key prefix, Cin, Cout, (kh, kw)) of the 94 BasicConv2d, in forward order."""
    return [(st["key"], st["cin"], st["cout"], st["k"]) for st in plan()[0] if st["kind"] == "conv"]


def workspace_floats() -> int:
    """fp32 workspace per frame: ``workspace_floats() * 4`` bytes = 10.2 MB (B holds the 147x147x64 map of
    Conv2d_2b_3x3, A the 71x71x192 of Conv2d_4a_3x3)."""
    return sum(plan()[1].values())


LAUNCHES_PER_CHUNK = len(plan()[0])
DEFAULT_CHUNK = WORKSPACE_BUDGET // (4 * workspace_floats())


def _prefix(sd, key: str) -> str:
    """The state_dict prefix of unit ``key`` (torchvision name): itself, or its ``blocks.*`` name in the reference
    wrapper's layout."""
    if not any(k.startswith("blocks.") for k in sd):
        return key
    top, _, rest = key.partition(".")
    return BLOCK_PREFIX[top] + ("." + rest if rest else "")


def pack_weights(state_dict_or_path) -> dict:
    """{unit key: (w, bias)} fp32 on the CPU for the 94 BasicConv2d, in the layout ``MCVD_OP_CONV2D`` reads, with
    their BatchNorm2d (eps 1e-3) folded in (``eval_weights.fold_bn``).  Raises ``ValueError`` naming the first
    missing or misshapen key."""
    sd = EW.load(state_dict_or_path, "InceptionV3", "Inception")
    return {key: EW.fold_bn(sd, "InceptionV3", _prefix(sd, key), ".conv.weight", (cout, cin, *k), BN_EPS)
            for key, cin, cout, k in units()}


class InceptionV3:
    """2048-d pool features of frames, as the reference's ``InceptionV3([3])`` computes them
    (evaluation/inception.py:129-162, fid_PR.py:calculate_activations).

    ``state_dict_or_path``: torchvision-``Inception3`` or reference-wrapper state_dict, see the module docstring.
    Batch norm is folded and the weights are packed once, onto ``device`` (default: the current CUDA device).
    Frames are processed in chunks of at most ``max_chunk_frames``; a chunk needs ``workspace_floats() * 4`` bytes
    (10.2 MB) per frame, so the default (``DEFAULT_CHUNK`` = 210 frames) keeps it under 2 GiB.

    ``tf32``: run the 94 convolutions on the TF32 tensor cores (``MCVD_OP_CONV2D_TF32``).  Activations (after the
    fused branch pools) and weights are rounded once to TF32 (round to nearest, ties away from zero) and the products
    summed in fp32, so the features differ from the default fp32 ones by about the TF32 rounding (cuDNN's
    ``allow_tf32`` class of numerics); a frame's features still do not depend on its batch or chunk.  The packed TF32
    weights are made once here and take 90.8 MB of device memory on top of the 87.0 MB of folded fp32 weights.  The
    default (False) is the fp32 FFMA path, unchanged.
    """

    def __init__(self, state_dict_or_path, device: Optional[Union[str, torch.device]] = None,
                 max_chunk_frames: int = DEFAULT_CHUNK, tf32: bool = False):
        if not 1 <= int(max_chunk_frames) <= 65535:
            raise ValueError(f"InceptionV3: max_chunk_frames={max_chunk_frames} must be in [1, 65535]")
        self.device = torch.device(device if device is not None else "cuda")
        self.max_chunk_frames = int(max_chunk_frames)
        self.weights = {k: tuple(t.to(self.device) for t in v) for k, v in pack_weights(state_dict_or_path).items()}
        self.tf32 = bool(tf32)
        self.packed = {}
        if self.tf32:
            from . import lib
            self.packed = {key: lib.tf32_pack_weights(self.weights[key][0]) for key, _, _, _ in units()}

    def program(self, frames: torch.Tensor, out: torch.Tensor, ws: torch.Tensor):
        """The ops of one chunk: ``frames`` [n, C, S, S] fp32 CUDA, ``out`` fp64 [n, 2048], ``ws`` at least
        ``n * workspace_floats()`` floats."""
        from . import lib
        n, C, S = frames.shape[0], frames.shape[1], frames.shape[-1]
        steps, size = plan()
        bufs, lo = {}, 0
        for name, per in size.items():
            bufs[name] = ws[lo:lo + n * per]
            lo += n * per
        ops = []
        for st in steps:
            op = lib.McvdOp()
            op.B = n
            if st["kind"] == "prep":
                op.kind, op.H, op.W, op.C0, op.i1 = lib.OP_FID_PREP, SIDE, SIDE, C, S
                op.src0, op.dst = frames.data_ptr(), bufs[st["dst"]].data_ptr()
            elif st["kind"] == "head":
                op.kind, op.H, op.W, op.C0, op.i5 = lib.OP_FID_HEAD, 1, 1, st["c"], st["s"]
                op.src0, op.dst = bufs[st["src"]].data_ptr(), out.data_ptr()
            elif st["kind"] == "pool":
                op.kind, op.C0, op.i5, op.i6, op.i7 = lib.OP_MAXPOOL2D, st["c"], st["s"], st["pitch"], st["off"]
                op.H = op.W = pool_out(st["s"])
                op.src0, op.dst = bufs[st["src"]].data_ptr(), bufs[st["dst"]].data_ptr()
            else:
                w, b = self.weights[st["key"]]
                if self.tf32:
                    w = self.packed[st["key"]]
                (kh, kw), (ph, pw) = st["k"], st["pad"]
                op.kind = lib.OP_CONV2D_TF32 if self.tf32 else lib.OP_CONV2D
                op.C0, op.Cout = st["c"], st["cout"]
                op.H, op.W = conv_out(st["s"], kh, st["stride"], ph), conv_out(st["s"], kw, st["stride"], pw)
                op.i0, op.i1, op.i2, op.i3, op.i4, op.i5 = kh, kw, st["stride"], ph, pw, st["s"]
                op.i6, op.i7 = st["pitch"], st["off"]
                if st["pool"] is not None:
                    op.flags = lib.F_POOL | (lib.F_AVG if st["pool"] == "avg" else 0)
                op.src0, op.dst = bufs[st["src"]].data_ptr(), bufs[st["dst"]].data_ptr()
                op.w, op.bias = w.data_ptr(), b.data_ptr()
            ops.append(op)
        return ops

    @torch.no_grad()
    def __call__(self, frames: torch.Tensor, channels: int) -> torch.Tensor:
        """float64 [N*T, 2048] on the device: the features of ``frames`` [N, C, S, S], or of videos [B, C*T, S, S]
        (frame-major) in frame order, C = ``channels`` = 1 or 3, values in [0, 1] (not clamped, as the reference
        does not clamp either).  CPU input is copied to the device one chunk at a time."""
        from . import lib
        if self.device.type != "cuda":
            raise RuntimeError("mcvd_b200.fid.InceptionV3 runs on CUDA only (no CPU fallback)")
        if channels not in (1, 3):
            raise ValueError(f"InceptionV3: {channels} channels per frame (1 or 3)")
        if frames.dim() != 4 or frames.shape[1] % channels or frames.shape[2] != frames.shape[3]:
            raise ValueError(f"InceptionV3: frames {tuple(frames.shape)} must be [N, {channels}*T, S, S]")
        S = frames.shape[-1]
        x = frames.reshape(-1, channels, S, S)
        N = x.shape[0]
        out = torch.empty(N, DIMS, dtype=torch.float64, device=self.device)
        if N == 0:
            return out
        chunk = min(self.max_chunk_frames, N)
        ws = torch.empty(chunk * workspace_floats(), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            for lo in range(0, N, chunk):
                hi = min(N, lo + chunk)
                xc = x[lo:hi].to(self.device, torch.float32).contiguous()
                ops = self.program(xc, out[lo:hi], ws)
                lib.run_program(lib.make_ops(ops), len(ops), stream)
        return out


# ---- Fréchet distance ------------------------------------------------------------------------------------------
def frechet_distance_stats(mu1, sigma1, mu2, sigma2, eps: float = 1e-6) -> float:
    """``calculate_frechet_distance`` (evaluation/fid_PR.py:53-109): ``|mu1 - mu2|^2 + tr(sigma1 + sigma2 -
    2 sqrtm(sigma1 sigma2))`` with SciPy's ``sqrtm``; if the root is not finite, ``eps`` is added to both diagonals
    and the root retaken; an imaginary part above 1e-3 on its diagonal raises ``ValueError``, else the real part is
    used.  fp64 on the host."""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    if mu1.shape != mu2.shape or sigma1.shape != sigma2.shape:
        raise ValueError(f"FID: statistics of different sizes ({mu1.shape}, {sigma1.shape} vs {mu2.shape}, "
                         f"{sigma2.shape})")
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        print(f"FID: fid calculation produces singular product; adding {eps} to diagonal of cov estimates")
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(covmean.imag))}")
        covmean = covmean.real
    return float(diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean))


def _np(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 2:
        raise ValueError(f"FID: features must be [N, D], got shape {x.shape}")
    return x


def stats(feats) -> tuple:
    """(mu, sigma) of features [N, D]: the mean and the unbiased covariance (``np.cov(rowvar=False)``), fp64."""
    f = _np(feats)
    return f.mean(0), np.cov(f, rowvar=False)


def fid(fake_feats, real_feats) -> float:
    """FID of two feature sets [N, D], as ``get_fid_PR`` forms it (real statistics first)."""
    mu_r, sigma_r = stats(real_feats)
    mu_g, sigma_g = stats(fake_feats)
    return frechet_distance_stats(mu_r, sigma_r, mu_g, sigma_g)


# ---- precision / recall -----------------------------------------------------------------------------------------
def _knn_feats(x, device) -> torch.Tensor:
    """fp32 [N, D4] on ``device``, D padded to a multiple of 4 with zeros (zero pairs add exactly 0)."""
    x = torch.as_tensor(x).to(device, torch.float32)
    if x.dim() != 2 or x.shape[0] < 1:
        raise ValueError(f"precision_recall: features must be a non-empty [N, D], got shape {tuple(x.shape)}")
    pad = -x.shape[1] % 4
    if pad:
        x = torch.nn.functional.pad(x, (0, pad))
    return x.contiguous()


def knn_radii(feats: torch.Tensor, k: int) -> torch.Tensor:
    """fp32 [N]: the distance of every row of ``feats`` (fp32 [N, D4] CUDA) to its (k+1)-th nearest row, itself
    included, as ``kthvalue(k + 1)`` of the reference's distance matrix."""
    from . import lib
    out = torch.empty(feats.shape[0], dtype=torch.float32, device=feats.device)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i0, op.i1 = lib.OP_KNN_RADIUS, feats.shape[0], 1, 1, feats.shape[1], \
        feats.shape[0], k + 1
    op.src0, op.src1, op.dst = feats.data_ptr(), feats.data_ptr(), out.data_ptr()
    with torch.cuda.device(feats.device):
        lib.run_program(lib.make_ops([op]), 1, torch.cuda.current_stream(feats.device).cuda_stream)
    return out


def knn_cover(a: torch.Tensor, b: torch.Tensor, radii_b: torch.Tensor) -> torch.Tensor:
    """int32 [Na]: 1 where a row of ``a`` lies within the radius of some row of ``b`` (d <= radius), else 0."""
    from . import lib
    out = torch.empty(a.shape[0], dtype=torch.int32, device=a.device)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i0 = lib.OP_KNN_COVER, a.shape[0], 1, 1, a.shape[1], b.shape[0]
    op.src0, op.src1, op.aux0, op.dst = a.data_ptr(), b.data_ptr(), radii_b.data_ptr(), out.data_ptr()
    with torch.cuda.device(a.device):
        lib.run_program(lib.make_ops([op]), 1, torch.cuda.current_stream(a.device).cuda_stream)
    return out


def _share(flags: torch.Tensor) -> float:
    """The fp32 mean of 0/1 flags as a Python float, as the reference's ``.float().mean().item()`` gives it (the
    count is exact, so the mean is the once-rounded fp32 quotient)."""
    return float(np.float32(int(flags.sum())) / np.float32(flags.numel()))


def precision_recall(real, fake, k: int = 3, device=None) -> tuple:
    """(precision, recall) of ``calculate_precision_recall_full`` (evaluation/fid_PR.py:251-260) on the GPU:
    precision is the share of fake rows within the k-NN radius of some real row, recall the converse.  ``real``
    and ``fake`` are [N, D] features (tensors or arrays; computed in fp32).  Four launches, O(N) memory."""
    if not 0 <= int(k) <= 7:
        raise ValueError(f"precision_recall: k={k} must be in [0, 7]")
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise RuntimeError("mcvd_b200.fid.precision_recall runs on CUDA only (no CPU fallback)")
    r, g = _knn_feats(real, dev), _knn_feats(fake, dev)
    if r.shape[1] != g.shape[1]:
        raise ValueError(f"precision_recall: feature sizes differ ({r.shape[1]} vs {g.shape[1]})")
    if min(r.shape[0], g.shape[0]) < k + 1:
        raise ValueError(f"precision_recall: k={k} needs at least {k + 1} rows per set")
    radii_r, radii_g = knn_radii(r, k), knn_radii(g, k)
    return _share(knn_cover(g, r, radii_r)), _share(knn_cover(r, g, radii_g))


# ---- drop-ins for evaluation/fid_PR.py ----------------------------------------------------------------------------
def default_weights_path() -> str:
    """Where the reference's ``load_state_dict_from_url`` keeps the FID weights: the torch hub cache."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)


def native_unsupported(device, dims) -> Optional[str]:
    """None when the drop-ins can run natively for this call, else why not (the reference should run)."""
    if dims != DIMS:
        return f"dims={dims} (only the 2048-d pool features are native)"
    if torch.device(device).type != "cuda":
        return f"device {device} is not CUDA"
    if not os.path.exists(default_weights_path()):
        return f"the FID weights are not in the torch hub cache ({default_weights_path()})"
    return None


@functools.lru_cache(maxsize=2)
def _model(path: str, device: str, tf32: bool = False) -> InceptionV3:
    return InceptionV3(path, device=device, tf32=tf32)


def env_tf32() -> bool:
    """True when ``MCVD_EVAL_TF32=1``: the drop-ins then compute features on the TF32 tensor cores."""
    return os.environ.get("MCVD_EVAL_TF32", "0") == "1"


def model_for(device) -> InceptionV3:
    """The ``InceptionV3`` of the hub-cache weights on ``device``, built once per process (and per ``MCVD_EVAL_TF32``
    setting: with ``MCVD_EVAL_TF32=1`` it runs its convolutions in TF32)."""
    path = default_weights_path()
    if not os.path.exists(path):
        raise FileNotFoundError(f"FID weights not found at {path}; mcvd_b200 never downloads them (place "
                                f"{WEIGHTS_FILE} there)")
    dev = torch.device(device)
    if dev.type == "cuda" and dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return _model(path, str(dev), env_tf32())


def _check_dims(dims):
    if dims != DIMS:
        raise NotImplementedError(f"mcvd_b200.fid: dims={dims}; only the 2048-d pool features are implemented")


def _features(samples, device) -> torch.Tensor:
    if not isinstance(samples, torch.Tensor):
        raise ValueError("sample is not tensor!")
    if samples.dim() != 4 or samples.shape[1] not in (1, 3):
        raise ValueError(f"FID: samples {tuple(samples.shape)} must be [N, 1 | 3, S, S]")
    return model_for(device)(samples, samples.shape[1])


def _activations(path_or_samples, device) -> torch.Tensor:
    """``get_activations``: a ``.pt`` / ``.pth`` feature file (fp32 [N, 2048]) or the features of samples."""
    if isinstance(path_or_samples, str):
        if not (path_or_samples.endswith(".pt") or path_or_samples.endswith(".pth")):
            raise ValueError("path is not .pt or .pth!")
        return torch.load(path_or_samples, map_location="cpu", weights_only=True)
    return _features(path_or_samples, device)


def _statistics(path_or_samples, device) -> tuple:
    """``_compute_statistics_of_path_or_samples``: a ``.npz`` with ``mu`` and ``sigma``, or the samples' stats."""
    if isinstance(path_or_samples, str):
        if not path_or_samples.endswith(".npz"):
            raise ValueError("path is not .npz!")
        with np.load(path_or_samples) as f:
            return f["mu"][:], f["sigma"][:]
    return stats(_features(path_or_samples, device))


def get_fid(path_or_samples1, path_or_samples2, device=torch.device("cuda"), batch_size=50, dims=2048) -> float:
    """``fid_PR.get_fid``: FID between two ``.npz`` statistics files or sample tensors [N, C, S, S] in [0, 1].
    ``batch_size`` is accepted for compatibility; the features do not depend on it."""
    _check_dims(dims)
    m1, s1 = _statistics(path_or_samples1, device)
    m2, s2 = _statistics(path_or_samples2, device)
    return frechet_distance_stats(m1, s1, m2, s2)


def get_fid_PR(real_path_or_samples, fake_path_or_samples, device=torch.device("cuda"), batch_size=50, dims=2048,
               k=3, save_feats_path=None) -> tuple:
    """``fid_PR.get_fid_PR``: (FID, precision, recall) of ``.pt`` feature files or sample tensors.  With
    ``save_feats_path`` the fake features are saved as fp32 CPU [N, 2048], the reference's format."""
    _check_dims(dims)
    feat_r = _activations(real_path_or_samples, device)
    feat_g = _activations(fake_path_or_samples, device)
    if save_feats_path is not None:
        torch.save(feat_g.detach().float().cpu(), save_feats_path)
    precision, recall = precision_recall(feat_r, feat_g, k, device)
    return fid(feat_g, feat_r), precision, recall


def get_PR(real_path_or_samples, fake_path_or_samples, device=torch.device("cuda"), batch_size=50, dims=2048) -> tuple:
    """``fid_PR.get_PR``: (precision, recall) with k = 3."""
    _check_dims(dims)
    feat_r = _activations(real_path_or_samples, device)
    feat_g = _activations(fake_path_or_samples, device)
    return precision_recall(feat_r, feat_g, 3, device)
