"""FVD (Fréchet Video Distance) of generated videos against real ones, with I3D features computed on the GPU.

MCVD's ``video_gen`` reports FVD next to MSE, PSNR, SSIM and LPIPS (reference runners/ncsn_runner.py:1311-1332,
1918-1982, 2217-2229).  It scores each video with an Inception-v1 I3D network (models/fvd/pytorch_i3d.py
``InceptionI3d``, 400 Kinetics classes, eval mode) after ``preprocess_single`` (models/fvd/fvd.py:160-186: bilinear
resize of the shorter side to 224, centre crop, ``(x - 0.5) * 2``), takes the 400-d pre-softmax output as the
video's feature and compares the feature sets of fake and real videos with the Fréchet distance of two Gaussians.

``I3D`` computes the same features for whole batches with the library's own kernels (``MCVD_OP_I3D_PREP``,
``MCVD_OP_CONV3D``, ``MCVD_OP_MAXPOOL3D``, ``MCVD_OP_I3D_HEAD``): ``LAUNCHES_PER_CHUNK`` launches per chunk of
videos, whatever its size.  A video's features do not depend on the batch or chunk it is computed in.
``I3D(..., tf32=True)`` runs the convolutions on the TF32 tensor cores instead (``MCVD_OP_CONV3D_TF32``): both
operands rounded once to TF32, fp32 accumulation, the numerics class of cuDNN with ``allow_tf32``.

Weights are never downloaded.  ``I3D`` takes an ``InceptionI3d`` state_dict (``Conv3d_1a_7x7.conv3d.weight``,
``Conv3d_1a_7x7.bn.{weight,bias,running_mean,running_var}``, ``Mixed_3b.b1b.conv3d.weight``, ...,
``logits.conv3d.{weight,bias}``), as a dict of tensors or a path for ``torch.load``.  The reference downloads a
TorchScript detector (``i3d_torchscript.pt``) instead; mapping that file's parameters is not supported.

``frechet_distance`` and ``fvd_summary`` run on the host in fp64 (numpy / scipy): the covariances are 400 x 400.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Union

import numpy as np
import torch

from . import eval_weights as EW

SIDE = 224                         # preprocess_single(resolution=224)
MIN_FRAMES = 9                     # at 8 frames the last time extent is 1, too short for the [2, 7, 7] average pool
FVD_MIN_FRAMES = 10                # video_gen computes a task's FVD only for videos of at least 10 frames (:1311-1332)
NUM_CLASSES = 400
BN_EPS = 1e-5

# InceptionI3d.__init__ (models/fvd/pytorch_i3d.py:204-285), in forward order:
#   ("conv", key, Cin, Cout, kernel, stride)       Unit3D with BatchNorm3d and ReLU, cubic kernel and stride
#   ("pool", (kt, ks), (st, ss))                   MaxPool3dSamePadding
#   ("mixed", key, Cin, [b0, b1a, b1b, b2a, b2b, b3b] output channels)
ARCH = [
    ("conv", "Conv3d_1a_7x7", 3, 64, 7, 2),
    ("pool", (1, 3), (1, 2)),
    ("conv", "Conv3d_2b_1x1", 64, 64, 1, 1),
    ("conv", "Conv3d_2c_3x3", 64, 192, 3, 1),
    ("pool", (1, 3), (1, 2)),
    ("mixed", "Mixed_3b", 192, [64, 96, 128, 16, 32, 32]),
    ("mixed", "Mixed_3c", 256, [128, 128, 192, 32, 96, 64]),
    ("pool", (3, 3), (2, 2)),
    ("mixed", "Mixed_4b", 480, [192, 96, 208, 16, 48, 64]),
    ("mixed", "Mixed_4c", 512, [160, 112, 224, 24, 64, 64]),
    ("mixed", "Mixed_4d", 512, [128, 128, 256, 24, 64, 64]),
    ("mixed", "Mixed_4e", 512, [112, 144, 288, 32, 64, 64]),
    ("mixed", "Mixed_4f", 528, [256, 160, 320, 32, 128, 128]),
    ("pool", (2, 2), (2, 2)),
    ("mixed", "Mixed_5b", 832, [256, 160, 320, 32, 128, 128]),
    ("mixed", "Mixed_5c", 832, [384, 192, 384, 48, 128, 128]),
]
HEAD_CHANNELS = 1024


def units() -> List[tuple]:
    """(state_dict key prefix, Cin, Cout, kernel) of every Unit3D with batch norm, in forward order (57)."""
    out = []
    for layer in ARCH:
        if layer[0] == "conv":
            out.append(layer[1:5])
        elif layer[0] == "mixed":
            _, key, cin, o = layer
            out += [(f"{key}.b0", cin, o[0], 1), (f"{key}.b1a", cin, o[1], 1), (f"{key}.b1b", o[1], o[2], 3),
                    (f"{key}.b2a", cin, o[3], 1), (f"{key}.b2b", o[3], o[4], 3), (f"{key}.b3b", cin, o[5], 1)]
    return out


def same_pad(n: int, k: int, s: int) -> int:
    """Total TF-"SAME" padding of one axis (``compute_pad``, pytorch_i3d.py:9-13, 71-75); the front gets half."""
    return max(k - (s if n % s == 0 else n % s), 0)


def same_out(n: int, k: int, s: int) -> int:
    return (n + same_pad(n, k, s) - k) // s + 1


def resize_target(S: int):
    """(height, width) ``preprocess_single`` resizes a square S x S frame to before its centre crop: the shorter side
    becomes 224 and the other ``ceil(S * (224 / S))``, which float rounding can make 225."""
    scale = SIDE / min(S, S)
    return math.ceil(S * scale), SIDE


def pack_weights(state_dict_or_path) -> dict:
    """{unit key: (w, bias)} for the 57 Unit3D plus ``"logits"``: (w [1024, 400], bias [400]) fp32 on the CPU.
    A Unit3D's (w, bias) is in the layout ``MCVD_OP_CONV3D`` reads, with its BatchNorm3d (eps 1e-5) folded in
    (``eval_weights.fold_bn``).  Raises ``ValueError`` naming the first missing or misshapen key."""
    sd = EW.load(state_dict_or_path, "I3D", "InceptionI3d")
    packed = {key: EW.fold_bn(sd, "I3D", key, ".conv3d.weight", (cout, cin, k, k, k), BN_EPS)
              for key, cin, cout, k in units()}
    w = EW.get(sd, "logits.conv3d.weight", (NUM_CLASSES, HEAD_CHANNELS, 1, 1, 1), "I3D", torch.float64)
    b = EW.get(sd, "logits.conv3d.bias", (NUM_CLASSES,), "I3D", torch.float64)
    packed["logits"] = (w.reshape(NUM_CLASSES, HEAD_CHANNELS).t().float().contiguous(), b.float().contiguous())
    return packed


def plan(T: int) -> tuple:
    """(steps, floats per video of each workspace buffer) of one video of T frames.

    A step is a dict: ``kind`` (prep | conv | pool | head), ``src`` / ``dst`` buffer names, the input geometry
    ``t``, ``s`` (time, side) and ``c`` (channels), and for conv / pool ``kt, ks, st, ss``, for conv ``key``,
    ``cout``, ``pitch``, ``off``.  The main chain ping-pongs between buffers A and B; an Inception block keeps
    its b1a, b2a and b3a outputs in t1, t2 and t3 and writes its four branches into channel slices of its output."""
    steps = []
    size = {"A": 0, "B": 0, "t1": 0, "t2": 0, "t3": 0}

    def need(buf, n):
        size[buf] = max(size[buf], n)

    def conv(key, src, dst, t, s, c, cout, k, st, pitch=None, off=0):
        steps.append(dict(kind="conv", key=key, src=src, dst=dst, t=t, s=s, c=c, cout=cout, kt=k, ks=k, st=st,
                          ss=st, pitch=pitch or cout, off=off))
        to, so = same_out(t, k, st), same_out(s, k, st)
        need(dst, to * so * so * (pitch or cout))
        return to, so

    def pool(src, dst, t, s, c, kt, ks, st, ss):
        steps.append(dict(kind="pool", src=src, dst=dst, t=t, s=s, c=c, kt=kt, ks=ks, st=st, ss=ss))
        to, so = same_out(t, kt, st), same_out(s, ks, ss)
        need(dst, to * so * so * c)
        return to, so

    t, s, c = T, SIDE, 4
    need("A", t * s * s * c)
    steps.append(dict(kind="prep", src=None, dst="A", t=T, s=SIDE, c=c))
    cur, oth = "A", "B"
    for layer in ARCH:
        if layer[0] == "conv":
            _, key, _, cout, k, st = layer
            t, s = conv(key, cur, oth, t, s, c, cout, k, st)
            c = cout
        elif layer[0] == "pool":
            _, (kt, ks), (st, ss) = layer
            t, s = pool(cur, oth, t, s, c, kt, ks, st, ss)
        else:
            _, key, cin, o = layer
            width = o[0] + o[2] + o[4] + o[5]
            conv(f"{key}.b0", cur, oth, t, s, c, o[0], 1, 1, width, 0)
            conv(f"{key}.b1a", cur, "t1", t, s, c, o[1], 1, 1)
            conv(f"{key}.b1b", "t1", oth, t, s, o[1], o[2], 3, 1, width, o[0])
            conv(f"{key}.b2a", cur, "t2", t, s, c, o[3], 1, 1)
            conv(f"{key}.b2b", "t2", oth, t, s, o[3], o[4], 3, 1, width, o[0] + o[2])
            pool(cur, "t3", t, s, c, 3, 3, 1, 1)
            conv(f"{key}.b3b", "t3", oth, t, s, c, o[5], 1, 1, width, o[0] + o[2] + o[4])
            c = width
        cur, oth = oth, cur
    steps.append(dict(kind="head", src=cur, dst=None, t=t, s=s, c=c))
    return steps, size


def workspace_floats(T: int) -> int:
    """fp32 workspace per video of T frames (``workspace_floats(25) * 4`` = 85.8 MiB: A holds the 224x224 input
    and every second activation, B the 7x7x7 stem's output, 13 x 112 x 112 x 64 floats = 40 MiB at T = 25)."""
    return sum(plan(T)[1].values())


LAUNCHES_PER_CHUNK = len(plan(MIN_FRAMES)[0])


class I3D:
    """400-d I3D features of videos, as the reference's ``get_fvd_feats`` computes them (models/fvd/fvd.py:41-49).

    ``state_dict_or_path``: an ``InceptionI3d`` state_dict, see the module docstring.  Batch norm is folded and the
    weights are packed once, onto ``device`` (default: the current CUDA device).  Videos are processed in chunks of
    at most ``max_chunk_videos``; a chunk needs ``workspace_floats(T) * 4`` bytes per video (33 MiB at T = 10,
    86 MiB at T = 25, 99 MiB at T = 30), so the default of 16 keeps it under 1.6 GiB up to T = 30.

    ``tf32``: run the 57 convolutions on the TF32 tensor cores (``MCVD_OP_CONV3D_TF32``).  Activations and weights
    are rounded once to TF32 (round to nearest, ties away from zero) and the products summed in fp32, so the features
    differ from the default fp32 ones by about the TF32 rounding (cuDNN's ``allow_tf32`` class of numerics); a video's
    features still do not depend on its batch or chunk.  The packed TF32 weights are made once here and take 52.9 MB
    of device memory on top of the 49.2 MB of folded fp32 weights.  The default (False) is the fp32 FFMA path,
    unchanged.
    """

    def __init__(self, state_dict_or_path, device: Optional[Union[str, torch.device]] = None,
                 max_chunk_videos: int = 16, tf32: bool = False):
        if not 1 <= int(max_chunk_videos) <= 4096:
            raise ValueError(f"I3D: max_chunk_videos={max_chunk_videos} must be in [1, 4096]")
        self.device = torch.device(device if device is not None else "cuda")
        self.max_chunk_videos = int(max_chunk_videos)
        self.weights = {k: tuple(t.to(self.device) for t in v) for k, v in pack_weights(state_dict_or_path).items()}
        self.tf32 = bool(tf32)
        self.packed = {}
        if self.tf32:
            from . import lib
            self.packed = {key: lib.tf32_pack_weights(self.weights[key][0]) for key, _, _, _ in units()}

    def program(self, videos: torch.Tensor, channels: int, out: torch.Tensor, ws: torch.Tensor):
        """The ops of one chunk: ``videos`` [n, channels*T, S, S] fp32 CUDA, ``out`` fp64 [n, 400], ``ws`` at least
        ``n * workspace_floats(T)`` floats."""
        from . import lib
        n, S = videos.shape[0], videos.shape[-1]
        T = videos.shape[1] // channels
        steps, size = plan(T)
        bufs, lo = {}, 0
        for name, per in size.items():
            bufs[name] = ws[lo:lo + n * per]
            lo += n * per
        Ht, Wt = resize_target(S)
        ops = []
        for st in steps:
            op = lib.McvdOp()
            op.B = n
            if st["kind"] == "prep":
                op.kind, op.H, op.W, op.C0 = lib.OP_I3D_PREP, SIDE, SIDE, channels
                op.i0, op.i1, op.i2, op.i3 = T, S, Ht, Wt
                op.src0, op.dst = videos.data_ptr(), bufs[st["dst"]].data_ptr()
            elif st["kind"] == "head":
                w, b = self.weights["logits"]
                op.kind, op.H, op.W, op.C0, op.Cout, op.i4, op.i5 = (lib.OP_I3D_HEAD, 1, 1, st["c"], NUM_CLASSES,
                                                                     st["t"], st["s"])
                op.src0, op.w, op.bias, op.dst = bufs[st["src"]].data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr()
            else:
                so = same_out(st["s"], st["ks"], st["ss"])
                op.H = op.W = so
                op.C0 = st["c"]
                op.i0, op.i1, op.i2, op.i3, op.i4, op.i5 = st["kt"], st["ks"], st["st"], st["ss"], st["t"], st["s"]
                op.src0, op.dst = bufs[st["src"]].data_ptr(), bufs[st["dst"]].data_ptr()
                if st["kind"] == "pool":
                    op.kind = lib.OP_MAXPOOL3D
                else:
                    w, b = self.weights[st["key"]]
                    if self.tf32:
                        w = self.packed[st["key"]]
                    op.kind = lib.OP_CONV3D_TF32 if self.tf32 else lib.OP_CONV3D
                    op.Cout, op.i6, op.i7 = st["cout"], st["pitch"], st["off"]
                    op.w, op.bias = w.data_ptr(), b.data_ptr()
            ops.append(op)
        return ops

    @torch.no_grad()
    def __call__(self, videos: torch.Tensor, channels: int) -> torch.Tensor:
        """float64 [B, 400]: the features of ``videos`` [B, channels*T, S, S] in [0, 1] on the GPU (frame-major,
        the layout of ``video_gen``'s frames; values are not clamped, as the reference does not clamp either)."""
        from . import lib
        if videos.device.type != "cuda" or self.device.type != "cuda":
            raise RuntimeError("mcvd_b200.fvd.I3D runs on CUDA tensors only (no CPU fallback)")
        if channels not in (1, 3):
            raise ValueError(f"I3D: {channels} channels per frame (1 or 3)")
        if videos.dim() != 4 or videos.shape[1] % channels or videos.shape[2] != videos.shape[3]:
            raise ValueError(f"I3D: videos {tuple(videos.shape)} must be [B, {channels}*T, S, S]")
        B, S = videos.shape[0], videos.shape[-1]
        T = videos.shape[1] // channels
        if T < MIN_FRAMES:
            raise ValueError(f"I3D: {T} frames; InceptionI3d needs at least {MIN_FRAMES}")
        v = videos.to(self.device).contiguous().float()
        out = torch.empty(B, NUM_CLASSES, dtype=torch.float64, device=self.device)
        if B == 0:
            return out
        chunk = min(self.max_chunk_videos, B, max(1, 65535 // T))
        ws = torch.empty(chunk * workspace_floats(T), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            for lo in range(0, B, chunk):
                hi = min(B, lo + chunk)
                ops = self.program(v[lo:hi], channels, out[lo:hi], ws)
                lib.run_program(lib.make_ops(ops), len(ops), stream)
        return out


def _feats(x) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    x = np.asarray(x, dtype=np.float64)
    if x.ndim != 2:
        raise ValueError(f"FVD: features must be [N, D], got shape {x.shape}")
    return x


def frechet_distance(fake, real) -> float:
    """Fréchet distance between Gaussians fitted to two feature sets [N, D] (models/fvd/fvd.py:275-287):
    ``|mu_f - mu_r|^2 + tr(S_f + S_r - 2 sqrtm(S_f S_r))`` with unbiased covariances (``np.cov(rowvar=False)``),
    scipy's ``sqrtm`` and the real part of the result, in fp64 on the host."""
    from scipy import linalg
    f, r = _feats(fake), _feats(real)
    if f.shape[1] != r.shape[1]:
        raise ValueError(f"FVD: feature sizes differ ({f.shape[1]} vs {r.shape[1]})")
    mu_f, mu_r = f.mean(0), r.mean(0)
    cov_f, cov_r = np.cov(f, rowvar=False), np.cov(r, rowvar=False)
    root = linalg.sqrtm(cov_f @ cov_r)
    diff = mu_f - mu_r
    return float(np.real(diff @ diff + np.trace(cov_f) + np.trace(cov_r) - 2.0 * np.trace(root)))


def fvd_summary(fake, real, preds_per_test: int) -> Dict[str, float]:
    """``fvd_stuff`` of the reference (runners/ncsn_runner.py:2217-2229): ``fvd`` over all fake videos [B*p, D]
    against the real ones [B, D]; with ``preds_per_test`` p > 1 also the mean, standard deviation (ddof 0) and
    95% normal half-interval (1.96 standard errors, ddof 1) of the p per-trajectory FVDs ``fake[j::p]``, else
    -1 for those three.  Trajectories are taken in order; the reference's random permutation of them changes
    none of the four values."""
    import scipy.stats as st
    f, r = _feats(fake), _feats(real)
    p = int(preds_per_test)
    if p < 1 or f.shape[0] != r.shape[0] * p:
        raise ValueError(f"FVD: {f.shape[0]} fake videos are not {p} per each of {r.shape[0]} real ones")
    out = {"fvd": frechet_distance(f, r), "fvd_traj_mean": -1.0, "fvd_traj_std": -1.0, "fvd_traj_conf95": -1.0}
    if p > 1:
        trajs = [frechet_distance(f[j::p], r) for j in range(p)]
        mean = float(np.mean(trajs))
        out["fvd_traj_mean"], out["fvd_traj_std"] = mean, float(np.std(trajs))
        out["fvd_traj_conf95"] = mean - float(st.norm.interval(0.95, loc=mean, scale=st.sem(trajs))[0])
    return out
