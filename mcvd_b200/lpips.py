"""LPIPS (v0.1, net-lin, AlexNet backbone) of generated frames against real ones, on the GPU.

MCVD's ``video_gen`` reports LPIPS next to MSE, PSNR and SSIM (reference runners/ncsn_runner.py:1427-1431,
1602-1609): per frame pair it makes two PIL images, resizes them to 128x128, runs ``PerceptualLoss(model='net-lin',
net='alex')`` at batch size 1 and sums the distances.  ``LPIPS`` computes the same per-frame distances for whole
batches with the library's own kernels (``MCVD_OP_LPIPS_PREP``, ``MCVD_OP_CONV_RELU``, ``MCVD_OP_LPIPS_LAYER``):
11 launches per chunk of frame pairs.  ``LPIPS(..., tf32=True)`` runs the five convolutions on the TF32 tensor cores
instead (``MCVD_OP_CONV_RELU_TF32``): both operands rounded once to TF32, fp32 accumulation, the numerics class of
cuDNN with ``allow_tf32``.

Weights are never downloaded.  ``LPIPS`` takes either
  * a torchvision AlexNet state_dict (``features.{0,3,6,8,10}.{weight,bias}``, e.g. the torch hub cache's
    ``alexnet-owt-7be5be79.pth``) and the LPIPS v0.1 linear layers (``lin{0..4}.model.1.weight``, the reference's
    ``models/weights/v0.1/alex.pth``), or
  * one state_dict of the reference's ``PNetLin`` (``net.slice{1..5}.N.{weight,bias}`` and ``lin{0..4}...``).
Each may be given as a dict of tensors or as a path for ``torch.load``.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Union

import numpy as np
import torch

from . import eval_weights as EW

SIDE = 128                         # Resize((128, 128)) of the reference's T2 transform
_PREC = 22                         # Pillow's PRECISION_BITS for 8-bit images

# torchvision alexnet().features[0:12]: (index, Cin, Cout, kernel, stride, padding, max-pool before the conv)
LAYERS = [(0, 3, 64, 11, 4, 2, False), (3, 64, 192, 5, 1, 2, True), (6, 192, 384, 3, 1, 1, True),
          (8, 384, 256, 3, 1, 1, False), (10, 256, 256, 3, 1, 1, False)]
_PNET_SLICE = {0: 1, 3: 2, 6: 3, 8: 4, 10: 5}     # features index -> PNetLin slice (models/pretrained_networks.py:65-74)


def pil_bilinear_table(size: int, out: int = SIDE) -> np.ndarray:
    """Pillow's bilinear resampling coefficients for ``size`` -> ``out`` pixels along one axis, int32
    [out, 2 + taps]: per output pixel the first source pixel, the number of source pixels used and ``taps``
    coefficients in 22-bit fixed point (zero past the used ones).  Restates ``precompute_coeffs`` and
    ``normalize_coeffs_8bpc`` of Pillow's Resample.c: the support widens by the scale when downscaling and each
    output's weights are renormalised to sum to 1 before rounding."""
    scale = size / out
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale                       # the bilinear filter's support is 1
    taps = int(math.ceil(support)) * 2 + 1
    table = np.zeros((out, 2 + taps), dtype=np.int32)
    for xx in range(out):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), size) - xmin
        w = [max(0.0, 1.0 - abs((x + xmin - center + 0.5) * (1.0 / filterscale))) for x in range(xmax)]
        ww = sum(w)
        table[xx, 0], table[xx, 1] = xmin, xmax
        for x in range(xmax):
            k = w[x] / ww if ww != 0.0 else w[x]
            table[xx, 2 + x] = int(-0.5 + k * (1 << _PREC)) if k < 0 else int(0.5 + k * (1 << _PREC))
    return table


def pack_weights(backbone, lin=None) -> List[tuple]:
    """[(w [k*k*Cin4, Cout], bias [Cout], lin [Cout])] per AlexNet layer, fp32 on the CPU, in the layout
    ``MCVD_OP_CONV_RELU`` reads (Cin padded to a multiple of 4 with zero weights).  Raises ``ValueError`` naming
    the first missing or misshapen key."""
    sd = EW.load(backbone, "LPIPS", "backbone")
    pnet = any(k.startswith("net.slice") for k in sd)
    if pnet:
        if lin is not None:
            raise ValueError("LPIPS: a PNetLin state_dict already holds the lin weights; do not pass lin")
        lsd = sd
    else:
        if lin is None:
            raise ValueError("LPIPS: a torchvision AlexNet state_dict needs the LPIPS lin weights (alex.pth)")
        lsd = EW.load(lin, "LPIPS", "lin")
    packed = []
    for li, (idx, cin, cout, k, _, _, _) in enumerate(LAYERS):
        pre = f"net.slice{_PNET_SLICE[idx]}.{idx}." if pnet else f"features.{idx}."
        w = EW.get(sd, pre + "weight", (cout, cin, k, k), "LPIPS", torch.float32)
        b = EW.get(sd, pre + "bias", (cout,), "LPIPS", torch.float32)
        lw = EW.get(lsd, f"lin{li}.model.1.weight", (1, cout, 1, 1), "LPIPS", torch.float32).reshape(cout)
        packed.append((EW.kmajor(w), b.contiguous(), lw.contiguous()))
    return packed


# floats of ping-pong workspace per image: A holds the network input, relu2 and relu4; B relu1, relu3 and relu5
_WS_A = SIDE * SIDE * 4
_WS_B = 31 * 31 * 64


class LPIPS:
    """Per-frame LPIPS of generated clips against real ones (``PerceptualLoss(model='net-lin', net='alex')``).

    ``backbone`` / ``lin``: see the module docstring.  The weights are packed once, onto ``device`` (default: the
    current CUDA device).  Frame pairs are processed in chunks of at most ``max_chunk_frames``; a chunk needs
    ``(128*128*4 + 31*31*64) * 4 * 2`` bytes (0.97 MiB) of workspace per frame pair, so the default of 256 pairs
    bounds it at 248 MiB.

    ``tf32``: run the five convolutions on the TF32 tensor cores (``MCVD_OP_CONV_RELU_TF32``).  Activations (after
    the max-pool of layers 2 and 3) and weights are rounded once to TF32 (round to nearest, ties away from zero) and
    the products summed in fp32, so the distances differ from the default fp32 ones by about the TF32 rounding
    (cuDNN's ``allow_tf32`` class of numerics); a frame pair's distance still does not depend on its batch or chunk.
    The packed TF32 weights are made once here and take 9.9 MB of device memory on top of the 9.9 MB of fp32
    weights; the workspace and the 11 launches per chunk are unchanged.  The default (False) is the fp32 FFMA path,
    unchanged.
    """

    def __init__(self, backbone, lin=None, device: Optional[Union[str, torch.device]] = None,
                 max_chunk_frames: int = 256, tf32: bool = False):
        if not 1 <= int(max_chunk_frames) <= 32767:
            raise ValueError(f"LPIPS: max_chunk_frames={max_chunk_frames} must be in [1, 32767]")
        self.device = torch.device(device if device is not None else "cuda")
        self.max_chunk_frames = int(max_chunk_frames)
        self.weights = [tuple(t.to(self.device) for t in layer) for layer in pack_weights(backbone, lin)]
        self.tf32 = bool(tf32)
        self.packed: List[torch.Tensor] = []
        if self.tf32:
            from . import lib
            self.packed = [lib.tf32_pack_weights(w) for w, _, _ in self.weights]
        self._tables: Dict[int, torch.Tensor] = {}

    def _table(self, size: int) -> torch.Tensor:
        if size not in self._tables:
            self._tables[size] = torch.from_numpy(pil_bilinear_table(size)).to(self.device)
        return self._tables[size]

    def program(self, pred: torch.Tensor, real: torch.Tensor, channels: int, out: torch.Tensor, ws: torch.Tensor):
        """The 11 ops of one chunk: ``pred`` / ``real`` [n, channels, S, S] fp32 CUDA, ``out`` fp64 [n],
        ``ws`` at least ``n * 2 * (_WS_A + _WS_B)`` floats."""
        from . import lib
        n, S = pred.shape[0], pred.shape[-1]
        A, B = ws[:2 * n * _WS_A], ws[2 * n * _WS_A:2 * n * (_WS_A + _WS_B)]
        ops = []
        op = lib.McvdOp()
        op.kind, op.B, op.H, op.W, op.C0 = lib.OP_LPIPS_PREP, n, SIDE, SIDE, channels
        op.i0, op.i1, op.i2 = 1, S, self._table(S).shape[1] - 2
        op.src0, op.src1, op.w, op.dst = pred.data_ptr(), real.data_ptr(), self._table(S).data_ptr(), A.data_ptr()
        ops.append(op)
        src, dst, side, cin = A, B, SIDE, 4
        for li, (_, _, cout, k, stride, pad, pool) in enumerate(LAYERS):
            w, b, lw = self.weights[li]
            if self.tf32:
                w = self.packed[li]
            hc = (side - 3) // 2 + 1 if pool else side
            oh = (hc + 2 * pad - k) // stride + 1
            op = lib.McvdOp()
            op.kind, op.flags, op.B, op.H, op.W, op.C0, op.Cout = (lib.OP_CONV_RELU_TF32 if self.tf32 else
                                                                   lib.OP_CONV_RELU, lib.F_POOL if pool else 0, 2 * n,
                                                                   oh, oh, cin, cout)
            op.i0, op.i1, op.i2, op.i3, op.i4 = k, stride, pad, side, side
            op.src0, op.w, op.bias, op.dst = src.data_ptr(), w.data_ptr(), b.data_ptr(), dst.data_ptr()
            ops.append(op)
            half = n * oh * oh * cout
            op = lib.McvdOp()
            op.kind, op.B, op.H, op.W, op.C0, op.i0 = lib.OP_LPIPS_LAYER, n, oh, oh, cout, li
            op.src0, op.src1, op.w, op.dst = dst.data_ptr(), dst[half:].data_ptr(), lw.data_ptr(), out.data_ptr()
            ops.append(op)
            src, dst, side, cin = dst, src, oh, cout
        return ops

    @torch.no_grad()
    def __call__(self, pred: torch.Tensor, real: torch.Tensor, channels: int) -> torch.Tensor:
        """float64 [B, F]: LPIPS of every frame of ``pred`` against the same frame of ``real``, both
        [B, channels*F, S, S] in [0, 1] on the GPU (values outside are clamped, as ``inverse_data_transform`` does
        before the reference sees them)."""
        from . import lib
        if pred.device.type != "cuda" or self.device.type != "cuda":
            raise RuntimeError("mcvd_b200.lpips.LPIPS runs on CUDA tensors only (no CPU fallback)")
        if channels not in (1, 3):
            raise ValueError(f"LPIPS: {channels} channels per frame (1 or 3)")
        if pred.dim() != 4 or pred.shape != real.shape or pred.shape[1] % channels or pred.shape[2] != pred.shape[3]:
            raise ValueError(f"LPIPS: pred {tuple(pred.shape)} and real {tuple(real.shape)} must both be "
                             f"[B, {channels}*F, S, S]")
        Bc, S = pred.shape[0], pred.shape[-1]
        F = pred.shape[1] // channels
        N = Bc * F
        p = pred.to(self.device).contiguous().float().reshape(N, channels, S, S)
        r = real.to(self.device).contiguous().float().reshape(N, channels, S, S)
        out = torch.empty(N, dtype=torch.float64, device=self.device)
        chunk = min(self.max_chunk_frames, N)
        ws = torch.empty(2 * chunk * (_WS_A + _WS_B), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device).cuda_stream
            for lo in range(0, N, chunk):
                hi = min(N, lo + chunk)
                ops = self.program(p[lo:hi], r[lo:hi], channels, out[lo:hi], ws)
                lib.run_program(lib.make_ops(ops), len(ops), stream)
        return out.reshape(Bc, F)
