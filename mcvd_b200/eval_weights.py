"""Weight loading and packing shared by the evaluation feature networks (``lpips``, ``fvd``, ``fid``).

Their convolutions (``MCVD_OP_CONV_RELU``, ``MCVD_OP_CONV3D``, ``MCVD_OP_CONV2D`` and the ``_TF32`` kinds, which pack
from the same image) read K-major weights: fp32 ``[taps][Cin4][Cout]`` with the taps in (dt, dy, dx) order and Cin
padded to a multiple of 4 with zero weights.
"""
from __future__ import annotations

from typing import Dict

import torch


def load(obj, net: str, what: str) -> Dict[str, torch.Tensor]:
    """``obj`` itself if it is a state_dict, else ``torch.load(obj)``; ``ValueError`` when that fails."""
    if isinstance(obj, dict):
        return obj
    try:
        return torch.load(obj, map_location="cpu", weights_only=True)
    except Exception as e:                          # noqa: BLE001 -- any unreadable file is a bad weight file
        raise ValueError(f"{net}: cannot read the {what} weights from {obj!r}: {e}") from e


def get(sd: Dict[str, torch.Tensor], key: str, shape, net: str, dtype: torch.dtype) -> torch.Tensor:
    """``sd[key]`` as a CPU tensor of ``dtype``; ``ValueError`` naming the key when it is missing or misshapen."""
    if key not in sd:
        raise ValueError(f"{net}: weight {key!r} missing")
    t = sd[key]
    if not isinstance(t, torch.Tensor) or tuple(t.shape) != tuple(shape):
        got = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
        raise ValueError(f"{net}: weight {key!r} has shape {got}, expected {tuple(shape)}")
    return t.detach().cpu().to(dtype)


def kmajor(w: torch.Tensor) -> torch.Tensor:
    """fp32 [taps * Cin4, Cout] of a convolution weight [Cout, Cin, *kernel]: permuted and zero-padded in ``w``'s
    dtype (both exact), then rounded once to fp32."""
    cout, cin, *kernel = w.shape
    cin4 = -(-cin // 4) * 4
    out = torch.zeros(*kernel, cin4, cout, dtype=w.dtype)
    out[..., :cin, :] = w.permute(*range(2, w.dim()), 1, 0)
    return out.reshape(-1, cout).float().contiguous()


def fold_bn(sd: Dict[str, torch.Tensor], net: str, prefix: str, conv_key: str, shape, eps: float) -> tuple:
    """(w [taps * Cin4, Cout], bias [Cout]) fp32 of a bias-free convolution ``prefix + conv_key`` of ``shape``
    followed by BatchNorm ``prefix + ".bn.*"`` (running statistics): the norm is folded into the convolution in fp64
    and each value rounded once."""
    w = get(sd, prefix + conv_key, shape, net, torch.float64)
    gamma, beta, mean, var = (get(sd, f"{prefix}.bn.{name}", shape[:1], net, torch.float64)
                              for name in ("weight", "bias", "running_mean", "running_var"))
    scale = gamma / torch.sqrt(var + eps)
    return kmajor(w * scale.view(-1, *[1] * (w.dim() - 1))), (beta - mean * scale).float().contiguous()
