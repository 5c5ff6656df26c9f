"""Interpreter of McvdOp programs in plain torch.  TEST INFRASTRUCTURE ONLY.

Executes the op arrays produced by ``mcvd_b200.program.Engine`` following the op semantics documented in
``include/mcvd_b200.h``, on whichever device the program's buffers live.  With the default fp32 compute type it lets
the ``-m "not gpu"`` suite check the host-side lowering (module walk, skip stack, FiLM offsets, virtual concats, SPADE
wiring, sampler coefficient plumbing) against the oracle without a GPU.  With ``compute_dtype=torch.float64`` every op
reads its buffers, computes in float64 and rounds once when it stores: the per-op reference of the GPU replay
(tests/program_replay.py).  It is NOT a fallback: the product never imports it, and ``Engine`` refuses to run without
the CUDA library unless a test passes an explicit ``_test_backend``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from mcvd_b200 import lib

# Range of the conv-epilogue GroupNorm statistics (include/mcvd_b200.h, MCVD_OP_CONV_UMMA2 dst2): |x| <= 2^12 keeps
# round(x * 2^16) inside int32 and the sum of 128 squares inside the unsigned 64-bit accumulator.
STATS_MAX = 4096.0
SILU_LIPSCHITZ = 1.1            # max |silu'(x)| = 1.0998


def silu(x):
    return x * torch.sigmoid(x)


def tile_geometry(B, H, W, ks):
    """(positions per image, image slots per 128-position tile, tiles) of the padded-flat position space of a
    tensor-core conv of kernel size ks (csrc/conv_umma.cu)"""
    pimg = (H + 1) * (W + 1) if ks == 3 else H * W
    return pimg, 127 // pimg + 2, 2 * ((B * pimg + 255) // 256)


def tile_slots(B, H, W, ks, device=None):
    """(image of slot jj of tile t, whether tile t holds rows of that image), both [tiles][NJ]: the slots a
    GN_FINALIZE reads; the others are never written"""
    pimg, nj, ntiles = tile_geometry(B, H, W, ks)
    t = torch.arange(ntiles, device=device).view(-1, 1)
    b = torch.arange(nj, device=device).view(1, -1) + torch.clamp((t * 128) // pimg, max=B - 1)
    return b, (b < B) & (t >= (b * pimg) // 128) & (t <= ((b + 1) * pimg - 1) // 128)


def tile_stats(y, ks):
    """Conv-epilogue statistics of a stored output y [B,H,W,C]: int64 [tiles][NJ][2][C] = sum, sum of squares of
    round(y * 2^16) over the rows of a 128-position tile that belong to one image.  Outputs outside the documented
    range |y| <= 2^12 (or NaN) have no defined statistics and raise ValueError."""
    B, H, W, C = y.shape
    if not bool((y.abs() <= STATS_MAX).all()):
        raise ValueError(f"conv output outside the epilogue-statistics range |x| <= {STATS_MAX:g}: "
                         f"max |x| = {float(y.abs().max()):.6g}")
    dev = y.device
    pimg, nj, ntiles = tile_geometry(B, H, W, ks)
    xi = torch.round(y.double() * 65536.0).to(torch.int64).reshape(B * H * W, C)
    yy, xx = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing="ij")
    r = (((yy + 1) * (W + 1) + xx + 1) if ks == 3 else (yy * W + xx)).reshape(1, -1)
    b = torch.arange(B, device=dev).reshape(-1, 1)
    t = (b * pimg + r) // 128
    jj = b - torch.clamp((t * 128) // pimg, max=B - 1)
    idx = (t.reshape(-1), jj.reshape(-1))
    st = torch.zeros(ntiles, nj, 2, C, dtype=torch.int64, device=dev)
    st[:, :, 0].index_put_(idx, xi, accumulate=True)
    st[:, :, 1].index_put_(idx, xi * xi, accumulate=True)
    return st


class Interpreter:
    def __init__(self, compute_dtype=torch.float32):
        self.tensors = {}
        self.cdt = compute_dtype

    # -- registry ---------------------------------------------------------------------------------
    def register(self, t: torch.Tensor):
        self.tensors[t.data_ptr()] = t

    def get(self, ptr, n=None, dtype=torch.float32):
        if not ptr:
            return None
        t = self.tensors[ptr]
        assert t.dtype == dtype, (t.dtype, dtype)
        flat = t.view(-1)
        return flat if n is None else flat[:n]

    def rd(self, ptr, n=None):
        """an fp32 buffer as a compute-type tensor (the buffer itself in fp32 mode)"""
        t = self.get(ptr, n)
        return None if t is None else t.to(self.cdt)

    # -- backend protocol used by Engine -----------------------------------------------------------
    def device_arch(self):
        return 100

    def umma_kblock(self, c0, c1):
        if c0 % 32 == 0 and c1 % 32 == 0:
            return 32
        if c0 % 16 == 0 and c1 % 16 == 0:
            return 16
        return 0

    def pack_umma(self, taps, nt, kb):
        t = taps.contiguous().float()
        self.register(t)
        return t, 1.0

    def run(self, ops, n):
        for i in range(n):
            self.exec(ops[i])

    # -- helpers ----------------------------------------------------------------------------------
    def _src(self, op, Hin, Win):
        """virtually concatenated NHWC input -> [B, Hin, Win, C]"""
        B = op.B
        a = self.rd(op.src0, B * Hin * Win * op.C0).view(B, Hin, Win, op.C0)
        if op.C1 > 0:
            b = self.rd(op.src1, B * Hin * Win * op.C1).view(B, Hin, Win, op.C1)
            a = torch.cat([a, b], dim=3)
        return a

    def _conv(self, op, x, taps_shape_out, mag=False):
        """x [B,H,W,Cin] NHWC; weights [taps][Cin][OP]; returns [B,H,W,Cout]"""
        B, H, W, Cin = x.shape
        ks, Cout = op.i0, op.Cout
        OP = taps_shape_out
        w = self.rd(op.w, ks * ks * Cin * OP).view(ks, ks, Cin, OP)[..., :Cout]
        if mag:
            w = w.abs()
        wt = w.permute(3, 2, 0, 1).contiguous()                     # OIHW
        y = F.conv2d(x.permute(0, 3, 1, 2), wt, None, padding=ks // 2)
        return y.permute(0, 2, 3, 1)

    def _fir_store(self, op, xc, dst, B, C, H, W, Hin, Win):
        if op.flags & (lib.F_UP | lib.F_DOWN):
            k1 = torch.tensor([1.0, 3.0, 3.0, 1.0], dtype=xc.dtype, device=xc.device)
            k2 = torch.outer(k1, k1) / 64.0
            xx = xc.reshape(B * C, 1, Hin, Win)
            if op.flags & lib.F_DOWN:
                y = F.conv2d(F.pad(xx, (1, 1, 1, 1)), k2.view(1, 1, 4, 4))[:, :, ::2, ::2]
            else:
                z = xx.new_zeros(B * C, 1, 2 * Hin, 2 * Win)
                z[:, :, ::2, ::2] = xx
                y = F.conv2d(F.pad(z, (2, 1, 2, 1)), (k2 * 4).view(1, 1, 4, 4))
            xc = y.reshape(B, C, H, W)
        self.get(dst, B * H * W * C).copy_(xc.permute(0, 2, 3, 1).reshape(-1))

    def _tile_stats(self, op):
        """epilogue statistics of the output the conv op just stored"""
        B, H, W, Cout = op.B, op.H, op.W, op.Cout
        pimg, nj, ntiles = tile_geometry(B, H, W, op.i0)
        y = self.get(op.dst, B * H * W * Cout).view(B, H, W, Cout)
        self.get(op.dst2, ntiles * nj * 2 * Cout, torch.int64).copy_(tile_stats(y, op.i0).reshape(-1))

    # -- ops ----------------------------------------------------------------------------------------
    def exec(self, op, magnitude=False):
        """Run one op.  magnitude=True evaluates instead the magnitude of its terms, the scale of its rounding error
        (the same op on absolute values: e.g. |f0| * (|act(norm(x))| * |w| + |bias| + |residual|) for a conv, with
        SILU_LIPSCHITZ in place of an output SiLU); for the kinds listed in MAGNITUDE_KINDS only."""
        k = op.kind
        B, H, W = op.B, op.H, op.W
        m = (lambda t: t.abs()) if magnitude else (lambda t: t)
        if magnitude:
            assert k in MAGNITUDE_KINDS, k
        if k == lib.OP_NCHW_TO_NHWC:
            a = self.rd(op.src0, B * op.C0 * H * W).view(B, op.C0, H, W)
            if op.C1 > 0:
                a = torch.cat([a, self.rd(op.src1, B * op.C1 * H * W).view(B, op.C1, H, W)], 1)
            a = a.permute(0, 2, 3, 1)
            pitch = op.Cout if op.Cout > 0 else a.shape[3]
            if pitch > a.shape[3]:
                a = F.pad(a, (0, pitch - a.shape[3]))
            self.get(op.dst, a.numel()).copy_(a.reshape(-1))
        elif k == lib.OP_NHWC_TO_NCHW:
            pitch = op.C1 if op.C1 > 0 else op.C0
            a = self.rd(op.src0, B * H * W * pitch).view(B, H, W, pitch)[..., :op.C0]
            self.get(op.dst, a.numel()).copy_(a.permute(0, 3, 1, 2).reshape(-1))
        elif k == lib.OP_TIMESTEP_EMBED:
            dim = op.Cout
            half = dim // 2
            t = self.rd(op.src0, B)
            f = self.rd(op.w, half)
            e = t[:, None] * f[None, :]
            if magnitude:                                           # sin/cos of an argument rounded to fp32
                e = torch.cat([e.abs() + 1, e.abs() + 1], 1)
            else:
                e = torch.cat([torch.sin(e), torch.cos(e)], 1)
            if dim % 2:
                e = F.pad(e, (0, 1))
            self.get(op.dst, B * dim).copy_(e.reshape(-1))
        elif k == lib.OP_LINEAR:
            x = self.rd(op.src0, B * op.C0).view(B, op.C0)
            if op.flags & lib.F_ACT_IN:
                x = silu(x)
            w = self.rd(op.w, op.Cout * op.C0).view(op.Cout, op.C0)
            y = F.linear(m(x), m(w), m(self.rd(op.bias, op.Cout)))
            if op.flags & lib.F_ACT_OUT:
                y = y * SILU_LIPSCHITZ if magnitude else silu(y)
            self.get(op.dst, B * op.Cout).copy_(y.reshape(-1))
        elif k == lib.OP_GN_PARTIAL:
            x = m(self._src(op, H, W).double())
            C = op.C0 + op.C1
            nchunk = op.i0
            ppc = -(-(H * W) // nchunk)
            x = x.view(B, H * W, C)
            out = self.get(op.dst, B * nchunk * C * 2, torch.float64).view(B, nchunk, C, 2)
            for c in range(nchunk):
                seg = x[:, c * ppc:(c + 1) * ppc]
                out[:, c, :, 0] = seg.sum(1)
                out[:, c, :, 1] = (seg * seg).sum(1)
        elif k == lib.OP_GN_FINALIZE:
            C, nchunk, cg = op.C0 + op.C1, op.i0, op.i1
            dev = self.tensors[op.dst].device

            def chan_sums(ptr, Cs, kind):
                """per (b, channel) sum / sum of squares as float64 [B, Cs, 2]"""
                if kind == 0:
                    return self.get(ptr, B * nchunk * Cs * 2, torch.float64).view(B, nchunk, Cs, 2).sum(1)
                pimg, nj, ntiles = tile_geometry(B, H, W, kind)
                st = self.get(ptr, ntiles * nj * 2 * Cs, torch.int64).view(ntiles, nj, 2, Cs).double()
                st[:, :, 1] += (st[:, :, 1] < 0) * 2.0 ** 64          # sums of squares are unsigned
                st = st * torch.tensor([2.0 ** -16, 2.0 ** -32], dtype=torch.float64, device=dev).view(1, 1, 2, 1)
                b, ok = tile_slots(B, H, W, kind, dev)
                out = torch.zeros(B, Cs, 2, dtype=torch.float64, device=dev)
                out.index_add_(0, b[ok], st[ok].transpose(1, 2))
                return out

            part = chan_sums(op.src0, op.C0, op.i4)
            if op.C1 > 0:
                part = torch.cat([part, chan_sums(op.src1, op.C1, op.i5)], dim=1)
            s = part.view(B, C // cg, cg, 2).sum(2)                 # [B, G, 2]
            cnt = H * W * cg
            mean = s[..., 0] / cnt
            var = (s[..., 1] / cnt - mean * mean).clamp_min(0)
            rstd = 1.0 / torch.sqrt(var + float(op.f0))
            mean_c = mean.to(self.cdt).repeat_interleave(cg, 1)
            rstd_c = rstd.to(self.cdt).repeat_interleave(cg, 1)
            G = torch.ones(B, C, dtype=self.cdt, device=dev)
            S = torch.zeros(B, C, dtype=self.cdt, device=dev)
            if op.aux0:
                if op.flags & lib.F_FILM:
                    if op.i2 == 0:          # batch stride 0: one shared FiLM row (uniform timestep)
                        film = self.rd(op.aux0)[None, :].expand(B, -1)
                    else:
                        film = self.rd(op.aux0, B * op.i2).view(B, op.i2)
                    G = 1.0 + film[:, op.i3:op.i3 + C]
                    S = film[:, op.i3 + C:op.i3 + 2 * C]
                else:
                    G = self.rd(op.aux0, C)[None].expand(B, C)
                    S = self.rd(op.aux1, C)[None].expand(B, C)
            tab = torch.stack([mean_c, rstd_c, G, S], dim=2)
            self.get(op.dst, B * C * 4).copy_(tab.reshape(-1))
            if op.dst2:                                             # planar table read by CONV_UMMA2
                self.get(op.dst2, B * 3 * C).copy_(torch.stack([mean_c, rstd_c * G, S], dim=1).reshape(-1))
        elif k == lib.OP_APPLY:
            Hin, Win = H, W
            if op.flags & lib.F_DOWN:
                Hin, Win = 2 * H, 2 * W
            if op.flags & lib.F_UP:
                Hin, Win = H // 2, W // 2
            x = self._src(op, Hin, Win)
            C = op.C0 + op.C1
            if op.dst2:
                self._fir_store(op, m(x).permute(0, 3, 1, 2), op.dst2, B, C, H, W, Hin, Win)
            if op.aux0:
                tab = self.rd(op.aux0, B * C * 4).view(B, 1, 1, C, 4)
                n = (x - tab[..., 0]) * tab[..., 1] if not magnitude else (x.abs() + tab[..., 0].abs()) * tab[..., 1]
                if op.aux1:
                    g = self.rd(op.aux1, B * Hin * Win * C).view(B, Hin, Win, C)
                    b = self.rd(op.aux2, B * Hin * Win * C).view(B, Hin, Win, C)
                    n = n * (1 + g) + b if not magnitude else n * (1 + g.abs()) + b.abs()
                n = n * m(tab[..., 2]) + m(tab[..., 3])
                if op.flags & lib.F_ACT_OUT:
                    n = n * SILU_LIPSCHITZ if magnitude else silu(n)
                x = n
            self._fir_store(op, m(x).permute(0, 3, 1, 2), op.dst, B, C, H, W, Hin, Win)
        elif k in (lib.OP_CONV_SIMT, lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
            x = self._src(op, H, W)
            C = op.C0 + op.C1
            if k in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
                OP = op.Cout
                scale, wscale = float(op.f0), float(op.f1)
                if op.aux1:
                    if k == lib.OP_CONV_UMMA2:                      # planar [B][3][C]: mean | rstd*G | S
                        t3 = self.rd(op.aux1, B * 3 * C).view(B, 3, 1, 1, C)
                        x = (x - t3[:, 0]) * t3[:, 1] + t3[:, 2]
                    else:
                        tab = self.rd(op.aux1, B * C * 4).view(B, 1, 1, C, 4)
                        x = ((x - tab[..., 0]) * tab[..., 1]) * tab[..., 2] + tab[..., 3]
                    if op.flags & lib.F_ACT_IN:
                        x = silu(x)
            else:
                OP = op.i1
                scale, wscale = float(op.f0), 1.0
            y = self._conv(op, m(x), OP, magnitude) * wscale
            if k in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2) and op.src2:
                # second K-segment: raw 1x1 conv of (src2|src3); its [1][C2+C3][Cout] weights follow the main ones
                Hs = H
                a2 = self.rd(op.src2, B * Hs * W * op.C2).view(B, Hs, W, op.C2)
                if op.C3 > 0:
                    a2 = torch.cat([a2, self.rd(op.src3, B * Hs * W * op.C3).view(B, Hs, W, op.C3)], 3)
                Cs = op.C2 + op.C3
                w_all = self.rd(op.w)
                n_main = op.i0 * op.i0 * C * op.Cout
                w2 = w_all[n_main:n_main + Cs * op.Cout].view(Cs, op.Cout)
                y = y + torch.einsum("bhwc,co->bhwo", m(a2), m(w2))
            y = y + m(self.rd(op.bias, op.Cout))
            if op.aux0:
                y = y + m(self.rd(op.aux0, B * H * W * op.Cout).view(B, H, W, op.Cout))
            y = y * (abs(scale) if magnitude else scale)
            if op.flags & lib.F_ACT_OUT:
                y = y * SILU_LIPSCHITZ if magnitude else silu(y)
            self.get(op.dst, y.numel()).copy_(y.reshape(-1))
            if k in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2) and op.dst2 and not magnitude:
                self._tile_stats(op)
        elif k == lib.OP_CONV_SMALLN:
            x = self.rd(op.src0, B * H * W * op.C0).view(B, H, W, op.C0)
            if op.aux0:
                tab = self.rd(op.aux0, B * op.C0 * 4).view(B, 1, 1, op.C0, 4)
                x = ((x - tab[..., 0]) * tab[..., 1]) * tab[..., 2] + tab[..., 3]
                if op.flags & lib.F_ACT_OUT:
                    x = silu(x)
            w = self.rd(op.w, 9 * op.C0 * op.i1).view(3, 3, op.C0, op.i1)[..., :op.Cout]
            y = F.conv2d(m(x).permute(0, 3, 1, 2), m(w).permute(3, 2, 0, 1).contiguous(),
                         m(self.rd(op.bias, op.Cout)), padding=1).permute(0, 2, 3, 1)
            self.get(op.dst, y.numel()).copy_(y.reshape(-1))
        elif k in (lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA):
            C, heads, d = op.C0, op.i0, op.i1
            T = H * W
            qkv = self.rd(op.src0, B * T * 3 * C).view(B, T, 3, heads, d)
            q, kk, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]          # [B, T, heads, d]
            if magnitude:
                # softmax(s) v moves by at most 2 max|ds| max|v| when the logits move by ds, and |ds| scales with the
                # logit magnitude scale * sum_d |q| |k|; the weighted sum itself with max|v|
                logit = torch.einsum("bthd,bshd->bhts", q.abs(), kk.abs()).amax(-1) * abs(float(op.f0))  # [B,h,T]
                vmax = v.abs().amax(dim=(1, 3))                                                         # [B,h]
                o = ((1 + 2 * logit) * vmax[:, :, None]).permute(0, 2, 1)[..., None].expand(B, T, heads, d)
                o = o.reshape(B, T, C)
            else:
                s = torch.einsum("bthd,bshd->bhts", q, kk) * float(op.f0)
                p = torch.softmax(s, dim=-1)
                o = torch.einsum("bhts,bshd->bthd", p, v).reshape(B, T, C)
            self.get(op.dst, o.numel()).copy_(o.reshape(-1))
        elif k == lib.OP_RESIZE_NEAREST:
            x = self.rd(op.src0, B * op.i0 * op.i1 * op.C0).view(B, op.i0, op.i1, op.C0).permute(0, 3, 1, 2)
            y = F.interpolate(x, size=(H, W), mode="nearest").permute(0, 2, 3, 1)
            self.get(op.dst, y.numel()).copy_(y.reshape(-1))
        elif k == lib.OP_DIFFUSION_UPDATE:
            C = op.C0
            xbuf = self.get(op.dst, B * C * H * W).view(B, C, H, W)
            x = m(xbuf.to(self.cdt))
            pitch = op.Cout if op.Cout > 0 else C
            eps = m(self.rd(op.src0, B * H * W * pitch).view(B, H, W, pitch)[..., :C].permute(0, 3, 1, 2))
            if magnitude:
                f = [abs(float(getattr(op, f"f{i}"))) for i in range(6)]
                x0 = f[0] * (x + f[1] * eps)
            else:
                f = [float(getattr(op, f"f{i}")) for i in range(6)]
                x0 = f[0] * (x - f[1] * eps)
                if op.flags & lib.F_CLIP:
                    x0 = x0.clamp(-1, 1)
            r = f[2] * x0 + f[3] * x
            if f[4] != 0.0:
                r = r + f[4] * eps
            if f[5] != 0.0:
                assert not (op.flags & lib.F_PHILOX), "interpreter has no Philox"
                r = r + f[5] * m(self.rd(op.src1, B * C * H * W).view(B, C, H, W))
            xbuf.copy_(r)
        elif k == lib.OP_COPY:
            n = op.i0
            self.get(op.dst, n).copy_(self.get(op.src0, n))
        else:
            raise NotImplementedError(f"op kind {k}")


# op kinds whose rounding error scales with the magnitude of their terms (Interpreter.exec(magnitude=True))
MAGNITUDE_KINDS = (lib.OP_TIMESTEP_EMBED, lib.OP_LINEAR, lib.OP_GN_PARTIAL, lib.OP_APPLY, lib.OP_CONV_SIMT,
                   lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2, lib.OP_CONV_SMALLN, lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA,
                   lib.OP_DIFFUSION_UPDATE)
