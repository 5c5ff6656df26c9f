"""CPU interpreter of McvdOp programs.  TEST INFRASTRUCTURE ONLY.

Executes the op arrays produced by ``mcvd_b200.program.Engine`` with plain torch fp32 on the CPU,
following the op semantics documented in ``include/mcvd_b200.h``.  It lets the ``-m "not gpu"`` suite
check the host-side lowering (module walk, skip stack, FiLM offsets, virtual concats, SPADE wiring,
sampler coefficient plumbing) against the oracle without a GPU.  It is NOT a fallback: the product
never imports it, and ``Engine`` refuses to run without the CUDA library unless a test passes an
explicit ``_test_backend``.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from mcvd_b200 import lib


def silu(x):
    return x * torch.sigmoid(x)


class Interpreter:
    def __init__(self):
        self.tensors = {}

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
        a = self.get(op.src0, B * Hin * Win * op.C0).view(B, Hin, Win, op.C0)
        if op.C1 > 0:
            b = self.get(op.src1, B * Hin * Win * op.C1).view(B, Hin, Win, op.C1)
            a = torch.cat([a, b], dim=3)
        return a

    def _conv(self, op, x, taps_shape_out):
        """x [B,H,W,Cin] NHWC; weights [taps][Cin][OP]; returns [B,H,W,Cout]"""
        B, H, W, Cin = x.shape
        ks, Cout = op.i0, op.Cout
        OP = taps_shape_out
        w = self.get(op.w, ks * ks * Cin * OP).view(ks, ks, Cin, OP)[..., :Cout]
        wt = w.permute(3, 2, 0, 1).contiguous()                     # OIHW
        y = F.conv2d(x.permute(0, 3, 1, 2), wt, None, padding=ks // 2)
        return y.permute(0, 2, 3, 1)

    def _fir_store(self, op, xc, dst, B, C, H, W, Hin, Win):
        if op.flags & (lib.F_UP | lib.F_DOWN):
            k1 = torch.tensor([1.0, 3.0, 3.0, 1.0])
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

    @staticmethod
    def _tile_geometry(B, H, W, ks):
        """(positions per image, image slots per 128-position tile, tiles) of the padded-flat position space of a
        CONV_UMMA2 of kernel size ks (csrc/conv_umma.cu)"""
        pimg = (H + 1) * (W + 1) if ks == 3 else H * W
        return pimg, 127 // pimg + 2, 2 * ((B * pimg + 255) // 256)

    def _tile_stats(self, op, y):
        """CONV_UMMA2 epilogue statistics: int64 [tiles][NJ][2][Cout] = sum, sum of squares of round(y * 2^16) over
        the rows of a 128-position tile that belong to one image"""
        B, H, W, Cout, ks = op.B, op.H, op.W, op.Cout, op.i0
        pimg, nj, ntiles = self._tile_geometry(B, H, W, ks)
        st = self.get(op.dst2, ntiles * nj * 2 * Cout, torch.int64).view(ntiles, nj, 2, Cout)
        st.zero_()
        xi = torch.round(y.double() * 65536.0).clamp(-(1 << 28), 1 << 28).to(torch.int64)
        yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
        r = ((yy + 1) * (W + 1) + xx + 1) if ks == 3 else (yy * W + xx)
        for b in range(B):
            q = (b * pimg + r).reshape(-1)
            t = q // 128
            jj = b - torch.clamp((t * 128) // pimg, max=B - 1)
            v = xi[b].reshape(H * W, Cout)
            st[:, :, 0].index_put_((t, jj), v, accumulate=True)
            st[:, :, 1].index_put_((t, jj), v * v, accumulate=True)

    # -- ops ----------------------------------------------------------------------------------------
    def exec(self, op):
        k = op.kind
        B, H, W = op.B, op.H, op.W
        if k == lib.OP_NCHW_TO_NHWC:
            a = self.get(op.src0, B * op.C0 * H * W).view(B, op.C0, H, W)
            if op.C1 > 0:
                a = torch.cat([a, self.get(op.src1, B * op.C1 * H * W).view(B, op.C1, H, W)], 1)
            a = a.permute(0, 2, 3, 1)
            pitch = op.Cout if op.Cout > 0 else a.shape[3]
            if pitch > a.shape[3]:
                a = F.pad(a, (0, pitch - a.shape[3]))
            self.get(op.dst, a.numel()).copy_(a.reshape(-1))
        elif k == lib.OP_NHWC_TO_NCHW:
            pitch = op.C1 if op.C1 > 0 else op.C0
            a = self.get(op.src0, B * H * W * pitch).view(B, H, W, pitch)[..., :op.C0]
            self.get(op.dst, a.numel()).copy_(a.permute(0, 3, 1, 2).reshape(-1))
        elif k == lib.OP_TIMESTEP_EMBED:
            dim = op.Cout
            half = dim // 2
            t = self.get(op.src0, B)
            f = self.get(op.w, half)
            e = t[:, None] * f[None, :]
            e = torch.cat([torch.sin(e), torch.cos(e)], 1)
            if dim % 2:
                e = F.pad(e, (0, 1))
            self.get(op.dst, B * dim).copy_(e.reshape(-1))
        elif k == lib.OP_LINEAR:
            x = self.get(op.src0, B * op.C0).view(B, op.C0)
            if op.flags & lib.F_ACT_IN:
                x = silu(x)
            w = self.get(op.w, op.Cout * op.C0).view(op.Cout, op.C0)
            y = F.linear(x, w, self.get(op.bias, op.Cout))
            if op.flags & lib.F_ACT_OUT:
                y = silu(y)
            self.get(op.dst, B * op.Cout).copy_(y.reshape(-1))
        elif k == lib.OP_GN_PARTIAL:
            x = self._src(op, H, W).double()
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

            def chan_sums(ptr, Cs, kind):
                """per (b, channel) sum / sum of squares as float64 [B, Cs, 2]"""
                if kind == 0:
                    return self.get(ptr, B * nchunk * Cs * 2, torch.float64).view(B, nchunk, Cs, 2).sum(1)
                pimg, nj, ntiles = self._tile_geometry(B, H, W, kind)
                st = self.get(ptr, ntiles * nj * 2 * Cs, torch.int64).view(ntiles, nj, 2, Cs)
                out = torch.zeros(B, Cs, 2, dtype=torch.float64)
                for b in range(B):
                    for t in range((b * pimg) // 128, ((b + 1) * pimg - 1) // 128 + 1):
                        jj = b - min(B - 1, (t * 128) // pimg)
                        out[b, :, 0] += st[t, jj, 0].double() / 65536.0
                        out[b, :, 1] += st[t, jj, 1].double() / 4294967296.0
                return out

            part = chan_sums(op.src0, op.C0, op.i4)
            if op.C1 > 0:
                part = torch.cat([part, chan_sums(op.src1, op.C1, op.i5)], dim=1)
            s = part.view(B, C // cg, cg, 2).sum(2)                 # [B, G, 2]
            cnt = H * W * cg
            mean = s[..., 0] / cnt
            var = (s[..., 1] / cnt - mean * mean).clamp_min(0)
            rstd = 1.0 / torch.sqrt(var + float(op.f0))
            mean_c = mean.float().repeat_interleave(cg, 1)
            rstd_c = rstd.float().repeat_interleave(cg, 1)
            G = torch.ones(B, C)
            S = torch.zeros(B, C)
            if op.aux0:
                if op.flags & lib.F_FILM:
                    if op.i2 == 0:          # batch stride 0: one shared FiLM row (uniform timestep)
                        film = self.get(op.aux0)[None, :].expand(B, -1)
                    else:
                        film = self.get(op.aux0, B * op.i2).view(B, op.i2)
                    G = 1.0 + film[:, op.i3:op.i3 + C]
                    S = film[:, op.i3 + C:op.i3 + 2 * C]
                else:
                    G = self.get(op.aux0, C)[None].expand(B, C)
                    S = self.get(op.aux1, C)[None].expand(B, C)
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
                self._fir_store(op, x.permute(0, 3, 1, 2), op.dst2, B, C, H, W, Hin, Win)
            if op.aux0:
                tab = self.get(op.aux0, B * C * 4).view(B, 1, 1, C, 4)
                n = (x - tab[..., 0]) * tab[..., 1]
                if op.aux1:
                    g = self.get(op.aux1, B * Hin * Win * C).view(B, Hin, Win, C)
                    b = self.get(op.aux2, B * Hin * Win * C).view(B, Hin, Win, C)
                    n = n * (1 + g) + b
                n = n * tab[..., 2] + tab[..., 3]
                if op.flags & lib.F_ACT_OUT:
                    n = silu(n)
                x = n
            self._fir_store(op, x.permute(0, 3, 1, 2), op.dst, B, C, H, W, Hin, Win)
        elif k in (lib.OP_CONV_SIMT, lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
            x = self._src(op, H, W)
            C = op.C0 + op.C1
            if k in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
                OP = op.Cout
                scale, wscale = float(op.f0), float(op.f1)
                if op.aux1:
                    if k == lib.OP_CONV_UMMA2:                      # planar [B][3][C]: mean | rstd*G | S
                        t3 = self.get(op.aux1, B * 3 * C).view(B, 3, 1, 1, C)
                        x = (x - t3[:, 0]) * t3[:, 1] + t3[:, 2]
                    else:
                        tab = self.get(op.aux1, B * C * 4).view(B, 1, 1, C, 4)
                        x = ((x - tab[..., 0]) * tab[..., 1]) * tab[..., 2] + tab[..., 3]
                    if op.flags & lib.F_ACT_IN:
                        x = silu(x)
            else:
                OP = op.i1
                scale, wscale = float(op.f0), 1.0
            y = self._conv(op, x, OP) * wscale
            if k in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2) and op.src2:
                # second K-segment: raw 1x1 conv of (src2|src3); its [1][C2+C3][Cout] weights follow the main ones
                Hs = H
                a2 = self.get(op.src2, B * Hs * W * op.C2).view(B, Hs, W, op.C2)
                if op.C3 > 0:
                    a2 = torch.cat([a2, self.get(op.src3, B * Hs * W * op.C3).view(B, Hs, W, op.C3)], 3)
                Cs = op.C2 + op.C3
                w_all = self.get(op.w)
                n_main = op.i0 * op.i0 * C * op.Cout
                w2 = w_all[n_main:n_main + Cs * op.Cout].view(Cs, op.Cout)
                y = y + torch.einsum("bhwc,co->bhwo", a2, w2)
            y = y + self.get(op.bias, op.Cout)
            if op.aux0:
                y = y + self.get(op.aux0, B * H * W * op.Cout).view(B, H, W, op.Cout)
            y = y * scale
            if op.flags & lib.F_ACT_OUT:
                y = silu(y)
            self.get(op.dst, y.numel()).copy_(y.reshape(-1))
            if k in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2) and op.dst2:
                self._tile_stats(op, y.reshape(B, H, W, op.Cout))
        elif k == lib.OP_CONV_SMALLN:
            x = self.get(op.src0, B * H * W * op.C0).view(B, H, W, op.C0)
            if op.aux0:
                tab = self.get(op.aux0, B * op.C0 * 4).view(B, 1, 1, op.C0, 4)
                x = ((x - tab[..., 0]) * tab[..., 1]) * tab[..., 2] + tab[..., 3]
                if op.flags & lib.F_ACT_OUT:
                    x = silu(x)
            op_ = op
            w = self.get(op.w, 9 * op.C0 * op.i1).view(3, 3, op.C0, op.i1)[..., :op.Cout]
            y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1).contiguous(), self.get(op_.bias, op.Cout),
                         padding=1).permute(0, 2, 3, 1)
            self.get(op.dst, y.numel()).copy_(y.reshape(-1))
        elif k in (lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA):
            C, heads, d = op.C0, op.i0, op.i1
            T = H * W
            qkv = self.get(op.src0, B * T * 3 * C).view(B, T, 3, heads, d)
            q, kk, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]          # [B, T, heads, d]
            s = torch.einsum("bthd,bshd->bhts", q, kk) * float(op.f0)
            p = torch.softmax(s, dim=-1)
            o = torch.einsum("bhts,bshd->bthd", p, v).reshape(B, T, C)
            self.get(op.dst, o.numel()).copy_(o.reshape(-1))
        elif k == lib.OP_RESIZE_NEAREST:
            x = self.get(op.src0, B * op.i0 * op.i1 * op.C0).view(B, op.i0, op.i1, op.C0).permute(0, 3, 1, 2)
            y = F.interpolate(x, size=(H, W), mode="nearest").permute(0, 2, 3, 1)
            self.get(op.dst, y.numel()).copy_(y.reshape(-1))
        elif k == lib.OP_DIFFUSION_UPDATE:
            C = op.C0
            x = self.get(op.dst, B * C * H * W).view(B, C, H, W)
            pitch = op.Cout if op.Cout > 0 else C
            eps = self.get(op.src0, B * H * W * pitch).view(B, H, W, pitch)[..., :C].permute(0, 3, 1, 2)
            x0 = op.f0 * (x - op.f1 * eps)
            if op.flags & lib.F_CLIP:
                x0 = x0.clamp(-1, 1)
            r = op.f2 * x0 + op.f3 * x
            if op.f4 != 0.0:
                r = r + op.f4 * eps
            if op.f5 != 0.0:
                assert not (op.flags & lib.F_PHILOX), "interpreter has no Philox"
                r = r + op.f5 * self.get(op.src1, B * C * H * W).view(B, C, H, W)
            x.copy_(r)
        elif k == lib.OP_COPY:
            n = op.i0
            self.get(op.dst, n).copy_(self.get(op.src0, n))
        else:
            raise NotImplementedError(f"op kind {k}")
