"""Per-kernel parity on the H100, through the C-ABI: every op kind against a torch fp32 CPU evaluation
of the same op (tests/op_interpreter.py semantics == include/mcvd_b200.h)."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from mcvd_b200 import lib
from mcvd_b200.lib import McvdOp

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return (torch.randn(*shape, generator=g) * scale)


def mk(kind, B, **kw):
    o = McvdOp()
    o.kind, o.B = kind, B
    for k, v in kw.items():
        setattr(o, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return o


def make_table(B, C, seed=3):
    tab = torch.stack([rnd(B, C, seed=seed) * 0.3, 0.5 + torch.rand(B, C), 1 + 0.3 * rnd(B, C, seed=seed + 1),
                       0.2 * rnd(B, C, seed=seed + 2)], dim=2).contiguous()
    return tab


def ref_norm(x_nhwc, tab, act):
    t = tab.view(tab.shape[0], 1, 1, tab.shape[1], 4)
    y = ((x_nhwc - t[..., 0]) * t[..., 1]) * t[..., 2] + t[..., 3]
    return y * torch.sigmoid(y) if act else y


def conv_ref(x_nhwc, w_oihw, bias, res, scale, act_out):
    y = F.conv2d(x_nhwc.permute(0, 3, 1, 2).double(), w_oihw.double(), bias.double(),
                 padding=w_oihw.shape[-1] // 2).permute(0, 2, 3, 1)
    if res is not None:
        y = y + res.double()
    y = y * scale
    if act_out:
        y = y * torch.sigmoid(y)
    return y.float()


def taps_of(w):
    O, I, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw, I, O).contiguous()


CONV_CASES = [
    # B, H, C0, C1, Cout, ks, tab, act_in, res, act_out
    (2, 8, 32, 0, 32, 3, False, False, False, False),
    (2, 16, 32, 0, 64, 3, True, True, True, False),
    (3, 8, 64, 32, 96, 3, True, True, True, False),
    (2, 32, 32, 0, 32, 3, True, True, False, False),
    (1, 64, 32, 0, 48, 3, False, False, False, True),
    (2, 16, 48, 48, 144, 3, True, True, True, False),      # KB = 16 path
    (2, 16, 64, 0, 192, 1, True, False, False, False),     # 1x1 (qkv-like)
    (2, 8, 96, 0, 96, 1, False, False, True, False),
    (4, 8, 128, 128, 256, 3, True, True, True, False),
    (2, 16, 32, 0, 512, 3, False, False, False, False),    # two n tiles of 256
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("kind", ["simt", "umma"])
def test_conv(case, kind):
    B, H, C0, C1, Cout, ks, use_tab, act_in, use_res, act_out = case
    Cin = C0 + C1
    x0 = rnd(B, H, H, C0, seed=1)
    x1 = rnd(B, H, H, C1, seed=2) if C1 else None
    w = rnd(Cout, Cin, ks, ks, seed=5) / math.sqrt(Cin * ks * ks)
    bias = rnd(Cout, seed=6) * 0.1
    res = rnd(B, H, H, Cout, seed=7) if use_res else None
    tab = make_table(B, Cin) if use_tab else None
    scale = 0.7071
    xin = x0 if x1 is None else torch.cat([x0, x1], 3)
    xa = ref_norm(xin, tab, act_in) if use_tab else xin
    ref = conv_ref(xa, w, bias, res, scale, act_out)

    d = lambda t: None if t is None else t.to(DEV).contiguous()
    x0d, x1d, bd, rd, td = d(x0), d(x1), d(bias), d(res), d(tab)
    out = torch.zeros(B, H, H, Cout, device=DEV)
    taps = taps_of(w).to(DEV)
    ops = []
    if kind == "simt":
        src0, src1, c0, c1 = x0d, x1d, C0, C1
        if use_tab:
            a = torch.empty(B, H, H, Cin, device=DEV)
            ops.append(mk(lib.OP_APPLY, B, H=H, W=H, C0=C0, C1=C1, src0=x0d, src1=x1d, aux0=td, dst=a,
                          flags=lib.F_ACT_OUT if act_in else 0))
            src0, src1, c0, c1 = a, None, Cin, 0
        ops.append(mk(lib.OP_CONV_SIMT, B, H=H, W=H, C0=c0, C1=c1, Cout=Cout, i0=ks, i1=Cout, f0=scale, src0=src0,
                      src1=src1, w=taps, bias=bd, aux0=rd, dst=out, flags=lib.F_ACT_OUT if act_out else 0))
    else:
        kb = lib.umma_kblock(C0, C1)
        assert kb in (16, 32)
        nt = max(dd for dd in range(16, 257, 16) if Cout % dd == 0)
        pk = torch.empty(taps.numel() * 4, dtype=torch.uint8, device=DEV)
        k = int(math.floor(math.log2(512.0 / float(taps.abs().max()))))
        rc = lib.load().mcvd_umma_pack_weights(taps.data_ptr(), ks * ks, Cin, Cout, nt, kb, pk.data_ptr(), k,
                                               torch.cuda.current_stream().cuda_stream)
        assert rc > 0, lib.last_error()
        from test_gpu_conv2 import expected_stats
        pimg = (H + 1) * (H + 1) if ks == 3 else H * H
        for nacc in (1, 2):
            out.zero_()
            fl = (lib.F_ACT_IN if act_in else 0) | (lib.F_ACT_OUT if act_out else 0)
            # epilogue GroupNorm statistics (exact integers of the stored output), when the maps are large enough
            st = torch.full((lib.umma2_stats_bytes(B, H, H, ks, Cout) // 8,), -7, dtype=torch.int64,
                            device=DEV) if pimg >= 64 else None
            run([mk(lib.OP_CONV_UMMA, B, H=H, W=H, C0=C0, C1=C1, Cout=Cout, i0=ks, i1=nt, i2=nacc, f0=scale,
                    f1=2.0 ** (-k), src0=x0d, src1=x1d, w=pk, bias=bd, aux0=rd, aux1=td, dst=out, dst2=st, flags=fl)])
            err = (out.cpu() - ref).abs().max().item()
            assert err < 2e-5 * max(1.0, ref.abs().max().item()), (case, nacc, err)
            if st is not None:
                exp = expected_stats(out.cpu(), ks)
                ntile = -(-(B * pimg) // 128)          # 128-position tiles that hold positions (the array is sized in pairs)
                assert torch.equal(st.cpu().view(exp.shape)[:ntile], exp[:ntile]), (case, nacc)
        return
    run(ops)
    err = (out.cpu() - ref).abs().max().item()
    assert err < 2e-5 * max(1.0, ref.abs().max().item()), (case, err)


@pytest.mark.parametrize("B,H,C0,C1", [(2, 16, 32, 0), (3, 8, 96, 48), (2, 32, 64, 64), (1, 8, 768, 768)])
def test_groupnorm_table(B, H, C0, C1):
    from mcvd_b200.arch import num_groups
    C = C0 + C1
    x0 = rnd(B, H, H, C0, seed=1) * 2 + 0.5
    x1 = rnd(B, H, H, C1, seed=2) if C1 else None
    film = rnd(B, 3 * C + 5, seed=3)
    off = 5
    cg = C // num_groups(C)
    nchunk = max(1, H * H // 64)
    x = x0 if x1 is None else torch.cat([x0, x1], 3)
    xg = x.permute(0, 3, 1, 2).reshape(B, C // cg, cg * H * H).double()
    mean, var = xg.mean(2), xg.var(2, unbiased=False)
    rstd = 1 / torch.sqrt(var + 1e-5)
    ref = torch.stack([mean.float().repeat_interleave(cg, 1), rstd.float().repeat_interleave(cg, 1),
                       1 + film[:, off:off + C], film[:, off + C:off + 2 * C]], 2)
    d = lambda t: None if t is None else t.to(DEV).contiguous()
    part = torch.zeros(B * nchunk * C * 2, dtype=torch.float64, device=DEV)
    tab = torch.zeros(B, C, 4, device=DEV)
    x0d, x1d, fd = d(x0), d(x1), d(film)
    run([mk(lib.OP_GN_PARTIAL, B, H=H, W=H, C0=C0, C1=C1, i0=nchunk, src0=x0d, src1=x1d, dst=part),
         mk(lib.OP_GN_FINALIZE, B, H=H, W=H, C0=C, i0=nchunk, i1=cg, f0=1e-5, src0=part, dst=tab, aux0=fd,
            i2=film.shape[1], i3=off, flags=lib.F_FILM)])
    assert (tab.cpu() - ref).abs().max().item() < 2e-5
    if C1:
        # per-tensor partials (what the lowering emits): one scan per tensor, finalize reads both arrays
        pa = torch.zeros(B * nchunk * C0 * 2, dtype=torch.float64, device=DEV)
        pb = torch.zeros(B * nchunk * C1 * 2, dtype=torch.float64, device=DEV)
        tab2 = torch.zeros(B, C, 4, device=DEV)
        run([mk(lib.OP_GN_PARTIAL, B, H=H, W=H, C0=C0, i0=nchunk, src0=x0d, dst=pa),
             mk(lib.OP_GN_PARTIAL, B, H=H, W=H, C0=C1, i0=nchunk, src0=x1d, dst=pb),
             mk(lib.OP_GN_FINALIZE, B, H=H, W=H, C0=C0, C1=C1, i0=nchunk, i1=cg, f0=1e-5, src0=pa, src1=pb, dst=tab2,
                aux0=fd, i2=film.shape[1], i3=off, flags=lib.F_FILM)])
        assert torch.equal(tab2, tab)


def test_groupnorm_partials_are_float64():
    """|mean| >> std: the variance E[x^2] - mean^2 keeps its bits only if every partial sum is fp64 (sums of 8 pixels
    in fp32 were 2^-24 relative, which cost rstd its leading digits here)"""
    B, H, C, nchunk = 2, 16, 32, 4
    x = 300.0 + rnd(B, H, H, C, seed=4) * 0.01
    part = torch.zeros(B * nchunk * C * 2, dtype=torch.float64, device=DEV)
    run([mk(lib.OP_GN_PARTIAL, B, H=H, W=H, C0=C, i0=nchunk, src0=x.to(DEV).contiguous(), dst=part)])
    xd = x.double().view(B, nchunk, H * H // nchunk, C)
    ref = torch.stack([xd.sum(2), (xd * xd).sum(2)], 3).reshape(-1)
    assert ((part.cpu() - ref).abs() <= 1e-12 * ref).all()


@pytest.mark.parametrize("mode", ["none", "down", "up"])
@pytest.mark.parametrize("spade", [False, True])
@pytest.mark.parametrize("B,Hin,C0,C1", [(2, 16, 32, 16),     # 48 channels: a full and a half 32-channel chunk
                                         (3, 6, 8, 4),        # tiles larger than the image, odd output size (down -> 3)
                                         (1, 36, 64, 0)])     # several tiles with a ragged edge, single source
def test_apply_fir(mode, spade, B, Hin, C0, C1):
    from oracle import mcvd_oracle as O
    C = C0 + C1
    x0 = rnd(B, Hin, Hin, C0, seed=1)
    x1 = rnd(B, Hin, Hin, C1, seed=2) if C1 else torch.zeros(B, Hin, Hin, 0)
    tab = make_table(B, C)
    gam, bet = rnd(B, Hin, Hin, C, seed=8) * 0.2, rnd(B, Hin, Hin, C, seed=9) * 0.2
    x = torch.cat([x0, x1], 3)
    t = tab.view(B, 1, 1, C, 4)
    n = (x - t[..., 0]) * t[..., 1]
    if spade:
        n = n * (1 + gam) + bet
    n = n * t[..., 2] + t[..., 3]
    n = (n * torch.sigmoid(n)).permute(0, 3, 1, 2)
    raw = x.permute(0, 3, 1, 2)
    H = Hin
    fl = 0
    if mode == "down":
        n, raw, H, fl = O.fir_downsample(n), O.fir_downsample(raw), Hin // 2, lib.F_DOWN
    elif mode == "up":
        n, raw, H, fl = O.fir_upsample(n), O.fir_upsample(raw), Hin * 2, lib.F_UP
    d = lambda t_: t_.to(DEV).contiguous()
    x0d, x1d, td, gd, bd = d(x0), (d(x1) if C1 else None), d(tab), d(gam), d(bet)
    o1 = torch.zeros(B, H, H, C, device=DEV)
    o2 = torch.zeros(B, H, H, C, device=DEV)
    o3 = torch.zeros(B, H, H, C, device=DEV)
    run([mk(lib.OP_APPLY, B, H=H, W=H, C0=C0, C1=C1, src0=x0d, src1=x1d, aux0=td, aux1=gd if spade else None,
            aux2=bd if spade else None, dst=o1, dst2=o3, flags=lib.F_ACT_OUT | fl),      # fused dual output
         mk(lib.OP_APPLY, B, H=H, W=H, C0=C0, C1=C1, src0=x0d, src1=x1d, dst=o2, flags=fl)])
    assert torch.equal(o2, o3)
    assert (o1.cpu() - n.permute(0, 2, 3, 1)).abs().max().item() < 1e-5
    assert (o2.cpu() - raw.permute(0, 2, 3, 1)).abs().max().item() < 1e-5


@pytest.mark.parametrize("B,H,heads,d", [(2, 8, 1, 32), (2, 16, 2, 48), (1, 32, 2, 96), (2, 8, 4, 96), (1, 16, 1, 192),
                                         (2, 16, 2, 64), (1, 16, 1, 128), (2, 32, 2, 192), (2, 8, 3, 192)])
@pytest.mark.parametrize("kind", ["simt", "umma"])
def test_attention(B, H, heads, d, kind):
    if kind == "umma" and d not in (32, 48, 64, 96, 128, 192):
        pytest.skip("tensor-core attention supports head dims 32..192")
    C, T = heads * d, H * H
    qkv = rnd(B, T, 3 * C, seed=4)
    scale = float(int(d) ** (-0.5))
    q, k, v = qkv.view(B, T, 3, heads, d).unbind(2)
    s = torch.einsum("bthd,bshd->bhts", q.double(), k.double()) * scale
    ref = torch.einsum("bhts,bshd->bthd", torch.softmax(s, -1), v.double()).reshape(B, T, C).float()
    qd = qkv.to(DEV)
    out = torch.zeros(B, T, C, device=DEV)
    if kind == "simt":
        run([mk(lib.OP_ATTENTION, B, H=H, W=H, C0=C, i0=heads, i1=d, f0=scale, src0=qd, dst=out)])
    else:
        scratch = torch.empty(lib.attention_scratch_bytes(B, T, C), dtype=torch.uint8, device=DEV)
        assert scratch.numel() == 4 * B * C * (-(-T // 128) * 128 + 2 * T)
        op = mk(lib.OP_ATTENTION_UMMA, B, H=H, W=H, C0=C, i0=heads, i1=d, f0=scale, src0=qd, dst=out, dst2=scratch)
        assert lib.load().mcvd_count_launches(ctypes.byref(op), 1) == 2        # pre-split + attention
        run([op])
    assert (out.cpu() - ref).abs().max().item() < 2e-5


def test_linear_embed_layout_update():
    B, nf = 5, 32
    t = torch.tensor([0.0, 10.0, 500.5, 990.0, 99.0])
    half = nf // 2
    freqs = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
    e_ref = torch.cat([torch.sin(t[:, None] * freqs), torch.cos(t[:, None] * freqs)], 1)
    w, b = rnd(48, nf, seed=1) * 0.2, rnd(48, seed=2)
    y_ref = F.silu(F.linear(e_ref, w, b))
    td, fd, wd, bd = t.to(DEV), freqs.to(DEV), w.to(DEV), b.to(DEV)
    e = torch.zeros(B, nf, device=DEV)
    y = torch.zeros(B, 48, device=DEV)
    run([mk(lib.OP_TIMESTEP_EMBED, B, Cout=nf, src0=td, w=fd, dst=e),
         mk(lib.OP_LINEAR, B, C0=nf, Cout=48, src0=e, w=wd, bias=bd, dst=y, flags=lib.F_ACT_OUT)])
    assert (e.cpu() - e_ref).abs().max().item() < 2e-6
    assert (y.cpu() - y_ref).abs().max().item() < 1e-5
    # single-row GEMV path (uniform-timestep sampling: the FiLM projection of one temb row), K % 4 == 0 and not
    for K in (384, 30):
        xs, ws, bs = rnd(1, K, seed=5), rnd(77, K, seed=6) * 0.1, rnd(77, seed=7)
        ys_ref = F.linear(F.silu(xs), ws, bs)
        ys = torch.zeros(1, 77, device=DEV)
        run([mk(lib.OP_LINEAR, 1, C0=K, Cout=77, src0=xs.to(DEV), w=ws.to(DEV).contiguous(), bias=bs.to(DEV), dst=ys,
                flags=lib.F_ACT_IN)])
        assert (ys.cpu() - ys_ref).abs().max().item() < 1e-5
    # batched rows (per-clip timesteps): staged-activation kernel; a row equals the single-row evaluation bit for bit
    Bb, K, N = 37, 384, 203
    xb, wb, bb = rnd(Bb, K, seed=8), rnd(N, K, seed=9) * 0.1, rnd(N, seed=10)
    yb_ref = F.silu(F.linear(F.silu(xb), wb, bb))
    xbd, wbd, bbd = xb.to(DEV), wb.to(DEV).contiguous(), bb.to(DEV)
    yb = torch.zeros(Bb, N, device=DEV)
    run([mk(lib.OP_LINEAR, Bb, C0=K, Cout=N, src0=xbd, w=wbd, bias=bbd, dst=yb, flags=lib.F_ACT_IN | lib.F_ACT_OUT)])
    assert (yb.cpu() - yb_ref).abs().max().item() < 1e-5
    y1 = torch.zeros(1, N, device=DEV)
    run([mk(lib.OP_LINEAR, 1, C0=K, Cout=N, src0=xbd[20:21].contiguous(), w=wbd, bias=bbd, dst=y1,
            flags=lib.F_ACT_IN | lib.F_ACT_OUT)])
    assert torch.equal(y1[0], yb[20])
    # layout round trip + diffusion update
    B, C, S = 2, 5, 16
    x, c = rnd(B, C, S, S, seed=3), rnd(B, 3, S, S, seed=4)
    xd, cd = x.to(DEV), c.to(DEV)
    nhwc = torch.zeros(B, S, S, C + 3, device=DEV)
    run([mk(lib.OP_NCHW_TO_NHWC, B, H=S, W=S, C0=C, C1=3, src0=xd, src1=cd, dst=nhwc)])
    assert torch.equal(nhwc.cpu(), torch.cat([x, c], 1).permute(0, 2, 3, 1))
    eps = rnd(B, S, S, C, seed=5)
    z = rnd(B, C, S, S, seed=6)
    k0, k1, ca, cb, cc, sg = 1.3, 0.4, 0.6, 0.35, 0.0, 0.2
    x0 = (k0 * (x - k1 * eps.permute(0, 3, 1, 2))).clamp(-1, 1)
    ref = ca * x0 + cb * x + sg * z
    ed, zd = eps.to(DEV), z.to(DEV)
    run([mk(lib.OP_DIFFUSION_UPDATE, B, H=S, W=S, C0=C, f0=k0, f1=k1, f2=ca, f3=cb, f4=cc, f5=sg, src0=ed, src1=zd,
            dst=xd, flags=lib.F_CLIP)])
    assert (xd.cpu() - ref).abs().max().item() < 1e-5
    back = torch.zeros(B, C, S, S, device=DEV)
    run([mk(lib.OP_NHWC_TO_NCHW, B, H=S, W=S, C0=C, src0=ed, dst=back)])
    assert torch.equal(back.cpu(), eps.permute(0, 3, 1, 2))


def test_philox_noise_statistics_and_sharding_invariance():
    B, C, S = 4, 5, 64
    x = torch.zeros(B, C, S, S, device=DEV)
    eps = torch.zeros(B, S, S, C, device=DEV)
    run([mk(lib.OP_DIFFUSION_UPDATE, B, H=S, W=S, C0=C, f3=1.0, f5=1.0, src0=eps, dst=x, flags=lib.F_PHILOX, i0=1234,
            i1=0, i2=0, i3=7)])
    z = x.cpu()
    assert abs(z.mean().item()) < 0.02 and abs(z.std().item() - 1.0) < 0.02
    assert abs((z ** 4).mean().item() - 3.0) < 0.2
    # clips 2..3 drawn as a separate shard (clip offset 2) must equal rows 2..3 of the full batch
    x2 = torch.zeros(2, C, S, S, device=DEV)
    run([mk(lib.OP_DIFFUSION_UPDATE, 2, H=S, W=S, C0=C, f3=1.0, f5=1.0, src0=eps, dst=x2, flags=lib.F_PHILOX, i0=1234,
            i1=0, i2=2, i3=7)])
    assert torch.equal(x2.cpu(), z[2:4])


def test_resize_and_smalln():
    B, S, C = 2, 32, 10
    x = rnd(B, S, S, C, seed=1)
    xd = x.to(DEV)
    for H in (16, 8, 32):
        out = torch.zeros(B, H, H, C, device=DEV)
        run([mk(lib.OP_RESIZE_NEAREST, B, H=H, W=H, C0=C, i0=S, i1=S, src0=xd, dst=out)])
        ref = F.interpolate(x.permute(0, 3, 1, 2), size=(H, H), mode="nearest").permute(0, 2, 3, 1)
        assert torch.equal(out.cpu(), ref)
    Cin, Cout = 32, 5
    x = rnd(B, S, S, Cin, seed=2)
    tab = make_table(B, Cin)
    w = rnd(Cout, Cin, 3, 3, seed=3) / math.sqrt(9 * Cin)
    bias = rnd(Cout, seed=4)
    ref = conv_ref(ref_norm(x, tab, True), w, bias, None, 1.0, False)
    taps = taps_of(w)
    tp = torch.zeros(9, Cin, 8)
    tp[:, :, :Cout] = taps
    xd, td, wd, bd = x.to(DEV), tab.to(DEV), tp.to(DEV), bias.to(DEV)
    out = torch.zeros(B, S, S, Cout, device=DEV)
    run([mk(lib.OP_CONV_SMALLN, B, H=S, W=S, C0=Cin, Cout=Cout, i1=8, src0=xd, w=wd, bias=bd, aux0=td, dst=out,
            flags=lib.F_ACT_OUT)])
    assert (out.cpu() - ref).abs().max().item() < 2e-5


FUSED_CASES = [
    # B, H, Cmain, Cout, Cs0, Cs1   (main: 3x3 on act(norm(h)); shortcut: raw 1x1 on (x0|x1), fused as 2nd K-segment)
    (2, 16, 64, 64, 32, 0),        # shortcut of a single K-block (table-buffer hazard case)
    (2, 8, 96, 96, 96, 96),        # concat shortcut source
    (3, 16, 48, 48, 48, 48),       # KB = 16
    (2, 32, 32, 96, 64, 0),
    (2, 8, 128, 256, 128, 64),
]


@pytest.mark.parametrize("case", FUSED_CASES)
def test_conv_umma_fused_shortcut(case):
    B, H, Cm, Cout, Cs0, Cs1 = case
    Cs = Cs0 + Cs1
    h = rnd(B, H, H, Cm, seed=1)
    x0 = rnd(B, H, H, Cs0, seed=2)
    x1 = rnd(B, H, H, Cs1, seed=3) if Cs1 else None
    w1 = rnd(Cout, Cm, 3, 3, seed=4) / math.sqrt(9 * Cm)
    w2 = rnd(Cout, Cs, 1, 1, seed=5) / math.sqrt(Cs)
    b1, b2 = rnd(Cout, seed=6) * 0.1, rnd(Cout, seed=7) * 0.1
    tab = make_table(B, Cm)
    xs = x0 if x1 is None else torch.cat([x0, x1], 3)
    ref = conv_ref(ref_norm(h, tab, True), w1, b1, None, 1.0, False) + conv_ref(xs, w2, b2, None, 1.0, False)
    ref = ref * 0.7071
    kb = min(lib.umma_kblock(Cm, 0), lib.umma_kblock(Cs0, Cs1))
    nt = max(dd for dd in range(16, 257, 16) if Cout % dd == 0)
    t1, t2 = taps_of(w1).to(DEV), taps_of(w2).to(DEV)
    k = int(math.floor(math.log2(512.0 / float(max(t1.abs().max(), t2.abs().max())))))
    parts = []
    for t in (t1, t2):
        pk = torch.empty(t.numel() * 4, dtype=torch.uint8, device=DEV)
        rc = lib.load().mcvd_umma_pack_weights(t.data_ptr(), t.shape[0], t.shape[1], Cout, nt, kb, pk.data_ptr(), k,
                                               torch.cuda.current_stream().cuda_stream)
        assert rc > 0, lib.last_error()
        parts.append(pk.view(Cout // nt, -1))
    wpk = torch.cat(parts, 1).contiguous().view(-1)
    d = lambda t: None if t is None else t.to(DEV).contiguous()
    hd, x0d, x1d, td, bd = d(h), d(x0), d(x1), d(tab), d(b1 + b2)
    out = torch.zeros(B, H, H, Cout, device=DEV)
    for nacc in (0, 1, 2):
        out.zero_()
        run([mk(lib.OP_CONV_UMMA, B, H=H, W=H, C0=Cm, Cout=Cout, i0=3, i1=nt, i2=nacc, f0=0.7071, f1=2.0 ** (-k),
                src0=hd, w=wpk, bias=bd, aux1=td, dst=out, flags=lib.F_ACT_IN, src2=x0d, src3=x1d, C2=Cs0, C3=Cs1)])
        err = (out.cpu() - ref).abs().max().item()
        assert err < 2e-5 * max(1.0, ref.abs().max().item()), (case, nacc, err)


@pytest.mark.parametrize("B,C,nf,S,rnd", [(3, 1, 4, 64, True), (2, 3, 2, 64, False), (1, 3, 2, 128, False), (2, 1, 3, 32, False)])
def test_frame_metrics_vs_oracle(B, C, nf, S, rnd):
    """MCVD_OP_FRAME_METRICS (per-frame MSE + SSIM of generated clips) against the CPU restatement of the reference's
    metric loop (oracle/metrics_oracle.py: runners/ncsn_runner.py:1581-1600 + skimage's SSIM algorithm)."""
    import numpy as np
    from oracle import metrics_oracle as M
    g = torch.Generator().manual_seed(B * 100 + S)
    real = torch.rand(B, C * nf, S, S, generator=g)
    real = torch.nn.functional.avg_pool2d(real, 5, 1, 2)                       # some spatial structure
    real = (real - real.min()) / (real.max() - real.min())
    pred = (real + 0.08 * torch.randn(real.shape, generator=g)).clamp(0, 1)
    pred[0, :C] = real[0, :C]                                                  # one identical frame: MSE 0, SSIM 1
    out = torch.zeros(B, nf, 2, dtype=torch.float64, device=DEV)
    run([mk(lib.OP_FRAME_METRICS, B, H=S, W=S, C0=C, i0=nf, src0=pred.to(DEV), src1=real.to(DEV), dst=out,
            flags=lib.F_ROUND if rnd else 0)])
    ref = M.frame_metrics(pred.numpy(), real.numpy(), C, round_first=rnd)
    got = out.cpu().numpy()
    assert got[0, 0, 0] == 0.0 and abs(got[0, 0, 1] - 1.0) < 1e-12
    assert np.abs(got[..., 0] - ref[..., 0]).max() < 1e-12
    assert np.abs(got[..., 1] - ref[..., 1]).max() < 1e-9


K1_CASES = [
    # B, H, C0, C1, Cout, tab, act_in, res, act_out      -- 1x1 convs, input-stationary and streaming (conv_umma.cu)
    (2, 16, 64, 0, 192, True, False, False, False),
    (2, 8, 96, 0, 96, False, False, True, False),
    (3, 8, 96, 96, 96, False, False, False, False),        # concatenated sources, 192 rows: a partial last tile
    (2, 16, 192, 0, 576, True, False, False, False),       # q/k/v projection: 3 n tiles spread over CTA groups
    (1, 8, 288, 0, 864, True, True, False, False),         # n tile 144 (16-wide tail block), 9 K-blocks, half a tile
    (2, 32, 96, 96, 96, False, False, True, True),
    (5, 32, 192, 0, 192, False, False, True, False),
    (40, 16, 192, 0, 576, True, False, False, False),      # 80 m tiles x 3 n tiles per CTA
    (8, 64, 96, 96, 96, False, False, False, False),       # 256 m tiles: several work items per CTA (phase wrap)
    (6, 64, 96, 0, 288, True, False, True, False),
    (2, 8, 384, 0, 96, False, False, False, False),        # 12 K-blocks, still resident next to small weight stages
    (4, 8, 384, 0, 1152, True, False, False, False),       # 8x8 q/k/v: ring of operand stages, one n tile per item
    (3, 8, 384, 384, 192, False, False, True, False),      # 24 K-blocks from two sources through the ring, residual
    (2, 16, 512, 0, 256, True, True, False, True),
    (10, 64, 32, 0, 64, True, False, False, False),        # one K-block (a single operand stage), 320 m tiles
    (3, 16, 32, 32, 32, False, False, True, False),
]


@pytest.mark.parametrize("case", K1_CASES)
def test_conv1x1_stationary(case):
    """1x1 convolutions through OP_CONV_UMMA in each work organisation (i2 = 2: the m tile's input resident while
    every n tile's weights stream past; i2 = 1: one n tile per work item; i2 = 0: the launcher's choice), with and
    without epilogue statistics: each against the fp64 reference, and all bit-identical (same K order per output)."""
    B, H, C0, C1, Cout, use_tab, act_in, use_res, act_out = case
    Cin = C0 + C1
    x0 = rnd(B, H, H, C0, seed=11)
    x1 = rnd(B, H, H, C1, seed=12) if C1 else None
    w = rnd(Cout, Cin, 1, 1, seed=15) / math.sqrt(Cin)
    bias = rnd(Cout, seed=16) * 0.1
    res = rnd(B, H, H, Cout, seed=17) if use_res else None
    tab = make_table(B, Cin) if use_tab else None
    scale = 0.7071
    xin = x0 if x1 is None else torch.cat([x0, x1], 3)
    xa = ref_norm(xin, tab, act_in) if use_tab else xin
    ref = conv_ref(xa, w, bias, res, scale, act_out)
    d = lambda t: None if t is None else t.to(DEV).contiguous()
    x0d, x1d, bd, rd, td = d(x0), d(x1), d(bias), d(res), d(tab)
    taps = taps_of(w).to(DEV)
    kb = lib.umma_kblock(C0, C1)
    nt = max(dd for dd in range(16, 257, 16) if Cout % dd == 0)
    pk = torch.empty(taps.numel() * 4, dtype=torch.uint8, device=DEV)
    k = int(math.floor(math.log2(512.0 / float(taps.abs().max()))))
    rc = lib.load().mcvd_umma_pack_weights(taps.data_ptr(), 1, Cin, Cout, nt, kb, pk.data_ptr(), k,
                                           torch.cuda.current_stream().cuda_stream)
    assert rc > 0, lib.last_error()
    fl = (lib.F_ACT_IN if act_in else 0) | (lib.F_ACT_OUT if act_out else 0)
    outs = []
    stats = []
    for mode, with_stats in ((2, False), (1, False), (0, False), (2, True), (1, True)):
        out = torch.full((B, H, H, Cout), float("nan"), device=DEV)
        st = torch.zeros(lib.umma2_stats_bytes(B, H, H, 1, Cout) // 8, dtype=torch.int64, device=DEV) \
            if with_stats and H * H >= 64 else None
        run([mk(lib.OP_CONV_UMMA, B, H=H, W=H, C0=C0, C1=C1, Cout=Cout, i0=1, i1=nt, i2=mode, f0=scale, f1=2.0 ** (-k),
                src0=x0d, src1=x1d, w=pk, bias=bd, aux0=rd, aux1=td, dst=out, dst2=st, flags=fl)])
        o = out.cpu()
        err = (o - ref).abs().max().item()
        assert err < 2e-5 * max(1.0, ref.abs().max().item()), (case, mode, with_stats, err)
        outs.append(o)
        if st is not None:
            stats.append(st.cpu())
    assert all(torch.equal(outs[0], o) for o in outs[1:]), case
    assert all(torch.equal(stats[0], s_) for s_ in stats[1:]), case
