"""Tensor-core conv with the planar norm table (MCVD_OP_CONV_UMMA2, csrc/conv_umma.cu) through the C-ABI: parity against a float64
torch evaluation of the reference ops (nn.Conv2d / NIN after get_act_norm, models/better/layers.py:89-113,541-544,
layerspp.py:518-549, fused Conv_2 shortcut layerspp.py:618-619), the exact integer GroupNorm statistics of its
epilogue, and their use by MCVD_OP_GN_FINALIZE (nn.GroupNorm, layerspp.py:474-477)."""
import math

import pytest
import torch
import torch.nn.functional as F

from mcvd_b200 import lib
from mcvd_b200.lib import McvdOp
from op_interpreter import tile_stats

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def rnd(*shape, seed=0):
    g = torch.Generator().manual_seed(seed + sum(shape))
    return torch.randn(*shape, generator=g)


def mk(kind, B, **kw):
    o = McvdOp()
    o.kind, o.B = kind, B
    for k, v in kw.items():
        setattr(o, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return o


def taps_of(w):
    O, I, kh, kw = w.shape
    return w.permute(2, 3, 1, 0).reshape(kh * kw, I, O).contiguous()


def make_table(B, C, seed=3):
    return torch.stack([rnd(B, C, seed=seed) * 0.3, 0.5 + torch.rand(B, C), 1 + 0.3 * rnd(B, C, seed=seed + 1),
                        0.2 * rnd(B, C, seed=seed + 2)], dim=2).contiguous()


def planar(tab):
    """(mean, rstd, G, S) [B,C,4] -> the planar [B,3,C] table CONV_UMMA2 reads: mean | rstd*G | S"""
    return torch.stack([tab[..., 0], tab[..., 1] * tab[..., 2], tab[..., 3]], 1).contiguous()


def pack2(t_main, t_sc, nt, kb):
    T, I, O = t_main.shape
    isc = 0 if t_sc is None else t_sc.shape[1]
    amax = float(max(t_main.abs().max(), t_sc.abs().max() if isc else 0))
    k = int(math.floor(math.log2(512.0 / amax)))
    per_unit = (I // kb) * T + isc // kb
    pk = torch.empty((T * I + isc) * O * 4, dtype=torch.uint8, device=DEV)
    L, s = lib.load(), torch.cuda.current_stream().cuda_stream
    assert L.mcvd_umma2_pack_weights(t_main.data_ptr(), T, I, O, nt, kb, pk.data_ptr(), k, 0, per_unit, s) > 0, lib.last_error()
    if isc:
        assert L.mcvd_umma2_pack_weights(t_sc.data_ptr(), 1, isc, O, nt, kb, pk.data_ptr(), k, (I // kb) * T, per_unit,
                                         s) > 0, lib.last_error()
    return pk, 2.0 ** (-k)


def expected_stats(y, ks):
    """what the epilogue must have written for the stored output y [B,H,W,C] (tests/op_interpreter.py semantics;
    raises ValueError outside the statistics' range |y| <= 2^12)"""
    return tile_stats(y, ks)


CASES = [
    # B, H, C0, C1, Cout, ks, tab(+SiLU), res, shortcut (C2, C3), stats
    (2, 8, 32, 0, 32, 3, False, False, (0, 0), True),
    (2, 16, 32, 0, 64, 3, True, True, (0, 0), True),
    (3, 8, 64, 32, 96, 3, True, True, (0, 0), True),          # virtual concat, images straddle tiles
    (2, 32, 32, 0, 32, 3, True, False, (0, 0), False),
    (1, 64, 32, 0, 48, 3, False, False, (0, 0), True),
    (2, 16, 48, 48, 144, 3, True, True, (0, 0), True),        # K-block 16, 16-wide epilogue tail
    (2, 16, 64, 0, 192, 1, True, False, (0, 0), True),        # 1x1 (qkv-like)
    (2, 8, 96, 0, 96, 1, False, True, (0, 0), True),          # NIN_3-like
    (4, 8, 128, 128, 256, 3, True, True, (0, 0), True),
    (2, 16, 32, 0, 512, 3, False, False, (0, 0), True),       # two n tiles
    (2, 16, 64, 0, 64, 3, True, False, (32, 0), True),        # fused 1x1 shortcut
    (2, 8, 96, 0, 96, 3, True, False, (96, 96), True),
    (3, 16, 48, 0, 48, 3, True, False, (48, 48), False),      # K-block 16 shortcut
    (2, 8, 128, 0, 256, 3, True, False, (128, 64), True),
    (5, 4, 32, 0, 32, 3, True, True, (0, 0), False),          # 4x4 maps: a tile spans six images
    (37, 16, 32, 0, 32, 3, True, True, (0, 0), True),         # more units than clusters would get one of: odd batch
    (2, 32, 16, 0, 96, 3, False, False, (0, 0), True),        # first conv (Cin padded to 16)
    (2, 32, 96, 0, 16, 3, True, False, (0, 0), False),        # last conv (Cout padded to 16)
]


@pytest.mark.parametrize("case", CASES)
def test_conv_umma2(case):
    B, H, C0, C1, Cout, ks, use_tab, use_res, (C2, C3), use_stats = case
    Cin, Cs = C0 + C1, C2 + C3
    x0 = rnd(B, H, H, C0, seed=1)
    x1 = rnd(B, H, H, C1, seed=2) if C1 else None
    y0 = rnd(B, H, H, C2, seed=11) if C2 else None
    y1 = rnd(B, H, H, C3, seed=12) if C3 else None
    w = rnd(Cout, Cin, ks, ks, seed=5) / math.sqrt(Cin * ks * ks)
    w2 = rnd(Cout, Cs, 1, 1, seed=15) / math.sqrt(Cs) if Cs else None
    bias = rnd(Cout, seed=6) * 0.1
    res = rnd(B, H, H, Cout, seed=7) if use_res else None
    tab = make_table(B, Cin) if use_tab else None
    scale = 0.7071
    xin = x0 if x1 is None else torch.cat([x0, x1], 3)
    if use_tab:
        t = tab.view(B, 1, 1, Cin, 4)
        xin = ((xin - t[..., 0]) * t[..., 1]) * t[..., 2] + t[..., 3]
        xin = xin * torch.sigmoid(xin)
    ref = F.conv2d(xin.permute(0, 3, 1, 2).double(), w.double(), bias.double(), padding=ks // 2).permute(0, 2, 3, 1)
    if Cs:
        ys = y0 if y1 is None else torch.cat([y0, y1], 3)
        ref = ref + F.conv2d(ys.permute(0, 3, 1, 2).double(), w2.double()).permute(0, 2, 3, 1)
    if use_res:
        ref = ref + res.double()
    ref = (ref * scale).float()

    nt = lib.umma2_pick_nt(Cout, ks)
    pimg = (H + 1) * (H + 1) if ks == 3 else H * H
    use_stats = use_stats and pimg >= 64
    kb = lib.umma2_plan(H, H, ks, C0, C1, C2, C3, nt, use_stats)
    assert kb in (16, 32)
    d = lambda t_: None if t_ is None else t_.to(DEV).contiguous()
    pk, wscale = pack2(taps_of(w).to(DEV), taps_of(w2).to(DEV) if Cs else None, nt, kb)
    x0d, x1d, y0d, y1d, bd, rd = d(x0), d(x1), d(y0), d(y1), d(bias), d(res)
    t3 = d(planar(tab)) if use_tab else None
    out = torch.zeros(B, H, H, Cout, device=DEV)
    st = torch.full((lib.umma2_stats_bytes(B, H, H, ks, Cout) // 8,), -7, dtype=torch.int64, device=DEV) if use_stats else None
    run([mk(lib.OP_CONV_UMMA2, B, H=H, W=H, C0=C0, C1=C1, Cout=Cout, i0=ks, i1=nt, i2=kb, f0=scale, f1=wscale, src0=x0d,
            src1=x1d, w=pk, bias=bd, aux0=rd, aux1=t3, dst=out, dst2=st, flags=lib.F_ACT_IN if use_tab else 0,
            src2=y0d, src3=y1d, C2=C2, C3=C3)])
    err = (out.cpu() - ref).abs().max().item()
    assert err < 2e-5 * max(1.0, ref.abs().max().item()), (case, err)
    if use_stats:
        exp = expected_stats(out.cpu(), ks)
        assert torch.equal(st.cpu().view(exp.shape), exp), case


@pytest.mark.parametrize("B,H,C0,C1,ks0,ks1", [(4, 16, 64, 0, 3, 0), (3, 8, 96, 48, 3, 1), (4, 32, 32, 32, 1, 3),
                                               (5, 8, 768, 768, 3, 3)])
def test_finalize_from_epilogue_statistics(B, H, C0, C1, ks0, ks1):
    """identity 1x1 / centre-tap 3x3 convs write x and its tile statistics; GN_FINALIZE on those statistics must
    give the float64 GroupNorm statistics of x, the planar table, and must not depend on the batch placement"""
    from mcvd_b200.arch import num_groups
    C = C0 + C1
    xs = [rnd(B, H, H, C0, seed=1) * 2 + 0.5] + ([rnd(B, H, H, C1, seed=2)] if C1 else [])
    film = rnd(B, 3 * C + 5, seed=3)
    off = 5
    cg = C // num_groups(C)

    def produce(xd, ks, Bn):
        """copy xd through an identity conv of kernel size ks with epilogue statistics"""
        Cc = xd.shape[3]
        w = torch.zeros(Cc, Cc, ks, ks)
        w[:, :, ks // 2, ks // 2] = torch.eye(Cc)
        nt = lib.umma2_pick_nt(Cc, ks)
        kb = lib.umma2_plan(H, H, ks, Cc, 0, 0, 0, nt, True)
        pk, wscale = pack2(taps_of(w).to(DEV), None, nt, kb)
        out = torch.zeros(Bn, H, H, Cc, device=DEV)
        st = torch.zeros(lib.umma2_stats_bytes(Bn, H, H, ks, Cc) // 8, dtype=torch.int64, device=DEV)
        zero = torch.zeros(Cc, device=DEV)
        run([mk(lib.OP_CONV_UMMA2, Bn, H=H, W=H, C0=Cc, Cout=Cc, i0=ks, i1=nt, i2=kb, f0=1.0, f1=wscale, src0=xd, w=pk,
                bias=zero, dst=out, dst2=st)])
        assert (out - xd).abs().max().item() < 1e-5      # hi + lo keeps ~22 bits of every input
        return out, st

    def table(lo, hi):
        Bn = hi - lo
        xd = [x[lo:hi].to(DEV).contiguous() for x in xs]
        outs, sts = zip(*([produce(xd[0], ks0, Bn)] + ([produce(xd[1], ks1, Bn)] if C1 else [])))
        tab = torch.zeros(Bn, C, 4, device=DEV)
        tab3 = torch.zeros(Bn, 3, C, device=DEV)
        fd = film[lo:hi].to(DEV).contiguous()
        run([mk(lib.OP_GN_FINALIZE, Bn, H=H, W=H, C0=C0, C1=C1, i0=0, i1=cg, f0=1e-5, src0=sts[0],
                src1=sts[1] if C1 else None, dst=tab, dst2=tab3, aux0=fd, i2=film.shape[1], i3=off, flags=lib.F_FILM,
                i4=ks0, i5=ks1)])
        return tab.cpu(), tab3.cpu(), torch.cat([o.cpu() for o in outs], 3)

    tab, tab3, x = table(0, B)
    xg = x.permute(0, 3, 1, 2).reshape(B, C // cg, cg * H * H).double()
    mean, var = xg.mean(2), xg.var(2, unbiased=False)
    rstd = 1 / torch.sqrt(var + 1e-5)
    ref = torch.stack([mean.float().repeat_interleave(cg, 1), rstd.float().repeat_interleave(cg, 1),
                       1 + film[:, off:off + C], film[:, off + C:off + 2 * C]], 2)
    assert (tab - ref).abs().max().item() < 2e-5
    assert torch.equal(tab3, planar(tab))
    # clips 1.. as their own batch: other tile boundaries, other warps, same integers -> identical tables
    tab_s, _, x_s = table(1, B)
    assert torch.equal(x_s, x[1:])
    assert torch.equal(tab_s, tab[1:])


def test_out_of_range_activations_stay_finite():
    """|x| above the fp16 range (65504): hi and lo saturate (F2FP.SATFINITE), hi + lo still carries the value up to
    131008 with >= 11 bits, beyond that it clamps -- never inf - inf = NaN as in the round-1 split"""
    B, H, C = 2, 8, 32
    w = rnd(C, C, 3, 3, seed=2) / math.sqrt(9 * C)
    bias = torch.zeros(C)
    kb = lib.umma2_plan(H, H, 3, C, 0, 0, 0, C, False)
    pk, wscale = pack2(taps_of(w).to(DEV), None, C, kb)
    for big, exact in ((1.2e5, True), (1.0e7, False)):
        x = rnd(B, H, H, C, seed=1)
        x[0, 3, 3, 5] = big
        x[1, 0, 0, 0] = -1.0e5
        ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), padding=1).permute(0, 2, 3, 1).float()
        out = torch.zeros(B, H, H, C, device=DEV)
        run([mk(lib.OP_CONV_UMMA2, B, H=H, W=H, C0=C, Cout=C, i0=3, i1=C, i2=kb, f0=1.0, f1=wscale, src0=x.to(DEV),
                w=pk, bias=bias.to(DEV), dst=out)])
        o = out.cpu()
        assert torch.isfinite(o).all()
        if exact:        # lo = fp16(x - hi) rounds to a multiple of 32 here: error <= 16 * |w| per term
            assert (o - ref).abs().max().item() < 64.0 * float(w.abs().max())
        far = torch.ones(B, H, H, dtype=torch.bool)
        far[0, 2:5, 2:5] = False
        far[1, 0:2, 0:2] = False
        assert (o[far] - ref[far]).abs().max().item() < 2e-5 * max(1.0, ref[far].abs().max().item())
