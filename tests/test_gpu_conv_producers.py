"""Producer side of the wgmma conv (csrc/conv_umma.cu): each producer thread converts one 8-channel chunk over a run of
slab positions and keeps the norm-table row of the current image in registers.  Every case runs at each forced tile
height (CONV_UMMA i4 = 128, 192) and slab-stage count (i5 = 2, 3) that fits, and at the launcher's own choice; with a
norm table it also runs through CONV_UMMA2 with the planar table.  Each result is held to the float64 reference within
the tolerance of test_gpu_conv_tma, and all of them must give identical bits."""
import math

import pytest
import torch
import torch.nn.functional as F

from mcvd_b200 import lib
import test_gpu_conv2 as C2

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

CASES = [
    # B, H, C0, C1, Cout, NT, tab, act_in, res, shortcut (C2, C3)
    (3, 8, 32, 0, 96, 96, True, True, False, (0, 0)),       # 8x8: a slab spans several images, last tile partial
    (2, 16, 64, 0, 96, 96, True, False, True, (0, 0)),      # norm without SiLU
    (3, 12, 32, 0, 96, 96, True, True, False, (0, 0)),      # 507 positions: last tile partly outside the batch
    (1, 64, 32, 0, 96, 96, True, True, False, (0, 0)),      # B = 1 at 64x64: two TMA boxes, slab reaches past the end
    (2, 64, 32, 0, 192, 192, False, False, False, (0, 0)),  # raw input, NT = 192, slab crossing the image boundary
    (1, 8, 16, 16, 96, 96, True, True, False, (0, 0)),      # K-block 16 over a virtual concat, B = 1
    (2, 16, 48, 0, 96, 96, True, True, False, (16, 0)),     # K-block 16 with a fused shortcut segment
    (2, 64, 32, 0, 96, 96, True, True, True, (32, 32)),     # 64x64 with a split C2|C3 shortcut and a residual
    (8, 64, 32, 0, 96, 96, True, True, False, (0, 0)),      # more tiles than SMs: a CTA's producers move on to a next tile
]


def forced_settings():
    return [(mt, sa) for mt in (128, 192) for sa in (2, 3)] + [(0, 0)]


@pytest.mark.parametrize("case", CASES)
def test_producers_bit_identical(case):
    B, H, C0, C1, Cout, nt, use_tab, act_in, use_res, (Ca, Cb) = case
    Cin, Cs = C0 + C1, Ca + Cb
    x0 = C2.rnd(B, H, H, C0, seed=1)
    x1 = C2.rnd(B, H, H, C1, seed=2) if C1 else None
    y0 = C2.rnd(B, H, H, Ca, seed=11) if Ca else None
    y1 = C2.rnd(B, H, H, Cb, seed=12) if Cb else None
    w = C2.rnd(Cout, Cin, 3, 3, seed=5) / math.sqrt(Cin * 9)
    w2 = C2.rnd(Cout, Cs, 1, 1, seed=15) / math.sqrt(Cs) if Cs else None
    bias = C2.rnd(Cout, seed=6) * 0.1
    res = C2.rnd(B, H, H, Cout, seed=7) if use_res else None
    tab = C2.make_table(B, Cin) if use_tab else None
    scale = 0.7071
    xin = x0 if x1 is None else torch.cat([x0, x1], 3)
    if use_tab:
        t = tab.view(B, 1, 1, Cin, 4)
        xin = ((xin - t[..., 0]) * t[..., 1]) * t[..., 2] + t[..., 3]
        if act_in:
            xin = xin * torch.sigmoid(xin)
    ref = F.conv2d(xin.permute(0, 3, 1, 2).double(), w.double(), bias.double(), padding=1).permute(0, 2, 3, 1)
    if Cs:
        ys = y0 if y1 is None else torch.cat([y0, y1], 3)
        ref = ref + F.conv2d(ys.permute(0, 3, 1, 2).double(), w2.double()).permute(0, 2, 3, 1)
    if use_res:
        ref = ref + res.double()
    ref = (ref * scale).float()

    kb = lib.umma2_plan(H, H, 3, C0, C1, Ca, Cb, nt, False)
    assert kb == (16 if (C0 % 32 or C1 % 32 or Ca % 32 or Cb % 32) else 32)
    d = lambda t_: None if t_ is None else t_.to(DEV).contiguous()
    pk, wscale = C2.pack2(C2.taps_of(w).to(DEV), C2.taps_of(w2).to(DEV) if Cs else None, nt, kb)
    x0d, x1d, y0d, y1d, bd, rd = d(x0), d(x1), d(y0), d(y1), d(bias), d(res)
    flags = lib.F_ACT_IN if act_in else 0
    common = dict(H=H, W=H, C0=C0, C1=C1, Cout=Cout, i0=3, i1=nt, f0=scale, f1=wscale, src0=x0d, src1=x1d, w=pk,
                  bias=bd, aux0=rd, dst=None, flags=flags, src2=y0d, src3=y1d, C2=Ca, C3=Cb)
    tol = 2e-5 * max(1.0, ref.abs().max().item())
    outs = {}

    def run(kind, key, tab_dev, **kw):
        out = torch.zeros(B, H, H, Cout, device=DEV)
        C2.run([C2.mk(kind, B, **{**common, "dst": out, "aux1": tab_dev, **kw})])
        outs[key] = out.cpu()
        err = (outs[key] - ref).abs().max().item()
        assert err < tol, (case, key, err)

    td = d(tab)
    for mt, sa in forced_settings():
        try:
            run(lib.OP_CONV_UMMA, (mt, sa), td, i2=1, i4=mt, i5=sa)
        except RuntimeError:
            # a forced height / stage count that does not fit shared memory; the 128 / 2 plan always does
            assert (mt, sa) not in ((128, 2), (0, 0)), case
    if use_tab:
        run(lib.OP_CONV_UMMA2, "planar", d(C2.planar(tab)), i2=kb)
    assert len(outs) >= 3, (case, list(outs))
    for key, out in outs.items():
        assert torch.equal(out, outs[(128, 2)]), (case, key)
