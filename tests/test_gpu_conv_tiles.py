"""Tile height of the wgmma conv (csrc/conv_umma.cu): every case runs at 128- and 192-position tiles (two and three
consumer warpgroups, forced through the CONV_UMMA i4 override) and at the launcher's own choice.  Each result is held
to the float64 reference of test_gpu_conv2 within the tolerance of test_gpu_conv_tma, and all heights must give
identical bits: an output sums the same products in the same order whichever tile it falls in."""
import math

import pytest
import torch
import torch.nn.functional as F

from mcvd_b200 import lib
import test_gpu_conv2 as C2

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

CASES = [
    # B, H, C0, C1, Cout, NT, ks, tab(+SiLU), res, shortcut (C2, C3)
    (3, 8, 32, 0, 96, 96, 3, True, False, (0, 0)),          # 8x8: a slab spans several images, last tile partial
    (2, 16, 64, 0, 144, 144, 3, True, True, (0, 0)),
    (2, 32, 32, 32, 192, 192, 3, True, False, (0, 0)),      # virtual concat
    (2, 64, 32, 0, 96, 96, 3, True, False, (0, 0)),         # HP > 256: two TMA boxes per K-block
    (1, 128, 32, 0, 96, 96, 3, True, False, (0, 0)),        # B = 1, 128x128: the largest slab (456 positions)
    (1, 128, 32, 0, 192, 192, 3, True, False, (0, 0)),      # 128x128 at NT = 192: one raw stage at MT = 192
    (3, 12, 32, 0, 96, 96, 3, True, True, (0, 0)),          # 507 positions: last tile partly outside the batch
    (1, 8, 16, 16, 96, 96, 3, True, False, (0, 0)),         # K-block 16, B = 1
    (2, 32, 16, 0, 96, 96, 3, False, False, (0, 0)),        # first conv: raw 16-channel input
    (2, 16, 64, 0, 96, 96, 3, True, False, (32, 32)),       # fused C2|C3 shortcut, centre-tap staging
    (2, 32, 32, 0, 144, 144, 3, True, True, (48, 16)),      # K-block 16 main + split shortcut
    (1, 64, 32, 0, 96, 96, 3, True, False, (32, 0)),        # HP > 256 with a shortcut segment, B = 1
    (5, 16, 96, 0, 192, 192, 1, True, False, (0, 0)),       # 1x1 with one n tile (streaming)
    (2, 8, 384, 0, 384, 192, 3, True, False, (0, 0)),       # two n tiles
]


@pytest.mark.parametrize("case", CASES)
def test_tile_heights_bit_identical(case):
    B, H, C0, C1, Cout, nt, ks, use_tab, use_res, (Ca, Cb) = case
    Cin, Cs = C0 + C1, Ca + Cb
    x0 = C2.rnd(B, H, H, C0, seed=1)
    x1 = C2.rnd(B, H, H, C1, seed=2) if C1 else None
    y0 = C2.rnd(B, H, H, Ca, seed=11) if Ca else None
    y1 = C2.rnd(B, H, H, Cb, seed=12) if Cb else None
    w = C2.rnd(Cout, Cin, ks, ks, seed=5) / math.sqrt(Cin * ks * ks)
    w2 = C2.rnd(Cout, Cs, 1, 1, seed=15) / math.sqrt(Cs) if Cs else None
    bias = C2.rnd(Cout, seed=6) * 0.1
    res = C2.rnd(B, H, H, Cout, seed=7) if use_res else None
    tab = C2.make_table(B, Cin) if use_tab else None
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

    kb = lib.umma2_plan(H, H, ks, C0, C1, Ca, Cb, nt, False)
    assert kb in (16, 32)
    d = lambda t_: None if t_ is None else t_.to(DEV).contiguous()
    pk, wscale = C2.pack2(C2.taps_of(w).to(DEV), C2.taps_of(w2).to(DEV) if Cs else None, nt, kb)
    x0d, x1d, y0d, y1d, bd, rd, td = d(x0), d(x1), d(y0), d(y1), d(bias), d(res), d(tab)
    outs = {}
    for mt in (128, 192, 0):
        out = torch.zeros(B, H, H, Cout, device=DEV)
        C2.run([C2.mk(lib.OP_CONV_UMMA, B, H=H, W=H, C0=C0, C1=C1, Cout=Cout, i0=ks, i1=nt, i2=1, i4=mt, f0=scale,
                      f1=wscale, src0=x0d, src1=x1d, w=pk, bias=bd, aux0=rd, aux1=td, dst=out,
                      flags=lib.F_ACT_IN if use_tab else 0, src2=y0d, src3=y1d, C2=Ca, C3=Cb)])
        outs[mt] = out.cpu()
        err = (outs[mt] - ref).abs().max().item()
        assert err < 2e-5 * max(1.0, ref.abs().max().item()), (case, mt, err)
    assert torch.equal(outs[128], outs[192]), case
    assert torch.equal(outs[0], outs[128]), case
