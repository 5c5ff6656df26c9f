"""Geometry of the TMA-staged input of the wgmma conv (csrc/conv_umma.cu): halo slabs that cross image boundaries
at every map size, a last tile only partly inside the batch, B = 1, split C2|C3 shortcut sources staged at the
centre tap only, K-block 16, the 16-channel padded first / last convs, input-stationary 1x1 and the planar table
with epilogue statistics.  Each case runs the float64-reference checks of test_gpu_ops / test_gpu_conv2."""
import math

import pytest
import torch

from mcvd_b200 import lib
import test_gpu_conv2 as C2
import test_gpu_ops as OPS

pytestmark = pytest.mark.gpu

DEV = "cuda:0"

UMMA_CASES = [
    # B, H, C0, C1, Cout, ks, tab, act_in, res, act_out
    (3, 8, 32, 0, 32, 3, True, True, False, False),        # 8x8: a slab spans three images
    (2, 16, 64, 0, 64, 3, True, True, True, False),
    (3, 32, 32, 32, 64, 3, True, True, False, True),
    (2, 64, 32, 0, 32, 3, True, False, False, False),       # HP > 256: two TMA boxes per K-block
    (1, 128, 32, 0, 32, 3, True, True, False, False),       # B = 1, 128x128
    (1, 128, 64, 0, 256, 3, True, True, False, False),      # 128x128 at NT = 256: one raw stage fits
    (3, 12, 32, 0, 48, 3, True, True, True, False),         # 3*13*13 = 507 positions: last tile partly outside
    (1, 8, 16, 16, 32, 3, True, True, False, False),        # K-block 16, B = 1
    (2, 32, 16, 0, 96, 3, False, False, False, False),      # first conv: 16 padded input channels
    (2, 32, 96, 0, 16, 3, True, True, False, False),        # last conv: 16 padded output channels
    (5, 16, 96, 0, 288, 1, True, True, False, False),       # 1x1, three n tiles (input-stationary with i2 = 2)
    (3, 12, 32, 32, 64, 1, True, False, True, False),       # 1x1, 432 positions: last tile partly outside
]


@pytest.mark.parametrize("case", UMMA_CASES)
def test_conv_umma_geometry(case):
    OPS.test_conv(case, "umma")          # i2 = 1 (streaming) and i2 = 2 against the float64 reference


PLANAR_CASES = [
    # B, H, C0, C1, Cout, ks, tab(+SiLU), res, shortcut (C2, C3), stats
    (2, 16, 64, 0, 64, 3, True, False, (32, 32), True),     # split shortcut sources, centre-tap staging
    (2, 32, 32, 0, 64, 3, True, True, (48, 16), True),      # K-block 16 main + split shortcut
    (1, 64, 32, 0, 32, 3, True, False, (32, 0), True),      # HP > 256 with a shortcut segment, B = 1
    (3, 12, 32, 0, 32, 3, True, True, (0, 0), True),        # last tile partly outside, statistics
    (1, 128, 32, 0, 32, 3, True, False, (0, 0), True),
    (2, 16, 96, 0, 192, 1, True, False, (0, 0), True),      # 1x1 with statistics
]


@pytest.mark.parametrize("case", PLANAR_CASES)
def test_conv_umma2_geometry(case):
    C2.test_conv_umma2(case)


@pytest.mark.parametrize("B,H,C0,Cout,ks", [(5, 16, 96, 288, 1), (3, 12, 64, 128, 1), (2, 16, 64, 64, 3)])
def test_work_organisations_bit_identical(B, H, C0, Cout, ks):
    """i2 = 1 (streaming) and i2 = 2 (input-stationary where it applies) stage the same input: identical bits"""
    x = C2.rnd(B, H, H, C0, seed=1).to(DEV)
    w = C2.rnd(Cout, C0, ks, ks, seed=5) / math.sqrt(C0 * ks * ks)
    tab = C2.make_table(B, C0).to(DEV)
    bias = (C2.rnd(Cout, seed=6) * 0.1).to(DEV)
    taps = C2.taps_of(w).to(DEV)
    kb = lib.umma_kblock(C0, 0)
    nt = max(d for d in range(16, 257, 16) if Cout % d == 0)
    pk = torch.empty(taps.numel() * 4, dtype=torch.uint8, device=DEV)
    k = int(math.floor(math.log2(512.0 / float(taps.abs().max()))))
    assert lib.load().mcvd_umma_pack_weights(taps.data_ptr(), ks * ks, C0, Cout, nt, kb, pk.data_ptr(), k,
                                             torch.cuda.current_stream().cuda_stream) > 0, lib.last_error()
    outs = []
    for mode in (1, 2):
        out = torch.zeros(B, H, H, Cout, device=DEV)
        C2.run([C2.mk(lib.OP_CONV_UMMA, B, H=H, W=H, C0=C0, Cout=Cout, i0=ks, i1=nt, i2=mode, f0=0.7071,
                      f1=2.0 ** (-k), src0=x, w=pk, bias=bias, aux1=tab, dst=out, flags=lib.F_ACT_IN)])
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
