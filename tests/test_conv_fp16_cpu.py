"""The fp16 convolution mode (model.conv_precision = "fp16") checked on the CPU.

Error model.  A half-mode conv rounds each operand once to fp16 (activations unscaled, weights after the per-layer
2^k pre-scale of mcvd_b200.program.umma_scale_log2, both saturating at 65504) and sums the products hi*hi in fp32.
One product then errs by at most (2u + u^2)|x||w| with u = 2^-11 while both operands are normal fp16 numbers, plus
(1 + u) times the absolute error of a subnormal operand, 2^-25 for an activation and 2^-25 * 2^-k for a weight, times
the other operand.  The per-element bound is therefore

    TAU_HALF * A + u_fp32 |ref| + (1 + u) 2^-25 (sum |w| over the products + 2^-k sum |x| over the products)

with TAU_HALF = 2u + u^2 + TAU_MATMUL (the fp32 accumulation term of the replay) and A, the floors and the pre-scale
as in tests/test_value_ranges_cpu.py.  Below, a float64 emulation of the half product stays inside the bound on the
input families of the default mode's model, and two deliberately wrong emulations leave it: weights rounded to 9
significand bits, and a pre-scale one power of two too small (the weights' subnormal floor doubles).

Lowering.  On the op interpreter, "fp16" gives MCVD_F_HALF to exactly the tensor-core convs that lower one of the
reference's nn.Conv2d layers (first and final conv, Conv_0, Conv_1, the Conv_2 skip projection fused or separate,
SPADE), never to the NIN projections, attention or CUDA-core ops; launch counts equal the default mode's, and the two
modes never share a program, a packed-weight key or a weight-cache file.
"""
import copy
import re

import pytest
import torch

from common import make_module
from mcvd_b200 import arch, configs, detfill, lib
from mcvd_b200.model import UNetMore_DDPM
from mcvd_b200.program import Engine, umma_scale_log2
from op_interpreter import Interpreter, round_fp16 as interp_round_fp16
from program_replay import TAU_HALF, TAU_MATMUL, U_FP16
from test_value_ranges_cpu import (CONV_FAMILIES, FP16_MAX, SHORTCUT_FAMILIES, SPLIT_FLOOR, U_FP32, conv_case,
                                   conv_scale_log2, interp_conv, worst_ratio)



def half_bound(case):
    """(float64 reference, per-element bound of the one-product conv) of a conv case"""
    ref = interp_conv(case)
    bound = TAU_HALF * interp_conv(case, magnitude=True) + U_FP32 * ref.abs()
    ones = lambda n: None if case.get(n) is None else torch.ones_like(case[n])
    zero_bias = torch.zeros_like(case["bias"])
    fw = interp_conv(case, True, x0=ones("x0"), x1=ones("x1"), y=ones("y"), tab=None, res=None, bias=zero_bias,
                     flags=case.get("flags", 0) & ~lib.F_ACT_IN)
    fx = interp_conv(case, True, taps=ones("taps"), taps_sc=ones("taps_sc"), res=None, bias=zero_bias)
    return ref, bound + (1 + U_FP16) * SPLIT_FLOOR * (fw + 2.0 ** -conv_scale_log2(case) * fx)


def round_fp16(x):
    """the kernel's saturating fp16 rounding (cvt.rn.satfinite) as a float64 tensor"""
    return interp_round_fp16(x.double())


def round_bits(x, bits):
    """x rounded to nearest-even with ``bits`` significand bits (a deliberately coarse weight image)"""
    m, e = torch.frexp(x.double())
    return torch.ldexp(torch.round(torch.ldexp(m, torch.full_like(e, bits))), e - bits)


def emulate_half(case, k=None, wround=round_fp16):
    """the one-product conv in float64: fp16 activations times pre-scaled fp16 weights (``wround`` replaces the
    weights' rounding), bias and scale afterwards.  Cases without a norm table, residual or output activation."""
    assert case.get("tab") is None and case.get("res") is None and not case.get("flags", 0)
    k = conv_scale_log2(case) if k is None else k
    over = {n: round_fp16(case[n]).float() for n in ("x0", "x1", "y") if case.get(n) is not None}
    over.update({n: (wround(case[n].double() * 2.0 ** k) * 2.0 ** -k).float()
                 for n in ("taps", "taps_sc") if case.get(n) is not None})
    out = interp_conv(case, bias=torch.zeros_like(case["bias"]), f0=1.0, **over)
    return (out + case["bias"].double()) * case["f0"]


def aligned_case(B=2, H=8, C=32, Cout=32, ks=3):
    """positive activations and weights, so that every product's rounding error has the same sign: output channels
    [0, Cout/2) have weights 256.5 * 2^-k (exact in fp16, a tie at 9 significand bits), channels [Cout/2, Cout)
    weights 2^-24 * 2^-k (the smallest fp16 subnormal after the pre-scale, a tie between 0 and it one power of two
    lower)"""
    k = 8
    w = torch.empty(ks * ks, C, Cout)
    w[..., : Cout // 2] = 256.5 * 2.0 ** -k
    w[..., Cout // 2:] = 2.0 ** (-24 - k)
    assert umma_scale_log2(float(w.abs().max())) == k
    x = 1.0 + detfill.uniform("aligned:x", (B, H, H, C), 0.0, 1.0)
    x = x.half().float()                                       # exact in fp16: only the weights round
    return dict(ks=ks, f0=1.0, bias=torch.zeros(Cout), x0=x, taps=w.contiguous(), flags=0)


EMU_SHAPES = [  # B, H, C0, Cout, ks, C2
    (2, 8, 32, 48, 3, 0),
    (2, 8, 64, 32, 1, 0),
    (2, 8, 32, 32, 3, 32),
]


@pytest.mark.parametrize("shape", EMU_SHAPES, ids=lambda s: "B{}H{}C{}-{}k{}sc{}".format(*s))
def test_emulated_half_product_meets_its_bound(shape):
    B, H, C0, Cout, ks, C2 = shape
    for fam in CONV_FAMILIES + (SHORTCUT_FAMILIES if C2 else ()):
        case = conv_case(fam, B, H, C0, Cout, ks, C2=C2)
        assert float(case["x0"].abs().max()) < FP16_MAX              # the families stay below saturation
        ref, bound = half_bound(case)
        r = worst_ratio(emulate_half(case), ref, bound)
        assert r <= 1.0, (fam, r)


def test_half_bound_is_wider_than_the_split_bound_only_by_the_rounding():
    """the relative term is 2^-10 (one rounding of each operand), about 100x the hi/lo split's TAU"""
    assert 0.9e-3 < TAU_HALF < 1.0e-3 and TAU_HALF / TAU_MATMUL > 90


@pytest.mark.parametrize("ks", [1, 3])
def test_coarse_weights_leave_the_half_bound(ks):
    """weights rounded to 9 significand bits instead of fp16's 11 leave the bound where the errors align"""
    case = aligned_case(ks=ks)
    ref, bound = half_bound(case)
    assert worst_ratio(emulate_half(case), ref, bound) <= 1.0
    r = worst_ratio(emulate_half(case, wround=lambda v: round_bits(v, 9)), ref, bound)
    assert r > 1.5, r


def test_small_prescale_leaves_the_half_bound():
    """a pre-scale one power of two too small doubles the weights' subnormal error"""
    case = aligned_case()
    ref, bound = half_bound(case)
    k = conv_scale_log2(case)
    assert worst_ratio(emulate_half(case, k=k), ref, bound) <= 1.0
    r = worst_ratio(emulate_half(case, k=k - 1), ref, bound)
    assert r > 1.5, r


def test_half_rounding_saturates():
    x = torch.tensor([7e4, -1e6, 65504.0, 1.0 + 2.0 ** -12])
    assert round_fp16(x).tolist() == [65504.0, -65504.0, 65504.0, 1.0]


# ------------------------------------------------------------------------------------ rounding offsets on a grid
# Offsets, in fp16 ulps of a grid value, that tests/test_gpu_conv_half_paths.py adds to the half kernel's operands:
# +-1/2 is a tie (round-to-nearest-even keeps a grid value, whose significand is even), the others are nearer to it.
DELTAS = (2.0 ** -2, -2.0 ** -2, 2.0 ** -1 - 2.0 ** -12, -(2.0 ** -1 - 2.0 ** -12), 2.0 ** -1, -2.0 ** -1)


def ulp_fp16(v):
    """the smaller of the fp16 spacings on either side of each normal value of v (float64): below a power of two it
    is half the spacing above"""
    m, e = torch.frexp(v.double().abs())
    u = torch.ldexp(torch.ones_like(m), e - 11)
    return torch.where(m == 0.5, u / 2, u)


def nudge(v, g):
    """v (float64, normal fp16 values or zero) plus an offset from DELTAS, drawn per element from generator g, times
    ulp_fp16(v); zeros stay zero"""
    i = torch.randint(0, len(DELTAS), v.shape, generator=g)
    d = torch.tensor(DELTAS, dtype=torch.float64)[i]
    return torch.where(v == 0, v, v + d * ulp_fp16(v))


def trunc_fp16(x):
    """x (float64, fp16 normal range) rounded toward zero to 11 significand bits: a deliberately wrong rounding"""
    m, e = torch.frexp(x.double())
    return torch.ldexp(torch.trunc(torch.ldexp(m, torch.full_like(e, 11))), e - 11)


def grid_values(n=4096, seed=1):
    g = torch.Generator().manual_seed(seed)
    v = torch.randint(-128, 129, (n,), generator=g).double() * 2.0 ** -6
    w = torch.randint(-4, 5, (n,), generator=g).double() * 2.0 ** 6          # pre-scaled weights (k = 10)
    return torch.cat([v, w]), g


def test_nudged_grid_values_round_back_to_nearest():
    v, g = grid_values()
    x = nudge(v, g)
    assert torch.equal(x.float().double(), x)                              # exact fp32 inputs
    assert torch.equal(round_fp16(x), v)
    frac = ((x - v) / ulp_fp16(v))[v != 0]
    assert set(frac.unique().tolist()) == set(DELTAS)
    ties = frac.abs() == 0.5
    assert ties.any() and torch.equal(round_fp16(x)[v != 0][ties], v[v != 0][ties])


def test_truncation_is_off_by_one_ulp_where_the_offset_points_to_zero():
    """the wrong rounding the GPU test rules out: toward zero it lands one ulp below the grid value exactly where the
    offset's sign is opposite to the value's, and on it elsewhere"""
    v, g = grid_values(seed=2)
    x = nudge(v, g)
    t = trunc_fp16(x)
    inward = (x.abs() < v.abs())
    assert inward.any() and (~inward & (v != 0)).any()
    assert torch.equal(t[~inward], v[~inward])
    assert torch.equal((v - t)[inward].abs(), ulp_fp16(v)[inward])
    # an exact-grid conv through the two roundings: the outputs differ
    xs, ws = x[:64].view(8, 8), torch.ones(8, 8, dtype=torch.float64)
    assert not torch.equal(round_fp16(xs) @ ws, trunc_fp16(xs) @ ws)


# ----------------------------------------------------------------------------------------------------- config key
def test_config_key_default_and_validation():
    cfg = configs.workload("tiny")
    assert not hasattr(cfg.model, "conv_precision")
    assert arch.conv_precision(cfg) == "fp32"
    assert UNetMore_DDPM(cfg).conv_precision == "fp32"
    for p in ("fp32", "fp16"):
        cfg.model.conv_precision = p
        assert UNetMore_DDPM(cfg).conv_precision == p
    for bad in ("bf16", "FP16", "tf32", None, 16):
        cfg.model.conv_precision = bad
        with pytest.raises(ValueError, match="'fp32' or 'fp16'"):
            UNetMore_DDPM(cfg)


def test_state_dict_is_the_same_in_both_modes():
    cfg = configs.workload("tiny")
    a = UNetMore_DDPM(cfg)
    cfg16 = copy.deepcopy(cfg)
    cfg16.model.conv_precision = "fp16"
    b = UNetMore_DDPM(cfg16)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(sa[k].shape == sb[k].shape for k in sa)
    b.load_state_dict(sa, strict=True)
    a.load_state_dict(sb, strict=True)
    assert all(torch.equal(v, b.state_dict()[k]) for k, v in sa.items())


# ----------------------------------------------------------------------------------------------------- lowering
def lowered(name, precision):
    cfg = configs.workload(name)
    cfg.model.conv_precision = precision
    cfg, net, sd = make_module(cfg, "cpu")
    eng = Engine(net, _test_backend=Interpreter())
    eng.conv_mode = "umma"
    net._engine = eng
    return cfg, net, eng, eng.program(1 if name == "tiny128" else cfg.bench_batch)


def conv2d_layers(net):
    """parameter names of the reference's nn.Conv2d layers (4-D weights; NIN and linear weights are 2-D)"""
    return [n for n, p in net.named_parameters() if p.dim() == 4]


@pytest.mark.parametrize("name", ["tiny", "tiny_spade", "tiny_general", "tiny128"])
def test_half_flag_marks_exactly_the_conv2d_layers(name):
    cfg, net, e32, p32 = lowered(name, "fp32")
    _, _, e16, p16 = lowered(name, "fp16")
    for P32, P16 in ((p32.step_ops, p16.step_ops), (p32.cond_ops, p16.cond_ops)):
        assert len(P32) == len(P16)
        for a, b in zip(P32, P16):
            assert a.kind == b.kind
            assert not (a.flags & lib.F_HALF)
            assert b.flags & ~lib.F_HALF == a.flags
    assert p32.step_launches == p16.step_launches and p32.cond_launches == p16.cond_launches
    assert p16.n_umma == p32.n_umma and p16.n_simt == p32.n_simt

    tc = [o for o in p16.step_ops + p16.cond_ops if o.kind in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2)]
    half = [o for o in tc if o.flags & lib.F_HALF]
    nin_ops = [o for o in tc if not o.flags & lib.F_HALF]
    assert all(o.i3 == 3 for o in half)
    # every op without the flag is an attention block's qkv or NIN_3 projection: 1x1 at an attention resolution
    # whose channel count is the block's (qkv: 3C out)
    attn = [ms for ms in net.spec.mods if ms.kind == "attn"]
    assert len(nin_ops) == 2 * len(attn)
    for o in nin_ops:
        assert o.i0 == 1 and not o.src2 and any(o.H == ms.res and o.C0 == ms.in_ch and o.Cout in (ms.in_ch, 3 * ms.in_ch)
                                                for ms in attn)
    # the flagged ops are the nn.Conv2d layers: one op per 3x3 conv (first, Conv_0, Conv_1, SPADE, final) plus the
    # separate 1x1 Conv_2 ops; fused Conv_2 ride inside a Conv_1 op
    # (3x3 convs with a fused norm below 8x8 run on the CUDA cores, unchanged)
    convs = conv2d_layers(net)
    n3 = sum(1 for n in convs if not n.endswith("Conv_2.weight"))
    n_sc = sum(1 for n in convs if n.endswith("Conv_2.weight"))
    ops = p16.step_ops + p16.cond_ops
    simt3 = sum(1 for o in ops if (o.kind == lib.OP_CONV_SIMT and o.i0 == 3) or o.kind == lib.OP_CONV_SMALLN)
    simt1 = sum(1 for o in ops if o.kind == lib.OP_CONV_SIMT and o.i0 == 1)
    fused = sum(1 for o in half if o.src2)
    assert sum(1 for o in half if o.i0 == 3) + simt3 == n3
    assert fused + sum(1 for o in half if o.i0 == 1) + simt1 == n_sc
    # CUDA-core convs, attention and linear layers never carry the flag
    for o in p16.step_ops + p16.cond_ops:
        if o.kind not in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
            assert not o.flags & lib.F_HALF


def test_separate_skip_projection_takes_the_half_mode():
    cfg = configs.workload("tiny")
    cfg.model.conv_precision = "fp16"
    cfg, net, sd = make_module(cfg, "cpu")
    eng = Engine(net, _test_backend=Interpreter())
    eng.conv_mode, eng.fuse_shortcut = "umma", "0"
    P = eng.program(cfg.bench_batch)
    sc = [o for o in P.step_ops if o.kind == lib.OP_CONV_UMMA and o.i0 == 1 and o.flags & lib.F_HALF]
    assert sc and not any(o.src2 for o in P.step_ops)


@pytest.mark.parametrize("name", ["tiny", "tiny_spade"])
def test_half_lowering_computes_the_same_network(name):
    """the interpreter ignores MCVD_F_HALF (fp32 everywhere): the half-mode program is the same network"""
    cfg, net, eng, P = lowered(name, "fp16")
    _, net32, _, _ = lowered(name, "fp32")
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    t = torch.full((B,), 37, dtype=torch.long)
    assert torch.equal(net(x, t, cond=cond), net32(x, t, cond=cond))


def test_modes_never_share_keys(tmp_path):
    _, _, e32, p32 = lowered("tiny", "fp32")
    _, _, e16, p16 = lowered("tiny", "fp16")
    assert p32.conv_precision == "fp32" and p16.conv_precision == "fp16"
    k32 = {k for k in e32.packed if isinstance(k, tuple) and k[1] == "umma"}
    k16 = {k for k in e16.packed if isinstance(k, tuple) and k[1] == "umma"}
    # only the NIN projections' images (hi/lo in both modes) share a key; every half image is tagged
    shared = k32 & k16
    assert shared and all(re.search(r"\.(qkv|NIN_3)$", k[0]) for k in shared)
    assert all(k[-1] == "fp16" for k in k16 - shared) and len(k16 - shared) == len(k32 - shared)
    # weight-cache file names (the interpreter backend has none: compute them as a CUDA engine would)
    paths = []
    for e in (e32, e16):
        e.cache_dir, e.backend = str(tmp_path), None
        paths.append(e._cache_path())
    assert paths[0] and paths[1] and paths[0] != paths[1]


# ------------------------------------------------------------------------------------------- tile heights (README)
# The conv groups (ks, H, Cin, Csc, Cout, n tile) that half mode moves from 128- to 192-position tiles at the benchmark
# batch on an H100 SXM (132 SMs), as the README's "Half-precision convolutions" section lists them
HALF_MT192 = {
    "cfg2": {(3, 64, 192, 0, 192, 192), (3, 64, 192, 192, 192, 192)},
    "cfg3": {(3, 64, 128, 0, 384, 192)},
    "cfg4": {(3, 64, 32, 0, 192, 192), (3, 64, 192, 0, 192, 192), (3, 64, 192, 384, 192, 192),
             (3, 64, 192, 576, 192, 192), (3, 64, 384, 0, 192, 192), (3, 64, 384, 0, 384, 192),
             (3, 64, 384, 384, 384, 192), (3, 64, 576, 0, 192, 192)},
    "cfg5": {(3, 64, 384, 0, 384, 192), (3, 64, 384, 384, 384, 192)},
}


@pytest.mark.parametrize("name", sorted(HALF_MT192))
def test_half_mode_tile_heights_match_the_readme(name):
    """every tensor-core conv of the lowered forward keeps its tile height in half mode except the README's groups,
    which go from 128 to 192 positions (the launcher's own plan, mcvd_conv_umma_launch_info, at 132 SMs)"""
    heights = {}
    for precision in ("fp32", "fp16"):
        cfg = configs.workload(name)
        cfg.model.conv_precision = precision
        cfg, net, sd = make_module(cfg, "cpu")
        eng = Engine(net, _test_backend=Interpreter())
        P = eng.program(cfg.bench_batch)
        heights[precision] = [((o.i0, o.H, o.C0 + o.C1, o.C2 + o.C3, o.Cout, o.i1), lib.conv_umma_launch_info(o, 132)["mt"])
                              for o in P.step_ops + P.cond_ops if o.kind in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2)]
        del P, eng, net
    assert [g for g, _ in heights["fp32"]] == [g for g, _ in heights["fp16"]]
    changed = {g32 for (g32, m32), (_, m16) in zip(heights["fp32"], heights["fp16"]) if m32 != m16}
    assert changed == HALF_MT192[name]
    assert all(m32 == 128 and m16 == 192 for (g, m32), (_, m16) in zip(heights["fp32"], heights["fp16"])
               if g in changed)
