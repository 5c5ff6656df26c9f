"""The tensor-core conv and attention on the H100 at trained-like value ranges, judged element by element.

Op level: every case of the input families of tests/test_value_ranges_cpu.py (activations spanning 2^-24 .. 2^11,
per-channel weight scales down to 2^-24, layers with max |w| from 2^-40 to 2^44, cancelling outputs, lopsided fused
shortcuts; attention logits up to 80, running maxima that jump by 100, ties, constant rows, v offset by 1e3) runs on
the kernels and is compared with the float64 Interpreter: the tensor-core kinds against the split error model
(conv_bound / attention_bound), the CUDA-core kinds against the replay's TAU*A + u|ref|.  Dropping either cross
product (i3 = 1 / 2) must leave the conv bound, and an attention scale off by 2^-12 the attention bound.

Network level: the op-by-op replay (tests/program_replay.py) of networks with a trained-like weight profile and with
the reference's fresh initialisation, held to the replay's bounds, after checking that each profile reaches the
value regimes it exists for.
"""
import gc
import math
import time

import pytest
import torch

from common import make_module
from mcvd_b200 import detfill, lib
from mcvd_b200.program import Engine
from program_replay import replay_program, twin_engine
from test_value_ranges_cpu import (ATTN_FAMILIES, CONV_FAMILIES, SHORTCUT_FAMILIES, attention_bound, attention_op,
                                   attention_qkv, conv_bound, conv_case, conv_op, perturbation_families,
                                   worst_ratio, SCALE_PERTURBATION)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run(op):
    arr = lib.make_ops([op])
    lib.validate_program(arr, 1)
    lib.run_program(arr, 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def packer():
    """an engine whose weight packing (power-of-two pre-scale included) serves the op-level cases"""
    return Engine(make_module("tiny", DEV)[1])


# ---------------------------------------------------------------------------------------------------------- conv
CONV_SHAPES = [
    # kind, B, H, C0, C1, Cout, ks, C2, i2 (work organisation), tab, res
    ("umma", 2, 16, 64, 0, 96, 3, 0, 1, True, True),          # streaming 3x3, fused norm, residual
    ("umma", 3, 8, 32, 32, 64, 3, 0, 1, False, False),        # virtual concat
    ("umma", 2, 16, 96, 0, 192, 1, 0, 1, True, False),        # 1x1 streaming (qkv-like)
    ("umma", 4, 8, 64, 0, 64, 1, 0, 2, False, True),          # 1x1 input-stationary (NIN_3-like)
    ("umma", 2, 16, 64, 0, 64, 3, 32, 1, True, False),        # fused 1x1 shortcut
    ("umma2", 2, 16, 64, 0, 64, 3, 32, 0, True, False),       # planar-table variant, fused shortcut
    ("umma2", 2, 8, 48, 48, 96, 3, 0, 0, False, True),        # planar-table variant, K-block 16
    ("simt", 2, 16, 64, 0, 96, 3, 0, 0, False, True),
]


def planar(tab):
    return torch.stack([tab[..., 0], tab[..., 1] * tab[..., 2], tab[..., 3]], 1).contiguous()


def run_conv(packer, kind, case, split=3, nacc=0):
    """the case on the kernel of ``kind``: output [B,H,W,Cout] fp32"""
    B, H, W, C0 = case["x0"].shape
    C1 = 0 if case.get("x1") is None else case["x1"].shape[3]
    Cout, ks = case["taps"].shape[2], case["ks"]
    dst = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    taps, sc = case["taps"], case.get("taps_sc")
    if kind == "simt":
        assert sc is None and case.get("tab") is None
        op = conv_op(case, lib.OP_CONV_SIMT, taps, 1.0, dst)
        op.i1 = Cout
        run(op)
        return dst
    if kind == "umma":
        nt = max(d for d in range(16, 257, 16) if Cout % d == 0)
        kb = lib.umma_kblock(C0, C1)
        w, f1 = packer._pack_umma(taps, nt, kb) if sc is None else packer._pack_umma_fused(taps, sc, nt, kb)
        op = conv_op(case, lib.OP_CONV_UMMA, w, f1, dst)
        op.i1, op.i2 = nt, nacc
    else:
        nt = lib.umma2_pick_nt(Cout, ks)
        C2 = 0 if sc is None else sc.shape[1]
        kb = lib.umma2_plan(H, W, ks, C0, C1, C2, 0, nt, False)
        w, f1 = packer._pack_umma2(taps, sc, nt, kb)
        tab3 = None if case.get("tab") is None else planar(case["tab"])
        op = conv_op(dict(case, tab=tab3), lib.OP_CONV_UMMA2, w, f1, dst)
        op.i1, op.i2 = nt, kb
    op.i3 = split
    run(op)
    return dst


def conv_cases(shape):
    kind, B, H, C0, C1, Cout, ks, C2, nacc, tab, res = shape
    fams = CONV_FAMILIES + (SHORTCUT_FAMILIES if C2 else ())
    for fam in fams:
        case = conv_case(fam, B, H, C0, Cout, ks, C1=C1, C2=C2, tab=tab, res=res)
        yield fam, {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in case.items()}


@pytest.mark.parametrize("shape", CONV_SHAPES, ids=lambda s: "{}-B{}H{}C{}+{}-{}k{}sc{}n{}".format(*s[:9]))
def test_conv_value_ranges(packer, shape):
    kind, nacc = shape[0], shape[8]
    report = []
    for fam, case in conv_cases(shape):
        ref, bound = conv_bound(case, tensor_core=kind != "simt")
        out = run_conv(packer, kind, case, nacc=nacc)
        r = worst_ratio(out, ref, bound)
        report.append(f"{fam} {r:.3g}")
    print(f"\n{shape}: worst err/bound " + ", ".join(report))
    assert all(float(s.split()[1]) <= 1.0 for s in report), report


@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("shape", [s for s in CONV_SHAPES if s[0] != "simt"],
                         ids=lambda s: "{}-B{}H{}C{}+{}-{}k{}sc{}n{}".format(*s[:9]))
def test_conv_bound_sees_a_dropped_product(packer, shape, split):
    for fam, case in conv_cases(shape):
        if fam == "zero":
            continue
        ref, bound = conv_bound(case)
        r = worst_ratio(run_conv(packer, shape[0], case, split=split, nacc=shape[8]), ref, bound)
        assert r > 1.0, (fam, r)


# ----------------------------------------------------------------------------------------------------- attention
HEAD_DIMS = (32, 48, 64, 96, 128, 192)
TOKENS = {64: (34, 4), 256: (2, 2), 1024: (1, 1)}          # T -> (B, heads): 136 CTAs at T = 64


def run_attention(kind, qkv, heads, d, scale):
    B, T, C3 = qkv.shape
    dst = torch.full((B, T, C3 // 3), float("nan"), device=DEV)
    scratch = None
    if kind == "umma":
        scratch = torch.empty(lib.attention_scratch_bytes(B, T, C3 // 3), dtype=torch.uint8, device=DEV)
    run(attention_op(lib.OP_ATTENTION_UMMA if kind == "umma" else lib.OP_ATTENTION, B, T, heads, d, scale, qkv, dst,
                     scratch))
    return dst


@pytest.mark.parametrize("kind", ["umma", "simt"])
@pytest.mark.parametrize("T", sorted(TOKENS))
@pytest.mark.parametrize("d", HEAD_DIMS)
def test_attention_value_ranges(kind, T, d):
    B, heads = TOKENS[T]
    report = []
    for fam in ATTN_FAMILIES:
        qkv, scale = attention_qkv(fam, B, T, heads, d)
        qkv = qkv.to(DEV)
        ref, bound = attention_bound(qkv, heads, d, scale, tensor_core=kind == "umma")
        out = run_attention(kind, qkv, heads, d, scale)
        report.append(f"{fam} {worst_ratio(out, ref, bound):.3g}")
        if kind == "umma" and fam in perturbation_families(d):
            off = run_attention(kind, qkv, heads, d, scale * (1 + SCALE_PERTURBATION))
            assert worst_ratio(off, ref, bound) > 1.0, (fam, "a perturbed logit scale stays inside the bound")
    print(f"\n{kind} T={T} d={d}: worst err/bound " + ", ".join(report))
    assert all(float(s.split()[1]) <= 1.0 for s in report), report


# ------------------------------------------------------------------------------------------------ stressed replay
def zero_init_layers(net):
    """weights the reference initialises with init_scale = 0, i.e. default_init(1e-10) (reference
    models/better/layers.py:77-80): every ResBlock's Conv_1 (layerspp.py:586), every attention block's NIN_3
    (layerspp.py:219) and the last conv"""
    last = f"unet.all_modules.{net.spec.mods[-1].idx}.weight"
    return lambda k: k.endswith("Conv_1.weight") or k.endswith("NIN_3.W") or k == last


FILM_W = 0.25


def stressed_state_dict(net, sd, variant, seed=1234):
    """Re-draw a state_dict in place, deterministically (detfill):
      trained  conv / linear / NIN weights: the detfill draw times a per-output-channel 2^U(-8, 2), about 1 % of the
               channels another x8; GroupNorm weight U(-0.5, 3), bias U(-1, 1); the FiLM projections (Dense_0): the
               detfill draw x FILM_W, bias U(-1.5, 2.5) on the scale half and U(-1, 1) on the shift half, so that
               1 + scale spans about [-1, 4]; the reference's zero-init layers at 2^-4 of the rest.  The q and k
               projections need no extra factor: the channel scales and GroupNorm gains alone peak the softmax, with
               largest scaled logits of 122 (cfg1) to 317 (cfg3) in the replayed rows; measured FiLM gains
               1 + scale span [-0.70, 3.71]
      fresh    the detfill profile, but the zero-init layers at the reference's default_init(1e-10) magnitude:
               U(+-sqrt(3e-10 / fan_avg)), fan_avg = (fan_in + fan_out) / 2"""
    detfill.randomize_state_dict(sd, seed)
    zero_init = zero_init_layers(net)
    for k, v in sd.items():
        if not torch.is_floating_point(v) or k.split(".")[-1] in ("betas", "alphas", "alphas_prev", "sigmas"):
            continue
        leaf = k.split(".")[-1]
        matrix = leaf == "W" or (leaf == "weight" and v.dim() >= 2)
        if variant == "fresh":
            if matrix and zero_init(k):
                fan_in, fan_out = (v.shape[0], v.shape[1]) if leaf == "W" else (v[0].numel(), v.shape[0] * v[0, 0].numel())
                a = math.sqrt(3e-10 / ((fan_in + fan_out) / 2))
                v.copy_(detfill.uniform(k + ":fresh", tuple(v.shape), -a, a, seed))
            continue
        if matrix and ".Dense_0." in k:
            v.mul_(FILM_W)
        elif matrix:
            n_out = v.shape[1] if leaf == "W" else v.shape[0]
            f = torch.exp2(detfill.uniform(k + ":chan", (n_out,), -8.0, 2.0, seed))
            f = torch.where(detfill.uniform(k + ":outlier", (n_out,), 0.0, 1.0, seed) < 0.01, f * 8.0, f)
            v.mul_(f.view(1, -1) if leaf == "W" else f.view(-1, *([1] * (v.dim() - 1))))
            if zero_init(k):
                v.mul_(2.0 ** -4)
        elif leaf == "weight":                                   # GroupNorm affine scale
            v.copy_(detfill.uniform(k + ":gn", tuple(v.shape), -0.5, 3.0, seed))
        elif ".Dense_0." in k:                                   # FiLM bias: scale half, shift half
            half = v.shape[0] // 2
            v[:half] = detfill.uniform(k + ":film", (half,), -1.5, 2.5, seed)
            v[half:] = detfill.uniform(k + ":shift", (v.shape[0] - half,), -1.0, 1.0, seed)
        elif "GroupNorm" in k or "Norm_0" in k:
            v.copy_(detfill.uniform(k + ":gnb", tuple(v.shape), -1.0, 1.0, seed))
    return sd


def stressed_module(name, variant, dev=DEV):
    cfg, net, _ = make_module(name, dev)
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    net.load_state_dict(stressed_state_dict(net, sd, variant))
    return cfg, net


def regimes(spec, P):
    """value ranges a lowered program met in its last run: largest scaled attention logit, FiLM gains 1 + scale of
    the first clip (None without FiLM), an upper bound on the smallest max |w| of a tensor-core conv (its pre-scale
    puts max |w| below 512 * f1), largest |x| of a conv output"""
    out = dict(logit=0.0, film=None, tc_wmax=float("inf"), conv_absmax=0.0)
    bufs = {t.data_ptr(): t for t in P.keep}
    for op in P.step_ops:
        if op.kind in (lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA):
            q, k, _ = bufs[op.src0].view(op.B, op.H * op.W, 3, op.i0, op.i1).double().unbind(2)
            out["logit"] = max(out["logit"], float(torch.einsum("bthd,bshd->bhts", q, k).amax()) * op.f0)
        if op.kind in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2):
            out["tc_wmax"] = min(out["tc_wmax"], 512.0 * op.f1)
        if op.kind in (lib.OP_CONV_UMMA, lib.OP_CONV_UMMA2, lib.OP_CONV_SIMT, lib.OP_CONV_SMALLN):
            out["conv_absmax"] = max(out["conv_absmax"], float(bufs[op.dst].abs().max()))
    offs = [(o, ms.out_ch if i else ms.in_ch) for ms in spec.mods if ms.kind == "res" for i, o in enumerate(ms.film_off)]
    if offs:
        gains = 1.0 + torch.cat([P.film.view(-1)[o:o + c] for o, c in offs])   # row 0: every clip shares one t
        out["film"] = (float(gains.min()), float(gains.max()))
    return out


STRESSED_ROWS = [
    ("cfg1", "trained", "umma"),
    ("cfg1", "trained", "simt"),
    ("cfg2", "trained", "umma"),
    ("cfg3", "trained", "umma"),       # SPADE
    ("cfg4", "trained", "umma"),       # head dim 192
    ("cfg1", "fresh", "umma"),
]


def stressed_replay(name, variant, mode, dev=DEV, backend=None):
    """replay of one row at B = 4 -> (Replay, regimes met)"""
    gc.collect()
    t0 = time.perf_counter()
    cfg, net = stressed_module(name, variant, dev)
    real = Engine(net, _test_backend=backend)
    real.conv_mode = mode
    real.epilogue_stats = False
    real.attn_mode = "simt" if mode == "simt" else "umma"
    twin = twin_engine(real, net)
    B = 4
    x, cond = detfill.synthetic_inputs(cfg, B)
    R = replay_program(real, twin, B, x.to(dev), cond.to(dev), 437.0, detfill.normal("replay_z", x.shape).to(dev))
    seen = regimes(real.spec, real.program(B))
    R.release()
    del real, twin, net
    gc.collect()
    film = "none" if seen["film"] is None else "[{:.3g}, {:.3g}]".format(*seen["film"])
    print(f"\n{name} B={B} {variant} {mode}: {R.n_ops} ops, {time.perf_counter() - t0:.1f} s; largest scaled logit "
          f"{seen['logit']:.3g}, FiLM gains {film}, smallest tensor-core max|w| < {seen['tc_wmax']:.3g}, "
          f"largest |conv output| {seen['conv_absmax']:.4g}\n{R.table()}")
    return R, seen


@pytest.mark.parametrize("name,variant,mode", STRESSED_ROWS, ids=["-".join(r) for r in STRESSED_ROWS])
def test_stressed_replay(name, variant, mode):
    torch.cuda.empty_cache()
    R, seen = stressed_replay(name, variant, mode)
    if variant == "trained":
        assert seen["logit"] >= 20.0
        if seen["film"] is not None:
            assert seen["film"][0] <= -0.5 and seen["film"][1] >= 3.0
    elif mode != "simt":
        assert seen["tc_wmax"] <= 2.0 ** -20
    assert not R.failures, f"{len(R.failures)} outputs over their bound:\n" + "\n".join(R.failures[:20])
    assert R.whole_program_identical
