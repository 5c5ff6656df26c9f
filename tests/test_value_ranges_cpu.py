"""Error model of the tensor-core kinds' fp16 hi/lo split, checked on the CPU against a torch emulation of the split.

The tensor-core conv and attention carry each operand as v = hi + lo (hi = fp16(v), lo = fp16(v - hi), both
saturating) and sum the products hi*hi + lo*hi + hi*lo in fp32.  A pair is exact to about 2^-22 |v| while lo is a
normal fp16 number, and to an absolute 2^-25 (half the smallest fp16 subnormal) below that.  Activations, q, k, v and
P are split unscaled, so they keep that floor; the conv's weights are split after a per-layer power-of-two pre-scale
2^k (mcvd_b200.program.umma_scale_log2) that puts the layer's max |w| in [256, 512), so their floor is 2^-25 * 2^-k.
The per-element bound of the tensor-core kinds is therefore the replay's relative bound (tests/program_replay.py)
plus a floor term:

    conv:       TAU*A + u|ref| + 2^-25 * (sum |w| over the products + 2^-k * sum |x| over the products)
    attention:  TAU * sum_s p_ts (M_ts |v_s - o_t| + |v_s|) + u|ref|
                + 2^-25 * (2 * scale * (sum_d |q_t| + max_s sum_d |k_s|) * max|v|                logits
                           + sum_s |v_s| / l                                                      P
                           + 1)                                                                   v

with A the op evaluated on absolute values (Interpreter.exec(magnitude=True)), p the softmax, M_ts = |scale| *
sum_d |q_td||k_sd| and l the softmax denominator sum_s exp(s - max).  The conv floors come from the float64 Interpreter on a ones-mask with |w| and on |x| with unit
weights.  CUDA-core kinds keep the replay's TAU*A + u|ref|.

The attention's relative term is not the Interpreter's magnitude (2 * TAU * max logit magnitude * max|v|, too loose
to see a dropped product) but the first-order propagation of TAU through the logits and P.V (attention_bound).

The tests below show the model is tight on the input families the GPU tests use (tests/test_gpu_value_ranges.py):
the emulated split stays inside it (at most 0.03 of it for attention), and dropping any one cross product leaves it
(the conv kernels' i3 = 1 / 2 experiments; q_lo*k_hi, q_hi*k_lo, P_lo*V_hi or P_hi*V_lo for attention), and so does
an attention scale off by 2^-12.
"""
import math

import pytest
import torch

from mcvd_b200 import detfill, lib
from mcvd_b200.lib import McvdOp
from mcvd_b200.program import umma_scale_log2
from op_interpreter import Interpreter
from program_replay import TAU_MATMUL

FP16_MAX = 65504.0
SPLIT_FLOOR = 2.0 ** -25          # absolute error of a hi/lo pair below the fp16 normal range
U_FP32 = 2.0 ** -23               # rounding of the reference and of the kernel's output to fp32


def split_fp16(x):
    """(hi, lo) of the kernels' saturating split (cvt.rn.satfinite) as float64 tensors"""
    x = x.float()
    hi = x.clamp(-FP16_MAX, FP16_MAX).half().float()
    lo = (x - hi).clamp(-FP16_MAX, FP16_MAX).half().float()
    return hi.double(), lo.double()


# ---------------------------------------------------------------------------------------------------------- conv
# A conv case is a dict of fp32 tensors on one device: x0 [B,H,W,C0], optional x1 [B,H,W,C1] (virtual concat),
# taps [ks*ks][C0+C1][Cout], bias [Cout], optional res [B,H,W,Cout], tab [B,C0+C1,4] (norm table; flags carry
# F_ACT_IN), y [B,H,W,C2] + taps_sc [1][C2][Cout] (fused 1x1 shortcut), and the ints / floats ks, f0, flags.

def conv_op(case, kind, w, f1, dst, **over):
    """the McvdOp of a case; ``over`` replaces tensors (or drops them with None)"""
    t = dict(case, **over)
    B, H, W, C0 = t["x0"].shape
    o = McvdOp()
    o.kind, o.B, o.H, o.W, o.C0, o.Cout = kind, B, H, W, C0, t["taps"].shape[2]
    o.i0, o.f0, o.f1, o.flags = t["ks"], t["f0"], f1, t.get("flags", 0)
    o.src0, o.w, o.dst, o.bias = t["x0"].data_ptr(), w.data_ptr(), dst.data_ptr(), t["bias"].data_ptr()
    if t.get("x1") is not None:
        o.C1, o.src1 = t["x1"].shape[3], t["x1"].data_ptr()
    if t.get("res") is not None:
        o.aux0 = t["res"].data_ptr()
    if t.get("tab") is not None:
        o.aux1 = t["tab"].data_ptr()
    if t.get("y") is not None:
        o.C2, o.src2 = t["y"].shape[3], t["y"].data_ptr()
    return o


def interp_conv(case, magnitude=False, **over):
    """CONV_UMMA of a case in float64 (stored to fp32): the reference, or with magnitude=True the magnitude A of
    its terms.  Weights are the case's fp32 taps (f1 = 1)."""
    t = dict(case, **over)
    it = Interpreter(torch.float64)
    w = t["taps"].reshape(-1) if t.get("y") is None else torch.cat([t["taps"].reshape(-1), t["taps_sc"].reshape(-1)])
    dst = torch.empty(t["x0"].shape[:3] + (t["taps"].shape[2],), device=w.device)
    for v in list(t.values()) + [w, dst]:
        if isinstance(v, torch.Tensor):
            it.register(v)
    it.exec(conv_op(t, lib.OP_CONV_UMMA, w, 1.0, dst), magnitude=magnitude)
    return dst.double()


def conv_scale_log2(case):
    """the pre-scale the error model assumes: the one that puts the conv's max |w| in [256, 512)"""
    amax = float(case["taps"].abs().max())
    if case.get("y") is not None:
        amax = max(amax, float(case["taps_sc"].abs().max()))
    return umma_scale_log2(amax)


def conv_bound(case, tensor_core=True):
    """(float64 reference, per-element bound) of a conv case"""
    ref = interp_conv(case)
    bound = TAU_MATMUL * interp_conv(case, magnitude=True) + U_FP32 * ref.abs()
    if tensor_core:
        ones = lambda n: None if case.get(n) is None else torch.ones_like(case[n])
        zero_bias = torch.zeros_like(case["bias"])
        # sum |w| over the products with a real (non-padding) input: the activations' floor
        fw = interp_conv(case, True, x0=ones("x0"), x1=ones("x1"), y=ones("y"), tab=None, res=None, bias=zero_bias,
                         flags=case.get("flags", 0) & ~lib.F_ACT_IN)
        # sum |x| over the products: the weights' floor, 2^-k of it in the unscaled domain
        fx = interp_conv(case, True, taps=ones("taps"), taps_sc=ones("taps_sc"), res=None, bias=zero_bias)
        bound = bound + SPLIT_FLOOR * (fw + 2.0 ** -conv_scale_log2(case) * fx)
    return ref, bound


def worst_ratio(out, ref, bound):
    err = (out.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(torch.nan_to_num(r, nan=float("inf")).max())


def emulate_conv(case, split=3, k=None):
    """the tensor-core conv's arithmetic in float64: split activations and pre-scaled weights, the hi*hi product plus
    lo*hi (split bit 0) and hi*lo (split bit 1).  Cases without a norm table, residual or output activation."""
    assert case.get("tab") is None and case.get("res") is None and not case.get("flags", 0)
    k = conv_scale_log2(case) if k is None else k
    zero_bias = torch.zeros_like(case["bias"])
    parts = {n: split_fp16(case[n]) for n in ("x0", "x1", "y") if case.get(n) is not None}
    wparts = {n: split_fp16(case[n] * 2.0 ** k) for n in ("taps", "taps_sc") if case.get(n) is not None}
    total = 0
    for a, b, on in ((0, 0, True), (1, 0, bool(split & 1)), (0, 1, bool(split & 2))):
        if on:
            over = {n: p[a].float() for n, p in parts.items()}
            over.update({n: p[b].float() * 2.0 ** -k for n, p in wparts.items()})
            total = total + interp_conv(case, bias=zero_bias, f0=1.0, **over)
    return (total + case["bias"].double()) * case["f0"]


def _pow2(name, shape, lo, hi):
    return torch.exp2(detfill.uniform(name, shape, lo, hi))


CONV_FAMILIES = ("unit", "wide_acts", "channel_scales", "zero", "max_2^-30", "max_2^-40", "max_2^36", "max_2^44",
                 "cancel")
SHORTCUT_FAMILIES = ("sc_main_tiny", "sc_shortcut_tiny")


def conv_case(family, B, H, C0, Cout, ks, C1=0, C2=0, tab=False, res=False, act_out=False, seed=""):
    """one conv case of an input family (deterministic, CPU tensors):
      unit            x ~ N(0,1), w ~ U(+-sqrt(3/fan_in)) (the detfill profile)
      wide_acts       |x| spans 2^-24 .. 2^11 in one tensor, with whole channels and one whole image of tiny values
      channel_scales  per-output-channel weight scales 2^U(-24, 0) of the layer max
      zero            an all-zero layer
      max_2^e         the layer (weights, bias and residual) rescaled to max |w| = 2^e
      cancel          duplicated input channels against +-w column pairs: half the outputs are exactly 0 with large A
      sc_*_tiny       the fused shortcut's main (or shortcut) weights 1e-6 of the other segment's"""
    key = f"vr:{family}:{B}:{H}:{C0}:{C1}:{C2}:{Cout}:{ks}:{seed}"
    Cin = C0 + C1
    res_scale = 4.0
    x = detfill.normal(key + ":x", (B, H, H, Cin))
    w = detfill.uniform(key + ":w", (ks * ks, Cin, Cout), -1.0, 1.0) * math.sqrt(3.0 / (Cin * ks * ks))
    case = dict(ks=ks, f0=0.7071 if res else 1.0, bias=detfill.uniform(key + ":b", (Cout,), -0.1, 0.1))
    if family == "wide_acts":
        x = x * _pow2(key + ":xs", (B, H, H, Cin), -24.0, 11.0)
        x[..., : Cin // 8] *= 2.0 ** -20                       # channels of tiny values
        x[0] = detfill.normal(key + ":x0", (H, H, Cin)) * 2.0 ** -22   # an image of tiny values
    elif family == "channel_scales":
        w = w * _pow2(key + ":ws", (1, 1, Cout), -24.0, 0.0)
    elif family == "zero":
        w = torch.zeros_like(w)
    elif family.startswith("max_2^"):
        c = 2.0 ** int(family[6:]) / float(w.abs().max())
        w, case["bias"], res_scale = w * c, case["bias"] * c, c
    elif family == "cancel":
        h = Cin // 2
        x[..., h:2 * h] = x[..., :h]
        w[:, h:2 * h, : Cout // 2] = -w[:, :h, : Cout // 2]
        case["bias"][: Cout // 2] = 0.0
    if C2:
        case["y"] = detfill.normal(key + ":y", (B, H, H, C2))
        case["taps_sc"] = detfill.uniform(key + ":wsc", (1, C2, Cout), -1.0, 1.0) * math.sqrt(3.0 / C2)
        if family == "sc_main_tiny":
            w = w * 1e-6
        elif family == "sc_shortcut_tiny":
            case["taps_sc"] = case["taps_sc"] * 1e-6
    case["x0"] = x[..., :C0].contiguous()
    if C1:
        case["x1"] = x[..., C0:].contiguous()
    case["taps"] = w.contiguous()
    flags = 0
    if tab:
        case["tab"] = torch.stack([detfill.normal(key + ":m", (B, Cin)) * 0.3,
                                   detfill.uniform(key + ":r", (B, Cin), 0.5, 1.5),
                                   detfill.uniform(key + ":g", (B, Cin), -0.5, 3.0),
                                   detfill.uniform(key + ":s", (B, Cin), -1.0, 1.0)], 2).contiguous()
        flags |= lib.F_ACT_IN
    if res:
        case["res"] = detfill.normal(key + ":res", (B, H, H, Cout)) * res_scale
    if act_out:
        flags |= lib.F_ACT_OUT
    case["flags"] = flags
    return case


EMU_SHAPES = [  # B, H, C0, Cout, ks, C2
    (2, 8, 32, 48, 3, 0),
    (2, 8, 64, 32, 1, 0),
    (2, 8, 32, 32, 3, 32),
]


@pytest.mark.parametrize("shape", EMU_SHAPES, ids=lambda s: "B{}H{}C{}-{}k{}sc{}".format(*s))
def test_emulated_split_meets_the_conv_bound(shape):
    B, H, C0, Cout, ks, C2 = shape
    for fam in CONV_FAMILIES + (SHORTCUT_FAMILIES if C2 else ()):
        case = conv_case(fam, B, H, C0, Cout, ks, C2=C2)
        ref, bound = conv_bound(case)
        r = worst_ratio(emulate_conv(case), ref, bound)
        assert r <= 1.0, (fam, r)


@pytest.mark.parametrize("shape", EMU_SHAPES, ids=lambda s: "B{}H{}C{}-{}k{}sc{}".format(*s))
@pytest.mark.parametrize("split", [1, 2])
def test_dropped_products_leave_the_conv_bound(shape, split):
    """the bound resolves one dropped cross product (about 2^-12 of each term) on every family with nonzero
    weights, the floor-dominated ones included"""
    B, H, C0, Cout, ks, C2 = shape
    for fam in CONV_FAMILIES + (SHORTCUT_FAMILIES if C2 else ()):
        if fam == "zero":
            continue
        case = conv_case(fam, B, H, C0, Cout, ks, C2=C2)
        ref, bound = conv_bound(case)
        r = worst_ratio(emulate_conv(case, split=split), ref, bound)
        assert r > 1.0, (fam, r)
        if fam == "unit":
            assert r > 4.0, r


def test_clamped_weight_scale_leaves_the_bound():
    """a pre-scale clamped to |k| <= 24 (the first implementation) puts a layer with max |w| = 2^-40 into fp16
    subnormals: the model reports it, while the [256, 512) scale meets it"""
    case = conv_case("max_2^-40", 2, 8, 32, 32, 3)
    ref, bound = conv_bound(case)
    assert worst_ratio(emulate_conv(case, k=24), ref, bound) > 10.0
    assert worst_ratio(emulate_conv(case), ref, bound) <= 1.0


def test_weight_scale_puts_every_layer_in_range():
    for e in range(-117, 128):
        for f in (0.5, 0.75, 0.999999):
            amax = math.ldexp(f, e)
            k = umma_scale_log2(amax)
            assert abs(k) <= 126 and 256.0 <= math.ldexp(amax, k) < 512.0, (amax, k)
    assert umma_scale_log2(0.0) == 0
    assert umma_scale_log2(2.0 ** -126) == 126          # the smallest normal weights stay short of 256


# ----------------------------------------------------------------------------------------------------- attention
def attention_op(kind, B, T, heads, d, scale, qkv, dst, scratch=None):
    side = int(round(math.sqrt(T)))
    o = McvdOp()
    o.kind, o.B, o.H, o.W, o.C0, o.i0, o.i1, o.f0 = kind, B, side, T // side, heads * d, heads, d, scale
    o.src0, o.dst = qkv.data_ptr(), dst.data_ptr()
    if scratch is not None:
        o.dst2 = scratch.data_ptr()
    return o


def interp_attention(qkv, heads, d, scale, magnitude=False):
    B, T, C3 = qkv.shape
    it = Interpreter(torch.float64)
    dst = torch.empty(B, T, C3 // 3, device=qkv.device)
    it.register(qkv)
    it.register(dst)
    it.exec(attention_op(lib.OP_ATTENTION, B, T, heads, d, scale, qkv, dst), magnitude=magnitude)
    return dst.double()


def attention_bound(qkv, heads, d, scale, tensor_core=True):
    """(float64 reference, per-element bound) of an attention over qkv [B, T, 3C] fp32.

    CUDA-core: the replay's TAU*A + u|ref| (A from Interpreter.exec(magnitude=True)).  Tensor-core: the first-order
    propagation of a relative error TAU in every product.  Logits s_ts off by at most TAU * M_ts, M_ts = |scale| *
    sum_d |q_td||k_sd|, move o_t = sum_s p_ts v_s by sum_s p_ts ds_ts (v_s - o_t), so by at most
    TAU * sum_s p_ts M_ts |v_s - o_t|; the P.V products add TAU * sum_s p_ts |v_s|; then u|ref| and the split floors.
    Weighting by p and by |v_s - o_t| instead of max|v| is what lets it see a logit error of 2^-12."""
    ref = interp_attention(qkv, heads, d, scale)
    if not tensor_core:
        return ref, TAU_MATMUL * interp_attention(qkv, heads, d, scale, magnitude=True) + U_FP32 * ref.abs()
    B, T, C3 = qkv.shape
    q, k, v = qkv.double().view(B, T, 3, heads, d).permute(2, 0, 3, 1, 4)        # [B, heads, T, d] each
    s = q @ k.transpose(-1, -2) * scale
    p = torch.softmax(s, -1)
    o = p @ v
    pm = p * (abs(scale) * (q.abs() @ k.abs().transpose(-1, -2)))              # p_ts M_ts
    logit_term = torch.empty_like(o)
    for t0 in range(0, T, 64):                                                  # [B, heads, 64, T, d] at a time
        dv = (v[:, :, None] - o[:, :, t0:t0 + 64, None]).abs()
        logit_term[:, :, t0:t0 + 64] = torch.einsum("bhts,bhtsd->bhtd", pm[:, :, t0:t0 + 64], dv)
    rel = TAU_MATMUL * (logit_term + p @ v.abs())
    # split floors: q and k (through the logits, <= 2 max|ds| max|v|), P (unnormalised p <= 1, divided by l), v
    l = torch.exp(s - s.amax(-1, keepdim=True)).sum(-1, keepdim=True)           # [B, heads, T, 1]
    ds = abs(scale) * (q.abs().sum(-1, keepdim=True) + k.abs().sum(-1).amax(-1)[..., None, None])
    vmax = v.abs().amax(dim=(2, 3), keepdim=True)
    floor = 2 * ds * vmax + v.abs().sum(2, keepdim=True) / l + 1.0
    bound = rel + SPLIT_FLOOR * floor
    return ref, bound.permute(0, 2, 1, 3).reshape(B, T, C3 // 3) + U_FP32 * ref.abs()


ATTN_PRODUCTS = ("q_lo*k_hi", "q_hi*k_lo", "p_lo*v_hi", "p_hi*v_lo")


def emulate_attention(qkv, heads, d, scale, drop=None):
    """the tensor-core attention's arithmetic in float64: S from split q, k (three products), P = exp(S*scale - max)
    split, O = (P_hi V_hi + P_lo V_hi + P_hi V_lo) / sum P; ``drop`` leaves out one of ATTN_PRODUCTS"""
    B, T, C3 = qkv.shape
    (qh, ql), (kh, kl), (vh, vl) = (split_fp16(t) for t in qkv.view(B, T, 3, heads, d).unbind(2))
    on = lambda name: 0.0 if drop == name else 1.0
    mm = lambda a, b: torch.einsum("bthd,bshd->bhts", a, b)
    s = (mm(qh, kh) + on("q_lo*k_hi") * mm(ql, kh) + on("q_hi*k_lo") * mm(qh, kl)) * scale
    p = torch.exp(s - s.amax(-1, keepdim=True))
    ph, pl = split_fp16(p)
    pv = lambda a, b: torch.einsum("bhts,bshd->bthd", a, b)
    o = (pv(ph, vh) + on("p_lo*v_hi") * pv(pl, vh) + on("p_hi*v_lo") * pv(ph, vl))
    o = o / p.sum(-1).permute(0, 2, 1)[..., None]
    return o.reshape(B, T, C3 // 3)


ATTN_FAMILIES = ("unit", "logit_0.1", "logit_10", "logit_40", "logit_80", "peak_first", "peak_last", "ties_const",
                 "v_offset")
PEAK_LOGIT = 100.0             # a jump of the running maximum by 100: exp(-100) of the online rescale is below fp32's


def attention_qkv(family, B, T, heads, d):
    """(qkv [B, T, 3C] fp32, scale d^-1/2) of an input family (deterministic, CPU):
      unit          q, k, v ~ N(0, 1)
      logit_L       q, k rescaled so the largest scaled logit is L
      peak_first    every query's maximum on one key of the first (peak_last: the last) key tile, PEAK_LOGIT above
                    the rest, so the online rescale of the other tiles underflows
      ties_const    exactly tied keys (pairs), and queries of zero: constant rows
      v_offset      v = 1e3 + U(-1, 1): the output is a mean near 1e3, which exposes errors in 1/l"""
    key = f"vr:attn:{family}:{B}:{T}:{heads}:{d}"
    scale = float(d) ** -0.5
    q, k = detfill.normal(key + ":q", (B, T, heads, d)), detfill.normal(key + ":k", (B, T, heads, d))
    v = detfill.normal(key + ":v", (B, T, heads, d))

    def to_max(L):
        m = float((torch.einsum("bthd,bshd->bhts", q.double(), k.double()) * scale).amax())
        return math.sqrt(L / m)
    if family.startswith("logit_"):
        c = to_max(float(family[6:]))
        q, k = q * c, k * c
    elif family in ("peak_first", "peak_last"):
        q, k = q * 0.2, k * 0.2
        u = detfill.normal(key + ":u", (1, 1, heads, d))
        u = u / u.norm(dim=-1, keepdim=True)
        q = q + u * 4.0
        s_star = 3 if family == "peak_first" else T - 2
        k[:, s_star] = u[:, 0] * (PEAK_LOGIT / (4.0 * scale))
    elif family == "ties_const":
        c = to_max(10.0)
        q, k = q * c, k * c
        k[:, 1::2] = k[:, 0::2]
        q[:, ::5] = 0.0
    elif family == "v_offset":
        c = to_max(10.0)
        q, k = q * c, k * c
        v = 1e3 + detfill.uniform(key + ":vo", (B, T, heads, d), -1.0, 1.0)
    qkv = torch.stack([q, k, v], 2).reshape(B, T, 3 * heads * d).contiguous()
    return qkv, scale


@pytest.mark.parametrize("T,d,heads", [(64, 32, 2), (256, 64, 1), (64, 192, 1)])
def test_emulated_split_meets_the_attention_bound(T, d, heads):
    for fam in ATTN_FAMILIES:
        qkv, scale = attention_qkv(fam, 2, T, heads, d)
        ref, bound = attention_bound(qkv, heads, d, scale)
        r = worst_ratio(emulate_attention(qkv, heads, d, scale), ref, bound)
        assert r <= 1.0, (fam, r)


@pytest.mark.parametrize("T,d,heads,families", [
    (64, 32, 2, ("unit", "logit_10", "logit_40")),
    (256, 64, 1, ("unit", "logit_10", "logit_40")),
    (256, 48, 1, ("unit", "logit_10", "logit_40")),
    (64, 192, 1, ("unit", "logit_10", "logit_40")),
    (1024, 96, 1, ("logit_10", "logit_40")),        # unit scale over 1024 keys: a dropped P_lo*V_hi is 0.76 of it
])
def test_dropped_products_leave_the_attention_bound(T, d, heads, families):
    for fam in families:
        qkv, scale = attention_qkv(fam, 2, T, heads, d)
        ref, bound = attention_bound(qkv, heads, d, scale)
        for drop in ATTN_PRODUCTS:
            r = worst_ratio(emulate_attention(qkv, heads, d, scale, drop=drop), ref, bound)
            assert r > 1.0, (fam, drop, r)


# Logits off by 2^-12 of their size (the attention scale f0 perturbed by 1 + 2^-12) leave the bound at unit scale,
# at logit maxima of 10, with ties and constant rows at every head dim, and with logit maxima of 40 up to head dim 64.
# The bound allows each logit an error of TAU * |scale| * sum_d |q||k|.  With random q and k the largest logit is a
# fraction of that sum that shrinks like d^-1/2, so at logit maxima of 40 the exact float64 attention with the perturbed
# scale measured 0.73 .. 1.1 of the bound for head dims 96 .. 192 (0.37 .. 1.0 at 80).  Fully peaked rows
# (peak_first / peak_last) are one-hot: no logit error of that size moves their output.
SCALE_PERTURBATION = 2.0 ** -12


def perturbation_families(d):
    return ("unit", "logit_10", "ties_const") + (("logit_40",) if d <= 64 else ())


@pytest.mark.parametrize("T,d,heads", [(64, 32, 2), (256, 64, 1), (1024, 96, 1), (64, 192, 1)])
def test_perturbed_scale_leaves_the_attention_bound(T, d, heads):
    for fam in perturbation_families(d):
        qkv, scale = attention_qkv(fam, 2, T, heads, d)
        ref, bound = attention_bound(qkv, heads, d, scale)
        r = worst_ratio(interp_attention(qkv, heads, d, scale * (1 + SCALE_PERTURBATION)), ref, bound)
        assert r > 1.0, (fam, r)
