"""The wgmma conv (csrc/conv_umma.cu) on every launcher path, in both precisions, on inputs whose exact result is known.

The shapes are the case tables of the default mode's conv tests (test_gpu_ops, test_gpu_conv2, test_gpu_conv_tiles,
test_gpu_conv_producers, test_gpu_conv_tma), run through CONV_UMMA in each work organisation, tile height and slab-stage
count the table exercises, and through CONV_UMMA2 with the planar norm table and epilogue statistics where the shape
allows; plus the plans that exist only in half mode (MCVD_F_HALF), whose launch plans are pinned through
mcvd_conv_umma_launch_info in both modes.

Inputs on a grid.  The conv's operands (the transformed activations when there is a norm table) are x = m * 2^-6 with
|x| <= 2, the weights small integers times 2^-4, so both are exact in fp16 after the power-of-two pre-scale.  Norm-table
means and shifts lie on the 2^-6 grid and rstd, G vary over powers of two per (image, channel), so reading another
image's row changes the result; the raw input is built from the operand through the inverse transform, and the
kernel's fp32 forward transform is emulated to confirm it returns the operand exactly.  Bias and residual lie on the
grid and f0 = 1/2; there is no SiLU (inexact).  Every product is then a multiple of g = 2^-10 (times the pre-scale) and
every partial sum stays below 2^24 g, so an fp32 accumulation drops no bits and the output must equal the float64
conv bit for bit, at either tile height and in any order.  The epilogue statistics must equal those of the stored
output (|y| <= 4096).

Half mode also tests the rounding of both operands: the activations (after the transform) and the pre-scaled weights
carry an offset delta in {+-2^-2, +-(2^-1 - 2^-12), +-2^-1} of an fp16 ulp of the grid value.  +-2^-1 is a tie, which
round-to-nearest-even sends back to the grid value (whose significand is even); the others round to it as well.  A
kernel that truncated either operand instead would land one ulp off wherever delta points toward zero, and the tests
check that such a kernel's output differs from the one measured.  The default mode runs the same inputs without the
offset, which gives its data movement bit-exact coverage."""
import pytest
import torch

from mcvd_b200 import lib
from mcvd_b200.lib import McvdOp
from test_conv_fp16_cpu import DELTAS, nudge, trunc_fp16, ulp_fp16
import test_gpu_conv2 as CV2
import test_gpu_conv_producers as PROD
import test_gpu_conv_tiles as TILES
import test_gpu_conv_tma as TMA
import test_gpu_ops as OPS

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
W_LOG2 = -4                  # the weights' power of two: |w| <= 4 * 2^-4, so |y| <= 2 * 0.25 * 3456 + 4 < 4096


def _pick_nt(cout):
    return max(d for d in range(16, 257, 16) if cout % d == 0)


def _gen(*key):
    return torch.Generator().manual_seed(hash(tuple(key)) % (2 ** 31))


def _grid(g, shape, m, step):
    """integers in [-m, m] times ``step``, float64"""
    return torch.randint(-m, m + 1, shape, generator=g, dtype=torch.int64).double() * step


class Inputs:
    """the tensors of one conv case on the exact grid.  ``half``: with the rounding offsets (see the module doc)."""

    def __init__(self, B, H, C0, C1, Cout, ks, tab, res, C2=0, C3=0, half=False, seed=0):
        self.B, self.H, self.C0, self.C1, self.Cout, self.ks, self.C2, self.C3 = B, H, C0, C1, Cout, ks, C2, C3
        self.half = half
        g = _gen(B, H, C0, C1, Cout, ks, tab, res, C2, C3, seed)
        Cin, Cs = C0 + C1, C2 + C3
        self.xhat = _grid(g, (B, H, H, Cin), 128, 2.0 ** -6)          # the conv's operand (after the transform)
        self.what = _grid(g, (ks * ks, Cin, Cout), 4, 2.0 ** W_LOG2)
        self.yhat = _grid(g, (B, H, H, Cs), 128, 2.0 ** -6) if Cs else None
        self.wschat = _grid(g, (1, Cs, Cout), 4, 2.0 ** W_LOG2) if Cs else None
        self.bias = _grid(g, (Cout,), 64, 2.0 ** -6)
        self.res = _grid(g, (B, H, H, Cout), 128, 2.0 ** -6) if res else None
        amax = float(max(self.what.abs().max(), self.wschat.abs().max() if Cs else 0.0))
        from mcvd_b200.program import umma_scale_log2
        self.k = umma_scale_log2(amax)
        # operands as the kernel reads them: offsets in half mode
        x_op = nudge(self.xhat, g) if half else self.xhat
        self.w = (nudge(self.what * 2.0 ** self.k, g) * 2.0 ** -self.k if half else self.what).float()
        self.y = (nudge(self.yhat, g) if half else self.yhat).float() if Cs else None
        self.wsc = (nudge(self.wschat * 2.0 ** self.k, g) * 2.0 ** -self.k if half else self.wschat).float() if Cs else None
        self.tab = self.tab3 = None
        if tab:
            mean = _grid(g, (B, Cin), 64, 2.0 ** -6)
            rstd = torch.exp2(torch.randint(-1, 2, (B, Cin), generator=g).double())
            G = torch.exp2(torch.randint(-1, 3, (B, Cin), generator=g).double())
            S = _grid(g, (B, Cin), 32, 2.0 ** -6)
            mul = (rstd * G).view(B, 1, 1, Cin)
            m4, s4 = mean.view(B, 1, 1, Cin), S.view(B, 1, 1, Cin)

            def forward(x32):      # the kernel's transform: fmaf(x - mean, rstd * G, S), each step in fp32
                d = (x32.double() - m4).float().double()
                return (d * mul + s4).float().double()

            x = (m4 + (x_op - s4) / mul).float()
            ok = forward(x) == x_op
            # where the offset does not survive the fp32 inverse (small |x| next to a large shift), drop it
            x = torch.where(ok, x, (m4 + (self.xhat - s4) / mul).float())
            x_op = torch.where(ok, x_op, self.xhat)
            assert torch.equal(forward(x), x_op)
            self.x = x
            self.kept = float((ok & (self.xhat != 0)).double().mean())
            self.tab = torch.stack([mean, rstd, G, S], 2).float().contiguous()
            self.tab3 = torch.stack([mean, rstd * G, S], 1).float().contiguous()
        else:
            self.x = x_op.float()
        self.x_op = x_op
        assert torch.equal(self.x_op.float().double(), self.x_op)

    def reference(self):
        """the float64 conv of the grid operands, + bias + residual, times f0 = 1/2: what the kernel must store"""
        F = torch.nn.functional
        y = F.conv2d(self.xhat.permute(0, 3, 1, 2), _oihw(self.what, self.ks), padding=self.ks // 2).permute(0, 2, 3, 1)
        if self.yhat is not None:
            y = y + torch.einsum("bhwc,co->bhwo", self.yhat, self.wschat[0])
        y = y + self.bias
        if self.res is not None:
            y = y + self.res
        return y * 0.5


def _oihw(taps, ks):
    """[taps][Cin][Cout] -> OIHW"""
    T, I, O = taps.shape
    return taps.view(ks, ks, I, O).permute(3, 2, 0, 1)


class Device:
    """one Inputs case on the GPU, packed for one n tile and K-block"""

    def __init__(self, inp: Inputs):
        self.inp = inp
        d = lambda t: None if t is None else t.float().to(DEV).contiguous()
        C0, C1, C2 = inp.C0, inp.C1, inp.C2
        self.x0, self.x1 = d(inp.x[..., :C0]), (d(inp.x[..., C0:]) if C1 else None)
        self.y0 = d(inp.y[..., :C2]) if inp.y is not None else None
        self.y1 = d(inp.y[..., C2:]) if inp.y is not None and inp.C3 else None
        self.bias, self.res, self.tab, self.tab3 = d(inp.bias), d(inp.res), d(inp.tab), d(inp.tab3)
        self.w, self.wsc = d(inp.w), d(inp.wsc)
        self.packed = {}

    def pack(self, nt, kb):
        key = (nt, kb)
        if key not in self.packed:
            inp = self.inp
            T, I, O = self.w.shape
            isc = 0 if self.wsc is None else self.wsc.shape[1]
            per_unit = (I // kb) * T + isc // kb
            parts = 1 if inp.half else 2
            out = torch.empty((T * I + isc) * O * 2 * parts, dtype=torch.uint8, device=DEV)
            L, s = lib.load(), torch.cuda.current_stream().cuda_stream
            assert L.mcvd_umma_pack_weights_ex(self.w.data_ptr(), T, I, O, nt, kb, out.data_ptr(), inp.k, 0, per_unit,
                                               parts, s) > 0, lib.last_error()
            if isc:
                assert L.mcvd_umma_pack_weights_ex(self.wsc.data_ptr(), 1, isc, O, nt, kb, out.data_ptr(), inp.k,
                                                   (I // kb) * T, per_unit, parts, s) > 0, lib.last_error()
            self.packed[key] = out
        return self.packed[key]

    def op(self, kind, nt, stats=False, **fields):
        """(McvdOp, output, statistics buffer or None, buffers to keep alive)"""
        inp = self.inp
        B, H = inp.B, inp.H
        kb = lib.umma_kblock(inp.C0, inp.C1) if not inp.C2 + inp.C3 else \
            min(lib.umma_kblock(inp.C0, inp.C1), lib.umma_kblock(inp.C2, inp.C3))
        w = self.pack(nt, kb)
        out = torch.full((B, H, H, inp.Cout), float("nan"), device=DEV)
        st = torch.full((lib.umma2_stats_bytes(B, H, H, inp.ks, inp.Cout) // 8,), -7, dtype=torch.int64,
                        device=DEV) if stats else None
        o = McvdOp()
        o.kind, o.B, o.H, o.W, o.C0, o.C1, o.Cout, o.i0, o.i1 = kind, B, H, H, inp.C0, inp.C1, inp.Cout, inp.ks, nt
        o.f0, o.f1, o.flags = 0.5, 2.0 ** -inp.k, lib.F_HALF if inp.half else 0
        tab = self.tab3 if kind == lib.OP_CONV_UMMA2 else self.tab
        for f, t in (("src0", self.x0), ("src1", self.x1), ("w", w), ("bias", self.bias), ("aux0", self.res),
                     ("aux1", tab), ("dst", out), ("dst2", st), ("src2", self.y0), ("src3", self.y1)):
            setattr(o, f, 0 if t is None else t.data_ptr())
        o.C2, o.C3 = inp.C2, inp.C3
        if kind == lib.OP_CONV_UMMA2:
            o.i2 = kb
        for f, v in fields.items():
            setattr(o, f, v)
        return o, out, st


def run_op(o):
    arr = lib.make_ops([o])
    lib.validate_program(arr, 1)
    lib.run_program(arr, 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def check_case(desc, variants, seed=0):
    """run every variant (kind, n tile, statistics, op fields) of a case in both modes: each output equals the
    float64 reference bit for bit, and its statistics those of the stored output"""
    B, H, C0, C1, Cout, ks, tab, res, C2, C3 = desc
    pimg = (H + 1) * (H + 1) if ks == 3 else H * H
    ref = None
    report = []
    for half in (False, True):
        inp = Inputs(B, H, C0, C1, Cout, ks, tab, res, C2, C3, half=half, seed=seed)
        if ref is None:
            ref = inp.reference().float()
        dev = Device(inp)
        for kind, nt, stats, fields in variants:
            stats = stats and pimg >= 64
            o, out, st = dev.op(kind, nt, stats, **fields)
            info = lib.conv_umma_launch_info(o)
            run_op(o)
            got = out.cpu()
            label = (desc, "half" if half else "default", lib_kind(kind), nt, stats, fields, info)
            bad = (got != ref)
            assert not bad.any(), (label, int(bad.sum()), float((got.double() - ref.double()).abs().max()))
            if stats:
                exp = CV2.expected_stats(got, ks)
                ntile = -(-(B * pimg) // 128) if kind == lib.OP_CONV_UMMA else exp.shape[0]
                assert torch.equal(st.cpu().view(exp.shape)[:ntile], exp[:ntile]), label
            report.append((half, lib_kind(kind), info["mt"], info["sa"], info["nb"], info["ra"], info["npi"]))
        if half and tab:
            assert inp.kept > 0.2, (desc, inp.kept)        # most table operands carry their rounding offset
    return report


def lib_kind(kind):
    return "UMMA2" if kind == lib.OP_CONV_UMMA2 else "UMMA"


def umma2_variant(Cout, ks, stats=True):
    return (lib.OP_CONV_UMMA2, lib.umma2_pick_nt(Cout, ks), stats, {})


# ------------------------------------------------------------------------------------------------- the case tables
def conv_desc(case):
    B, H, C0, C1, Cout, ks, tab, _act_in, res, _act_out = case
    return (B, H, C0, C1, Cout, ks, tab, res, 0, 0)


@pytest.mark.parametrize("case", OPS.CONV_CASES + TMA.UMMA_CASES)
def test_conv_cases(case):
    desc = conv_desc(case)
    nt = _pick_nt(desc[4])
    U = lib.OP_CONV_UMMA
    check_case(desc, [(U, nt, False, dict(i2=1)), (U, nt, True, dict(i2=2)), umma2_variant(desc[4], desc[5])])


@pytest.mark.parametrize("case", OPS.K1_CASES)
def test_conv1x1_cases(case):
    B, H, C0, C1, Cout, tab, _act_in, res, _act_out = case
    nt = _pick_nt(Cout)
    U = lib.OP_CONV_UMMA
    check_case((B, H, C0, C1, Cout, 1, tab, res, 0, 0),
               [(U, nt, False, dict(i2=2)), (U, nt, False, dict(i2=1)), (U, nt, False, dict(i2=0)),
                (U, nt, True, dict(i2=2)), (U, nt, True, dict(i2=1))])


@pytest.mark.parametrize("case", OPS.FUSED_CASES)
def test_fused_shortcut_cases(case):
    B, H, Cm, Cout, Cs0, Cs1 = case
    nt = _pick_nt(Cout)
    U = lib.OP_CONV_UMMA
    check_case((B, H, Cm, 0, Cout, 3, True, False, Cs0, Cs1),
               [(U, nt, False, dict(i2=i2)) for i2 in (0, 1, 2)] + [umma2_variant(Cout, 3)])


@pytest.mark.parametrize("case", CV2.CASES + TMA.PLANAR_CASES)
def test_planar_cases(case):
    B, H, C0, C1, Cout, ks, tab, res, (C2, C3), stats = case
    check_case((B, H, C0, C1, Cout, ks, tab, res, C2, C3),
               [umma2_variant(Cout, ks, stats), (lib.OP_CONV_UMMA, _pick_nt(Cout), False, dict(i2=1))])


@pytest.mark.parametrize("case", TILES.CASES)
def test_tile_height_cases(case):
    B, H, C0, C1, Cout, nt, ks, tab, res, (C2, C3) = case
    check_case((B, H, C0, C1, Cout, ks, tab, res, C2, C3),
               [(lib.OP_CONV_UMMA, nt, False, dict(i2=1, i4=mt)) for mt in (128, 192, 0)])


def fitting(desc, nt, settings):
    """the forced (tile height, slab stages) settings whose plan fits, by the launcher's own planning, in each mode"""
    return {half: [(mt, sa) for mt, sa in settings if _info_or_error(desc, nt, half, dict(i2=1, i4=mt, i5=sa)) != "error"]
            for half in (False, True)}


@pytest.mark.parametrize("case", PROD.CASES)
def test_producer_cases(case):
    B, H, C0, C1, Cout, nt, tab, _act_in, res, (C2, C3) = case
    desc = (B, H, C0, C1, Cout, 3, tab, res, C2, C3)
    fit = fitting(desc, nt, PROD.forced_settings())
    assert set(fit[False]) <= set(fit[True])          # half mode's plans are never larger
    variants = [(lib.OP_CONV_UMMA, nt, False, dict(i2=1, i4=mt, i5=sa)) for mt, sa in fit[True]]
    if tab:
        variants.append(umma2_variant(Cout, 3, False))
    check_case(desc, variants)


# ------------------------------------------------------------------------------------------ plans only half mode has
def info(desc, nt, half, kind=lib.OP_CONV_UMMA, stats=False, sms=132, **fields):
    """the launch plan of a case; host arithmetic only (the pointers are placeholders)"""
    B, H, C0, C1, Cout, ks, tab, res, C2, C3 = desc
    o = McvdOp()
    o.kind, o.B, o.H, o.W, o.C0, o.C1, o.Cout, o.i0, o.i1 = kind, B, H, H, C0, C1, Cout, ks, nt
    o.src0 = o.w = o.dst = 256
    o.src1 = 256 if C1 else 0
    o.aux1 = 256 if tab else 0
    o.aux0 = 256 if res else 0
    o.dst2 = 256 if stats else 0
    o.src2, o.C2, o.src3, o.C3 = (256 if C2 else 0), C2, (256 if C3 else 0), C3
    o.flags = lib.F_HALF if half else 0
    for f, v in fields.items():
        setattr(o, f, v)
    return lib.conv_umma_launch_info(o, sms)


HALF_ONLY = [
    # (name, case desc, n tile, op fields, {field: (default mode, half mode)}); "error" = the plan does not fit
    ("1x1 12 K-blocks input-stationary", (2, 16, 384, 0, 192, 1, True, False, 0, 0), 96, dict(i2=2),
     dict(npi=(1, 2), sa=(2, 12), nb=(None, 10))),
    ("128x128 two raw stages", (1, 128, 128, 0, 128, 3, True, False, 0, 0), 128, dict(i2=1),
     dict(ra=(1, 2))),
    ("128x128 three slab stages", (1, 128, 32, 0, 96, 3, True, False, 0, 0), 96, dict(i2=1, i4=192, i5=3),
     dict(sa=("error", 3))),
    ("input-stationary 1x1, Cout 192 at NT 64", (4, 8, 64, 0, 192, 1, False, True, 0, 0), 64, dict(i2=2),
     dict(npi=(3, 3), nb=(None, 10))),
]


def _info_or_error(desc, nt, half, fields):
    try:
        return info(desc, nt, half, **fields)
    except RuntimeError:
        return "error"


@pytest.mark.parametrize("row", HALF_ONLY, ids=[r[0] for r in HALF_ONLY])
def test_half_only_plans(row):
    """each plan is reached in half mode (and differs from the default mode's as stated), and computes exactly"""
    name, desc, nt, fields, expect = row
    got = {half: _info_or_error(desc, nt, half, fields) for half in (False, True)}
    print(f"\n{name}: default {got[False]}, half {got[True]}")
    assert got[True] != "error"
    for f, (d32, d16) in expect.items():
        if d32 == "error":
            assert got[False] == "error", got[False]
        elif d32 is not None:
            assert got[False][f] == d32, (f, got[False])
        if d16 is not None:
            assert got[True][f] == d16, (f, got[True])
    variants = [(lib.OP_CONV_UMMA, nt, False, fields)]
    report = []
    for half in (False, True):
        if got[half] == "error":
            continue
        inp = Inputs(*desc, half=half)
        ref = inp.reference().float()
        dev = Device(inp)
        o, out, _ = dev.op(lib.OP_CONV_UMMA, nt, False, **fields)
        run_op(o)
        assert torch.equal(out.cpu(), ref), (name, half)
        report.append(half)
    assert True in report


def test_half_plans_reach_the_weight_stage_cap():
    """nearly every half-mode plan of the conv table holds the cap of 10 weight stages, more than in the default mode"""
    descs = [conv_desc(c) for c in OPS.CONV_CASES + TMA.UMMA_CASES]
    nb = {half: [info(d, _pick_nt(d[4]), half, i2=1)["nb"] for d in descs] for half in (False, True)}
    print(f"\nweight stages: default {nb[False]}, half {nb[True]}")
    assert sum(n == 10 for n in nb[True]) >= 0.9 * len(descs)
    assert sum(n == 10 for n in nb[True]) > sum(n == 10 for n in nb[False])
    assert all(h >= d for h, d in zip(nb[True], nb[False]))


# --------------------------------------------------------------------------------------- the rounding is measured
def test_truncating_kernels_would_be_caught():
    """the half kernel's output differs from a kernel that truncated the activations, and from one that truncated
    the pre-scaled weights: the exact comparison above sees the direction of each rounding"""
    desc = (2, 16, 64, 0, 96, 3, False, False, 0, 0)
    inp = Inputs(*desc, half=True)
    dev = Device(inp)
    o, out, _ = dev.op(lib.OP_CONV_UMMA, 96, False, i2=1)
    run_op(o)
    got = out.cpu()
    assert torch.equal(got, inp.reference().float())
    xt = trunc_fp16(inp.x.double())
    wt = trunc_fp16(inp.w.double() * 2.0 ** inp.k) * 2.0 ** -inp.k
    for name, over in (("activations", dict(xhat=xt)), ("weights", dict(what=wt))):
        alt = Inputs(*desc, half=True)
        for f, v in over.items():
            setattr(alt, f, v)
        r = alt.reference().float()
        ndiff = int((r != got).sum())
        print(f"\ntruncated {name}: {ndiff} of {got.numel()} outputs differ")
        assert ndiff > got.numel() // 2, name


def test_rounding_offsets_are_one_ulp_fraction():
    """the offsets of the half inputs are the stated fractions of an fp16 ulp of the grid value"""
    inp = Inputs(2, 8, 32, 0, 32, 3, False, False, half=True)
    nz = inp.xhat != 0
    frac = ((inp.x_op - inp.xhat) / ulp_fp16(inp.xhat))[nz]
    assert set(frac.unique().tolist()) == set(DELTAS)
