"""The TF32 mode of LPIPS on the H100 (MCVD_OP_CONV_RELU_TF32, ``lpips.LPIPS(tf32=True)``).

Per op: each of the five AlexNet geometries is compared with an fp64 convolution of the TF32-rounded operands.  The
expected values are emulated on the CPU: the 3x3 / stride-2 max-pool first (exact in fp32), then both operands
rounded on the fp32 bit pattern to nearest with ties away from zero (cvt.rna), then the convolution in fp64.  The
kernel's only error is then the fp32 accumulation, so every output must satisfy
|y - ref| <= 2 (K + 1) 2^-24 (|x| * |w| + |b|).  Whole network: a pair's distance is the same bits at any chunk size
and batch position; the largest and the RMS deviation of the distances from the native fp32 ones are at most twice
those of the same AlexNet-LPIPS computed with cuDNN (``F.conv2d`` / ``F.max_pool2d``) with TF32 on against off."""
import pytest
import torch
import torch.nn.functional as Fn

from common import make_module
from mcvd_b200 import detfill, eval_weights as EW, lib, lpips as LP, runner
from oracle import lpips_oracle as LO, tasks_oracle as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rna(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> TF32, round to nearest, ties away from zero (cvt.rna.tf32.f32), as fp32."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def test_rna_matches_the_rounding_rule():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 2 ** -11 - 2 ** -23])
    assert rna(x).tolist() == [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -9, -(1.0 + 2 ** -10), 1.0]


# ---- per op -----------------------------------------------------------------------------------------------------
def conv_relu_tf32(x, w_kmajor, b, k, stride, pad, pool, cout):
    """dst [n, H, W, Cout] of one MCVD_OP_CONV_RELU_TF32 op on NHWC ``x``, with ``w_kmajor`` packed here"""
    n, side, _, cin = x.shape
    hc = (side - 3) // 2 + 1 if pool else side
    oh = (hc + 2 * pad - k) // stride + 1
    dst = torch.full((n, oh, oh, cout), float("nan"), device=DEV)
    packed = lib.tf32_pack_weights(w_kmajor)
    op = lib.McvdOp()
    op.kind, op.flags, op.B, op.H, op.W, op.C0, op.Cout = (lib.OP_CONV_RELU_TF32, lib.F_POOL if pool else 0, n, oh, oh,
                                                           cin, cout)
    op.i0, op.i1, op.i2, op.i3, op.i4 = k, stride, pad, side, side
    op.src0, op.w, op.bias, op.dst = x.data_ptr(), packed.data_ptr(), b.data_ptr(), dst.data_ptr()
    run([op])
    return dst


def layer_case(li, side, n, tag):
    _, cout, cin, k, stride, pad, pool = LO.CONVS[li]
    cin4 = 4 if cin == 3 else cin
    if li == 0:                                                 # the network input: about [-2, 2], channel 3 zero
        x = detfill.normal(f"lt32x{tag}", (n, side, side, cin4)).to(DEV)
        x[..., 3] = 0
    else:                                                       # a ReLU output
        x = torch.relu(detfill.normal(f"lt32x{tag}", (n, side, side, cin4))).to(DEV)
    wt = detfill.uniform(f"lt32w{tag}", (cout, cin, k, k), -1, 1) * (3.0 / (cin * k * k)) ** 0.5
    b = detfill.uniform(f"lt32b{tag}", (cout,), -0.1, 0.1).to(DEV)
    w = EW.kmajor(wt).to(DEV)
    got = conv_relu_tf32(x, w, b, k, stride, pad, pool, cout)
    assert bool(got.isfinite().all())
    h = x[..., :cin].permute(0, 3, 1, 2)
    if pool:
        h = Fn.max_pool2d(h, 3, 2)                               # exact: the max of fp32 values
    xr, wr, bd = rna(h).double().cpu(), rna(wt).double(), b.double().cpu()
    ref = torch.relu(Fn.conv2d(xr, wr, bd, stride=stride, padding=pad))
    mag = Fn.conv2d(xr.abs(), wr.abs(), bd.abs(), stride=stride, padding=pad)
    got64 = got.permute(0, 3, 1, 2).double().cpu()
    assert got64.shape == ref.shape
    err = (got64 - ref).abs()
    bound = 2.0 * (k * k * cin4 + 1) * 2.0 ** -24 * mag
    worst = float((err / bound.clamp_min(1e-300)).max())
    assert bool((err <= bound).all()), f"layer {li}: error / bound up to {worst:.3g}"
    assert float(ref.abs().max()) > 0
    return x, w, b, got


# (layer, input side, pairs' images): the full AlexNet geometry of a 128x128 input (stem 128 -> 31, conv2 pooled
# 31 -> 15, conv3 pooled 15 -> 7, conv4 and conv5 at 7), and small odd sides (partial M tiles, pools of odd maps)
FULL = [(0, 128, 3), (1, 31, 3), (2, 15, 5), (3, 7, 7), (4, 7, 7)]
SMALL = [(0, 37, 1), (1, 13, 3), (2, 9, 3), (3, 5, 1), (4, 3, 3)]


@pytest.mark.parametrize("li,side,n", FULL + SMALL)
def test_conv_relu_tf32_within_fp32_accumulation_of_the_rounded_product(li, side, n):
    layer_case(li, side, n, f"{li}_{side}_{n}")


def test_stem_zero_fourth_channel_contributes_nothing():
    """The network input's fourth channel is zero: whatever the packed weights hold there, the output is the same bits
    (and it matched the 3-channel reference above)."""
    x, w, b, got = layer_case(0, 128, 2, "ch4")
    w2 = w.clone().reshape(11, 11, 4, 64)
    w2[:, :, 3] = detfill.uniform("lt32ch4junk", (11, 11, 64), -5, 5).to(DEV)
    got2 = conv_relu_tf32(x, w2.reshape(-1, 64), b, 11, 4, 2, False, 64)
    assert torch.equal(got, got2)


# ---- network ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sd():
    return LO.synthetic_weights()


@pytest.fixture(scope="module")
def nets(sd):
    return LP.LPIPS(sd, device=DEV), LP.LPIPS(sd, device=DEV, tf32=True)


def pairs(n, S=64, C=1, seed=0):
    """seeded random frames [n, C, S, S] and noisy copies of them"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    real = torch.rand(n, C, S, S, device=DEV, generator=g)
    pred = (real + 0.2 * torch.randn(n, C, S, S, device=DEV, generator=g)).clamp(0, 1)
    return pred, real


def test_tf32_packing_and_program(nets):
    net32, net = nets
    assert net.tf32 and not net32.tf32 and len(net.packed) == 5
    for (w, _, _), p in zip(net.weights, net.packed):
        assert p.numel() * 4 == lib.tf32_packed_bytes(w.shape[0], w.shape[1])
        want = torch.sort(torch.cat([rna(w).flatten(), torch.zeros(p.numel() - w.numel(), device=DEV)]))[0]
        assert torch.equal(torch.sort(p)[0], want)               # every weight rounded once, plus zero padding


def test_distances_are_batch_invariant(sd, nets):
    net = nets[1]
    pred, real = pairs(300, S=32, seed=1)
    base = net(pred, real, 1)                                   # chunks of 256 and 44 pairs
    assert base.shape == (300, 1) and bool(base.isfinite().all()) and bool((base > 0).all())
    for chunk in (1, 7, 256):
        assert torch.equal(LP.LPIPS(sd, device=DEV, max_chunk_frames=chunk, tf32=True)(pred, real, 1), base), chunk
    for i in (0, 6, 7, 255, 256, 299):
        assert torch.equal(net(pred[i:i + 1], real[i:i + 1], 1), base[i:i + 1]), i
    assert torch.equal(net(pred.flip(0), real.flip(0), 1), base.flip(0))
    clips = net(pred.reshape(30, 10, 32, 32), real.reshape(30, 10, 32, 32), 1)
    assert torch.equal(clips.reshape(300, 1), base)
    assert not torch.equal(base, nets[0](pred, real, 1))        # a different numerics class


def network_inputs(net, pred, real, C):
    """NCHW [2n, 3, 128, 128] network inputs of the pairs (pred, then real), made by the native prep"""
    n = pred.shape[0]
    ws = torch.empty(2 * n * (LP._WS_A + LP._WS_B), device=DEV)
    out = torch.empty(n, dtype=torch.float64, device=DEV)
    run(net.program(pred, real, C, out, ws)[:1])
    return ws[:2 * n * LP._WS_A].reshape(2 * n, 128, 128, 4)[..., :3].permute(0, 3, 1, 2).contiguous()


def cudnn_lpips(sd, x):
    """per-pair LPIPS of NCHW inputs ``x`` [2n, 3, 128, 128] (pred, then real): the AlexNet from ``F.conv2d`` /
    ``F.max_pool2d`` under the caller's cuDNN TF32 setting, the head in fp64 (as the native LPIPS_LAYER)."""
    n = x.shape[0] // 2
    d = torch.zeros(n, dtype=torch.float64, device=DEV)
    h = x
    for li, (key, _, _, _, stride, pad, pool) in enumerate(LO.CONVS):
        if pool:
            h = Fn.max_pool2d(h, 3, 2)
        h = torch.relu(Fn.conv2d(h, sd[key + ".weight"].to(DEV), sd[key + ".bias"].to(DEV), stride=stride,
                                 padding=pad))
        f = h.double()
        f = f / (f.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
        lin = sd[f"lin{li}.model.1.weight"].to(DEV).double().reshape(1, -1, 1, 1)
        d += (lin * (f[:n] - f[n:]) ** 2).sum(1).mean((1, 2))
    return d


def with_tf32(flag, fn):
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = flag
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# the evaluation batches of the benchmark workloads: (clips, frames, side, channels)
CASES = {"cfg2": (64, 20, 64, 1), "cfg5": (32, 28, 128, 3)}


@pytest.mark.parametrize("case", list(CASES))
def test_tf32_deviation_is_within_twice_cudnns(sd, nets, case):
    B, F, S, C = CASES[case]
    N = B * F
    pred, real = pairs(N, S=S, C=C, seed=2 + list(CASES).index(case))
    d32, dtf = (net(pred, real, C).reshape(-1) for net in nets)
    e32, etf = [], []
    for lo in range(0, N, 256):
        x = network_inputs(nets[0], pred[lo:lo + 256], real[lo:lo + 256], C)
        e32.append(with_tf32(False, lambda: cudnn_lpips(sd, x)))
        etf.append(with_tf32(True, lambda: cudnn_lpips(sd, x)))
    e32, etf = torch.cat(e32), torch.cat(etf)
    assert float(((e32 - d32).abs() / d32).max()) < 1e-3          # the fp32 arms compute the same distances
    dn, dc = (dtf - d32).abs(), (etf - e32).abs()
    native = float(dn.max()), float(dn.pow(2).mean().sqrt())
    cudnn = float(dc.max()), float(dc.pow(2).mean().sqrt())
    assert 0 < native[0] <= 2 * cudnn[0], (native, cudnn)
    assert 0 < native[1] <= 2 * cudnn[1], (native, cudnn)


def test_evaluate_tasks_with_tf32_lpips(nets):
    net32, net = nets
    cfg, model, _ = make_module("tiny_general", DEV)
    X = T.golden_clips(cfg, batch=2).to(DEV)
    kw = dict(preds_per_test=2, philox_seed=5, init_seed=6)
    o32 = runner.evaluate_tasks(cfg, model, X, lpips=net32, **kw)
    out = runner.evaluate_tasks(cfg, model, X, lpips=net, **kw)
    C = cfg.data.channels
    assert list(out) == list(o32)
    for task, (frames, m) in out.items():
        frames0, m0 = o32[task]
        assert torch.equal(frames, frames0)
        if m0 is None:
            assert m is None
            continue
        assert set(m) == set(m0)
        for k in m0:
            assert m[k].shape == m0[k].shape and m[k].dtype == m0[k].dtype, (task, k)
            if "lpips" not in k:
                assert torch.equal(m[k], m0[k]), (task, k)
        real, _, _ = runner.task_inputs(cfg, X.repeat_interleave(2, dim=0), task)
        direct = net(frames, real.to(DEV), C)
        assert torch.equal(m["per_frame_lpips"], direct)
        assert torch.equal(m["lpips"], direct.mean(1).reshape(2, 2).min(-1).values)
        assert bool((net(frames, frames, C) == 0).all())          # identical pairs: exactly 0
    frames, m = runner.evaluate_clips(cfg, model, X, lpips=net, **kw)
    assert torch.equal(m["lpips"], out["interp"][1]["lpips"])
