"""The TF32 tensor-core convolutions of the FVD and FID feature networks on the H100 (MCVD_OP_CONV3D_TF32,
MCVD_OP_CONV2D_TF32, ``fvd.I3D(tf32=True)``, ``fid.InceptionV3(tf32=True)``).

Per op: the kernel is compared with an fp64 convolution of the TF32-rounded input and weights (rounded here on the
fp32 bit pattern, to nearest with ties away from zero, as cvt.rna does).  Its only error is then the fp32 accumulation,
so every output must satisfy |y - ref| <= 2 (K + 1) 2^-24 (|x| * |w| + |b|): K products and the bias, each with at
most one fp32 ulp.  End to end: the largest feature deviation from the native fp32 features, over the feature scale,
is at most twice cuDNN's own TF32-versus-fp32 deviation on the same inputs and folded weights, and so is the change
of FID / FVD."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from mcvd_b200 import detfill, fid as FD, fvd as FV, lib
from oracle import i3d_oracle as IO, inception_oracle as NO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rna(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> TF32, round to nearest, ties away from zero (cvt.rna.tf32.f32), as fp32."""
    b = x.float().contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def check_bound(got, ref, mag, K):
    """elementwise |got - ref| <= 2 (K + 1) 2^-24 mag"""
    err = (got - ref).abs()
    bound = 2.0 * (K + 1) * 2.0 ** -24 * mag
    worst = float((err / bound.clamp_min(1e-300)).max())
    assert bool((err <= bound).all()), f"error / bound up to {worst:.3g}"
    assert float(ref.abs().max()) > 0


def test_rna_matches_the_rounding_rule():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, -(1.0 + 2 ** -11), 1.0 + 2 ** -11 - 2 ** -23])
    assert rna(x).tolist() == [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -9, -(1.0 + 2 ** -10), 1.0]


def test_packing_rounds_every_weight_once():
    """The packed image is a permutation of the rounded weights plus zero padding."""
    for K, cout in ((36, 32), (1372, 64), (192, 208), (448, 80)):
        w = detfill.normal(f"tfpack{K}_{cout}", (K, cout)).to(DEV)
        p = lib.tf32_pack_weights(w)
        torch.cuda.synchronize()
        assert p.numel() * 4 == lib.tf32_packed_bytes(K, cout)
        want = torch.sort(torch.cat([rna(w).flatten(), torch.zeros(p.numel() - K * cout, device=DEV)]))[0]
        assert torch.equal(torch.sort(p)[0], want)


# ---- 3-D (I3D) ------------------------------------------------------------------------------------------------
def conv3d_case(cin, cout, k, s, T, S, n, off, pitch, tag):
    x = torch.relu(detfill.normal(f"t3x{tag}", (n, T, S, S, cin))).to(DEV)
    if cin == 4:
        x[..., 3] = 0
    wt = detfill.uniform(f"t3w{tag}", (cout, cin, k, k, k), -1, 1) * (3.0 / (cin * k ** 3)) ** 0.5
    b = detfill.uniform(f"t3b{tag}", (cout,), -0.1, 0.1)
    w = wt.permute(2, 3, 4, 1, 0).reshape(-1, cout).contiguous().to(DEV)
    To, So = FV.same_out(T, k, s), FV.same_out(S, k, s)
    dst = torch.full((n, To, So, So, pitch), float("nan"), device=DEV)
    op = lib.McvdOp()
    op.kind, op.B, op.C0, op.Cout, op.H, op.W = lib.OP_CONV3D_TF32, n, cin, cout, So, So
    op.i0, op.i1, op.i2, op.i3, op.i4, op.i5, op.i6, op.i7 = k, k, s, s, T, S, pitch, off
    packed = lib.tf32_pack_weights(w)
    op.src0, op.w, op.bias, op.dst = x.data_ptr(), packed.data_ptr(), b.to(DEV).data_ptr(), dst.data_ptr()
    run([op])
    xr = rna(x).permute(0, 4, 1, 2, 3).double().cpu()
    wr = rna(wt).double()

    def conv(a, ww, bb):
        return Fn.conv3d(IO.same_pad(a, (k,) * 3, (s,) * 3), ww, bb, stride=s)
    ref = torch.relu(conv(xr, wr, b.double()))
    mag = conv(xr.abs(), wr.abs(), b.double().abs())
    got = dst[..., off:off + cout].permute(0, 4, 1, 2, 3).double().cpu()
    check_bound(got, ref, mag, k ** 3 * cin)
    assert bool(dst[..., :off].isnan().all()) and bool(dst[..., off + cout:].isnan().all())


# (Cin, Cout, k, stride, T, S, n, off, pitch): the 7x7x7 stride-2 stem (Cin 4, K = 1372 not a multiple of 8), the
# 1x1x1 and 3x3x3 units with Couts of every n-tile width and remainder (16, 48, 80, 208, 320, 448), odd input sizes
# for the SAME padding, M not a multiple of the 128-position tile, and channel slices
CONV3D = [(4, 64, 7, 2, 9, 23, 2, 0, 64), (4, 64, 7, 2, 4, 17, 1, 8, 80), (64, 192, 3, 1, 3, 9, 2, 0, 192),
          (16, 48, 3, 1, 4, 7, 3, 64, 128), (192, 16, 1, 1, 3, 9, 2, 4, 28), (480, 208, 1, 1, 2, 7, 3, 192, 512),
          (832, 448, 1, 1, 1, 5, 2, 0, 448), (112, 224, 3, 1, 2, 6, 2, 8, 240), (96, 80, 3, 2, 5, 11, 1, 4, 88),
          (528, 320, 1, 1, 2, 7, 1, 0, 320)]


@pytest.mark.parametrize("cin,cout,k,s,T,S,n,off,pitch", CONV3D)
def test_conv3d_tf32_within_fp32_accumulation_of_the_rounded_product(cin, cout, k, s, T, S, n, off, pitch):
    conv3d_case(cin, cout, k, s, T, S, n, off, pitch, f"{cin}_{cout}_{k}_{s}_{T}_{S}")


# ---- 2-D (Inception) --------------------------------------------------------------------------------------------
def pool_fp32(x, pool):
    """The branch pool as the kernel forms it in fp32: max, or the in-map taps summed in (dy, dx) order over their
    count."""
    n, S, _, c = x.shape
    xp = Fn.pad(x, (0, 0, 1, 1, 1, 1))
    ones = Fn.pad(torch.ones(n, S, S, 1, device=x.device), (0, 0, 1, 1, 1, 1))
    acc = torch.full_like(x, -float("inf")) if pool == "max" else torch.zeros_like(x)
    count = torch.zeros(n, S, S, 1, device=x.device)
    for dy in range(3):
        for dx in range(3):
            u, inside = xp[:, dy:dy + S, dx:dx + S], ones[:, dy:dy + S, dx:dx + S]
            if pool == "max":
                acc = torch.where(inside > 0, torch.maximum(acc, u), acc)
            else:
                acc = acc + u                                   # a padding tap adds an exact 0
                count = count + inside
    return acc if pool == "max" else acc / count


def conv2d_case(cin, cout, k, stride, pad, pool, side, n, off, pitch, tag):
    x = torch.relu(detfill.normal(f"t2x{tag}", (n, side, side, cin))).to(DEV)
    if pool == "max":
        x = x - 0.5                                             # the padding must never win the max
    if cin == 4:
        x[..., 3] = 0
    fan = cin * k[0] * k[1]
    wt = detfill.uniform(f"t2w{tag}", (cout, cin, k[0], k[1]), -1, 1) * (3.0 / fan) ** 0.5
    b = detfill.uniform(f"t2b{tag}", (cout,), -0.1, 0.1)
    w = wt.permute(2, 3, 1, 0).reshape(-1, cout).contiguous().to(DEV)
    ho, wo = FD.conv_out(side, k[0], stride, pad[0]), FD.conv_out(side, k[1], stride, pad[1])
    dst = torch.full((n, ho, wo, pitch), float("nan"), device=DEV)
    op = lib.McvdOp()
    op.kind, op.B, op.C0, op.Cout, op.H, op.W = lib.OP_CONV2D_TF32, n, cin, cout, ho, wo
    op.flags = 0 if pool is None else lib.F_POOL | (lib.F_AVG if pool == "avg" else 0)
    op.i0, op.i1, op.i2, op.i3, op.i4, op.i5, op.i6, op.i7 = k[0], k[1], stride, pad[0], pad[1], side, pitch, off
    packed = lib.tf32_pack_weights(w)
    op.src0, op.w, op.bias, op.dst = x.data_ptr(), packed.data_ptr(), b.to(DEV).data_ptr(), dst.data_ptr()
    run([op])
    xin = x if pool is None else pool_fp32(x, pool)
    xr = rna(xin).permute(0, 3, 1, 2).double().cpu()
    wr = rna(wt).double()
    ref = torch.relu(Fn.conv2d(xr, wr, b.double(), stride=stride, padding=pad))
    mag = Fn.conv2d(xr.abs(), wr.abs(), b.double().abs(), stride=stride, padding=pad)
    got = dst[..., off:off + cout].permute(0, 3, 1, 2).double().cpu()
    check_bound(got, ref, mag, fan)
    assert bool(dst[..., :off].isnan().all()) and bool(dst[..., off + cout:].isnan().all())


# (Cin, Cout, (kh, kw), stride, (ph, pw), pool): every kernel shape and padding of the network, stride 2 without
# padding, the fused max / average pools, and Couts of every n-tile width and remainder
CONV2D = [(4, 32, (3, 3), 2, (0, 0), None), (32, 64, (3, 3), 1, (1, 1), None), (64, 80, (1, 1), 1, (0, 0), None),
          (48, 64, (5, 5), 1, (2, 2), None), (128, 128, (1, 7), 1, (0, 3), None), (160, 192, (7, 1), 1, (3, 0), None),
          (384, 384, (1, 3), 1, (0, 1), None), (384, 384, (3, 1), 1, (1, 0), None), (96, 96, (3, 3), 2, (0, 0), None),
          (288, 384, (3, 3), 2, (0, 0), None), (192, 32, (1, 1), 1, (0, 0), "avg"), (768, 192, (1, 1), 1, (0, 0), "avg"),
          (2048, 192, (1, 1), 1, (0, 0), "max"), (1280, 448, (1, 1), 1, (0, 0), None), (192, 320, (3, 3), 2, (0, 0), None),
          (288, 48, (1, 1), 1, (0, 0), None), (256, 16, (1, 1), 1, (0, 0), "avg")]


@pytest.mark.parametrize("cin,cout,k,stride,pad,pool", CONV2D)
@pytest.mark.parametrize("side", [8, 17])
def test_conv2d_tf32_within_fp32_accumulation_of_the_rounded_product(cin, cout, k, stride, pad, pool, side):
    conv2d_case(cin, cout, k, stride, pad, pool, side, 3, 8, cout + 16, f"{cin}_{cout}_{k}_{stride}_{pool}_{side}")


def test_conv2d_tf32_stem_at_full_size():
    """The Inception stem on 299x299 frames: M = 2 * 149 * 149 positions, a partial last tile."""
    conv2d_case(4, 32, (3, 3), 2, (0, 0), None, 299, 2, 0, 32, "stem299")


# ---- networks ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def i3d_sd():
    return IO.synthetic_weights()


@pytest.fixture(scope="module")
def inc_sd():
    return NO.synthetic_weights()


@pytest.fixture(scope="module")
def i3d_nets(i3d_sd):
    return FV.I3D(i3d_sd, device=DEV), FV.I3D(i3d_sd, device=DEV, tf32=True)


@pytest.fixture(scope="module")
def inc_nets(inc_sd):
    return FD.InceptionV3(inc_sd, device=DEV), FD.InceptionV3(inc_sd, device=DEV, tf32=True)


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def with_tf32(flag, fn):
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = flag
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def deviation(a, b):
    return float((a - b).abs().max() / b.abs().max())


def test_i3d_tf32_features_are_batch_invariant(i3d_sd, i3d_nets):
    net = i3d_nets[1]
    assert net.tf32 and not i3d_nets[0].tf32
    x = torch.from_numpy(IO.blob_videos("tf32chunk", 5, 10, 32, 1)).to(DEV)
    base = net(x, 1)
    assert base.shape == (5, 400) and bool(base.isfinite().all())
    for chunk in (1, 3, 16):
        assert torch.equal(FV.I3D(i3d_sd, device=DEV, max_chunk_videos=chunk, tf32=True)(x, 1), base), chunk
    for i in (0, 2, 4):
        assert torch.equal(net(x[i:i + 1], 1), base[i:i + 1])
    assert torch.equal(net(x.flip(0), 1), base.flip(0))
    assert not torch.equal(base, i3d_nets[0](x, 1))                # a different numerics class


def test_inception_tf32_features_are_batch_invariant(inc_sd, inc_nets):
    net = inc_nets[1]
    x = torch.from_numpy(NO.blob_frames("tf32chunk", 17, 64, 1)).to(DEV)
    base = net(x, 1)
    assert base.shape == (17, 2048) and bool(base.isfinite().all())
    for chunk in (1, 3, 16):
        assert torch.equal(FD.InceptionV3(inc_sd, device=DEV, max_chunk_frames=chunk, tf32=True)(x, 1), base), chunk
    for i in (0, 8, 16):
        assert torch.equal(net(x[i:i + 1], 1), base[i:i + 1])
    assert torch.equal(net(x.flip(0), 1), base.flip(0))
    assert torch.equal(net(x.repeat(1, 3, 1, 1), 3), base)
    assert not torch.equal(base, inc_nets[0](x, 1))


def test_i3d_tf32_deviation_is_within_twice_cudnns(i3d_sd, i3d_nets):
    ref = _tool("time_fvd").CudnnI3D(i3d_sd, DEV)
    real = torch.from_numpy(IO.blob_videos("tf32fvd_r", 16, 10, 64, 3)).to(DEV)
    fake = (real + 0.1 * detfill.normal("tf32fvd_f", tuple(real.shape)).to(DEV)).clamp(0, 1)
    videos = torch.cat([real, fake])
    f32, ftf = (net(videos, 3) for net in i3d_nets)
    c32 = with_tf32(False, lambda: ref(videos, 3))
    ctf = with_tf32(True, lambda: ref(videos, 3))
    dev_native, dev_cudnn = deviation(ftf, f32), deviation(ctf, c32)
    assert 0 < dev_native <= 2 * dev_cudnn, (dev_native, dev_cudnn)
    d32, dtf = FV.frechet_distance(f32[16:], f32[:16]), FV.frechet_distance(ftf[16:], ftf[:16])
    e32, etf = FV.frechet_distance(c32[16:], c32[:16]), FV.frechet_distance(ctf[16:], ctf[:16])
    assert abs(dtf - d32) / d32 <= 2 * abs(etf - e32) / e32 + 1e-9, (d32, dtf, e32, etf)


def test_inception_tf32_deviation_is_within_twice_cudnns(inc_sd, inc_nets):
    ref = _tool("time_fid").TorchInception(inc_sd, DEV)
    real = torch.from_numpy(NO.blob_frames("tf32fid_r", 24, 64, 3)).to(DEV)
    fake = (real + 0.1 * detfill.normal("tf32fid_f", tuple(real.shape)).to(DEV)).clamp(0, 1)
    frames = torch.cat([real, fake])
    f32, ftf = (net(frames, 3) for net in inc_nets)
    c32 = with_tf32(False, lambda: ref(frames))
    ctf = with_tf32(True, lambda: ref(frames))
    dev_native, dev_cudnn = deviation(ftf, f32), deviation(ctf, c32)
    assert 0 < dev_native <= 2 * dev_cudnn, (dev_native, dev_cudnn)
    d32, dtf = FD.fid(f32[24:], f32[:24]), FD.fid(ftf[24:], ftf[:24])
    e32, etf = FD.fid(c32[24:], c32[:24]), FD.fid(ctf[24:], ctf[:24])
    assert abs(dtf - d32) / d32 <= 2 * abs(etf - e32) / e32 + 1e-9, (d32, dtf, e32, etf)


def test_drop_ins_use_tf32_under_the_environment_switch(inc_sd, inc_nets, tmp_path, monkeypatch):
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    torch.save(inc_sd, tmp_path / "hub" / "checkpoints" / FD.WEIGHTS_FILE)
    real, fake = (torch.from_numpy(a) for a in NO.golden_cases()["grey64"])
    FD._model.cache_clear()
    try:
        monkeypatch.setenv("MCVD_EVAL_TF32", "1")
        assert FD.model_for(DEV).tf32
        fr, ff = inc_nets[1](real, 1), inc_nets[1](fake, 1)
        assert FD.get_fid(real, fake, DEV) == FD.frechet_distance_stats(*FD.stats(fr), *FD.stats(ff))
        monkeypatch.delenv("MCVD_EVAL_TF32")
        assert not FD.model_for(DEV).tf32
        fr, ff = inc_nets[0](real, 1), inc_nets[0](fake, 1)
        assert FD.get_fid(real, fake, DEV) == FD.frechet_distance_stats(*FD.stats(fr), *FD.stats(ff))
    finally:
        FD._model.cache_clear()
