"""FVD's I3D features on the H100 (mcvd_b200/fvd.py, MCVD_OP_I3D_PREP / CONV3D / MAXPOOL3D / I3D_HEAD) against the
golden written from the unmodified reference FVD code (tests/golden/fvd.npz) and the fp64 oracle.

Tolerances: the prep is within 1e-6 of the reference's fp32 F.interpolate; each convolution and pool is
within 1e-5 of its output's scale of an fp64 evaluation of the same input (fp32 FFMA accumulation); features are
within 1e-4 of the feature scale of the golden and the oracle (57 fp32 layers); FVD from the GPU features within
1e-3 relative of the golden's."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from common import golden, make_module
from mcvd_b200 import detfill, fvd as FV, lib, runner
from oracle import i3d_oracle as IO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def sd():
    return IO.synthetic_weights()


@pytest.fixture(scope="module")
def net(sd):
    return FV.I3D(sd, device=DEV)


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


@pytest.mark.parametrize("C,S,T", [(1, 32, 2), (3, 64, 3), (1, 48, 2), (3, 25, 2), (1, 128, 1)])
def test_prep_matches_f_interpolate(C, S, T):
    B = 2
    v = detfill.uniform(f"prep{C}_{S}", (B, C * T, S, S), -0.1, 1.1).to(DEV)   # out of [0, 1]: no clamp
    dst = torch.full((B, T, 224, 224, 4), float("nan"), device=DEV)
    Ht, Wt = FV.resize_target(S)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i0, op.i1, op.i2, op.i3 = lib.OP_I3D_PREP, B, 224, 224, C, T, S, Ht, Wt
    op.src0, op.dst = v.data_ptr(), dst.data_ptr()
    run([op])
    assert bool((dst[..., 3] == 0).all())
    x = IO.to_i3d(v.cpu(), C)                                   # [B, 3, T, S, S]
    h0 = (Ht - 224) // 2
    for b in range(B):
        got = dst[b, ..., :3].permute(3, 0, 1, 2).double().cpu()
        # the reference's fp32 call (preprocess_single), and fp64 (the fp32 source-index rounding: ~1e-5)
        for dtype, tol in ((torch.float32, 1e-6), (torch.float64, 3e-5)):
            want = Fn.interpolate(x[b].to(dtype), size=(Ht, Wt), mode="bilinear", align_corners=False)
            want = ((want[:, :, h0:h0 + 224] - 0.5) * 2).double()
            assert float((got - want).abs().max()) <= tol, (b, dtype, float((got - want).abs().max()))
        if C == 1:
            assert torch.equal(got[0], got[1]) and torch.equal(got[0], got[2])


def conv_op(x, w, b, k, s, cout, dst, pitch, off):
    n, t, side, _, cin = x.shape
    op = lib.McvdOp()
    op.kind, op.B, op.C0, op.Cout = lib.OP_CONV3D, n, cin, cout
    op.H = op.W = FV.same_out(side, k, s)
    op.i0, op.i1, op.i2, op.i3, op.i4, op.i5, op.i6, op.i7 = k, k, s, s, t, side, pitch, off
    op.src0, op.w, op.bias, op.dst = x.data_ptr(), w.data_ptr(), b.data_ptr(), dst.data_ptr()
    return op


# (Cin, Cout, kernel, stride): the stem, stage 2 and Inception shapes, with the odd Couts of the 4x blocks
CONVS = [(4, 64, 7, 2), (64, 64, 1, 1), (64, 192, 3, 1), (192, 16, 1, 1), (16, 32, 3, 1), (96, 128, 3, 1),
         (112, 224, 3, 1), (24, 64, 3, 1), (144, 288, 3, 1), (832, 48, 1, 1), (48, 128, 3, 1), (512, 112, 1, 1)]


@pytest.mark.parametrize("cin,cout,k,s", CONVS)
@pytest.mark.parametrize("t,side", [(6, 14), (7, 15)])
def test_conv3d_matches_fp64_and_writes_only_its_slice(cin, cout, k, s, t, side):
    n = 2
    x = torch.relu(detfill.normal(f"cx{cin}_{k}", (n, t, side, side, cin))).to(DEV)
    wt = detfill.uniform(f"cw{cin}_{cout}_{k}", (cout, cin, k, k, k), -1, 1) * (3.0 / (cin * k ** 3)) ** 0.5
    b = detfill.uniform(f"cb{cout}", (cout,), -0.1, 0.1)
    w = wt.permute(2, 3, 4, 1, 0).reshape(-1, cout).contiguous().to(DEV)
    off, pitch = 8, cout + 16
    to, so = FV.same_out(t, k, s), FV.same_out(side, k, s)
    dst = torch.full((n, to, so, so, pitch), float("nan"), device=DEV)
    bd = b.to(DEV)
    run([conv_op(x, w, bd, k, s, cout, dst, pitch, off)])
    xin = x.permute(0, 4, 1, 2, 3).double().cpu()
    want = torch.relu(Fn.conv3d(IO.same_pad(xin, (k,) * 3, (s,) * 3), wt.double(), b.double(), stride=s))
    got = dst[..., off:off + cout].permute(0, 4, 1, 2, 3).double().cpu()
    scale = float(want.abs().max())
    assert got.shape == want.shape and scale > 0
    assert float((got - want).abs().max()) <= 1e-5 * scale, float((got - want).abs().max())
    assert bool(dst[..., :off].isnan().all()) and bool(dst[..., off + cout:].isnan().all())


@pytest.mark.parametrize("k,s", [((1, 3, 3), (1, 2, 2)), ((3, 3, 3), (2, 2, 2)), ((2, 2, 2), (2, 2, 2)),
                                 ((3, 3, 3), (1, 1, 1))])
@pytest.mark.parametrize("t,side", [(6, 14), (7, 15), (13, 112)])
def test_maxpool3d_matches_zero_padded_max_pool(k, s, t, side):
    n, c = 2, 16
    x = detfill.normal(f"px{t}_{side}", (n, t, side, side, c)).to(DEV)      # negative values see the zero padding
    to, so = FV.same_out(t, k[0], s[0]), FV.same_out(side, k[1], s[1])
    dst = torch.full((n, to, so, so, c), float("nan"), device=DEV)
    op = lib.McvdOp()
    op.kind, op.B, op.C0, op.H, op.W = lib.OP_MAXPOOL3D, n, c, so, so
    op.i0, op.i1, op.i2, op.i3, op.i4, op.i5 = k[0], k[1], s[0], s[1], t, side
    op.src0, op.dst = x.data_ptr(), dst.data_ptr()
    run([op])
    want = IO.max_pool(x.permute(0, 4, 1, 2, 3).double().cpu(), k, s)
    assert torch.equal(dst.permute(0, 4, 1, 2, 3).double().cpu(), want)


def test_features_match_golden_and_oracle(net, sd):
    g = golden("fvd")
    for name, (real, fake, C, p) in IO.golden_cases().items():
        feats = {}
        for key, v in (("real", real), ("fake", fake)):
            got = net(torch.from_numpy(v).to(DEV), C)
            assert got.dtype == torch.float64 and got.shape == (v.shape[0], 400)
            got = got.cpu().numpy()
            want = g[f"{name}_{key}_feats"]
            scale = np.abs(want).max()
            assert np.abs(got - want).max() <= 1e-4 * scale, (name, key, np.abs(got - want).max(), scale)
            if key == "real":
                orc = IO.features(v[:1], C, sd)
                assert np.abs(got[:1] - orc).max() <= 1e-4 * scale
            feats[key] = got
        d = FV.frechet_distance(feats["fake"], feats["real"])
        assert abs(d - g[f"{name}_fvd"]) <= 1e-3 * g[f"{name}_fvd"], (name, d, g[f"{name}_fvd"])
        s = FV.fvd_summary(feats["fake"], feats["real"], p)
        if p > 1:
            assert abs(s["fvd_traj_mean"] - g[f"{name}_traj_fvd"].mean()) <= 1e-3 * g[f"{name}_traj_fvd"].mean()


def test_features_do_not_depend_on_chunk_or_position(sd, net, monkeypatch):
    v = torch.from_numpy(IO.blob_videos("chunking", 7, 10, 32, 1)).to(DEV)
    small = FV.I3D(sd, device=DEV, max_chunk_videos=3)
    programs = []
    real_run = lib.run_program

    def counting(arr, n, stream):
        programs.append(lib.load().mcvd_count_launches(arr, n))
        real_run(arr, n, stream)
    monkeypatch.setattr(lib, "run_program", counting)
    a = small(v, 1)
    assert programs == [FV.LAUNCHES_PER_CHUNK] * 3                       # 3 + 3 + 1 videos
    monkeypatch.setattr(lib, "run_program", real_run)
    b = net(v, 1)
    assert torch.equal(a, b)
    for i in (0, 3, 6):
        assert torch.equal(net(v[i:i + 1], 1), b[i:i + 1])
    assert torch.equal(net(v.flip(0), 1), b.flip(0))


def test_bad_videos_raise(net):
    with pytest.raises(ValueError, match="at least 9"):
        net(torch.zeros(1, 8, 32, 32, device=DEV), 1)
    with pytest.raises(ValueError, match="must be"):
        net(torch.zeros(1, 10, 32, 31, device=DEV), 1)
    with pytest.raises(ValueError, match="channels"):
        net(torch.zeros(1, 20, 32, 32, device=DEV), 2)


def test_evaluate_tasks_fvd_on_gpu(net):
    cfg, model, _ = make_module("tiny", DEV)
    X = detfill.uniform("fvd_gpu_clips", (2, 10, 1, 32, 32), 0.0, 1.0).to(DEV)
    kw = dict(preds_per_test=2, philox_seed=5, init_seed=6, num_frames_pred=7)
    plain = runner.evaluate_tasks(cfg, model, X, **kw)
    out = runner.evaluate_tasks(cfg, model, X, i3d=net, **kw)
    frames, m = out["pred"]
    frames0, m0 = plain["pred"]
    assert torch.equal(frames, frames0)
    assert set(m) == set(m0) | {"i3d_fake", "i3d_real", "fvd", "fvd_traj_mean", "fvd_traj_std", "fvd_traj_conf95"}
    for k in m0:
        assert torch.equal(m[k], m0[k]), k
    fake, real = runner.fvd_videos(cfg, "pred", runner.task_inputs(cfg, X.repeat_interleave(2, 0), "pred", 7)[1],
                                   frames, runner.task_inputs(cfg, X.repeat_interleave(2, 0), "pred", 7)[0])
    assert torch.equal(m["i3d_fake"], net(fake, 1)) and torch.equal(m["i3d_real"], net(real[::2], 1))
    assert m["i3d_fake"].shape == (4, 400) and m["fvd"] > 0 and m["fvd_traj_mean"] > 0
