"""FID, precision and recall on the H100 (mcvd_b200/fid.py, MCVD_OP_FID_PREP / CONV2D / MAXPOOL2D / FID_HEAD /
KNN_RADIUS / KNN_COVER) against the golden written from the unmodified reference (tests/golden/fid.npz) and the fp64
oracle.

Tolerances: the prep's resize is within 1e-6 of the reference's fp32 F.interpolate on the CPU and on the GPU; each
convolution is within 1e-5 of its output's scale of an fp64 evaluation of the same input (fp32 FFMA accumulation);
the max-pool is bit-exact; features are within 1e-4 of the feature scale of the golden and the oracle (94 fp32
layers); FID from the GPU features within 1e-3 relative of the golden's.  The k-NN ops are exact: on integer-valued features every squared distance is an exact
fp32 integer, so radii and flags must equal the oracle's bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from common import golden
from mcvd_b200 import detfill, fid as FD, lib
from oracle import inception_oracle as NO

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CASES = ("grey64", "rgb64", "rgb128", "dup_grey64")


@pytest.fixture(scope="module")
def sd():
    return NO.synthetic_weights()


@pytest.fixture(scope="module")
def net(sd):
    return FD.InceptionV3(sd, device=DEV)


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


@pytest.mark.parametrize("C,S", [(1, 64), (3, 64), (3, 128), (1, 32), (3, 299), (3, 400)])
def test_prep_matches_f_interpolate(C, S):
    N = 3
    x = detfill.uniform(f"fidprep{C}_{S}", (N, C, S, S), -0.1, 1.1).to(DEV)    # out of [0, 1]: no clamp
    dst = torch.full((N, 299, 299, 4), float("nan"), device=DEV)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i1 = lib.OP_FID_PREP, N, 299, 299, C, S
    op.src0, op.dst = x.data_ptr(), dst.data_ptr()
    run([op])
    assert bool((dst[..., 3] == 0).all())
    got = dst[..., :3].permute(0, 3, 1, 2).double().cpu()
    xin = x.repeat(1, 3 // C, 1, 1)
    for dev in ("cpu", DEV):                                        # the reference runs on either
        want = Fn.interpolate(xin.to(dev), size=(299, 299), mode="bilinear", align_corners=False).double().cpu()
        err = float(((got + 1) / 2 - want).abs().max())            # the resize, before 2x - 1
        assert err <= 1e-6, (dev, err)
        assert float((got - (2 * want.float() - 1).double()).abs().max()) <= 2e-6
    if C == 1:
        assert torch.equal(got[:, 0], got[:, 1]) and torch.equal(got[:, 0], got[:, 2])


def conv_op(x, w, b, k, stride, pad, cout, dst, pitch, off, flags=0):
    n, side, _, cin = x.shape
    op = lib.McvdOp()
    op.kind, op.B, op.C0, op.Cout, op.flags = lib.OP_CONV2D, n, cin, cout, flags
    op.H, op.W = FD.conv_out(side, k[0], stride, pad[0]), FD.conv_out(side, k[1], stride, pad[1])
    op.i0, op.i1, op.i2, op.i3, op.i4, op.i5, op.i6, op.i7 = k[0], k[1], stride, pad[0], pad[1], side, pitch, off
    op.src0, op.w, op.bias, op.dst = x.data_ptr(), w.data_ptr(), b.data_ptr(), dst.data_ptr()
    return op


# (Cin, Cout, (kh, kw), stride, (ph, pw), pool): every kernel shape and padding of the network, stride 2, and the
# fused pools of the branch_pool convs
CONVS = [(4, 32, (3, 3), 2, (0, 0), None), (32, 64, (3, 3), 1, (1, 1), None), (64, 80, (1, 1), 1, (0, 0), None),
         (48, 64, (5, 5), 1, (2, 2), None), (128, 128, (1, 7), 1, (0, 3), None), (160, 192, (7, 1), 1, (3, 0), None),
         (384, 384, (1, 3), 1, (0, 1), None), (384, 384, (3, 1), 1, (1, 0), None), (96, 96, (3, 3), 2, (0, 0), None),
         (288, 384, (3, 3), 2, (0, 0), None), (192, 32, (1, 1), 1, (0, 0), "avg"), (768, 192, (1, 1), 1, (0, 0), "avg"),
         (2048, 192, (1, 1), 1, (0, 0), "max"), (1280, 448, (1, 1), 1, (0, 0), None)]


@pytest.mark.parametrize("cin,cout,k,stride,pad,pool", CONVS)
@pytest.mark.parametrize("side", [8, 17])
def test_conv2d_matches_fp64_and_writes_only_its_slice(cin, cout, k, stride, pad, pool, side):
    n = 3
    x = torch.relu(detfill.normal(f"fc{cin}_{k}_{side}", (n, side, side, cin))).to(DEV)
    if pool == "max":
        x = x - 0.5                                   # negative values: the padding must never win the max
    fan = cin * k[0] * k[1]
    wt = detfill.uniform(f"fw{cin}_{cout}_{k}", (cout, cin, k[0], k[1]), -1, 1) * (3.0 / fan) ** 0.5
    b = detfill.uniform(f"fb{cout}", (cout,), -0.1, 0.1)
    w = wt.permute(2, 3, 1, 0).reshape(-1, cout).contiguous().to(DEV)
    off, pitch = 8, cout + 16
    ho, wo = FD.conv_out(side, k[0], stride, pad[0]), FD.conv_out(side, k[1], stride, pad[1])
    dst = torch.full((n, ho, wo, pitch), float("nan"), device=DEV)
    flags = 0 if pool is None else lib.F_POOL | (lib.F_AVG if pool == "avg" else 0)
    run([conv_op(x, w, b.to(DEV), k, stride, pad, cout, dst, pitch, off, flags)])
    xin = x.permute(0, 3, 1, 2).double().cpu()
    if pool == "avg":
        xin = Fn.avg_pool2d(xin, 3, 1, 1, count_include_pad=False)
    elif pool == "max":
        xin = Fn.max_pool2d(xin, 3, 1, 1)
    want = torch.relu(Fn.conv2d(xin, wt.double(), b.double(), stride=stride, padding=pad))
    got = dst[..., off:off + cout].permute(0, 3, 1, 2).double().cpu()
    scale = float(want.abs().max())
    assert got.shape == want.shape and scale > 0
    assert float((got - want).abs().max()) <= 1e-5 * scale, float((got - want).abs().max()) / scale
    assert bool(dst[..., :off].isnan().all()) and bool(dst[..., off + cout:].isnan().all())


@pytest.mark.parametrize("side,c", [(147, 64), (71, 192), (35, 288), (17, 768), (8, 16)])
def test_maxpool2d_is_bit_exact_into_a_slice(side, c):
    n = 2
    x = detfill.normal(f"mp{side}_{c}", (n, side, side, c)).to(DEV)
    so = (side - 3) // 2 + 1
    off, pitch = 4, c + 12
    dst = torch.full((n, so, so, pitch), float("nan"), device=DEV)
    op = lib.McvdOp()
    op.kind, op.B, op.C0, op.H, op.W, op.i5, op.i6, op.i7 = lib.OP_MAXPOOL2D, n, c, so, so, side, pitch, off
    op.src0, op.dst = x.data_ptr(), dst.data_ptr()
    run([op])
    want = Fn.max_pool2d(x.permute(0, 3, 1, 2), 3, 2).permute(0, 2, 3, 1)
    assert torch.equal(dst[..., off:off + c], want)
    assert bool(dst[..., :off].isnan().all()) and bool(dst[..., off + c:].isnan().all())


def test_head_is_the_fp64_mean():
    x = detfill.normal("fidhead", (3, 8, 8, 2048)).to(DEV)
    out = torch.empty(3, 2048, dtype=torch.float64, device=DEV)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i5 = lib.OP_FID_HEAD, 3, 1, 1, 2048, 8
    op.src0, op.dst = x.data_ptr(), out.data_ptr()
    run([op])
    want = x.double().mean((1, 2))
    assert float((out - want).abs().max()) <= 1e-15


def test_features_match_golden_and_oracle(net, sd):
    g = golden("fid")
    for name, (real, fake) in NO.golden_cases().items():
        feats = {}
        for key, frames in (("real", real), ("fake", fake)):
            got = net(torch.from_numpy(frames).to(DEV), frames.shape[1])
            assert got.dtype == torch.float64 and got.shape == (len(frames), 2048)
            got = got.cpu().numpy()
            want = g[f"{name}_{key}_feats"]
            scale = np.abs(want).max()
            assert np.abs(got - want).max() <= 1e-4 * scale, (name, key, np.abs(got - want).max(), scale)
            if key == "real":
                orc = NO.features(frames[:1], sd)
                assert np.abs(got[:1] - orc).max() <= 1e-4 * scale
            feats[key] = got
        d = FD.fid(feats["fake"], feats["real"])
        assert abs(d - g[f"{name}_fid"]) <= 1e-3 * g[f"{name}_fid"], (name, d, g[f"{name}_fid"])
        pr = FD.precision_recall(feats["real"], feats["fake"], 3, DEV)
        assert pr == (g[f"{name}_precision"], g[f"{name}_recall"]), name


def test_features_do_not_depend_on_chunk_position_or_channels(sd, net, monkeypatch):
    x = torch.from_numpy(NO.blob_frames("fidchunk", 9, 64, 1)).to(DEV)
    base = net(x, 1)
    programs = []
    real_run = lib.run_program

    def counting(arr, n, stream):
        programs.append(lib.load().mcvd_count_launches(arr, n))
        real_run(arr, n, stream)
    monkeypatch.setattr(lib, "run_program", counting)
    assert torch.equal(FD.InceptionV3(sd, device=DEV, max_chunk_frames=7)(x, 1), base)
    assert programs == [FD.LAUNCHES_PER_CHUNK] * 2                    # 7 + 2 frames
    monkeypatch.setattr(lib, "run_program", real_run)
    assert torch.equal(FD.InceptionV3(sd, device=DEV, max_chunk_frames=1)(x, 1), base)
    for i in (0, 4, 8):
        assert torch.equal(net(x[i:i + 1], 1), base[i:i + 1])
    assert torch.equal(net(x.flip(0), 1), base.flip(0))
    assert torch.equal(net(x.repeat(1, 3, 1, 1), 3), base)          # a grey frame = its RGB replica, bit for bit
    assert torch.equal(net(x.cpu(), 1), base)                        # CPU frames are copied per chunk
    video = x[:8].reshape(2, 4, 64, 64)                              # [B, C*T, S, S]: frames in frame order
    assert torch.equal(net(video, 1), base[:8])


def test_bad_frames_raise(net):
    with pytest.raises(ValueError, match="channels"):
        net(torch.zeros(1, 2, 32, 32, device=DEV), 2)
    with pytest.raises(ValueError, match="must be"):
        net(torch.zeros(1, 3, 32, 31, device=DEV), 3)
    assert net(torch.zeros(0, 3, 32, 32, device=DEV), 3).shape == (0, 2048)


# ---- k-NN --------------------------------------------------------------------------------------------------------
def int_feats(tag, n, d):
    """Integer-valued features in [-3, 3]: every squared distance is an exact fp32 integer (< 2^24)."""
    return torch.round(detfill.uniform(tag, (n, d), -3.49, 3.49)).float()


def oracle_knn(a, b, k):
    """(radii of b [Nb] float32, cover flags of a over b [Na]) from exact integer squared distances, checked in fp64."""
    a64, b64 = a.double().numpy(), b.double().numpy()
    d2_bb = ((b64[:, None] - b64[None]) ** 2).sum(-1)
    d2_ab = ((a64[:, None] - b64[None]) ** 2).sum(-1)
    r2 = np.sort(d2_bb, 1)[:, k]
    radii = np.sqrt(r2.astype(np.float32))
    assert np.array_equal(radii.astype(np.float64), np.sort(NO.distances(b64, b64), 1)[:, k].astype(np.float32))
    return radii, (d2_ab <= r2[None, :]).any(1).astype(np.int32)


@pytest.mark.parametrize("k", [1, 3, 5])
@pytest.mark.parametrize("na,nb,d", [(100, 130, 2048), (64, 200, 36), (1, 8, 4), (257, 65, 12)])
def test_knn_radius_and_cover_are_exact(k, na, nb, d):
    a = int_feats(f"knn_a{na}_{d}", na, d)
    b = int_feats(f"knn_b{nb}_{d}", nb, d)
    want_r, want_f = oracle_knn(a, b, k)
    ad, bd = a.to(DEV), b.to(DEV)
    radii = FD.knn_radii(bd, k)
    flags = FD.knn_cover(ad, bd, radii)
    torch.cuda.synchronize()
    assert np.array_equal(radii.cpu().numpy(), want_r)
    assert np.array_equal(flags.cpu().numpy(), want_f)
    again = FD.knn_radii(bd, k), FD.knn_cover(ad, bd, radii)
    assert torch.equal(again[0], radii) and torch.equal(again[1], flags)


def test_knn_counts_exact_duplicates_as_kthvalue_does():
    base = int_feats("knn_dup", 40, 20)
    x = base.repeat_interleave(3, 0).to(DEV)                        # three copies of every row
    for k, zero in ((0, True), (1, True), (2, True), (3, False)):
        r = FD.knn_radii(x, k).cpu()
        want = torch.from_numpy(NO.distances(x.cpu(), x.cpu())).kthvalue(k + 1, dim=1).values.float()
        assert bool((r == 0).all()) == zero and torch.equal(r, want), k
    a = int_feats("knn_dup_a", 30, 20).to(DEV)
    flags = FD.knn_cover(torch.cat([x[:5], a]), x, FD.knn_radii(x, 0))
    assert bool(flags[:5].all())                                    # radius 0: only the exact copies are covered


def test_precision_recall_of_golden_features_equal_the_golden():
    g = golden("fid")
    for name in CASES:
        rf, ff = g[f"{name}_real_feats"], g[f"{name}_fake_feats"]
        p, r = FD.precision_recall(torch.from_numpy(rf), ff, 3, DEV)
        assert (p, r) == (g[f"{name}_precision"], g[f"{name}_recall"]), name
        assert isinstance(p, float) and isinstance(r, float)


# ---- drop-ins ---------------------------------------------------------------------------------------------------
def test_drop_ins_read_the_hub_cache_and_never_download(sd, net, tmp_path, monkeypatch):
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    FD._model.cache_clear()
    real, fake = NO.golden_cases()["grey64"]
    real_t, fake_t = torch.from_numpy(real), torch.from_numpy(fake)
    with pytest.raises(FileNotFoundError, match="never downloads"):
        FD.get_fid_PR(real_t, fake_t, DEV)
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    torch.save(sd, tmp_path / "hub" / "checkpoints" / FD.WEIGHTS_FILE)
    fr, ff = net(real_t, 1), net(fake_t, 1)
    torch.save(fr.float().cpu(), tmp_path / "real_feats.pt")
    d, p, r = FD.get_fid_PR(str(tmp_path / "real_feats.pt"), fake_t, DEV, save_feats_path=str(tmp_path / "g.pt"))
    saved = torch.load(tmp_path / "g.pt")
    assert saved.dtype == torch.float32 and saved.device.type == "cpu" and torch.equal(saved, ff.float().cpu())
    assert abs(d - FD.fid(ff, fr.float())) <= 1e-9 * d
    assert (p, r) == FD.precision_recall(fr.float(), ff, 3, DEV) == FD.get_PR(str(tmp_path / "real_feats.pt"),
                                                                             fake_t, DEV)
    mu, sigma = FD.stats(fr)
    np.savez(tmp_path / "real_stats.npz", mu=mu, sigma=sigma)
    assert FD.get_fid(str(tmp_path / "real_stats.npz"), fake_t, DEV) == FD.fid(ff, fr)
    assert FD.get_fid(real_t, fake_t, "cuda") == FD.frechet_distance_stats(*FD.stats(fr), *FD.stats(ff))
    FD._model.cache_clear()
