"""FID, precision and recall on the CPU: the fp64 oracle against the golden written from the unmodified reference
(tests/golden/fid.npz, oracle/gen_golden_fid.py), the host Fréchet distance, weight loading and folding in both key
layouts, the chunk program's launch count and validation, and the ``patch.install()`` rebinding against a stub with
the reference's module layout."""
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from common import golden
from mcvd_b200 import detfill, fid as FD, lib
from oracle import inception_oracle as NO

CASES = ("grey64", "rgb64", "rgb128", "dup_grey64")


@pytest.fixture(scope="module")
def sd():
    return NO.synthetic_weights()


@pytest.fixture(scope="module")
def cases():
    return NO.golden_cases()


def test_golden_frames_regenerate(cases):
    g = golden("fid")
    assert tuple(cases) == CASES
    for name, (real, fake) in cases.items():
        assert NO.checksum(real) == str(g[f"{name}_real_sha"]) and NO.checksum(fake) == str(g[f"{name}_fake_sha"])
        assert g[f"{name}_real_feats"].shape == (len(real), 2048) and g[f"{name}_fake_feats"].shape == (len(fake), 2048)
    real = cases["dup_grey64"][0]
    assert np.array_equal(real[0::2], real[1::2])                 # every real frame of dup_grey64 appears twice


def test_oracle_matches_reference_golden(sd, cases):
    """fp64 oracle vs the fp32 reference network (grey cases: the reference was given the RGB replica), on the first
    two frames of every set: features within 1e-6 of the feature scale."""
    g = golden("fid")
    for name, (real, fake) in cases.items():
        for frames, key in ((real, "real"), (fake, "fake")):
            want = g[f"{name}_{key}_feats"][:2]
            got = NO.features(frames[:2], sd)
            scale = np.abs(want).max()
            assert scale > 1 and np.abs(got - want).max() <= 1e-6 * scale, (name, key, np.abs(got - want).max())


def test_host_fid_and_oracle_precision_recall_match_golden():
    """``fid`` of the golden features against the reference's get_fid_PR value, and the oracle's precision / recall
    (exact distances) against the reference's cdist-based ones: equal, since every comparison has a margin."""
    g = golden("fid")
    for name in CASES:
        rf, ff = g[f"{name}_real_feats"], g[f"{name}_fake_feats"]
        d = FD.fid(torch.from_numpy(ff), rf)
        assert d > 1 and abs(d - g[f"{name}_fid"]) <= 1e-6 * g[f"{name}_fid"], (name, d, g[f"{name}_fid"])
        assert g[f"{name}_margin"] > 1e-3 and abs(NO.cover_margin(rf, ff) - g[f"{name}_margin"]) < 1e-9
        assert NO.precision_recall(rf, ff) == (g[f"{name}_precision"], g[f"{name}_recall"]), name
    assert g["rgb128_precision"] == float(np.float32(4 / 6))    # the fp32 mean the reference's .item() returns


def test_frechet_distance_stats_matches_reference_including_the_singular_retry(capsys):
    g = golden("fid")
    cases = NO.frechet_cases()
    got = FD.frechet_distance_stats(*cases["full"])
    assert abs(got - g["fd_full"]) <= 1e-12 * g["fd_full"]
    assert "singular product" not in capsys.readouterr().out
    got = FD.frechet_distance_stats(*cases["singular"])
    assert "singular product; adding 1e-06" in capsys.readouterr().out
    assert abs(got - g["fd_singular"]) <= 1e-12 * g["fd_singular"]
    with pytest.raises(ValueError, match="different sizes"):
        FD.frechet_distance_stats(np.zeros(3), np.eye(3), np.zeros(4), np.eye(4))


def test_get_fid_from_two_stats_files(tmp_path):
    (m1, s1, m2, s2) = NO.frechet_cases()["full"]
    np.savez(tmp_path / "a.npz", mu=m1, sigma=s1)
    np.savez(tmp_path / "b.npz", mu=m2, sigma=s2)
    assert FD.get_fid(str(tmp_path / "a.npz"), str(tmp_path / "b.npz"), "cpu") == golden("fid")["fd_full"]
    with pytest.raises(ValueError, match="npz"):
        FD.get_fid(str(tmp_path / "a.pt"), str(tmp_path / "b.npz"), "cpu")
    with pytest.raises(NotImplementedError, match="dims=768"):
        FD.get_fid(str(tmp_path / "a.npz"), str(tmp_path / "b.npz"), "cpu", dims=768)
    with pytest.raises(NotImplementedError):
        FD.get_fid_PR(str(tmp_path / "a.pt"), str(tmp_path / "b.pt"), "cpu", 50, 192)


def test_oracle_precision_recall_follows_kthvalue_ties():
    """Duplicated rows: the (k+1)-th smallest distance counts every copy, as torch.kthvalue does."""
    base = detfill.normal("pr_ties", (5, 6)).numpy()
    real = np.repeat(base, 3, axis=0)                          # three copies of each row
    d = NO.distances(real, real)
    for k in (0, 1, 2, 3):
        want = torch.from_numpy(d).kthvalue(k + 1, dim=1).values.numpy()
        assert np.array_equal(np.sort(d, 1)[:, k], want)
        if k < 3:
            assert not want.any()                             # the copies (self included) are at distance 0
    assert NO.precision_recall(real, real) == (1.0, 1.0)


def test_folded_weights_equal_the_unfolded_network_in_both_layouts(sd):
    packed = FD.pack_weights(sd)
    assert len(packed) == 94 and list(packed) == [u[0] for u in FD.units()]
    wrapped = FD.pack_weights(NO.wrapper_state_dict(sd))
    assert all(torch.equal(packed[k][0], wrapped[k][0]) and torch.equal(packed[k][1], wrapped[k][1]) for k in packed)
    for key, cin, cout, (kh, kw) in FD.units():
        w, b = packed[key]
        cin4 = -(-cin // 4) * 4
        assert w.shape == (kh * kw * cin4, cout) and w.dtype == torch.float32 and b.shape == (cout,)
        wt = w.double().reshape(kh, kw, cin4, cout)[:, :, :cin].permute(3, 2, 0, 1)
        if cin4 != cin:
            assert not bool(w.reshape(kh, kw, cin4, cout)[:, :, cin:].any())
        g, bb = sd[key + ".bn.weight"].double(), sd[key + ".bn.bias"].double()
        m, v = sd[key + ".bn.running_mean"].double(), sd[key + ".bn.running_var"].double()
        scale = g / torch.sqrt(v + 1e-3)
        assert torch.equal(wt, (sd[key + ".conv.weight"].double() * scale.view(-1, 1, 1, 1)).float().double()), key
        assert torch.equal(b, (bb - m * scale).float()), key
    for key in ("Conv2d_1a_3x3", "Mixed_6b.branch7x7_2", "Mixed_7c.branch3x3_2b", "Mixed_5b.branch5x5_2"):
        _, cin, cout, (kh, kw) = next(u for u in FD.units() if u[0] == key)
        w, b = packed[key]
        cin4 = -(-cin // 4) * 4
        x = detfill.normal("fold_" + key, (1, cin, 9, 9)).double()
        pad = (kh // 2, kw // 2)
        want = NO.basic(x, sd, key, padding=pad)
        wt = w.double().reshape(kh, kw, cin4, cout)[:, :, :cin].permute(3, 2, 0, 1)
        got = torch.relu(Fn.conv2d(x, wt, padding=pad) + b.double().view(1, -1, 1, 1))
        assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max()), key


def test_bad_weight_files_raise(sd, tmp_path):
    with pytest.raises(ValueError, match="Mixed_6c.branch7x7dbl_3.conv.weight"):
        FD.pack_weights({k: v for k, v in sd.items() if k != "Mixed_6c.branch7x7dbl_3.conv.weight"})
    with pytest.raises(ValueError, match="Conv2d_1a_3x3.bn.running_var"):
        FD.pack_weights(dict(sd, **{"Conv2d_1a_3x3.bn.running_var": torch.ones(31)}))
    with pytest.raises(ValueError, match="Mixed_7b.branch3x3_2a.conv.weight"):
        FD.pack_weights(dict(sd, **{"Mixed_7b.branch3x3_2a.conv.weight": torch.zeros(384, 384, 3, 1)}))
    wrapped = NO.wrapper_state_dict(sd)
    with pytest.raises(ValueError, match="blocks.3.2.branch_pool.bn.bias"):
        FD.pack_weights({k: v for k, v in wrapped.items() if k != "blocks.3.2.branch_pool.bn.bias"})
    assert "fc.weight" not in wrapped and "fc.weight" in sd       # fc is ignored either way
    torch.save(sd, tmp_path / "pt_inception.pth")
    a, b = FD.pack_weights(sd), FD.pack_weights(str(tmp_path / "pt_inception.pth"))
    assert all(torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) for k in a)
    (tmp_path / "junk.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="cannot read"):
        FD.pack_weights(str(tmp_path / "junk.pth"))
    with pytest.raises(ValueError, match="max_chunk_frames"):
        FD.InceptionV3(sd, device="cpu", max_chunk_frames=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        FD.InceptionV3(sd, device="cpu")(torch.zeros(1, 3, 32, 32), 3)


def chunk_ops(n, S=64, C=1, sd=None):
    net = FD.InceptionV3(sd if sd is not None else NO.synthetic_weights(), device="cpu")
    frames = torch.zeros(n, C, S, S)
    out = torch.zeros(n, 2048, dtype=torch.float64)
    ws = torch.zeros(n * FD.workspace_floats())
    return net.program(frames, out, ws), (frames, out, ws, net)


@pytest.mark.parametrize("n,S,C", [(1, 64, 1), (7, 128, 3), (210, 32, 3)])
def test_chunk_program_validates_and_costs_a_fixed_number_of_launches(sd, n, S, C):
    ops, keep = chunk_ops(n, S, C, sd)
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    assert lib.load().mcvd_count_launches(arr, len(ops)) == len(ops) == FD.LAUNCHES_PER_CHUNK == 100
    kinds = [o.kind for o in ops]
    assert kinds[0] == lib.OP_FID_PREP and kinds[-1] == lib.OP_FID_HEAD
    assert kinds.count(lib.OP_CONV2D) == 94 and kinds.count(lib.OP_MAXPOOL2D) == 4
    pooled = [o.flags for o in ops if o.kind == lib.OP_CONV2D and o.flags]
    assert pooled == [lib.F_POOL | lib.F_AVG] * 8 + [lib.F_POOL]   # 3 A + 4 C + E_1 average, E_2 max
    head = ops[-1]
    assert (head.i5, head.C0, head.B) == (8, 2048, n)
    assert FD.DEFAULT_CHUNK * FD.workspace_floats() * 4 <= 2 << 30 < (FD.DEFAULT_CHUNK + 1) * FD.workspace_floats() * 4


def test_concat_slices_tile_each_block_output(sd):
    """The branches of every block write disjoint channel slices that cover its output exactly, in torchvision's
    concat order."""
    steps, _ = FD.plan()
    by_block, block = {}, None
    for st in steps:
        if st["kind"] == "conv":
            block = st["key"].split(".")[0]
        width = st["cout"] if st["kind"] == "conv" else st["c"]
        if st["kind"] in ("conv", "pool") and st["pitch"] != width:    # a write into a block's concat
            by_block.setdefault(block, []).append((st["off"], width, st["pitch"]))
    assert len(by_block) == 11
    for block, sl in by_block.items():
        pitch = sl[0][2]
        covered = sorted((o, o + c) for o, c, _ in sl)
        assert covered[0][0] == 0 and covered[-1][1] == pitch, block
        assert all(a[1] == b[0] for a, b in zip(covered, covered[1:])), block
    assert [o for o, _, _ in by_block["Mixed_7b"]] == [0, 320, 704, 1088, 1472, 1856]


def test_validate_program_rejects_bad_fid_ops(sd):
    ops, keep = chunk_ops(2, sd=sd)
    prep, stem, pool = ops[0], ops[1], ops[4]
    row = next(o for o in ops if (o.i0, o.i1) == (1, 7))
    pooled = next(o for o in ops if o.flags)
    head = ops[-1]
    assert (stem.i0, stem.i2, stem.i5, stem.H) == (3, 2, 299, 149) and (row.i3, row.i4) == (0, 3)

    def rejects(op, match):
        with pytest.raises(RuntimeError, match=match):
            lib.validate_program(lib.make_ops([op]), 1)

    def edit(op, **kw):
        o = lib.McvdOp.from_buffer_copy(op)
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    rejects(edit(prep, C0=2), "1 or 3")
    rejects(edit(prep, H=224, W=224), "299x299")
    rejects(edit(prep, B=65536), "grid")
    rejects(edit(prep, dst=None), "null")
    rejects(edit(stem, w=None), "null")
    rejects(edit(stem, C0=3), "multiple of 4")
    rejects(edit(stem, Cout=30), "multiple of 8")
    rejects(edit(stem, H=150, W=150), "geometry")
    rejects(edit(stem, i5=301), "geometry")                  # (301 - 3) / 2 + 1 = 150
    rejects(edit(stem, i2=0), "stride")
    rejects(edit(row, i4=7), "smaller than the kernel")
    rejects(edit(row, W=row.W - 1), "geometry")
    rejects(edit(row, i6=row.i7 + row.Cout - 4), "pitch")
    rejects(edit(row, i7=row.i7 + 2), "pitch")
    rejects(edit(stem, flags=lib.F_POOL), "1x1 stride-1")
    rejects(edit(pooled, flags=lib.F_AVG), "needs MCVD_F_POOL")
    rejects(edit(pooled, flags=lib.F_POOL | lib.F_GAMMA), "flags")
    rejects(edit(pool, C0=6), "multiple of 4")
    rejects(edit(pool, H=74, W=74), "3x3 / stride-2")
    rejects(edit(pool, i6=32), "pitch")
    rejects(edit(head, H=8, W=8), "1x1")
    rejects(edit(head, i5=0), "side")
    feats = torch.zeros(70, 12)
    radii = torch.zeros(70)
    out = torch.zeros(70)
    knn = lib.McvdOp(kind=lib.OP_KNN_RADIUS, B=70, H=1, W=1, C0=12, i0=70, i1=4, src0=feats.data_ptr(),
                     src1=feats.data_ptr(), dst=out.data_ptr())
    cover = edit(knn, kind=lib.OP_KNN_COVER, i1=0, aux0=radii.data_ptr())
    lib.validate_program(lib.make_ops([prep, stem, pool, row, pooled, head, knn, cover]), 8)
    rejects(edit(knn, i1=9), "1 .. 8")
    rejects(edit(knn, i1=0), "1 .. 8")
    rejects(edit(knn, i0=3), "larger than the second set")
    rejects(edit(knn, C0=10), "multiple of 4")
    rejects(edit(knn, src1=None), "null")
    rejects(edit(knn, flags=lib.F_POOL), "flags")
    rejects(edit(cover, aux0=None), "radii")
    rejects(edit(cover, i0=0), "empty")
    rejects(edit(cover, H=2), "1x1")


def test_header_and_binding_agree_on_fid_surface():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "mcvd_b200.h")).read()
    for name, val in (("FID_PREP", 28), ("CONV2D", 29), ("MAXPOOL2D", 30), ("FID_HEAD", 31), ("KNN_RADIUS", 32),
                      ("KNN_COVER", 33)):
        assert int(re.search(rf"MCVD_OP_{name}\s*=\s*(\d+)", hdr).group(1)) == getattr(lib, f"OP_{name}") == val
    assert int(re.search(r"#define MCVD_F_AVG\s+\(1 << (\d+)\)", hdr).group(1)) == 11 and lib.F_AVG == 1 << 11
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.load().mcvd_abi_version() == 5


# ---- drop-in ----------------------------------------------------------------------------------------------------
def test_patch_install_rebinds_fid_and_falls_back(tmp_path, monkeypatch):
    """A stub with the reference's layout (evaluation/fid_PR.py; runners/ncsn_runner.py importing get_fid and
    get_fid_PR) stands in for the reference tree.  The native functions run only when the weights file is in the
    torch hub cache, dims is 2048 and the device is CUDA; every other call gets the reference function."""
    for d in ("runners", "models", "evaluation"):
        (tmp_path / d).mkdir()
        (tmp_path / d / "__init__.py").write_text("")
    (tmp_path / "models" / "__init__.py").write_text(
        "def ddpm_sampler(x_mod, scorenet, **kw):\n    return 'reference ddpm'\n"
        "def ddim_sampler(x_mod, scorenet, **kw):\n    return 'reference ddim'\n"
        "def FPNDM_sampler(x_mod, scorenet, **kw):\n    return 'reference fpndm'\n")
    (tmp_path / "evaluation" / "fid_PR.py").write_text(
        "def get_fid(p1, p2, device='cuda', batch_size=50, dims=2048):\n    return 'reference fid'\n"
        "def get_fid_PR(r, f, device='cuda', batch_size=50, dims=2048, k=3, save_feats_path=None):\n"
        "    return 'reference fid_PR'\n"
        "def get_PR(r, f, device='cuda', batch_size=50, dims=2048):\n    return 'reference PR'\n")
    (tmp_path / "runners" / "ncsn_runner.py").write_text(
        "from evaluation.fid_PR import get_fid, get_fid_PR\n"
        "from models import ddpm_sampler, ddim_sampler, FPNDM_sampler\n"
        "def get_model(config):\n    return 'reference model'\n")
    hub = tmp_path / "hub"
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(hub))
    for name in ("get_fid", "get_fid_PR", "get_PR"):
        monkeypatch.setattr(FD, name, lambda *a, _n=name, **kw: ("native " + _n, a, kw))
    monkeypatch.syspath_prepend(str(tmp_path))
    mods = ("runners", "runners.ncsn_runner", "models", "evaluation", "evaluation.fid_PR")
    for m in mods:
        sys.modules.pop(m, None)
    try:
        from mcvd_b200 import patch
        patch.install(verbose=False)
        import importlib
        R = importlib.import_module("runners.ncsn_runner")
        EF = importlib.import_module("evaluation.fid_PR")
        assert R.get_fid is EF.get_fid and R.get_fid_PR is EF.get_fid_PR and not hasattr(R, "get_PR")
        x = torch.zeros(2, 3, 8, 8)
        assert EF.get_fid_PR("r.pt", x, torch.device("cuda")) == "reference fid_PR"     # no weights yet
        (hub / "checkpoints").mkdir(parents=True)
        (hub / "checkpoints" / FD.WEIGHTS_FILE).write_bytes(b"")
        assert FD.native_unsupported("cuda:0", 2048) is None
        assert R.get_fid_PR("r.pt", x, torch.device("cuda"), k=5)[0] == "native get_fid_PR"
        assert R.get_fid("s.npz", x, "cuda")[0] == "native get_fid"
        assert EF.get_PR("r.pt", x)[0] == "native get_PR"                              # device defaults to cuda
        assert R.get_fid("s.npz", x, "cpu") == "reference fid"
        assert R.get_fid_PR("r.pt", x, "cuda", 50, 768) == "reference fid_PR"           # dims, positional
        assert EF.get_PR("r.pt", x, device="cuda", dims=64) == "reference PR"
    finally:
        for m in mods:
            sys.modules.pop(m, None)
