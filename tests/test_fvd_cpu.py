"""FVD on the CPU: the fp64 oracle against the golden written from the unmodified reference FVD code
(tests/golden/fvd.npz, oracle/gen_golden_fvd.py), the host Fréchet distance and summary, the oracle's resize against
``F.interpolate``, weight loading and folding, op validation and launch counts, and the ``evaluate_tasks`` plumbing
with the oracle standing in for the GPU."""
import math
import os
import re

import numpy as np
import pytest
import scipy.stats as st
import torch
import torch.nn.functional as Fn

from common import golden
from mcvd_b200 import configs, detfill, fvd as FV, lib, runner
from oracle import i3d_oracle as IO
from test_tasks_cpu import cpu_metrics, recording_sampler


@pytest.fixture(scope="module")
def sd():
    return IO.synthetic_weights()


@pytest.fixture(scope="module")
def cases():
    return IO.golden_cases()


def test_golden_videos_regenerate(cases):
    g = golden("fvd")
    for name, (real, fake, C, p) in cases.items():
        assert IO.checksum(real) == str(g[f"{name}_real_sha"]) and IO.checksum(fake) == str(g[f"{name}_fake_sha"])
        assert int(g[f"{name}_channels"]) == C and int(g[f"{name}_p"]) == p
        assert fake.shape[0] == real.shape[0] * p


def test_oracle_matches_reference_golden(sd, cases):
    """fp64 oracle vs the fp32 reference network: features within 1e-6 of the feature scale, FVD within 1e-5."""
    g = golden("fvd")
    for name, (real, fake, C, p) in cases.items():
        rf, ff = IO.features(real, C, sd), IO.features(fake, C, sd)
        for got, key in ((rf, "real"), (ff, "fake")):
            want = g[f"{name}_{key}_feats"]
            assert got.shape == want.shape == (len(got), 400)
            scale = np.abs(want).max()
            assert scale > 1 and np.abs(got - want).max() <= 1e-6 * scale, (name, key, np.abs(got - want).max())
        assert abs(IO.frechet_distance(ff, rf) - g[f"{name}_fvd"]) <= 1e-5 * g[f"{name}_fvd"]


def test_host_frechet_distance_and_summary_match_golden():
    g = golden("fvd")
    for name in ("grey32_t10", "rgb64_t11", "grey64_t25_p2"):
        f, r, p = g[f"{name}_fake_feats"], g[f"{name}_real_feats"], int(g[f"{name}_p"])
        d = FV.frechet_distance(f, r)
        assert d > 0.5 and abs(d - g[f"{name}_fvd"]) <= 1e-12 * g[f"{name}_fvd"]
        assert abs(IO.frechet_distance(f, r) - d) <= 1e-6 * d       # the eigenvalue restatement agrees
        s = FV.fvd_summary(torch.from_numpy(f), torch.from_numpy(r), p)
        assert sorted(s) == ["fvd", "fvd_traj_conf95", "fvd_traj_mean", "fvd_traj_std"]
        assert abs(s["fvd"] - g[f"{name}_fvd"]) <= 1e-12 * g[f"{name}_fvd"]
        if p == 1:
            assert s["fvd_traj_mean"] == s["fvd_traj_std"] == s["fvd_traj_conf95"] == -1
            continue
        trajs = g[f"{name}_traj_fvd"]
        mean = trajs.mean()
        conf = mean - st.norm.interval(0.95, loc=mean, scale=st.sem(trajs))[0]
        for key, want in (("fvd_traj_mean", mean), ("fvd_traj_std", trajs.std()), ("fvd_traj_conf95", conf)):
            assert abs(s[key] - want) <= 1e-12 * abs(want), key
        assert abs(s["fvd_traj_conf95"] - 1.959963984540054 * trajs.std(ddof=1) / math.sqrt(p)) <= 1e-9


def test_fvd_summary_rejects_mismatched_sets():
    with pytest.raises(ValueError, match="per each"):
        FV.fvd_summary(np.zeros((5, 4)), np.zeros((2, 4)), 2)
    with pytest.raises(ValueError, match="feature sizes"):
        FV.frechet_distance(np.zeros((5, 4)), np.zeros((5, 3)))


@pytest.mark.parametrize("S", [16, 25, 32, 48, 64, 100, 128, 256])
def test_oracle_resize_matches_f_interpolate(S):
    """The oracle's interpolation matrices (and the 225-row target float rounding gives some sides) against the
    reference's own call, F.interpolate(size=target, bilinear, align_corners=False) and its centre crop."""
    v = detfill.uniform(f"resize{S}", (3, 2, S, S), 0.0, 1.0).double()
    Ht, Wt = FV.resize_target(S)
    scale = 224 / min(S, S)
    assert (Ht, Wt) == (math.ceil(S * scale), 224)
    want = Fn.interpolate(v, size=(Ht, Wt), mode="bilinear", align_corners=False)
    h0 = (Ht - 224) // 2
    want = (want[:, :, h0:h0 + 224, :224] - 0.5) * 2
    got = IO.preprocess(v)
    assert got.shape == want.shape == (3, 2, 224, 224)
    assert float((got - want).abs().max()) <= 1e-12


def test_folded_weights_equal_the_unfolded_network(sd):
    packed = FV.pack_weights(sd)
    assert len(packed) == 58
    for key, cin, cout, k in FV.units():
        w, b = packed[key]
        cin4 = -(-cin // 4) * 4
        assert w.shape == (k ** 3 * cin4, cout) and w.dtype == torch.float32 and b.shape == (cout,)
        if cin4 != cin:
            assert not bool(w.reshape(k ** 3, cin4, cout)[:, cin:].any())
        # conv + batch norm in fp64 vs the folded fp32 weights applied in fp64: equal to fp32 rounding
        xin = detfill.normal("fold_" + key, (1, cin, 3, 5, 5)).double()
        want = IO.unit(xin, sd, key, k) if k == 1 else None
        wt = w.double().reshape(k, k, k, cin4, cout)[..., :cin, :].permute(4, 3, 0, 1, 2)
        if want is not None:
            got = torch.relu(Fn.conv3d(xin, wt) + b.double().view(1, -1, 1, 1, 1))
            assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max()), key
        g, bb = sd[key + ".bn.weight"].double(), sd[key + ".bn.bias"].double()
        m, v = sd[key + ".bn.running_mean"].double(), sd[key + ".bn.running_var"].double()
        scale = g / torch.sqrt(v + 1e-5)
        ref_w = (sd[key + ".conv3d.weight"].double() * scale.view(-1, 1, 1, 1, 1))
        assert torch.equal(wt, ref_w.float().double()), key
        assert torch.equal(b, (bb - m * scale).float()), key
    w, b = packed["logits"]
    assert torch.equal(w, sd["logits.conv3d.weight"].reshape(400, 1024).t()) and torch.equal(b, sd["logits.conv3d.bias"])


def test_bad_weight_files_raise(sd, tmp_path):
    with pytest.raises(ValueError, match="Mixed_4c.b1b.conv3d.weight"):
        FV.pack_weights({k: v for k, v in sd.items() if k != "Mixed_4c.b1b.conv3d.weight"})
    with pytest.raises(ValueError, match="Conv3d_1a_7x7.bn.running_var"):
        FV.pack_weights(dict(sd, **{"Conv3d_1a_7x7.bn.running_var": torch.ones(63)}))
    with pytest.raises(ValueError, match="logits.conv3d.bias"):
        FV.pack_weights({k: v for k, v in sd.items() if k != "logits.conv3d.bias"})
    with pytest.raises(ValueError, match="Mixed_3b.b0.conv3d.weight"):
        FV.pack_weights(dict(sd, **{"Mixed_3b.b0.conv3d.weight": torch.zeros(64, 192, 3, 3, 3)}))
    torch.save(sd, tmp_path / "i3d.pt")
    a, b = FV.pack_weights(sd), FV.pack_weights(str(tmp_path / "i3d.pt"))
    assert all(torch.equal(a[k][0], b[k][0]) and torch.equal(a[k][1], b[k][1]) for k in a)
    (tmp_path / "junk.pt").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="cannot read"):
        FV.pack_weights(str(tmp_path / "junk.pt"))
    with pytest.raises(ValueError, match="max_chunk_videos"):
        FV.I3D(sd, device="cpu", max_chunk_videos=0)
    net = FV.I3D(sd, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        net(torch.zeros(1, 10, 32, 32), 1)


def chunk_ops(n, T=10, S=32, C=1, sd=None):
    net = FV.I3D(sd or IO.synthetic_weights(), device="cpu")
    videos = torch.zeros(n, C * T, S, S)
    out = torch.zeros(n, 400, dtype=torch.float64)
    ws = torch.zeros(n * FV.workspace_floats(T))
    return net.program(videos, C, out, ws), (videos, out, ws, net)


@pytest.mark.parametrize("n,T", [(1, 9), (2, 10), (5, 25), (16, 30)])
def test_chunk_program_validates_and_costs_a_fixed_number_of_launches(sd, n, T):
    ops, keep = chunk_ops(n, T, sd=sd)
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    assert lib.load().mcvd_count_launches(arr, len(ops)) == len(ops) == FV.LAUNCHES_PER_CHUNK == 72
    kinds = [o.kind for o in ops]
    assert kinds[0] == lib.OP_I3D_PREP and kinds[-1] == lib.OP_I3D_HEAD
    assert kinds.count(lib.OP_CONV3D) == 57 and kinds.count(lib.OP_MAXPOOL3D) == 4 + 9
    head = ops[-1]
    assert (head.i4, head.i5, head.C0, head.Cout) == (FV.same_out(FV.same_out(FV.same_out(T, 7, 2), 3, 2), 2, 2), 7,
                                                      1024, 400)


def test_validate_program_rejects_bad_i3d_ops(sd):
    ops, keep = chunk_ops(2, sd=sd)
    prep, stem, pool, b1b, head = ops[0], ops[1], ops[2], ops[8], ops[-1]
    assert (stem.i0, stem.i2, b1b.i0, b1b.i7, b1b.i6) == (7, 2, 3, 64, 256)

    def rejects(op, match):
        with pytest.raises(RuntimeError, match=match):
            lib.validate_program(lib.make_ops([op]), 1)

    def edit(op, **kw):
        o = lib.McvdOp.from_buffer_copy(op)
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    rejects(edit(prep, C0=2), "1 or 3")
    rejects(edit(prep, H=112, W=112), "224x224")
    rejects(edit(prep, i2=223), "crop")
    rejects(edit(prep, B=6554), "grid")                     # 6554 videos x 10 frames > 65535
    rejects(edit(prep, dst=None), "null")
    rejects(edit(stem, w=None), "null")
    rejects(edit(stem, bias=None), "null")
    rejects(edit(stem, C0=3), "multiple of 4")
    rejects(edit(stem, Cout=60), "multiple of 8")
    rejects(edit(stem, H=111, W=111), "SAME")
    rejects(edit(stem, i5=225), "SAME")                     # ceil(225 / 2) = 113
    rejects(edit(stem, H=112, W=111), "SAME")
    rejects(edit(stem, i3=0), "stride")
    rejects(edit(b1b, i6=191), "pitch")                     # offset 64 + 128 channels > pitch
    rejects(edit(b1b, i7=130), "pitch")                     # offset not a multiple of 4
    rejects(edit(pool, C0=6), "multiple of 4")
    rejects(edit(pool, H=55, W=55), "SAME")
    rejects(edit(pool, src0=None), "null")
    rejects(edit(head, i4=1), "2 time steps")
    rejects(edit(head, i5=8), "side must be 7")
    rejects(edit(head, w=None), "null")
    rejects(edit(head, Cout=513), "logits")
    lib.validate_program(lib.make_ops([prep, stem, pool, b1b, head]), 5)


def test_header_and_binding_agree_on_i3d_surface():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "mcvd_b200.h")).read()
    for name, val in (("I3D_PREP", 22), ("CONV3D", 23), ("MAXPOOL3D", 24), ("I3D_HEAD", 25)):
        assert int(re.search(rf"MCVD_OP_{name}\s*=\s*(\d+)", hdr).group(1)) == getattr(lib, f"OP_{name}") == val
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.load().mcvd_abi_version() == 5


# ---- evaluate_tasks ---------------------------------------------------------------------------------------------
def oracle_i3d(calls):
    """Stands in for fvd.I3D: records each call and returns cheap deterministic per-video "features" (the video's
    per-frame means in the first columns), so the test can see which frames each video holds."""
    def fn(videos, channels):
        calls.append((videos.clone(), channels))
        B, CT = videos.shape[:2]
        f = torch.zeros(B, 400, dtype=torch.float64)
        f[:, :CT] = videos.double().mean((2, 3))
        f[:, 399] = torch.arange(B, dtype=torch.float64) ** 1.5
        return f
    return fn


def clips(cfg, B, T, tag="fvd_clips"):
    d = cfg.data
    return detfill.uniform(tag, (B, T, d.channels, d.image_size, d.image_size), 0.0, 1.0)


def test_evaluate_tasks_fvd_videos_gate_and_keys(monkeypatch):
    """tiny_general (Fc 3, F 2, Ff 2) with num_frames_pred 7: interpolation videos have 3 + 2 + 2 = 7 frames (no
    FVD); prediction with the future zeroed has 3 + 7 = 10 (FVD); generation has 3 + 7 = 10 and is scored against
    task (2)'s real videos."""
    cfg = configs.workload("tiny_general")
    C, Fc = cfg.data.channels, cfg.data.num_frames_cond
    X = clips(cfg, 2, 10)
    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    kw = dict(preds_per_test=2, philox_seed=99, init_seed=7, num_frames_pred=7)
    plain = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, sampler=recording_sampler([]), **kw)
    calls = []
    out = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, i3d=oracle_i3d(calls), sampler=recording_sampler([]),
                                **kw)
    assert list(out) == list(plain) == ["interp", "pred", "gen"]
    keys = ["fvd", "fvd_traj_conf95", "fvd_traj_mean", "fvd_traj_std", "i3d_fake", "i3d_real"]
    for task, (frames, m) in out.items():
        assert torch.equal(frames, plain[task][0])
        if task == "interp":                                    # 7-frame videos: no FVD, metrics unchanged
            assert sorted(m) == sorted(plain[task][1])
            for k in m:
                assert torch.equal(m[k], plain[task][1][k])
    assert len(calls) == 4
    Xr = X.repeat_interleave(2, dim=0)
    # task (2): past + prediction, against past + real frames, deduplicated [::p]
    (fake, c0), (real, c1) = calls[0], calls[1]
    frames = out["pred"][0]
    assert c0 == c1 == C and fake.shape == (4, 10 * C, 32, 32) and real.shape == (2, 10 * C, 32, 32)
    past = Xr[:, :Fc].reshape(4, -1, 32, 32)
    assert torch.allclose(fake, torch.cat([past, frames], 1), atol=1e-6)
    assert torch.allclose(real, X[:, :Fc + 7].reshape(2, -1, 32, 32), atol=1e-6)
    m = out["pred"][1]
    assert sorted(m) == sorted(list(plain["pred"][1]) + keys)
    assert torch.equal(m["i3d_fake"], oracle_i3d([])(fake, C)) and torch.equal(m["i3d_real"], oracle_i3d([])(real, C))
    want = FV.fvd_summary(m["i3d_fake"], m["i3d_real"], 2)
    assert np.array_equal([m[k] for k in want], list(want.values()), equal_nan=True) and m["fvd_traj_mean"] != -1
    # task (3): the generated frames alone, against task (2)'s real videos
    (fake, _), (real, _) = calls[2], calls[3]
    assert torch.equal(fake, out["gen"][0]) and fake.shape == (4, 10 * C, 32, 32)
    assert torch.equal(real, calls[1][0])
    assert sorted(out["gen"][1]) == keys
    # evaluate_clips passes it on to task (1): interpolation with 7-frame videos gets no FVD
    calls = []
    _, m = runner.evaluate_clips(cfg, torch.nn.Linear(1, 1), X, i3d=oracle_i3d(calls), sampler=recording_sampler([]),
                                 **kw)
    assert calls == [] and "fvd" not in m


def test_evaluate_tasks_fvd_interpolation_and_short_real(monkeypatch):
    """An interpolation model with 10-frame videos (Fc 3, F 5, Ff 2) gets past + frames + future; a prediction that
    runs past the real frames of X gets neither metrics nor FVD; below 10 frames there is no FVD."""
    cfg = configs.workload("tiny_general")
    cfg.data.num_frames = 5
    cfg.data.prob_mask_cond, cfg.data.prob_mask_future = 0.0, 0.0          # interpolation only
    C, Fc, F = cfg.data.channels, cfg.data.num_frames_cond, cfg.data.num_frames
    X = clips(cfg, 3, Fc + F + 2, "fvd_interp")
    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    calls = []
    out = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, preds_per_test=1, i3d=oracle_i3d(calls),
                                sampler=recording_sampler([]), philox_seed=1)
    assert list(out) == ["interp"] and len(calls) == 2
    frames, m = out["interp"]
    (fake, _), (real, _) = calls
    assert fake.shape == real.shape == (3, 10 * C, 32, 32)
    Xf = X.reshape(3, -1, 32, 32)
    assert torch.allclose(real, Xf, atol=1e-6)
    assert torch.allclose(fake[:, :C * Fc], Xf[:, :C * Fc], atol=1e-6)
    assert torch.equal(fake[:, C * Fc:C * (Fc + F)], frames)
    assert torch.allclose(fake[:, C * (Fc + F):], Xf[:, C * (Fc + F):], atol=1e-6)
    assert m["fvd_traj_mean"] == m["fvd_traj_std"] == m["fvd_traj_conf95"] == -1 and m["i3d_real"].shape == (3, 400)
    # prediction past the real frames: no metrics, no I3D call
    cfg2 = configs.workload("tiny")
    calls = []
    out = runner.evaluate_tasks(cfg2, torch.nn.Linear(1, 1), clips(cfg2, 2, 8), preds_per_test=1, num_frames_pred=7,
                                i3d=oracle_i3d(calls), sampler=recording_sampler([]))
    assert out["pred"][1] is None and calls == []
    # 3 + 6 = 9 frames: metrics, no FVD; 3 + 7 = 10: FVD
    out = runner.evaluate_tasks(cfg2, torch.nn.Linear(1, 1), clips(cfg2, 2, 10), preds_per_test=1, num_frames_pred=6,
                                i3d=oracle_i3d(calls), sampler=recording_sampler([]))
    assert "fvd" not in out["pred"][1] and "mse" in out["pred"][1] and calls == []
    out = runner.evaluate_tasks(cfg2, torch.nn.Linear(1, 1), clips(cfg2, 2, 10), preds_per_test=1, num_frames_pred=7,
                                i3d=oracle_i3d(calls), sampler=recording_sampler([]))
    assert "fvd" in out["pred"][1] and len(calls) == 2


def test_evaluate_tasks_gen_real_set_is_task_one_without_task_two(monkeypatch):
    """A model that masks the past but has no future frames runs (1) prediction and (3) generation; generation is
    scored against task (1)'s real videos (runners/ncsn_runner.py:1975-1977)."""
    cfg = configs.workload("tiny")
    cfg.data.prob_mask_cond = 0.5
    assert runner.tasks_for(cfg) == ["pred", "gen"]
    X = clips(cfg, 2, 10, "fvd_gen1")
    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    calls = []
    out = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, preds_per_test=1, num_frames_pred=7,
                                i3d=oracle_i3d(calls), sampler=recording_sampler([]))
    assert len(calls) == 4
    assert torch.equal(calls[3][0], calls[1][0])            # gen's real set = pred's real set
    assert torch.equal(calls[2][0], out["gen"][0]) and "fvd" in out["gen"][1]
