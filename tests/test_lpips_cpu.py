"""LPIPS on the CPU: the host resize tables against Pillow, the oracle's network input against torchvision's transform
chain, the oracle against the golden written from the unmodified reference ``PerceptualLoss`` (tests/golden/lpips.npz,
oracle/gen_golden_lpips.py), weight loading, op validation and launch counts, and the ``evaluate_tasks`` plumbing
with the oracle standing in for the GPU."""
import numpy as np
import PIL.Image
import pytest
import torch

from common import golden
from mcvd_b200 import configs, lib, lpips as LP, runner
from oracle import lpips_oracle as LO, tasks_oracle as T
from test_tasks_cpu import cpu_metrics, recording_sampler


def apply_table(table: np.ndarray, u8: np.ndarray) -> np.ndarray:
    """The kernel's two-pass fixed-point resize of one [S, S] uint8 plane, with the host table, in numpy."""
    M = np.zeros((table.shape[0], u8.shape[1]), dtype=np.int64)
    for o, row in enumerate(table):
        M[o, row[0]:row[0] + row[1]] = row[2:2 + row[1]]
    clip8 = lambda v: np.where(v >= 1 << 30, 255, np.where(v <= 0, 0, v >> 22))
    h = clip8(u8.astype(np.int64) @ M.T + (1 << 21))
    return clip8(M @ h + (1 << 21)).astype(np.uint8)


@pytest.mark.parametrize("S", [16, 32, 48, 64, 96, 128, 256])
def test_host_resize_tables_equal_pil(S):
    rng = np.random.default_rng(S)
    table = LP.pil_bilinear_table(S)
    assert table.shape[0] == 128 and table.dtype == np.int32
    for u8 in (rng.integers(0, 256, (S, S), dtype=np.uint8), (rng.random((S, S)) > 0.7).astype(np.uint8) * 255,
               np.full((S, S), 255, np.uint8)):
        want = np.asarray(PIL.Image.fromarray(u8).resize((128, 128), PIL.Image.BILINEAR))
        assert np.array_equal(apply_table(table, u8), want)
        assert np.array_equal(LO.pil_resize(u8), want)


def torchvision_input(frame: torch.Tensor) -> torch.Tensor:
    """The reference loop's transform chain for one [C, S, S] frame, then PNetLin's ScalingLayer."""
    import torchvision.transforms as Tr
    T2 = Tr.Compose([Tr.Resize((128, 128)), Tr.ToTensor(), Tr.Normalize(mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))])
    x = T2(Tr.ToPILImage()(frame).convert("RGB"))
    shift = torch.Tensor([-.030, -.088, -.188])[:, None, None]
    scale = torch.Tensor([.458, .448, .450])[:, None, None]
    return (x - shift) / scale


def quantisation_edges(shape, seed=0):
    """[0, 1] values at k/255 and one ulp either side, where trunc(x * 255) changes."""
    k = np.random.default_rng(seed).integers(0, 256, shape).astype(np.float32) / np.float32(255)
    d = np.random.default_rng(seed + 1).integers(-1, 2, shape)
    return np.clip(np.where(d < 0, np.nextafter(k, np.float32(0)), np.where(d > 0, np.nextafter(k, np.float32(1)), k)),
                   0, 1).astype(np.float32)


@pytest.mark.parametrize("C,S", [(1, 32), (3, 64), (1, 128), (3, 128), (1, 48)])
def test_oracle_network_input_is_torchvision_bit_for_bit(C, S):
    for frame in (quantisation_edges((C, S, S), S), np.random.default_rng(C).random((C, S, S)).astype(np.float32)):
        want = torchvision_input(torch.from_numpy(frame)).numpy()
        got = LO.network_input(frame)
        assert got.dtype == np.float32 and np.array_equal(got, want)


def test_oracle_matches_reference_golden():
    """fp64 oracle vs the fp32 reference: 1e-6 relative, plus 1e-9 absolute for the fp32 rounding of the
    reference's own sums at the smallest distances (~1e-4)."""
    g = golden("lpips")
    sd = LO.synthetic_weights()
    seen = []
    for name in LO.golden_cases():
        C = int(g[f"{name}_channels"])
        d = LO.lpips(g[f"{name}_pred"], g[f"{name}_real"], C, sd)
        ref = g[f"{name}_frame"]
        assert d.shape == ref.shape
        assert np.all(np.abs(d - ref) <= 1e-6 * ref + 1e-9), (name, np.abs(d - ref).max())
        assert np.allclose(d.mean(1), g[f"{name}_clip"], rtol=1e-6, atol=1e-9)
        seen.append(ref)
    seen = np.concatenate([s.ravel() for s in seen])
    assert seen.min() < 2e-4 and seen.max() > 0.15


def test_both_weight_formats_pack_identically(tmp_path):
    sd = LO.synthetic_weights()
    tv, lin = LO.torchvision_format(sd)
    torch.save(tv, tmp_path / "alexnet.pth")
    torch.save(lin, tmp_path / "alex.pth")
    a = LP.pack_weights(sd)
    b = LP.pack_weights(str(tmp_path / "alexnet.pth"), str(tmp_path / "alex.pth"))
    assert len(a) == len(b) == 5
    for (wa, ba, la), (wb, bb, lb), (_, cin, cout, k, *_r) in zip(a, b, LP.LAYERS):
        assert torch.equal(wa, wb) and torch.equal(ba, bb) and torch.equal(la, lb)
        cin4 = -(-cin // 4) * 4
        assert wa.shape == (k * k * cin4, cout) and ba.shape == la.shape == (cout,)
    # layout: w[(ky * k + kx) * Cin4 + c, o] = weight[o, c, ky, kx]; the padded input channel has zero weights
    w = sd["net.slice1.0.weight"]
    assert float(a[0][0][(2 * 11 + 7) * 4 + 1, 5]) == float(w[5, 1, 2, 7])
    assert not bool(a[0][0].reshape(121, 4, 64)[:, 3].any())


def test_bad_weight_files_raise(tmp_path):
    sd = LO.synthetic_weights()
    tv, lin = LO.torchvision_format(sd)
    with pytest.raises(ValueError, match="features.6.weight"):
        LP.pack_weights({k: v for k, v in tv.items() if k != "features.6.weight"}, lin)
    with pytest.raises(ValueError, match="features.3.bias"):
        LP.pack_weights(dict(tv, **{"features.3.bias": torch.zeros(191)}), lin)
    with pytest.raises(ValueError, match="lin4.model.1.weight"):
        LP.pack_weights(tv, {k: v for k, v in lin.items() if k != "lin4.model.1.weight"})
    with pytest.raises(ValueError, match="net.slice2.3.weight"):
        LP.pack_weights(dict(sd, **{"net.slice2.3.weight": torch.zeros(192, 64, 3, 3)}))
    with pytest.raises(ValueError, match="lin weights"):
        LP.pack_weights(tv)
    with pytest.raises(ValueError, match="do not pass lin"):
        LP.pack_weights(sd, lin)
    (tmp_path / "junk.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="cannot read"):
        LP.pack_weights(str(tmp_path / "junk.pth"), lin)
    with pytest.raises(ValueError, match="max_chunk_frames"):
        LP.LPIPS(sd, device="cpu", max_chunk_frames=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        LP.LPIPS(sd, device="cpu")(torch.zeros(1, 1, 32, 32), torch.zeros(1, 1, 32, 32), 1)


def chunk_ops(n, S=64, C=1):
    net = LP.LPIPS(LO.synthetic_weights(), device="cpu")
    pred, real = torch.zeros(n, C, S, S), torch.zeros(n, C, S, S)
    out = torch.zeros(n, dtype=torch.float64)
    ws = torch.zeros(2 * n * (LP._WS_A + LP._WS_B))
    return net.program(pred, real, C, out, ws), (pred, real, out, ws, net)


@pytest.mark.parametrize("n", [1, 2, 37, 256])
def test_chunk_program_validates_and_costs_a_fixed_number_of_launches(n):
    ops, keep = chunk_ops(n)
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    assert lib.load().mcvd_count_launches(arr, len(ops)) == len(ops) == 11
    assert [o.kind for o in ops] == [lib.OP_LPIPS_PREP] + [lib.OP_CONV_RELU, lib.OP_LPIPS_LAYER] * 5
    assert [(o.H, o.Cout) for o in ops[1::2]] == [(31, 64), (15, 192), (7, 384), (7, 256), (7, 256)]


def test_validate_program_rejects_bad_lpips_ops():
    ops, keep = chunk_ops(2)
    prep, conv, layer = ops[0], ops[3], ops[2]            # conv2 reads the pooled relu1

    def rejects(op, match):
        with pytest.raises(RuntimeError, match=match):
            lib.validate_program(lib.make_ops([op]), 1)

    def edit(op, **kw):
        o = lib.McvdOp.from_buffer_copy(op)
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    rejects(edit(prep, w=None), "resize table")
    rejects(edit(prep, src1=None), "real frames")
    rejects(edit(prep, C0=2), "channels per frame")
    rejects(edit(prep, C0=4), "channels per frame")
    rejects(edit(prep, H=64, W=64), "128x128")
    rejects(edit(prep, W=127), "128x128")
    rejects(edit(conv, w=None), "null weights")
    rejects(edit(conv, bias=None), "null weights")
    rejects(edit(conv, H=14, W=14), "geometry")             # pool 31 -> 15, 5x5 pad 2 -> 15
    rejects(edit(conv, i3=30, i4=30), "geometry")           # pool 30 -> 14
    rejects(edit(conv, flags=0), "geometry")                # without the pool the 31x31 input gives 31x31
    rejects(edit(conv, i0=3), "geometry")
    rejects(edit(conv, C0=6), "multiple of 4")
    rejects(edit(conv, Cout=96), "multiple of 64")
    rejects(edit(conv, i1=0), "stride")
    rejects(edit(layer, w=None), "lin weights")
    rejects(edit(layer, src1=None), "real features")
    lib.validate_program(lib.make_ops([prep, conv, layer]), 3)


def test_header_and_binding_agree_on_lpips_surface():
    import os
    import re
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                            "mcvd_b200.h")).read()
    for name, val in (("LPIPS_PREP", 19), ("CONV_RELU", 20), ("LPIPS_LAYER", 21)):
        assert int(re.search(rf"MCVD_OP_{name}\s*=\s*(\d+)", hdr).group(1)) == getattr(lib, f"OP_{name}") == val
    assert int(re.search(r"#define MCVD_F_POOL\s+\(1 << (\d+)\)", hdr).group(1)) == 9 and lib.F_POOL == 1 << 9
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.load().mcvd_abi_version() == 5


def oracle_lpips(calls):
    sd = LO.synthetic_weights()

    def fn(pred, real, channels):
        calls.append((tuple(pred.shape), channels))
        return torch.from_numpy(LO.lpips(pred.numpy(), real.numpy(), channels, sd))
    return fn


def test_evaluate_tasks_lpips_reduction_and_keys(monkeypatch):
    cfg = configs.workload("tiny_general")
    C, F = cfg.data.channels, cfg.data.num_frames
    X = T.golden_clips(cfg, batch=2)
    monkeypatch.setattr(runner, "frame_metrics", cpu_metrics)
    kw = dict(preds_per_test=2, philox_seed=99, init_seed=7)
    plain = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, sampler=recording_sampler([]), **kw)
    calls = []
    out = runner.evaluate_tasks(cfg, torch.nn.Linear(1, 1), X, lpips=oracle_lpips(calls),
                                sampler=recording_sampler([]), **kw)
    assert list(out) == list(plain) == ["interp", "pred", "gen"]
    assert calls == [((4, C * F, 32, 32), C), ((4, C * 5, 32, 32), C)]
    for task, (frames, m) in out.items():
        frames0, m0 = plain[task]
        assert torch.equal(frames, frames0)
        if task == "gen":
            assert m is None and m0 is None
            continue
        assert sorted(m0) == ["mse", "per_frame", "psnr", "ssim"]
        assert sorted(m) == sorted(list(m0) + ["lpips", "per_frame_lpips"])
        for k in m0:
            assert torch.equal(m[k], m0[k]), k
        pf = m["per_frame_lpips"]
        assert pf.shape == (4, frames.shape[1] // C) and pf.dtype == torch.float64
        want = LO.clip_lpips(pf.numpy(), 2)
        assert m["lpips"].shape == (2,) and np.array_equal(m["lpips"].numpy(), want)
    # evaluate_clips passes it on to task (1)
    frames, m = runner.evaluate_clips(cfg, torch.nn.Linear(1, 1), X, lpips=oracle_lpips([]),
                                      sampler=recording_sampler([]), **kw)
    assert torch.equal(m["per_frame_lpips"], out["interp"][1]["per_frame_lpips"])
