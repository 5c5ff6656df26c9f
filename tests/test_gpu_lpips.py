"""LPIPS on the H100 (mcvd_b200/lpips.py, MCVD_OP_LPIPS_PREP / CONV_RELU / LPIPS_LAYER) against the golden written
from the unmodified reference ``PerceptualLoss`` (tests/golden/lpips.npz) and the fp64 oracle.

Tolerances: the network input is bit-exact (integer resize, fp32 normalisation in torchvision's order); each
convolution is within 1e-5 of its output's scale of an fp64 torch evaluation of the same input (fp32 FFMA
accumulation); per-frame distances are within 1e-5 + 1e-4 d of the golden and of the oracle."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from common import golden, make_module
from mcvd_b200 import lib, lpips as LP, runner
from oracle import lpips_oracle as LO, tasks_oracle as T
from test_lpips_cpu import quantisation_edges

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def net():
    return LP.LPIPS(LO.synthetic_weights(), device=DEV)


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def chunk(net, pred, real, C):
    """(network input [2n, 128, 128, 4], the five taps [2n, H, W, Cout] each, per-pair distances) of one chunk,
    with every tap kept (the product ping-pongs two buffers)."""
    n = pred.shape[0]
    ws = torch.zeros(2 * n * (LP._WS_A + LP._WS_B), device=DEV)
    out = torch.empty(n, dtype=torch.float64, device=DEV)
    ops = net.program(pred, real, C, out, ws)
    taps = [torch.empty(2 * n, o.H, o.W, o.Cout, device=DEV) for o in ops[1::2]]
    inp = torch.empty(2 * n, 128, 128, 4, device=DEV)
    ops[0].dst = inp.data_ptr()
    prev = inp
    for i, t in enumerate(taps):
        conv, layer = ops[1 + 2 * i], ops[2 + 2 * i]
        conv.src0, conv.dst = prev.data_ptr(), t.data_ptr()
        layer.src0, layer.src1 = t.data_ptr(), t[n:].data_ptr()
        prev = t
    run(ops)
    return inp, taps, out


@pytest.mark.parametrize("C,S", [(1, 32), (3, 64), (1, 128), (3, 128), (1, 48), (3, 256)])
def test_prep_is_the_torchvision_input_bit_for_bit(net, C, S):
    B, F = 2, 2
    pred = torch.from_numpy(quantisation_edges((B, C * F, S, S), S))
    real = torch.from_numpy(np.random.default_rng(S).random((B, C * F, S, S)).astype(np.float32) * 1.2 - 0.1)
    dst = torch.full((2 * B * F, 128, 128, 4), float("nan"), device=DEV)
    tab = net._table(S)
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W, op.C0, op.i0, op.i1, op.i2 = lib.OP_LPIPS_PREP, B, 128, 128, C, F, S, tab.shape[1] - 2
    p, r = pred.to(DEV), real.to(DEV)
    op.src0, op.src1, op.w, op.dst = p.data_ptr(), r.data_ptr(), tab.data_ptr(), dst.data_ptr()
    run([op])
    got = dst.cpu()
    assert not bool(got[..., 3].any())
    for i, src in enumerate((pred, real)):
        for b in range(B):
            for f in range(F):
                want = LO.network_input(src[b, f * C:(f + 1) * C].numpy())
                img = got[(i * B + b) * F + f, ..., :3].permute(2, 0, 1).numpy()
                assert np.array_equal(img, want), (i, b, f)


def test_each_conv_layer_matches_fp64(net):
    """Each layer from the kernel's own input: the error of one layer, not accumulated through the network."""
    g = golden("lpips")
    pred, real = (torch.from_numpy(g[f"rgb64_{k}"]).reshape(2, 3, 64, 64).to(DEV) for k in ("pred", "real"))
    inp, taps, _ = chunk(net, pred, real, 3)
    sd = LO.synthetic_weights()
    x = inp[..., :3].permute(0, 3, 1, 2)
    for i, (key, _, _, _, stride, pad, pool) in enumerate(LO.CONVS):
        h = x.double()
        if pool:
            h = Fn.max_pool2d(h, 3, 2)
        want = torch.relu(Fn.conv2d(h, sd[key + ".weight"].double().to(DEV), sd[key + ".bias"].double().to(DEV),
                                    stride=stride, padding=pad))
        got = taps[i].permute(0, 3, 1, 2).double()
        scale = float(want.abs().max())
        assert got.shape == want.shape and scale > 0
        assert float((got - want).abs().max()) <= 1e-5 * scale, (key, float((got - want).abs().max()), scale)
        x = taps[i].permute(0, 3, 1, 2)


def test_lpips_matches_golden_and_oracle(net):
    g = golden("lpips")
    sd = LO.synthetic_weights()
    for name in LO.golden_cases():
        C = int(g[f"{name}_channels"])
        pred, real = g[f"{name}_pred"], g[f"{name}_real"]
        d = net(torch.from_numpy(pred).to(DEV), torch.from_numpy(real).to(DEV), C)
        assert d.shape == g[f"{name}_frame"].shape and d.dtype == torch.float64
        d = d.cpu().numpy()
        for want in (g[f"{name}_frame"], LO.lpips(pred, real, C, sd)):
            assert np.all(np.abs(d - want) <= 1e-5 + 1e-4 * want), (name, d, want)


def test_identity_and_symmetry_are_exact(net):
    g = golden("lpips")
    a, b = (torch.from_numpy(g[f"rgb64_{k}"]).to(DEV) for k in ("pred", "real"))
    assert bool((net(a, a, 3) == 0).all()) and bool((net(b, b, 3) == 0).all())
    ab, ba = net(a, b, 3), net(b, a, 3)
    assert bool((ab > 0).all()) and torch.equal(ab, ba)


def pairs(n, S=64, C=1, seed=0):
    rng = np.random.default_rng(seed)
    real = rng.random((n, C, S, S)).astype(np.float32)
    pred = np.clip(real + 0.2 * rng.standard_normal(real.shape), 0, 1).astype(np.float32)
    return torch.from_numpy(pred).to(DEV), torch.from_numpy(real).to(DEV)


def test_batch_and_chunking_do_not_change_a_frame(net):
    small = LP.LPIPS(LO.synthetic_weights(), device=DEV, max_chunk_frames=5)
    pred, real = pairs(37)
    full = small(pred, real, 1)
    assert full.shape == (37, 1)
    assert torch.equal(full, net(pred, real, 1))
    for i in (0, 4, 5, 36):
        assert torch.equal(small(pred[i:i + 1], real[i:i + 1], 1), full[i:i + 1])
    # [B, C*F] clips: frame f of clip b is pair b*F + f
    clips = small(pred.reshape(1, 37, 64, 64), real.reshape(1, 37, 64, 64), 1)
    assert torch.equal(clips.reshape(37, 1), full)


def test_300_pairs_across_chunks_with_fixed_launches(net, monkeypatch):
    pred, real = pairs(300, S=32, seed=1)
    chunked = LP.LPIPS(LO.synthetic_weights(), device=DEV, max_chunk_frames=64)
    programs = []
    real_run = lib.run_program

    def counting(arr, n, stream):
        programs.append(lib.load().mcvd_count_launches(arr, n))
        real_run(arr, n, stream)
    monkeypatch.setattr(lib, "run_program", counting)
    d = chunked(pred.reshape(30, 10, 32, 32), real.reshape(30, 10, 32, 32), 1)
    assert programs == [11] * 5                               # 64, 64, 64, 64, 44 pairs
    monkeypatch.setattr(lib, "run_program", real_run)
    assert d.shape == (30, 10) and torch.equal(d.reshape(300, 1), net(pred, real, 1))
    sd = LO.synthetic_weights()
    for i in (0, 63, 64, 255, 256, 299):
        want = LO.lpips(pred[i:i + 1].cpu().numpy(), real[i:i + 1].cpu().numpy(), 1, sd)[0, 0]
        assert abs(float(d.reshape(-1)[i]) - want) <= 1e-5 + 1e-4 * want, i


def test_evaluate_tasks_with_lpips_on_gpu(net):
    cfg, model, _ = make_module("tiny_general", DEV)
    X = T.golden_clips(cfg, batch=2).to(DEV)
    kw = dict(preds_per_test=2, philox_seed=5, init_seed=6)
    plain = runner.evaluate_tasks(cfg, model, X, **kw)
    out = runner.evaluate_tasks(cfg, model, X, lpips=net, **kw)
    C = cfg.data.channels
    assert list(out) == list(plain)
    for task, (frames, m) in out.items():
        frames0, m0 = plain[task]
        assert torch.equal(frames, frames0)
        if m0 is None:
            assert m is None
            continue
        assert set(m) == set(m0) | {"lpips", "per_frame_lpips"}
        for k in m0:
            assert torch.equal(m[k], m0[k]), (task, k)
        real, _, _ = runner.task_inputs(cfg, X.repeat_interleave(2, dim=0), task)
        direct = net(frames, real.to(DEV), C)
        assert m["per_frame_lpips"].shape == (4, frames.shape[1] // C)
        assert torch.equal(m["per_frame_lpips"], direct)
        assert torch.equal(m["lpips"], direct.mean(1).reshape(2, 2).min(-1).values)
    frames, m = runner.evaluate_clips(cfg, model, X, lpips=net, **kw)
    assert torch.equal(m["lpips"], out["interp"][1]["lpips"])
