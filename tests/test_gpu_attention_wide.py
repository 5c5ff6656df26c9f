"""The tensor-core attention at head dims 256 and 288 on the H100 (Cityscapes SPADE and UCF-101 recipes): op parity
against float64, bit-stable outputs across batch composition and CUDA-graph replay, the trained-like value ranges of
tests/test_gpu_value_ranges.py, the op-by-op replay of the cfg6 / cfg7 forwards, a short DDPM sampler call on a
UCF-101-shaped module, and patch.install() handing the UCF-101 recipe to the native module."""
import ctypes

import pytest
import torch

from common import make_module, max_err, step_noise
from mcvd_b200 import configs, detfill, lib, samplers
from oracle import mcvd_oracle as O
from test_gpu_ops import mk, rnd, run
from test_gpu_program_replay import replay_row
from test_gpu_value_ranges import TOKENS, run_attention
from test_value_ranges_cpu import ATTN_FAMILIES, SCALE_PERTURBATION, attention_bound, attention_qkv, \
    perturbation_families, worst_ratio

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def attention_op(B, T, heads, d, qkv, out, scratch):
    side = int(T ** 0.5)
    return mk(lib.OP_ATTENTION_UMMA, B, H=side, W=side, C0=heads * d, i0=heads, i1=d, f0=float(d) ** -0.5, src0=qkv,
              dst=out, dst2=scratch)


def tc_attention(qkv, heads, d):
    B, T, C3 = qkv.shape
    out = torch.full((B, T, C3 // 3), float("nan"), device=DEV)
    scratch = torch.empty(lib.attention_scratch_bytes(B, T, C3 // 3), dtype=torch.uint8, device=DEV)
    run([attention_op(B, T, heads, d, qkv, out, scratch)])
    return out


# T = 64: one partial 128-row query tile; 256 / 1024: 2 / 8 query-tile CTAs per head
@pytest.mark.parametrize("B,T,heads", [(3, 64, 2), (2, 256, 3), (1, 1024, 2)])
@pytest.mark.parametrize("d", [256, 288])
def test_wide_attention_matches_float64(B, T, heads, d):
    C = heads * d
    qkv = rnd(B, T, 3 * C, seed=4)
    scale = float(d) ** -0.5
    q, k, v = qkv.view(B, T, 3, heads, d).unbind(2)
    s = torch.einsum("bthd,bshd->bhts", q.double(), k.double()) * scale
    ref = torch.einsum("bhts,bshd->bthd", torch.softmax(s, -1), v.double()).reshape(B, T, C).float()
    qd = qkv.to(DEV)
    out = torch.zeros(B, T, C, device=DEV)
    scratch = torch.empty(lib.attention_scratch_bytes(B, T, C), dtype=torch.uint8, device=DEV)
    assert scratch.numel() == 4 * B * C * (-(-T // 128) * 128 + 2 * T)
    op = attention_op(B, T, heads, d, qd, out, scratch)
    assert lib.load().mcvd_count_launches(ctypes.byref(op), 1) == 2        # pre-split + attention
    run([op])
    assert (out.cpu() - ref).abs().max().item() < 2e-5


@pytest.mark.parametrize("T,heads,d", [(256, 3, 288), (1024, 2, 256)])
def test_wide_attention_bits_do_not_depend_on_the_batch_or_graph_replay(T, heads, d):
    B = 3
    qkv = rnd(B, T, 3 * heads * d, seed=9).to(DEV)
    full = tc_attention(qkv, heads, d)
    for i in range(B):                                     # each clip alone
        assert torch.equal(tc_attention(qkv[i:i + 1].contiguous(), heads, d)[0], full[i])
    rev = tc_attention(qkv.flip(0).contiguous(), heads, d)   # clips at other positions
    assert torch.equal(rev.flip(0), full)
    out = torch.full_like(full, float("nan"))
    scratch = torch.empty(lib.attention_scratch_bytes(B, T, heads * d), dtype=torch.uint8, device=DEV)
    arr = lib.make_ops([attention_op(B, T, heads, d, qkv, out, scratch)])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        lib.run_program(arr, 1, s.cuda_stream)                   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        lib.run_program(arr, 1, torch.cuda.current_stream().cuda_stream)
    out.fill_(float("nan"))
    for _ in range(2):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, full)


@pytest.mark.parametrize("kind,d", [("umma", 256), ("umma", 288), ("simt", 256)])
@pytest.mark.parametrize("T", sorted(TOKENS))
def test_wide_attention_value_ranges(kind, T, d):
    B, heads = TOKENS[T]
    report = []
    for fam in ATTN_FAMILIES:
        qkv, scale = attention_qkv(fam, B, T, heads, d)
        qkv = qkv.to(DEV)
        ref, bound = attention_bound(qkv, heads, d, scale, tensor_core=kind == "umma")
        report.append(f"{fam} {worst_ratio(run_attention(kind, qkv, heads, d, scale), ref, bound):.3g}")
        if kind == "umma" and fam in perturbation_families(d):
            off = run_attention(kind, qkv, heads, d, scale * (1 + SCALE_PERTURBATION))
            assert worst_ratio(off, ref, bound) > 1.0, (fam, "a perturbed logit scale stays inside the bound")
    print(f"\n{kind} T={T} d={d}: worst err/bound " + ", ".join(report))
    assert all(float(r.split()[1]) <= 1.0 for r in report), report


@pytest.mark.parametrize("name", ["cfg6", "cfg7"])
def test_wide_recipe_program_replay(name, monkeypatch):
    """the full-width cfg6 / cfg7 forward, op by op against the float64 twin, at 4 clips instead of the benchmark
    batch (every layer's shape, attention included, but the batch; the twin's float64 buffers of 32 or 60 clips
    would not fit beside the engine's)"""
    workload = configs.workload

    def small(n):
        cfg = workload(n)
        cfg.bench_batch = 4
        return cfg
    monkeypatch.setattr(configs, "workload", small)
    R = replay_row(name, "umma")
    assert not R.failures, f"{len(R.failures)} outputs over their bound:\n" + "\n".join(R.failures[:20])
    assert R.whole_program_identical
    kinds = {k.split(".")[0] for k in R.stats}
    assert "ATTENTION_UMMA" in kinds and "ATTENTION" not in kinds


def test_ucf101_ddpm_sampler_vs_oracle():
    """cfg6 (UCF-101, 288-channel heads) at full width, one clip, a 4-step DDPM sampler call (+ denoise) with injected
    noise against the oracle's sampler: the tolerance of the cfg2 sampler test (PSNR >= 50 dB, max |diff| < 5e-3)"""
    torch.set_num_threads(min(torch.get_num_threads(), 16))
    cfg, net, sd = make_module("cfg6", DEV)
    L = 4
    x, cond = detfill.synthetic_inputs(cfg, 1, seed=21)
    zs = step_noise(x.shape, L, tag="c6z")
    out = samplers.ddpm_sampler(x.to(DEV), net, cond=cond.to(DEV), final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, noise_list=[z.to(DEV) for z in zs])[0].cpu()
    P = net.engine().program(1)
    assert {op.kind for op in P.step_ops} & {lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA} == {lib.OP_ATTENTION_UMMA}
    fn = lambda xx, tt, cc: O.unet_forward(cfg, sd, xx, tt, cc)
    ref = O.ddpm_sample(fn, O.make_schedule(cfg), x.clone(), cond, L, True, True, noise=zs)[0]
    to01 = lambda a: ((a + 1) / 2).clamp(0, 1)
    assert O.psnr01(to01(out), to01(ref)) >= 50.0
    assert max_err(out, ref) < 5e-3


def test_patch_install_gives_the_ucf101_recipe_the_native_module(tmp_path, monkeypatch):
    """patch.install() with the stubbed reference layout of test_gpu_model.py: get_model returns the native module"""
    import importlib
    import sys
    (tmp_path / "runners").mkdir()
    (tmp_path / "models").mkdir()
    (tmp_path / "runners" / "__init__.py").write_text("")
    (tmp_path / "models" / "__init__.py").write_text(
        "def ddpm_sampler(x_mod, scorenet, **kw):\n    return 'reference ddpm'\n"
        "def ddim_sampler(x_mod, scorenet, **kw):\n    return 'reference ddim'\n"
        "def FPNDM_sampler(x_mod, scorenet, **kw):\n    return 'reference fpndm'\n")
    (tmp_path / "runners" / "ncsn_runner.py").write_text(
        "from models import ddpm_sampler, ddim_sampler, FPNDM_sampler\n"
        "def get_model(config):\n    return 'reference model'\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    for m in ("runners", "runners.ncsn_runner", "models"):
        sys.modules.pop(m, None)
    try:
        from mcvd_b200 import patch, model as fast_model
        patch.install(verbose=False)
        R = importlib.import_module("runners.ncsn_runner")
        cfg = configs.workload("cfg6")
        cfg.device = torch.device(DEV)
        net = R.get_model(cfg)
        assert isinstance(net, fast_model.UNetMore_DDPM) and next(net.parameters()).is_cuda
        cfg = configs.workload("cfg6")
        cfg.model.n_head_channels = -1                   # one 576..1152-channel head: no kernel, the reference's model
        cfg.device = torch.device(DEV)
        assert R.get_model(cfg) == "reference model"
    finally:
        for m in ("runners", "runners.ncsn_runner", "models"):
            sys.modules.pop(m, None)
