"""Head dims 256 and 288 (the Cityscapes SPADE and UCF-101 recipes, n_head_channels = 256 / 288) on the host: the
lowering sends them to the tensor-core attention, the op interpreter matches the oracle, the support check names
head dims no kernel runs, and the float64 emulation of the split arithmetic stays inside (and a dropped cross
product outside) the attention bound at these widths."""
import pytest
import torch

from common import make_module, max_err
from mcvd_b200 import arch, configs, detfill, lib
from mcvd_b200.program import Engine
from op_interpreter import Interpreter
from oracle import mcvd_oracle as O
from test_value_ranges_cpu import (ATTN_FAMILIES, ATTN_PRODUCTS, attention_bound, attention_qkv, emulate_attention,
                                   worst_ratio)


def wide_config(ngf, ch_mult, nhc, attn=(16,)):
    """the 32x32 tiny test net with wider levels: its attention blocks at 16x16 get heads of nhc channels"""
    cfg = configs.workload("tiny")
    cfg.model.ngf, cfg.model.ch_mult, cfg.model.n_head_channels = ngf, list(ch_mult), nhc
    cfg.model.attn_resolutions = list(attn)
    return cfg


def attention_dims(cfg):
    spec = arch.build_spec(cfg)
    return [(ms.res * ms.res, ms.in_ch // ms.heads) for ms in spec.mods if ms.kind == "attn"]


def test_key_tiles_come_from_the_kernels():
    K = lambda kind, T, d: lib.load().mcvd_attention_key_tile(kind, T, d)
    for d in (256, 288):
        for T in (64, 256, 1024):
            assert K(lib.OP_ATTENTION_UMMA, T, d) == 32
        assert K(lib.OP_ATTENTION_UMMA, 16, d) == 0                 # 16 tokens: no key tile the kernel is built for
    assert K(lib.OP_ATTENTION_UMMA, 4096, 96) == 128 and K(lib.OP_ATTENTION_UMMA, 256, 128) == 64
    assert K(lib.OP_ATTENTION_UMMA, 1024, 384) == 0 and K(lib.OP_ATTENTION_UMMA, 1024, 16) == 0
    assert K(lib.OP_ATTENTION, 1024, 256) > 0 and K(lib.OP_ATTENTION, 16, 16) > 0
    assert K(lib.OP_ATTENTION, 1024, 288) == 0                     # no CUDA-core kernel at 288
    assert K(lib.OP_CONV_UMMA, 1024, 64) == 0
    assert lib.attention_kind(1024, 288) == lib.OP_ATTENTION_UMMA
    assert lib.attention_kind(1024, 256, "simt") == lib.OP_ATTENTION
    assert lib.attention_kind(16, 288) is None and lib.attention_kind(1024, 288, "simt") is None
    assert lib.attention_kind(16, 256) == lib.OP_ATTENTION                 # too few tokens for the tensor cores


@pytest.mark.parametrize("ngf,ch_mult,nhc,d", [(96, (1, 3), 288, 288), (128, (1, 2), 256, 256)])
def test_wide_heads_lower_to_the_tensor_core_attention(ngf, ch_mult, nhc, d):
    cfg = wide_config(ngf, ch_mult, nhc)
    assert arch.check_supported(cfg) is None
    assert {dd for _, dd in attention_dims(cfg)} == {d}
    cfg, net, sd = make_module(cfg, "cpu")
    eng = Engine(net, _test_backend=Interpreter())
    net._engine = eng
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    for t in (37, 990):
        tt = torch.full((B,), t, dtype=torch.long)
        assert max_err(net(x, tt, cond=cond), O.unet_forward(cfg, sd, x, tt, cond)) < 5e-5
    P = eng.program(B)
    att = [op for op in P.step_ops if op.kind in (lib.OP_ATTENTION, lib.OP_ATTENTION_UMMA)]
    assert att and all(op.kind == lib.OP_ATTENTION_UMMA and op.i1 == d for op in att)
    lib.validate_program(P.step_arr, len(P.step_ops))
    assert lib.load().mcvd_count_launches(P.step_arr, len(P.step_ops)) == P.step_launches == len(P.step_ops) + len(att)


def test_cuda_core_attention_at_288_fails_when_the_program_is_built():
    cfg, net, _ = make_module(wide_config(96, (1, 3), 288), "cpu")
    eng = Engine(net, _test_backend=Interpreter())
    eng.attn_mode = "simt"
    with pytest.raises(ValueError, match="head dim 288"):
        eng.program(cfg.bench_batch)


def test_check_supported_names_a_head_dim_no_kernel_runs():
    cfg = wide_config(96, (1, 4), -1)                # n_head_channels = -1: one 384-channel head at 16x16
    why = arch.check_supported(cfg)
    assert why is not None and "head dim 384" in why, why
    cfg = wide_config(96, (1, 1, 3), 288)
    cfg.data.image_size = 16                         # the middle block's 288-channel head over 4x4 = 16 tokens
    why = arch.check_supported(cfg)
    assert why is not None and "head dim 288" in why and "4x4" in why, why


@pytest.mark.parametrize("name,d", [("cfg6", 288), ("cfg7", 256)])
def test_published_wide_recipes_need_only_supported_head_dims(name, d):
    cfg = configs.workload(name)
    assert name in configs.ALL_WORKLOADS and arch.check_supported(cfg) is None
    dims = attention_dims(cfg)
    assert {dd for _, dd in dims} == {d} and {T for T, _ in dims} == {64, 256, 1024}
    assert all(lib.attention_kind(T, dd) == lib.OP_ATTENTION_UMMA for T, dd in dims)


@pytest.mark.parametrize("T,d,heads", [(64, 256, 1), (64, 288, 2)])
def test_emulated_split_meets_the_attention_bound_at_wide_heads(T, d, heads):
    for fam in ATTN_FAMILIES:
        qkv, scale = attention_qkv(fam, 2, T, heads, d)
        ref, bound = attention_bound(qkv, heads, d, scale)
        assert worst_ratio(emulate_attention(qkv, heads, d, scale), ref, bound) <= 1.0, fam
        if fam in ("unit", "logit_10", "logit_40"):
            for drop in ATTN_PRODUCTS:
                r = worst_ratio(emulate_attention(qkv, heads, d, scale, drop=drop), ref, bound)
                assert r > 1.0, (fam, drop, r)
