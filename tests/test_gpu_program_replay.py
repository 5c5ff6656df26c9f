"""The lowered forward of every benchmark workload, at its benchmark batch size, replayed op by op on the H100 against
a float64 twin (tests/program_replay.py): every op is run alone on the real engine's buffers and judged on its exact
inputs, so the shapes, launcher choices (n tile, tile height, input-stationary or streaming, stage counts, K-block)
and batch sizes the benchmark runs are each checked against a plain high-precision reference, and a failure names the
op.  Each row also replays the NHWC -> NCHW output op and a DDPM update (clipped x0, injected noise), and checks that
the op-by-op eps is bit-identical to one run of the whole program."""
import gc
import time

import pytest
import torch

from common import make_module
from mcvd_b200 import configs, detfill, lib
from mcvd_b200.program import Engine
from program_replay import TC_CONV_KINDS, KIND_NAME, replay_program, twin_engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def replay_row(name, mode, per_clip_t=False, split_mode=3, precision="fp32"):
    """mode: umma | umma+stats (GroupNorm partial sums from the conv epilogue) | umma2 | simt (CUDA-core convs and
    attention); precision: model.conv_precision (fp16: the nn.Conv2d layers' convs carry MCVD_F_HALF)"""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    cfg = configs.workload(name)
    cfg.model.conv_precision = precision
    cfg, net, _ = make_module(cfg, DEV)
    real = Engine(net)
    real.conv_mode = mode.split("+")[0]
    real.epilogue_stats = mode in ("umma2", "umma+stats")
    real.attn_mode = "simt" if mode == "simt" else "umma"
    real.split_mode = split_mode
    twin = twin_engine(real, net)
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    t = torch.linspace(5.0, 995.0, B) if per_clip_t else 437.0
    R = replay_program(real, twin, B, x.to(DEV), cond.to(DEV), t, detfill.normal("replay_z", x.shape).to(DEV))
    R.release()
    del real, twin, net
    gc.collect()                       # engines and interpreter registries hold each other's buffers
    torch.cuda.synchronize()
    R.wall_s = time.perf_counter() - t0
    R.peak_gb = torch.cuda.max_memory_allocated() / 2 ** 30
    torch.cuda.empty_cache()
    print(f"\n{name} B={B} {mode} {precision} {'per-clip' if per_clip_t else 'uniform'} t, split {split_mode}: {R.n_ops} ops, "
          f"{R.wall_s:.1f} s, peak {R.peak_gb:.1f} GiB, all clips\n{R.table()}")
    if R.range_max:
        print(f"  largest |x| of a statistics-writing conv output: {max(R.range_max.values()):.4g}")
    return R


ROWS = [
    ("cfg1", "umma", False, "fp32"),
    ("cfg1", "simt", False, "fp32"),
    ("cfg2", "umma", False, "fp32"),
    ("cfg2", "umma", True, "fp32"),            # per-clip t: batched LINEAR, FiLM stride film_total
    ("cfg2", "umma2", False, "fp32"),
    ("cfg2", "umma+stats", False, "fp32"),
    ("cfg3", "umma", False, "fp32"),           # SPADE cond_ops
    ("cfg4", "umma", False, "fp32"),           # head dim 192, key tile 32, 3 channels
    ("cfg5", "umma", False, "fp32"),           # 128x128 maps, one-raw-stage plans, 32x32 attention
    # model.conv_precision = fp16: the nn.Conv2d layers' convs by the one-product bound, their statistics exact
    ("cfg1", "umma", False, "fp16"),
    ("cfg2", "umma", False, "fp16"),
    ("cfg2", "umma2", False, "fp16"),
    ("cfg2", "umma+stats", False, "fp16"),
    ("cfg3", "umma", False, "fp16"),
    ("cfg4", "umma", False, "fp16"),
    ("cfg5", "umma", False, "fp16"),
]


@pytest.mark.parametrize("name,mode,per_clip_t,precision", ROWS,
                         ids=[f"{n}-{m}-{'perclip' if p else 'uniform'}" + ("" if c == "fp32" else "-" + c)
                              for n, m, p, c in ROWS])
def test_program_replay(name, mode, per_clip_t, precision):
    R = replay_row(name, mode, per_clip_t, precision=precision)
    assert not R.failures, f"{len(R.failures)} outputs over their bound:\n" + "\n".join(R.failures[:20])
    assert R.whole_program_identical, "op-by-op eps differs from one run of the whole program"
    kinds = {k.split(".")[0] for k in R.stats}
    assert {"GN_FINALIZE", "DIFFUSION_UPDATE", "NHWC_TO_NCHW"} <= kinds
    if mode == "simt":
        assert "CONV_SIMT" in kinds and "ATTENTION" in kinds and not kinds & {"CONV_UMMA", "ATTENTION_UMMA"}
    else:
        assert ("CONV_UMMA2" if mode == "umma2" else "CONV_UMMA") in kinds and "ATTENTION_UMMA" in kinds
    if mode in ("umma2", "umma+stats"):
        # every statistics-writing conv output lies inside the range the int64 statistics represent exactly
        assert R.range_max and max(R.range_max.values()) <= 4096.0
    if name == "cfg3":
        assert "RESIZE_NEAREST" in kinds
    assert (R.n_half > 0) == (precision == "fp16")


@pytest.mark.parametrize("name", ["cfg1", "cfg2"])
def test_replay_catches_a_dropped_partial_product(name):
    """split_mode 2 drops the lo(activation) * hi(weight) product of the tensor-core convs, an error of about 2^-12 of
    each product: the bounds must be tight enough to report it, on those convs only"""
    R = replay_row(name, "umma", split_mode=2)
    tc = [KIND_NAME[k] for k in TC_CONV_KINDS]
    assert max(R.stats.get(k, [0, 0.0])[1] for k in tc) > 1.0, R.table()
    assert all(f.split(":")[0].split(" ")[1].split(".")[0] in tc for f in R.failures), R.failures[:5]
    assert R.whole_program_identical
