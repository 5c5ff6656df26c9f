"""The op-by-op replay harness (tests/program_replay.py) on the CPU: an fp32 interpreter engine stands in for the
CUDA one and is replayed against the float64 twin.  Checks the program pairing and pointer map without a GPU, and that
a plain fp32 implementation of every op kind stays inside the replay's bounds."""
import pytest
import torch

from common import make_module
from mcvd_b200 import configs, detfill, lib
from mcvd_b200.program import Engine
from op_interpreter import Interpreter, tile_stats
from program_replay import HarnessError, Replay, replay_program, twin_engine


def cpu_pair(name, conv_mode, epilogue_stats=False, precision="fp32"):
    cfg = configs.workload(name)
    cfg.model.conv_precision = precision
    cfg, net, _ = make_module(cfg, "cpu")
    real = Engine(net, _test_backend=Interpreter(half=precision == "fp16"))
    real.conv_mode, real.epilogue_stats = conv_mode, epilogue_stats
    return cfg, net, real, twin_engine(real, net)


@pytest.mark.parametrize("name,conv_mode,stats", [("tiny", "umma", False), ("tiny", "umma2", True),
                                                  ("tiny", "simt", False), ("tiny_spade", "umma", True),
                                                  ("tiny_rgb", "umma", False)])
@pytest.mark.parametrize("per_clip_t", [False, True])
def test_fp32_interpreter_replays_within_bounds(name, conv_mode, stats, per_clip_t):
    cfg, net, real, twin = cpu_pair(name, conv_mode, stats)
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    t = torch.linspace(20.0, 900.0, B) if per_clip_t else 321.0
    R = replay_program(real, twin, B, x, cond, t, detfill.normal("replay_z", x.shape))
    assert not R.failures, "\n".join(R.failures[:10])
    assert R.whole_program_identical
    kinds = {k.split(".")[0] for k in R.stats}
    assert "GN_FINALIZE" in kinds and "DIFFUSION_UPDATE" in kinds and "NHWC_TO_NCHW" in kinds
    assert ("CONV_SIMT" if conv_mode == "simt" else "CONV_" + conv_mode.upper()) in kinds
    if stats:
        assert R.stats[("CONV_" + conv_mode.upper()) + ".dst2"][0] > 0
    if name == "tiny_spade":
        assert "RESIZE_NEAREST" in kinds
    # the fp32 arithmetic leaves visible error somewhere: the bounds are not vacuous comparisons of equal numbers
    assert max(w for k, (n, w) in R.stats.items() if k.startswith("CONV")) > 0


def test_pairing_rejects_mismatched_programs():
    cfg, net, real, twin = cpu_pair("tiny", "umma")
    twin.fuse_shortcut = "0"                     # another lowering: one more op per channel-changing ResBlock
    B = cfg.bench_batch
    P, Q = real.program(B), twin.program(B)
    with pytest.raises(HarnessError):
        Replay(real, P, twin, Q).pair("step", P.step_ops, Q.step_ops)
    cfg, net, real, twin = cpu_pair("tiny", "umma")
    P, Q = real.program(B), twin.program(B)
    R = Replay(real, P, twin, Q)
    R.pair("step", P.step_ops, Q.step_ops)
    Q.step_ops[5].dst = Q.step_ops[6].dst        # one real buffer would map to two twin buffers
    with pytest.raises(HarnessError):
        Replay(real, P, twin, Q).pair("step", P.step_ops, Q.step_ops)


def test_replay_flags_a_wrong_op():
    """a kernel that is subtly wrong -- here the real engine's weights of one conv scaled by 1 + 2^-10, about the
    error of dropping one of the fp16 hi/lo partial products -- is reported on that op and no other"""
    cfg, net, real, twin = cpu_pair("tiny", "umma")
    B = cfg.bench_batch
    P = real.program(B)
    i = next(j for j, o in enumerate(P.step_ops) if o.kind == lib.OP_CONV_UMMA and o.i0 == 3 and j > 10)
    real.backend.tensors[P.step_ops[i].w].mul_(1 + 2.0 ** -10)
    x, cond = detfill.synthetic_inputs(cfg, B)
    R = replay_program(real, twin, B, x, cond, 500.0, detfill.normal("replay_z", x.shape))
    assert R.failures and all(f.startswith(f"step[{i}] CONV_UMMA") for f in R.failures), R.failures[:3]


def test_epilogue_statistics_range_is_enforced():
    y = torch.zeros(2, 8, 8, 16)
    tile_stats(y + 4096.0, 3)
    for bad in (4096.5, -5000.0, float("nan")):
        y[1, 3, 4, 5] = bad
        with pytest.raises(ValueError):
            tile_stats(y, 3)


@pytest.mark.parametrize("name,conv_mode,stats", [("tiny", "umma", False), ("tiny_spade", "umma", False),
                                                  ("tiny", "umma2", True)])
def test_half_emulation_replays_within_the_one_product_bound(name, conv_mode, stats):
    """the interpreter's fp16 emulation of MCVD_F_HALF convs (operands rounded once to fp16) replayed against the
    float64 twin: inside the one-product bound, statistics exact"""
    cfg, net, real, twin = cpu_pair(name, conv_mode, stats, precision="fp16")
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    R = replay_program(real, twin, B, x, cond, 321.0, detfill.normal("replay_z", x.shape))
    assert not R.failures, "\n".join(R.failures[:10])
    assert R.n_half > 0
    if stats:
        assert R.stats["CONV_UMMA2.dst2"][0] > 0
    # the half rounding is visible: a worst ratio far above the default mode's TAU_MATMUL-sized errors
    assert max(w for k, (n, w) in R.stats.items() if k.startswith("CONV_UMMA")) > 0.01, R.table()


def test_replay_flags_a_wrong_half_op():
    """one half-mode conv whose weights are scaled by 1 + 2^-4 is reported on that op and no other"""
    cfg, net, real, twin = cpu_pair("tiny", "umma", precision="fp16")
    B = cfg.bench_batch
    P = real.program(B)
    i = next(j for j, o in enumerate(P.step_ops) if o.kind == lib.OP_CONV_UMMA and o.flags & lib.F_HALF and j > 10)
    real.backend.tensors[P.step_ops[i].w].mul_(1 + 2.0 ** -4)
    x, cond = detfill.synthetic_inputs(cfg, B)
    R = replay_program(real, twin, B, x, cond, 500.0, detfill.normal("replay_z", x.shape))
    assert R.failures and all(f.startswith(f"step[{i}] CONV_UMMA") for f in R.failures), R.failures[:3]
