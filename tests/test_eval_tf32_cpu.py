"""The TF32 convolutions of the FVD and FID feature networks on the CPU: the header, the Python binding and the
library agree on MCVD_OP_CONV3D_TF32 / MCVD_OP_CONV2D_TF32 and the packing entry points; the lowered I3D and
Inception programs with ``tf32=True`` validate, cost 72 and 100 launches and differ from the fp32 ones only in the conv
kinds and weight pointers; validation rejects what it rejects for the fp32 kinds, with the same reasons."""
import ctypes as C
import os
import re

import pytest
import torch

from mcvd_b200 import fid as FD, fvd as FV, lib
from oracle import i3d_oracle as IO, inception_oracle as NO

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "mcvd_b200.h")
FP32_KIND = {lib.OP_CONV3D_TF32: lib.OP_CONV3D, lib.OP_CONV2D_TF32: lib.OP_CONV2D}


def as_tf32(net, units):
    """``net`` (built on the CPU, where packing cannot run) lowered as ``tf32=True`` lowers it: the packed images are
    stand-ins of the size the library asks for, the pointers all validation looks at."""
    net.tf32 = True
    net.packed = {key: torch.zeros(lib.tf32_packed_bytes(net.weights[key][0].shape[0], cout) // 4)
                  for key, _, cout, _ in units}
    return net


def i3d_programs(n, T=10, S=32, C=1):
    net = FV.I3D(IO.synthetic_weights(), device="cpu")
    videos = torch.zeros(n, C * T, S, S)
    out = torch.zeros(n, 400, dtype=torch.float64)
    ws = torch.zeros(n * FV.workspace_floats(T))
    fp32 = net.program(videos, C, out, ws)
    tf32 = as_tf32(net, FV.units()).program(videos, C, out, ws)
    return fp32, tf32, (net, videos, out, ws)


def fid_programs(n, S=64, C=1):
    net = FD.InceptionV3(NO.synthetic_weights(), device="cpu")
    frames = torch.zeros(n, C, S, S)
    out = torch.zeros(n, 2048, dtype=torch.float64)
    ws = torch.zeros(n * FD.workspace_floats())
    fp32 = net.program(frames, out, ws)
    tf32 = as_tf32(net, FD.units()).program(frames, out, ws)
    return fp32, tf32, (net, frames, out, ws)


def fields(op):
    return {name: getattr(op, name) for name, _ in lib.McvdOp._fields_}


def test_header_binding_and_library_agree_on_the_tf32_surface():
    hdr = open(HEADER).read()
    for name, val in (("CONV3D_TF32", 34), ("CONV2D_TF32", 35)):
        assert int(re.search(rf"MCVD_OP_{name}\s*=\s*(\d+)", hdr).group(1)) == getattr(lib, f"OP_{name}") == val
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.load().mcvd_abi_version() == 5
    assert re.search(r"long long mcvd_tf32_packed_bytes\(int K, int Cout\);", hdr)
    assert re.search(r"int mcvd_tf32_pack_weights\(const float\* w_kmajor, int K, int Cout, void\* out, void\* stream\);",
                     hdr)
    so = lib.load()
    for sym in ("mcvd_tf32_packed_bytes", "mcvd_tf32_pack_weights"):
        assert sym in lib.EXPORTS and hasattr(so, sym)
    # kind 36 is unknown: the two new kinds are the last ones
    op = lib.McvdOp()
    op.kind, op.B, op.H, op.W = 36, 1, 1, 1
    with pytest.raises(RuntimeError, match="unknown kind 36"):
        lib.validate_program(lib.make_ops([op]), 1)


@pytest.mark.parametrize("K,cout", [(36, 32), (1372, 64), (64, 16), (192, 208), (2048, 448), (4, 8), (1, 8)])
def test_packed_size_covers_the_weights_in_whole_tiles(K, cout):
    n = lib.tf32_packed_bytes(K, cout)
    assert n % (32 * 4) == 0 and n >= K * cout * 4
    assert n <= (-(-K // 32) * 32) * (cout + 128) * 4            # K padded to a slab, at most one extra n tile


@pytest.mark.parametrize("K,cout", [(0, 8), (32, 0), (32, 12), (32, -8)])
def test_packing_rejects_bad_shapes(K, cout):
    assert lib.load().mcvd_tf32_packed_bytes(K, cout) < 0
    with pytest.raises(RuntimeError, match="tf32 packing"):
        lib.tf32_packed_bytes(K, cout)
    assert lib.load().mcvd_tf32_pack_weights(None, K, cout, None, None) < 0


def test_packing_rejects_null_and_misaligned_buffers():
    buf = (C.c_float * 64)()
    base = C.addressof(buf)
    assert lib.load().mcvd_tf32_pack_weights(None, 32, 8, C.c_void_p(base), None) < 0
    assert "null" in lib.last_error()
    assert lib.load().mcvd_tf32_pack_weights(C.c_void_p(base), 32, 8, C.c_void_p(base + 4), None) < 0
    assert "aligned" in lib.last_error()


def test_tf32_packing_needs_cuda_weights():
    with pytest.raises(ValueError, match="CUDA"):
        lib.tf32_pack_weights(torch.zeros(36, 32))
    with pytest.raises(ValueError, match="CUDA"):
        FV.I3D(IO.synthetic_weights(), device="cpu", tf32=True)
    with pytest.raises(ValueError, match="CUDA"):
        FD.InceptionV3(NO.synthetic_weights(), device="cpu", tf32=True)


@pytest.mark.parametrize("n,T", [(1, 9), (3, 10), (16, 30)])
def test_i3d_tf32_program_validates_costs_72_launches_and_differs_only_in_convs(n, T):
    fp32, tf32, keep = i3d_programs(n, T)
    net = keep[0]
    arr = lib.make_ops(tf32)
    lib.validate_program(arr, len(tf32))
    assert lib.load().mcvd_count_launches(arr, len(tf32)) == len(tf32) == FV.LAUNCHES_PER_CHUNK == 72
    assert [o.kind for o in tf32].count(lib.OP_CONV3D_TF32) == 57
    assert_only_convs_differ(fp32, tf32, net, [st for st in FV.plan(T)[0]])


@pytest.mark.parametrize("n,S,C", [(1, 64, 1), (7, 128, 3), (210, 32, 3)])
def test_inception_tf32_program_validates_costs_100_launches_and_differs_only_in_convs(n, S, C):
    fp32, tf32, keep = fid_programs(n, S, C)
    net = keep[0]
    arr = lib.make_ops(tf32)
    lib.validate_program(arr, len(tf32))
    assert lib.load().mcvd_count_launches(arr, len(tf32)) == len(tf32) == FD.LAUNCHES_PER_CHUNK == 100
    assert [o.kind for o in tf32].count(lib.OP_CONV2D_TF32) == 94
    pooled = [o.flags for o in tf32 if o.kind == lib.OP_CONV2D_TF32 and o.flags]
    assert pooled == [lib.F_POOL | lib.F_AVG] * 8 + [lib.F_POOL]
    assert_only_convs_differ(fp32, tf32, net, FD.plan()[0])


def assert_only_convs_differ(fp32, tf32, net, steps):
    assert len(fp32) == len(tf32) == len(steps)
    for a, b, st in zip(fp32, tf32, steps):
        fa, fb = fields(a), fields(b)
        if st["kind"] != "conv":
            assert fa == fb
            continue
        assert FP32_KIND[fb.pop("kind")] == fa.pop("kind")
        assert fa.pop("w") == net.weights[st["key"]][0].data_ptr()
        assert fb.pop("w") == net.packed[st["key"]].data_ptr()
        assert fa == fb


def rejects_alike(op, match):
    """``op`` as a TF32 kind is rejected with the reason its fp32 kind gives."""
    fp = lib.McvdOp.from_buffer_copy(op)
    fp.kind = FP32_KIND[op.kind]
    with pytest.raises(RuntimeError) as e32:
        lib.validate_program(lib.make_ops([fp]), 1)
    with pytest.raises(RuntimeError) as etf:
        lib.validate_program(lib.make_ops([op]), 1)
    m32 = re.search(r"op 0 CONV[23]D: (.*)$", str(e32.value))
    mtf = re.search(r"op 0 CONV[23]D_TF32: (.*)$", str(etf.value))
    assert m32 and mtf and m32.group(1) == mtf.group(1), (str(e32.value), str(etf.value))
    assert re.search(match, mtf.group(1)), mtf.group(1)


def edit(op, **kw):
    o = lib.McvdOp.from_buffer_copy(op)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_validation_rejects_bad_conv3d_tf32_ops_as_conv3d():
    _, ops, keep = i3d_programs(2)
    stem, b1b = ops[1], ops[8]
    assert stem.kind == b1b.kind == lib.OP_CONV3D_TF32 and (stem.i0, b1b.i0, b1b.i7, b1b.i6) == (7, 3, 64, 256)
    rejects_alike(edit(stem, w=None), "null")
    rejects_alike(edit(stem, bias=None), "null")
    rejects_alike(edit(stem, C0=3), "multiple of 4")
    rejects_alike(edit(stem, Cout=60), "multiple of 8")
    rejects_alike(edit(stem, H=111, W=111), "SAME")
    rejects_alike(edit(stem, i3=0), "stride")
    rejects_alike(edit(b1b, i6=191), "pitch")
    rejects_alike(edit(b1b, i7=130), "pitch")
    rejects_alike(edit(b1b, i7=-4), "pitch")
    with pytest.raises(RuntimeError, match="CONV3D_TF32: bias must be 16-byte aligned"):
        lib.validate_program(lib.make_ops([edit(stem, bias=stem.bias + 4)]), 1)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        lib.validate_program(lib.make_ops([edit(stem, w=stem.w + 4)]), 1)
    lib.validate_program(lib.make_ops([stem, b1b]), 2)


def test_validation_rejects_bad_conv2d_tf32_ops_as_conv2d():
    _, ops, keep = fid_programs(2)
    stem = ops[1]
    row = next(o for o in ops if (o.i0, o.i1) == (1, 7))
    pooled = next(o for o in ops if o.flags)
    sliced = next(o for o in ops if o.kind == lib.OP_CONV2D_TF32 and o.i7 > 0)
    assert stem.kind == lib.OP_CONV2D_TF32 and (stem.i0, stem.i2, stem.H) == (3, 2, 149)
    rejects_alike(edit(stem, w=None), "null")
    rejects_alike(edit(stem, C0=6), "multiple of 4")
    rejects_alike(edit(stem, Cout=36), "multiple of 8")
    rejects_alike(edit(stem, H=150), "geometry")
    rejects_alike(edit(row, i4=7), "padding")
    rejects_alike(edit(sliced, i6=sliced.i7 + sliced.Cout - 4), "pitch")
    rejects_alike(edit(sliced, i7=sliced.i7 + 2), "pitch")
    rejects_alike(edit(pooled, flags=lib.F_AVG), "MCVD_F_AVG needs MCVD_F_POOL")
    rejects_alike(edit(pooled, flags=lib.F_POOL | lib.F_L1), "flags other than")
    rejects_alike(edit(stem, flags=lib.F_POOL), "fused pool needs a 1x1")
    rejects_alike(edit(row, flags=lib.F_POOL | lib.F_AVG), "fused pool needs a 1x1")
    lib.validate_program(lib.make_ops([stem, row, pooled, sliced]), 4)


def test_drop_ins_choose_tf32_from_the_environment(monkeypatch):
    monkeypatch.delenv("MCVD_EVAL_TF32", raising=False)
    assert FD.env_tf32() is False
    monkeypatch.setenv("MCVD_EVAL_TF32", "0")
    assert FD.env_tf32() is False
    monkeypatch.setenv("MCVD_EVAL_TF32", "1")
    assert FD.env_tf32() is True
    built = []
    monkeypatch.setattr(FD, "InceptionV3", lambda path, device=None, tf32=False: built.append(tf32) or tf32)
    monkeypatch.setattr(FD, "default_weights_path", lambda: HEADER)       # any existing file
    FD._model.cache_clear()
    try:
        assert FD.model_for("cpu") is True
        monkeypatch.setenv("MCVD_EVAL_TF32", "0")
        assert FD.model_for("cpu") is False
        assert built == [True, False]
    finally:
        FD._model.cache_clear()
