"""The TF32 mode of LPIPS on the CPU: the header, the Python binding and the library agree on
MCVD_OP_CONV_RELU_TF32; a ``tf32=True`` chunk program validates, costs 11 launches and differs from the fp32 one only
in the conv kinds and weight pointers; validation rejects malformed kind-37 ops with the reasons it gives for the
matching MCVD_OP_CONV_RELU ops, word for word."""
import os
import re

import pytest
import torch

from mcvd_b200 import lib, lpips as LP
from oracle import lpips_oracle as LO

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "mcvd_b200.h")


def chunk_programs(n, S=64, C=1):
    """(fp32 ops, tf32 ops, what keeps their pointers alive) of one chunk.  The net is built on the CPU, where packing
    cannot run: the packed images are zero stand-ins of the size the library asks for, all validation looks at."""
    net = LP.LPIPS(LO.synthetic_weights(), device="cpu")
    pred, real = torch.zeros(n, C, S, S), torch.zeros(n, C, S, S)
    out = torch.zeros(n, dtype=torch.float64)
    ws = torch.zeros(2 * n * (LP._WS_A + LP._WS_B))
    fp32 = net.program(pred, real, C, out, ws)
    net.tf32 = True
    net.packed = [torch.zeros(lib.tf32_packed_bytes(w.shape[0], w.shape[1]) // 4) for w, _, _ in net.weights]
    tf32 = net.program(pred, real, C, out, ws)
    return fp32, tf32, (net, pred, real, out, ws)


def fields(op):
    return {name: getattr(op, name) for name, _ in lib.McvdOp._fields_}


def edit(op, **kw):
    o = lib.McvdOp.from_buffer_copy(op)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def test_header_binding_and_library_agree_on_the_lpips_tf32_kind():
    hdr = open(HEADER).read()
    assert int(re.search(r"MCVD_OP_CONV_RELU_TF32\s*=\s*(\d+)", hdr).group(1)) == lib.OP_CONV_RELU_TF32 == 37
    assert re.search(r"MCVD_OP_CONV_RELU_TF32 = 37,\s*MCVD_OP__COUNT", hdr)
    assert re.search(r"#define MCVD_ABI_VERSION 5\b", hdr) and lib.load().mcvd_abi_version() == 5
    _, ops, keep = chunk_programs(1)
    lib.validate_program(lib.make_ops([ops[1]]), 1)           # the library knows kind 37 ...
    for kind in (36, 38):                                       # ... 36 stays unassigned, and 37 is the last kind
        op = lib.McvdOp.from_buffer_copy(ops[1])
        op.kind = kind
        with pytest.raises(RuntimeError, match=f"unknown kind {kind}"):
            lib.validate_program(lib.make_ops([op]), 1)
        with pytest.raises(RuntimeError, match=f"unknown op kind {kind}"):
            lib.run_program(lib.make_ops([op]), 1, 0)


def test_tf32_packing_needs_cuda_weights():
    with pytest.raises(ValueError, match="CUDA"):
        LP.LPIPS(LO.synthetic_weights(), device="cpu", tf32=True)
    net = LP.LPIPS(LO.synthetic_weights(), device="cpu")
    assert net.tf32 is False and net.packed == []


@pytest.mark.parametrize("K,cout", [(484, 64), (1600, 192), (1728, 384), (3456, 256), (2304, 256)])
def test_alexnet_layers_pack_in_whole_tiles(K, cout):
    n = lib.tf32_packed_bytes(K, cout)
    assert n == -(-K // 32) * 32 * cout * 4                   # every AlexNet Cout is a whole number of n tiles


@pytest.mark.parametrize("n", [1, 2, 37, 256])
def test_tf32_chunk_program_validates_costs_11_launches_and_differs_only_in_convs(n):
    fp32, tf32, keep = chunk_programs(n)
    net = keep[0]
    arr = lib.make_ops(tf32)
    lib.validate_program(arr, len(tf32))
    assert lib.load().mcvd_count_launches(arr, len(tf32)) == len(tf32) == 11
    assert [o.kind for o in tf32] == [lib.OP_LPIPS_PREP] + [lib.OP_CONV_RELU_TF32, lib.OP_LPIPS_LAYER] * 5
    assert [o.flags for o in tf32[1::2]] == [0, lib.F_POOL, lib.F_POOL, 0, 0]
    assert len(fp32) == len(tf32)
    for i, (a, b) in enumerate(zip(fp32, tf32)):
        fa, fb = fields(a), fields(b)
        if a.kind != lib.OP_CONV_RELU:
            assert fa == fb
            continue
        li = (i - 1) // 2
        assert fa.pop("kind") == lib.OP_CONV_RELU and fb.pop("kind") == lib.OP_CONV_RELU_TF32
        assert fa.pop("w") == net.weights[li][0].data_ptr()
        assert fb.pop("w") == net.packed[li].data_ptr()
        assert fa == fb


def rejects_alike(op, match):
    """``op`` (kind 37) is rejected with the reason its CONV_RELU twin gives."""
    fp = edit(op, kind=lib.OP_CONV_RELU)
    with pytest.raises(RuntimeError) as e32:
        lib.validate_program(lib.make_ops([fp]), 1)
    with pytest.raises(RuntimeError) as etf:
        lib.validate_program(lib.make_ops([op]), 1)
    m32 = re.search(r"op 0 CONV_RELU: (.*)$", str(e32.value))
    mtf = re.search(r"op 0 CONV_RELU_TF32: (.*)$", str(etf.value))
    assert m32 and mtf and m32.group(1) == mtf.group(1), (str(e32.value), str(etf.value))
    assert re.search(match, mtf.group(1)), mtf.group(1)


def test_validation_rejects_bad_conv_relu_tf32_ops_as_conv_relu():
    _, ops, keep = chunk_programs(2)
    stem, conv2 = ops[1], ops[3]                               # conv2 reads the pooled relu1
    assert stem.kind == conv2.kind == lib.OP_CONV_RELU_TF32
    assert (stem.i0, stem.i1, stem.C0, stem.flags) == (11, 4, 4, 0) and conv2.flags == lib.F_POOL
    rejects_alike(edit(stem, C0=3), "input channels must be a positive multiple of 4")
    rejects_alike(edit(conv2, C0=66), "input channels must be a positive multiple of 4")
    rejects_alike(edit(stem, Cout=96), "output channels must be a positive multiple of 64")
    rejects_alike(edit(conv2, Cout=200), "output channels must be a positive multiple of 64")
    rejects_alike(edit(conv2, i3=2, i4=2), "pooled input smaller than the 3x3 window")
    rejects_alike(edit(conv2, i3=31, i4=2), "pooled input smaller than the 3x3 window")
    rejects_alike(edit(stem, w=None), "null weights or bias")
    rejects_alike(edit(conv2, bias=None), "null weights or bias")
    rejects_alike(edit(conv2, H=14, W=14), "geometry")
    rejects_alike(edit(conv2, flags=0), "geometry")
    rejects_alike(edit(stem, i1=0), "stride")
    with pytest.raises(RuntimeError, match="op 0 CONV_RELU_TF32: bias must be 16-byte aligned"):
        lib.validate_program(lib.make_ops([edit(stem, bias=stem.bias + 4)]), 1)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        lib.validate_program(lib.make_ops([edit(stem, w=stem.w + 4)]), 1)
    lib.validate_program(lib.make_ops(ops[1::2]), 5)
