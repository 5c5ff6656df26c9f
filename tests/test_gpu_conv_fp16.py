"""The fp16 convolution mode (model.conv_precision = "fp16", MCVD_F_HALF) on the H100.

Op level: the half-mode tensor-core conv against the float64 Interpreter within the one-product error model of
tests/test_conv_fp16_cpu.py, on the input families of tests/test_value_ranges_cpu.py, at both tile heights (forced
through i4), which must give the same bits.

Network level: the native half mode's error against a float64 forward of the oracle, relative to the output scale,
is held to twice the error of the oracle itself run on the GPU in fp32 with cuDNN's TF32 convolutions and fp32
matmuls (torch's defaults, the reference's numerics); the default mode stays far below both (1/20 of the TF32 error,
or within 4 fp32 ulps of the output scale: with the reference's fresh initialisation the zero-initialised last layers
keep every mode near fp32 rounding).  Sampler level: the same comparison of the deviation from the fp32 oracle for a
10-step DDPM call on cfg2 and for DDIM, F-PNDM and a Gamma-noise model on tiny networks.  The RMS deviation is held to
twice the TF32 oracle's everywhere, and so is the largest one except for DDIM: a deterministic sampler carries every
step's rounding to its output, and the largest element of the difference of two such runs is the noisiest statistic
here.  On an H100 its ratio reached 2.26 on tiny (RMS 1.56), so DDIM's largest deviation is held to 2.5 times.  Then
the invariances (graph replay, shards, batch position) and the weight images.
"""
import contextlib
import os

import pytest
import torch

from common import golden, make_module, step_noise
from mcvd_b200 import configs, detfill, lib, runner, samplers
from oracle import gen_golden_gamma as GG, mcvd_oracle as O
from test_conv_fp16_cpu import half_bound
import test_gpu_conv2 as C2
from test_gpu_value_ranges import stressed_state_dict
from test_value_ranges_cpu import CONV_FAMILIES, SHORTCUT_FAMILIES, conv_case, conv_op, worst_ratio

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def run(op):
    arr = lib.make_ops([op])
    lib.validate_program(arr, 1)
    lib.run_program(arr, 1, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def half_module(name, precision="fp16", dev=DEV, variant=None):
    cfg = configs.workload(name)
    cfg.model.conv_precision = precision
    cfg, net, sd = make_module(cfg, dev)
    if variant is not None:
        sd = stressed_state_dict(net, {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}, variant)
        net.load_state_dict(sd)
        sd = {k: v.detach().cpu().clone() for k, v in sd.items()}
    return cfg, net, sd


@pytest.fixture(scope="module")
def packer():
    return half_module("tiny")[1].engine()


# ---------------------------------------------------------------------------------------------------------- op level
HALF_SHAPES = [
    # B, H, C0, C1, Cout, ks, C2, i2 (work organisation), tab, res, tile heights, extra (n tile, i5, act_out, planar:
    # CONV_UMMA2 with the planar table and epilogue statistics)
    (2, 16, 64, 0, 96, 3, 0, 1, True, True, (128, 192), {}),      # streaming 3x3, fused norm, residual
    (3, 8, 32, 32, 64, 3, 0, 1, False, False, (128, 192), {}),    # virtual concat
    (2, 16, 96, 0, 192, 1, 0, 1, True, False, (128, 192), {}),    # 1x1 streaming
    (4, 8, 64, 0, 192, 1, 0, 2, False, True, (128,), dict(nt=64)),     # 1x1 input-stationary: three n tiles per item
    (2, 16, 64, 0, 64, 3, 32, 1, True, False, (128, 192), {}),    # fused 1x1 shortcut
    (2, 8, 48, 48, 96, 3, 0, 1, False, True, (128, 192), {}),     # K-block 16
    (2, 16, 64, 0, 96, 3, 0, 1, True, False, (128, 192), dict(act_out=True)),     # output SiLU
    (1, 128, 32, 0, 96, 3, 0, 1, True, False, (192,), dict(i5=3)),     # three slab stages at 128x128: half mode only
    (2, 16, 64, 0, 144, 3, 0, 1, True, True, (128, 192), dict(nt=144)),          # n tile 144
    (2, 8, 64, 0, 384, 3, 0, 1, True, False, (128, 192), dict(nt=192)),          # two n tiles
    (2, 16, 64, 0, 64, 3, 32, 0, True, False, (128,), dict(planar=True)),        # planar table, statistics
]


def run_half(packer, case, nacc, mt, extra):
    B, H, W, C0 = case["x0"].shape
    C1 = 0 if case.get("x1") is None else case["x1"].shape[3]
    Cout = case["taps"].shape[2]
    taps, sc = case["taps"], case.get("taps_sc")
    nt = extra.get("nt") or max(d for d in range(16, 257, 16) if Cout % d == 0)
    kb = lib.umma_kblock(C0, C1)
    w, f1 = packer._pack_umma(taps, nt, kb, True) if sc is None else packer._pack_umma_fused(taps, sc, nt, kb, True)
    assert w.numel() == 2 * (taps.numel() + (0 if sc is None else sc.numel()))        # hi only: 2 bytes a weight
    dst = torch.full((B, H, W, Cout), float("nan"), device=DEV)
    st = None
    if extra.get("planar"):
        st = torch.full((lib.umma2_stats_bytes(B, H, W, case["ks"], Cout) // 8,), -7, dtype=torch.int64, device=DEV)
        tab3 = C2.planar(case["tab"]).contiguous()
        op = conv_op(case, lib.OP_CONV_UMMA2, w, f1, dst, tab=tab3)
        op.dst2, op.i2 = st.data_ptr(), kb
    else:
        op = conv_op(case, lib.OP_CONV_UMMA, w, f1, dst)
        op.i2, op.i4, op.i5 = nacc, mt, extra.get("i5", 0)
    op.i1, op.flags = nt, op.flags | lib.F_HALF
    run(op)
    torch.cuda.synchronize()
    return dst, st


@pytest.mark.parametrize("shape", HALF_SHAPES,
                         ids=lambda s: "B{}H{}C{}+{}-{}k{}sc{}n{}".format(*s[:8]) + "".join(f"-{k}{v}" for k, v in s[11].items()))
def test_half_conv_meets_the_one_product_bound(packer, shape):
    B, H, C0, C1, Cout, ks, C2_, nacc, tab, res, heights, extra = shape
    report = []
    stats_checked = 0
    for fam in CONV_FAMILIES + (SHORTCUT_FAMILIES if C2_ else ()):
        case = conv_case(fam, B, H, C0, Cout, ks, C1=C1, C2=C2_, tab=tab, res=res, act_out=extra.get("act_out", False))
        case = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in case.items()}
        ref, bound = half_bound(case)
        outs = [run_half(packer, case, nacc, mt, extra) for mt in heights]
        for o, _ in outs[1:]:
            assert torch.equal(o, outs[0][0]), f"{fam}: MT = {heights} differ"
        out, st = outs[0]
        if st is not None and float(out.abs().max()) <= 4096.0:       # the statistics' documented range
            exp = C2.expected_stats(out.cpu(), ks)
            assert torch.equal(st.cpu().view(exp.shape), exp), fam
            stats_checked += 1
        report.append((fam, worst_ratio(out, ref, bound)))
    print(f"\n{shape}: worst err/bound " + ", ".join(f"{f} {r:.3g}" for f, r in report))
    assert all(r <= 1.0 for _, r in report), report
    assert not extra.get("planar") or stats_checked >= 3


def test_half_flag_rejects_a_split_experiment(packer):
    case = {k: v.to(DEV) if isinstance(v, torch.Tensor) else v for k, v in conv_case("unit", 2, 8, 32, 32, 3).items()}
    w, f1 = packer._pack_umma(case["taps"], 32, 32, True)
    dst = torch.empty(2, 8, 8, 32, device=DEV)
    op = conv_op(case, lib.OP_CONV_UMMA, w, f1, dst)
    op.i1, op.i3, op.flags = 32, 2, lib.F_HALF
    with pytest.raises(RuntimeError, match="F_HALF"):
        lib.validate_program(lib.make_ops([op]), 1)


# ----------------------------------------------------------------------------------------------------- network level
@contextlib.contextmanager
def oracle_on(device, dtype, tf32=False):
    """the oracle's forward on ``device`` in ``dtype``: its fp32 CPU constants (the timestep embedding, computed in
    fp32 as the reference does, and the FIR taps) follow the weights; ``tf32`` gives the reference's GPU numerics,
    cuDNN TF32 convolutions and fp32 matmuls (torch's defaults)"""
    emb, fir = O.timestep_embedding, O.fir_taps
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    O.timestep_embedding = lambda t, dim: emb(t.cpu(), dim).to(device, dtype)
    O.fir_taps = lambda up: fir(up).to(device, dtype)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32, False
    try:
        yield
    finally:
        O.timestep_embedding, O.fir_taps = emb, fir
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def f64_forward(cfg, sd, x, t, cond):
    with oracle_on("cpu", torch.float64):
        return O.unet_forward(cfg, {k: v.double() for k, v in sd.items()}, x.double(), t,
                              None if cond is None else cond.double())


def tf32_oracle(cfg, sd, x, t, cond):
    return tf32_fn(cfg, sd)(x, t, cond)


U32 = 2.0 ** -24                 # fp32 unit roundoff


def errors(out, ref):
    """(max |err|, RMS err) relative to the output scale (RMS of the float64 reference)"""
    d = out.double() - ref
    s = float(ref.pow(2).mean().sqrt())
    return float(d.abs().max()) / s, float(d.pow(2).mean().sqrt()) / s


NET_ROWS = [(n, v, "umma") for n in ("tiny", "tiny_spade", "tiny_rgb", "cfg2") for v in ("trained", "fresh")] + \
    [("cfg2", "trained", "umma2"), ("cfg2", "trained", "umma+stats")]


@pytest.mark.parametrize("name,variant,mode", NET_ROWS,
                         ids=["-".join(r[:2]) + ("" if r[2] == "umma" else "-" + r[2]) for r in NET_ROWS])
def test_network_error_within_twice_the_references_tf32(name, variant, mode):
    """mode: the lowering's conv mode, umma2 (planar-table convs) or umma+stats (GroupNorm statistics from the conv
    epilogue) besides the default"""
    torch.set_num_threads(min(torch.get_num_threads(), 16))
    cfg, net16, sd = half_module(name, "fp16", variant=variant)
    eng = net16.engine()
    eng.conv_mode = mode.split("+")[0]
    eng.epilogue_stats = mode in ("umma2", "umma+stats")
    _, net32, _ = half_module(name, "fp32", variant=variant)
    B = 1 if name == "cfg2" else 2
    x, cond = detfill.synthetic_inputs(cfg, B, seed=5)
    t = torch.tensor([437, 90][:B], dtype=torch.long)
    ref = f64_forward(cfg, sd, x, t, cond)
    xd, cd = x.to(DEV), None if cond is None else cond.to(DEV)
    e16 = errors(net16(xd, t.to(DEV), cond=cd).cpu(), ref)
    e32 = errors(net32(xd, t.to(DEV), cond=cd).cpu(), ref)
    etf = errors(tf32_oracle(cfg, sd, x, t, cond), ref)
    print(f"\n{name} {variant}: max/RMS error over the output scale: native fp16 {e16[0]:.3g}/{e16[1]:.3g}, "
          f"oracle TF32 {etf[0]:.3g}/{etf[1]:.3g}, native fp32 {e32[0]:.3g}/{e32[1]:.3g}; "
          f"ratios fp16/TF32 {e16[0] / etf[0]:.3g}/{e16[1] / etf[1]:.3g}")
    assert e16[0] <= 2 * etf[0] and e16[1] <= 2 * etf[1]
    peak = float(ref.abs().max() / ref.pow(2).mean().sqrt())          # max |ref| over the output scale
    assert e32[0] <= max(0.05 * etf[0], 4 * U32 * peak) and e32[1] <= max(0.05 * etf[1], 4 * U32)
    P = net16.engine().program(B)
    assert any(o.flags & lib.F_HALF for o in P.step_ops)
    if mode != "umma":
        assert any(o.flags & lib.F_HALF and o.dst2 for o in P.step_ops)       # half convs with epilogue statistics


# ----------------------------------------------------------------------------------------------------- samplers
def tf32_fn(cfg, sd):
    sdg = {k: v.to(DEV) for k, v in sd.items()}

    def fn(xx, tt, cc):
        with oracle_on(DEV, torch.float32, tf32=True):
            return O.unet_forward(cfg, sdg, xx.to(DEV), tt.to(DEV), None if cc is None else cc.to(DEV)).cpu()
    return fn


def deviation(a, b):
    d = (a.double() - b.double())
    return float(d.abs().max()), float(d.pow(2).mean().sqrt())


def check_deviation(label, native, tf32, ref, max_ratio=2.0):
    dn, dt = deviation(native, ref), deviation(tf32, ref)
    print(f"\n{label}: deviation from the fp32 oracle max/RMS: native fp16 {dn[0]:.3g}/{dn[1]:.3g}, "
          f"oracle TF32 {dt[0]:.3g}/{dt[1]:.3g}; ratios {dn[0] / dt[0]:.3g}/{dn[1] / dt[1]:.3g}")
    assert dn[0] <= max_ratio * dt[0] and dn[1] <= 2 * dt[1], (dn, dt)


def test_cfg2_ten_step_sampler_half_vs_tf32_oracle():
    torch.set_num_threads(min(torch.get_num_threads(), 16))
    cfg, net, sd = half_module("cfg2")
    L = 10
    x, cond = detfill.synthetic_inputs(cfg, 1, seed=21)
    zs = step_noise(x.shape, L, tag="c2z")
    out = samplers.ddpm_sampler(x.to(DEV), net, cond=cond.to(DEV), final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, noise_list=[z.to(DEV) for z in zs])[0].cpu()
    sched = O.make_schedule(cfg)
    ref = O.ddpm_sample(lambda xx, tt, cc: O.unet_forward(cfg, sd, xx, tt, cc), sched, x.clone(), cond, L, True, True,
                        noise=zs)[0]
    tf = O.ddpm_sample(tf32_fn(cfg, sd), sched, x.clone(), cond, L, True, True, noise=zs)[0]
    check_deviation("cfg2 DDPM 10 steps", out, tf, ref)


@pytest.mark.parametrize("name", ["tiny", "tiny_spade"])
def test_ddim_and_fpndm_half_vs_tf32_oracle(name):
    cfg, net, sd = half_module(name)
    B, L = cfg.bench_batch, cfg.sampling.subsample
    x, cond = detfill.synthetic_inputs(cfg, B)
    sched = O.make_schedule(cfg)
    f32 = lambda xx, tt, cc: O.unet_forward(cfg, sd, xx, tt, cc)
    ftf = tf32_fn(cfg, sd)
    out = samplers.ddim_sampler(x.to(DEV), net, cond=cond.to(DEV), final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, log=False)[0].cpu()
    check_deviation(f"{name} DDIM", out, O.ddim_sample(ftf, sched, x.clone(), cond, L, True, True)[0],
                    O.ddim_sample(f32, sched, x.clone(), cond, L, True, True)[0], max_ratio=2.5)
    out = samplers.FPNDM_sampler(x.to(DEV), net, cond=cond.to(DEV), final_only=True, subsample_steps=L,
                                 clip_before=True, log=False)[0].cpu()
    check_deviation(f"{name} F-PNDM", out, O.fpndm_sample(ftf, sched, x.clone(), cond, L, True)[0],
                    O.fpndm_sample(f32, sched, x.clone(), cond, L, True)[0])


def test_gamma_sampler_half_vs_tf32_oracle():
    """Gamma noise (tiny_gamma) with the reference's recorded draws injected: the update is the DDPM one with those z"""
    cfg, net, sd = half_module("tiny_gamma")
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    L = cfg.sampling.subsample
    _, zs = GG.reference_noise(net.k_cum.cpu(), net.theta_t.cpu(), net.alphas.cpu(), x.shape, L, "ddpm_g")
    out = samplers.ddpm_sampler(x.to(DEV), net, cond=cond.to(DEV), final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, gamma=True, noise_list=[z.to(DEV) for z in zs], log=False)[0].cpu()
    sched = O.make_schedule(cfg)
    ref = torch.from_numpy(golden("tiny_gamma")["ddpm"])                         # the reference itself, CPU fp32
    tf = O.ddpm_sample(tf32_fn(cfg, sd), sched, x.clone(), cond, L, True, True, noise=zs)[0]
    to01 = lambda a: ((a + 1) / 2).clamp(0, 1)
    assert O.psnr01(to01(tf), to01(ref)) >= 40.0                     # the oracle runs the same Gamma sampler
    check_deviation("tiny_gamma DDPM", out, tf, ref)


# ----------------------------------------------------------------------------------------------------- invariance
def test_graph_replay_equals_eager_launches():
    cfg, net, _ = half_module("tiny")
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    kw = dict(cond=cond.to(DEV), final_only=True, denoise=True, subsample_steps=cfg.sampling.subsample,
              philox_seed=3, log=False)
    graphed = samplers.ddpm_sampler(x.to(DEV), net, **kw)
    net.engine().use_graph = False
    eager = samplers.ddpm_sampler(x.to(DEV), net, **kw)
    assert torch.equal(graphed, eager)


def test_shards_reproduce_the_single_batch():
    cfg, net, _ = half_module("tiny")
    cfg.sampling.num_frames_pred = 4
    cond = detfill.synthetic_inputs(cfg, 5)[1].to(DEV)
    full = runner.video_gen_sharded(cfg, net, cond, 0, 1, philox_seed=99, init_seed=7)
    parts = [runner.video_gen_clips(cfg, net, cond[lo:hi], clip_offset=lo, philox_seed=99,
                                    init_fn=runner.clip_init_fn(7, lo, hi, DEV))
             for lo, hi in ((0, 2), (2, 5))]
    assert torch.equal(torch.cat(parts), full)


def test_clip_output_is_independent_of_batch_position():
    cfg, net, _ = half_module("cfg2")
    B = 4
    x, cond = detfill.synthetic_inputs(cfg, B)
    xd, cd = x.to(DEV), cond.to(DEV)
    t = torch.full((B,), 500, dtype=torch.long, device=DEV)
    a = net(xd, t, cond=cd)
    assert torch.equal(a, net(xd, t, cond=cd))
    assert torch.equal(torch.cat([net(xd[:1], t[:1], cond=cd[:1]), net(xd[1:], t[1:], cond=cd[1:])]), a)
    perm = torch.tensor([2, 0, 3, 1], device=DEV)
    assert torch.equal(net(xd[perm], t, cond=cd[perm]), a[perm])


# ----------------------------------------------------------------------------------------------------- weights
def image_bytes(eng):
    return {k[:5]: v[0].numel() for k, v in eng.packed.items()
            if isinstance(k, tuple) and len(k) > 1 and k[1] == "umma"}


def test_half_images_are_half_the_bytes():
    cfg, n16, _ = half_module("tiny")
    _, n32, _ = half_module("tiny", "fp32")
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    t = torch.full((cfg.bench_batch,), 5, dtype=torch.long, device=DEV)
    for n in (n16, n32):
        n(x.to(DEV), t, cond=cond.to(DEV))
    b16, b32 = image_bytes(n16.engine()), image_bytes(n32.engine())
    assert b16.keys() == b32.keys()
    nin = {k for k in b16 if k[0].endswith((".qkv", ".NIN_3"))}
    assert nin and all(b16[k] == b32[k] for k in nin)
    assert all(2 * b16[k] == b32[k] for k in b16.keys() - nin)


def test_ema_style_data_copy_repacks_half_images():
    cfg, net, _ = half_module("tiny")
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    t = torch.full((B,), 100, dtype=torch.long, device=DEV)
    a = net(x.to(DEV), t, cond=cond.to(DEV)).clone()
    sd2 = {k: v.clone() for k, v in net.state_dict().items()}
    detfill.randomize_state_dict(sd2, seed=77)
    for n, p in net.named_parameters():
        p.data.copy_(sd2[n].to(p.device))
    before = net.engine().packs_computed
    b = net(x.to(DEV), t, cond=cond.to(DEV))
    assert net.engine().packs_computed > before and not torch.equal(a, b)
    _, fresh, _ = half_module("tiny")
    fresh.load_state_dict(net.state_dict())
    assert torch.equal(fresh(x.to(DEV), t, cond=cond.to(DEV)), b)


def test_weight_cache_keeps_the_modes_apart(tmp_path, monkeypatch):
    monkeypatch.setenv("MCVD_WEIGHT_CACHE", str(tmp_path))
    cfg, _, _ = half_module("tiny")
    x, cond = detfill.synthetic_inputs(cfg, cfg.bench_batch)
    t = torch.full((cfg.bench_batch,), 5, dtype=torch.long, device=DEV)

    def forward(precision):
        _, net, _ = half_module("tiny", precision)
        out = net(x.to(DEV), t, cond=cond.to(DEV))
        e = net.engine()
        return out, e.packs_computed, e.packs_loaded, e._cache_path()

    o16, c16, l16, p16 = forward("fp16")
    o32, c32, l32, p32 = forward("fp32")
    assert p16 != p32 and os.path.exists(p16) and os.path.exists(p32)
    assert c16 > 0 and l16 == 0 and c32 > 0 and l32 == 0          # the fp32 engine did not read the fp16 file
    r16, c, l, _ = forward("fp16")
    assert c == 0 and l > 0 and torch.equal(r16, o16)
    r32, c, l, _ = forward("fp32")
    assert c == 0 and l > 0 and torch.equal(r32, o32)
    assert not torch.equal(o16, o32)
