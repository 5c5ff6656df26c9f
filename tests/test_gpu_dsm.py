"""Denoising score-matching test loss on the H100: MCVD_OP_DSM_PERTURB element by element against the Philox and Gamma
oracles (oracle/gamma_oracle.py), the injected-noise mode bit for bit against torch's fp32 expression, MCVD_OP_DSM_LOSS
against an fp64 sum and bit-stable across batch positions, golden parity with the reference's noise injected
(tests/golden/dsm.npz), the benchmark-size run against a recomputation from the same build's forward, bit-exact split
batches, reproducibility under torch.manual_seed and the launch count.

Tolerances: the normal draw 1e-5 absolute (fp32 logf / cospif of the same uniforms); the Gamma draw 1e-5 of its
standard deviation, with no acceptance test within 1e-12 of its threshold, as in tests/test_gpu_gamma.py.  Golden
losses 1e-4 relative (the forward agrees with the oracle to 5e-5 absolute and z - eps is O(1)).  At benchmark size
1e-12 relative: the same eps and z summed in another order."""
import math

import numpy as np
import pytest
import torch

from common import golden, make_module
from mcvd_b200 import detfill, dsm, lib, runner
from mcvd_b200.lib import McvdOp
from oracle import gamma_oracle as GO, gen_golden_dsm as GD

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SEED = 20261017


def run(ops):
    arr = lib.make_ops(ops)
    lib.validate_program(arr, len(ops))
    lib.run_program(arr, len(ops), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()


def table(net, labels, gamma=False):
    a = net.alphas[labels.to(net.alphas.device)]
    tab = torch.zeros(len(labels), 4, device=DEV)
    tab[:, 0], tab[:, 1] = a.sqrt(), (1 - a).sqrt()
    if gamma:
        tab[:, 2] = net.k_cum[labels]
        tab[:, 3] = net.theta_t[labels] / (1 - a).sqrt()
    return tab


def perturb(x, tab, flags, z_in=None, clip0=0, step=dsm.DSM_STEP):
    B, C, H, W = x.shape
    xt, z = torch.empty_like(x), torch.full_like(x, float("nan"))
    o = McvdOp()
    o.kind, o.flags, o.B, o.H, o.W, o.C0 = lib.OP_DSM_PERTURB, flags, B, H, W, C
    o.i0, o.i1 = GO.seed_words(SEED)
    o.i2, o.i3 = clip0, step
    o.src0, o.aux0, o.dst = x.data_ptr(), tab.data_ptr(), xt.data_ptr()
    if flags & lib.F_PHILOX:
        o.dst2 = z.data_ptr()
    else:
        o.src1 = z_in.data_ptr()
    run([o])
    return xt, (z if flags & lib.F_PHILOX else z_in)


def oracle_normal(clip, step, n):
    """philox_normal of elements 0..n-1: the kernel's fp32 uniforms, then Box-Muller in float64"""
    r0, r1, _, _ = GO.philox4x32_10(np.arange(n, dtype=np.uint32), clip, step, 0x4D435644, *GO.seed_words(SEED))
    inv = np.float32(2.3283064365386963e-10)
    u1 = (r0.astype(np.float32) + np.float32(1.0)) * inv
    u2 = (r1.astype(np.float32) + np.float32(0.5)) * inv
    u1 = np.minimum(np.maximum(u1, np.float32(1e-12)), np.float32(1.0))
    return np.sqrt(-2.0 * np.log(u1.astype(np.float64))) * np.cos(2.0 * np.pi * u2.astype(np.float64))


@pytest.mark.parametrize("gamma", [False, True])
def test_perturb_draws_equal_the_oracle_per_element(gamma):
    _, net, _ = make_module("tiny_gamma", DEV)
    labels = torch.tensor([0, 500, 999], device=DEV)
    B, C, S, clip0 = 3, 2, 32, 5
    x = detfill.uniform("dsm_px", (B, C, S, S)).to(DEV)
    tab = table(net, labels, gamma)
    xt, z = perturb(x, tab, lib.F_PHILOX | (lib.F_GAMMA if gamma else 0), clip0=clip0)
    n = C * S * S
    zc = z.reshape(B, n).double().cpu().numpy()
    for b in range(B):
        if gamma:
            k, s = float(tab[b, 2]), float(tab[b, 3])
            g, att, margin = GO.gamma_centred(k, SEED, clip0 + b, dsm.DSM_STEP, n)
            assert int((margin < 1e-12).sum()) == 0 and (att >= 0).all()
            err = np.abs(zc[b] - s * g).max()
            assert err <= 1e-5 * s * math.sqrt(k), (b, k, err)
        else:
            err = np.abs(zc[b] - oracle_normal(clip0 + b, dsm.DSM_STEP, n)).max()
            assert err <= 1e-5, (b, err)
    # x_t is torch's fp32 expression on the returned z, bit for bit
    assert torch.equal(xt, tab[:, 0].reshape(-1, 1, 1, 1) * x + tab[:, 1].reshape(-1, 1, 1, 1) * z)
    assert bool(torch.isfinite(z).all())


def test_injected_perturb_is_the_reference_expression_bit_for_bit():
    _, net, _ = make_module("tiny", DEV)
    labels = torch.tensor([0, 1, 333, 640, 998, 999], device=DEV)
    x = detfill.uniform("dsm_ix", (6, 2, 32, 32)).to(DEV)
    z = detfill.normal("dsm_iz", (6, 2, 32, 32)).to(DEV)
    xt, _ = perturb(x, table(net, labels), 0, z_in=z)
    used = net.alphas[labels].reshape(6, 1, 1, 1)
    assert torch.equal(xt, used.sqrt() * x + (1 - used).sqrt() * z)


def loss_op(eps, z, C, pitch, l1=False):
    B, _, H, W = z.shape
    out = torch.empty(B, dtype=torch.float64, device=DEV)
    o = McvdOp()
    o.kind, o.flags, o.B, o.H, o.W, o.C0, o.Cout = lib.OP_DSM_LOSS, lib.F_L1 if l1 else 0, B, H, W, C, pitch
    o.src0, o.src1, o.dst = eps.data_ptr(), z.data_ptr(), out.data_ptr()
    run([o])
    return out


@pytest.mark.parametrize("l1", [False, True])
def test_loss_op_equals_fp64_sum_and_is_stable_across_batch_positions(l1):
    B, C, S, pitch = 7, 10, 64, 16
    eps = detfill.normal("dsm_le", (B, S, S, pitch)).to(DEV)
    eps[..., C:] = float("nan")                                     # channel padding is never read
    z = detfill.normal("dsm_lz", (B, C, S, S)).to(DEV)
    got = loss_op(eps, z, C, pitch, l1)
    d = (z - eps[..., :C].permute(0, 3, 1, 2)).double()
    want = (d.abs() if l1 else 0.5 * d * d).sum(dim=(1, 2, 3))
    assert torch.allclose(got, want, rtol=1e-12, atol=0), (got, want)
    one = loss_op(eps[5:6].contiguous(), z[5:6].contiguous(), C, pitch, l1)
    assert torch.equal(one[0], got[5])


def gpu_module(name):
    return make_module(name, DEV)[:2]


@pytest.mark.parametrize("key,name,l1", GD.CASES)
def test_injected_dsm_matches_reference_golden(key, name, l1):
    g = golden("dsm")
    cfg, net = gpu_module(name)
    labels = torch.from_numpy(g["labels"])
    x, cond = GD.clean(cfg, len(labels))
    gamma = bool(cfg.model.gamma)
    z = GD.reference_noise(net.cpu(), labels, x.shape, gamma)
    net.to(DEV)
    hooked = {}
    mean = dsm.anneal_dsm_score_estimation(net, x.to(DEV), labels=labels.to(DEV), cond=cond.to(DEV), gamma=gamma,
                                           L1=l1, noise=z.to(DEV), hook=lambda loss, lab: hooked.update(loss=loss))
    x_t = net.engine().programs[len(labels)].x_in
    assert torch.equal(x_t.cpu(), torch.from_numpy(g[f"{'tiny' if key == 'tiny_l1' else key}_xt"]))
    want = torch.from_numpy(g[f"{key}_loss"]).double()
    assert torch.allclose(hooked["loss"].double().cpu(), want, rtol=1e-4, atol=0), (hooked["loss"], want)
    assert mean.is_cuda and mean.dtype == torch.float32
    assert abs(float(mean) / float(g[f"{key}_mean"]) - 1) < 1e-4


def test_benchmark_size_loss_equals_recomputation_from_the_forward():
    """cfg2, B = 64, labels spread over [0, 999], Philox noise: x_t is torch's fp32 expression on the returned z, and
    the per-clip loss is the fp64 sum of 0.5 (z - net(x_t, labels, cond))^2 of the same build."""
    cfg, net = gpu_module("cfg2")
    B = 64
    labels = torch.linspace(0, 999, B).round().long().to(DEV)
    x = detfill.uniform("dsm_bx", (B, 5, 64, 64)).to(DEV)
    cond = detfill.synthetic_inputs(cfg, B)[1].to(DEV)
    eng = net.engine()
    loss = eng.dsm(x, labels, cond, philox=(SEED, 0, dsm.DSM_STEP))
    P = eng.programs[B]
    x_t, z = P.x_in.clone(), P.dsm.z.clone()
    used = net.alphas[labels].reshape(B, 1, 1, 1)
    assert torch.equal(x_t, used.sqrt() * x + (1 - used).sqrt() * z)
    assert abs(float(z.std()) - 1) < 0.01
    assert eng.launches_last_dsm == P.cond_launches + P.step_launches + 2
    with torch.no_grad():
        eps = net(x_t, labels, cond)
    assert eng.launches_last_dsm == eng.launches_last_forward + 1          # + perturb + loss - layout change
    want = (0.5 * (z - eps).double() ** 2).sum(dim=(1, 2, 3))
    assert torch.allclose(loss, want, rtol=1e-12, atol=0), float(((loss - want) / want).abs().max())


@pytest.mark.parametrize("name", ["tiny", "tiny_gamma"])
def test_split_batches_are_bit_exact(name):
    """clips [0, 3) and [3, 7) with their clip_offset give the bits of one batch of 7"""
    cfg, net = gpu_module(name)
    X = detfill.uniform("dsm_X", (7, 5, 1, 32, 32), 0.0, 1.0)
    labels = torch.tensor([0, 999, 17, 500, 250, 998, 640], device=DEV)
    full = runner.test_loss(cfg, net, X, labels=labels, philox_seed=99)
    parts = [runner.test_loss(cfg, net, X[lo:hi], labels=labels[lo:hi], philox_seed=99, clip_offset=lo)["loss"]
             for lo, hi in ((0, 3), (3, 7))]
    assert torch.equal(torch.cat(parts), full["loss"])
    assert bool(torch.isfinite(full["loss"]).all()) and full["mean"].dtype == torch.float64
    per = runner.loss_per_level(full["loss"], labels, 1000)
    assert per[999] == full["loss"][1] and torch.isnan(per[1])


def test_runs_follow_torch_manual_seed_and_noise_is_paired_across_levels():
    cfg, net = gpu_module("tiny")
    x, cond = GD.clean(cfg, 4)
    x, cond = x.to(DEV), cond.to(DEV)
    outs = []
    for seed in (3, 3, 4):
        torch.manual_seed(seed)
        seen = {}
        outs.append(dsm.anneal_dsm_score_estimation(net, x, cond=cond, hook=lambda l, lab: seen.update(labels=lab)))
        outs.append(seen["labels"])
    assert torch.equal(outs[0], outs[2]) and torch.equal(outs[1], outs[3])
    assert not torch.equal(outs[0], outs[4])
    # the same seed perturbs with the same z whatever the labels: checkpoints and levels are compared paired
    P = net.engine().programs[4]
    zs = []
    for lab in ([0, 1, 2, 3], [999, 500, 7, 640]):
        dsm.anneal_dsm_score_estimation(net, x, labels=torch.tensor(lab, device=DEV), cond=cond, philox_seed=5)
        zs.append(P.dsm.z.clone())
    assert torch.equal(zs[0], zs[1])
