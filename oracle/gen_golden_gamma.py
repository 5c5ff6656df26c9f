"""Generate tests/golden/tiny_gamma.npz from the UNMODIFIED reference.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden_gamma

Workload ``tiny_gamma`` (``tiny`` trained with Gamma noise, ``model.gamma=True``).  The reference draws its Gamma noise
with ``torch.distributions.Gamma(...).sample()``, imported into ``models`` (models/__init__.py:11).  For the duration of
each call ``models.Gamma`` is replaced by ``GammaStub``, which returns ``mean + std * n`` with ``n`` from
``detfill.normal`` under a running tag, so the draws are recorded and ``reference_noise`` regenerates exactly the
standardised noise the reference computed from them.  Recorded:
  * ``ddpm``: ``ddpm_sampler(gamma=True)``; ``ddpm_tmin``: the same with the ``t_min`` warm start;
  * ``ddim_tmin``: ``ddim_sampler(gamma=True)`` with the warm start (its only Gamma draw);
  * ``video``: a 2-block AR loop (``mcvd_oracle.video_gen_loop``) around the reference ``ddpm_sampler``, x_T of block i
    ``Gamma(k_cum[0], 1/theta_t[0]).sample() - k_cum[0] * theta_t[0]`` as runners/ncsn_runner.py:1471-1474 forms it;
  * the reference's ``k`` / ``k_cum`` / ``theta_t`` buffers and its ``state_dict`` key list.
Inputs and weights regenerate from the hash, as for the other goldens.
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mcvd_b200 import configs, detfill                        # noqa: E402
from oracle import mcvd_oracle as O, ref_import               # noqa: E402
from oracle.gen_golden import OUT                             # noqa: E402

NAME = "tiny_gamma"
T_MIN = 0.35
NUM_FRAMES_PRED = 4                                           # two AR blocks of num_frames = 2


class GammaStub:
    """Stands in for ``torch.distributions.Gamma(concentration, rate)``: ``sample(shape)`` returns
    ``concentration / rate + sqrt(concentration) / rate * n`` (the distribution's mean and std), ``n`` the
    ``detfill.normal`` tensor of tag ``{prefix}{count}``, count running over every draw of this stub."""

    def __init__(self, prefix: str):
        self.prefix, self.count = prefix, 0

    def __call__(self, concentration, rate):
        stub = self

        class _Draw:
            def sample(self, sample_shape=torch.Size()):
                n = detfill.normal(f"{stub.prefix}{stub.count}", tuple(sample_shape) + tuple(concentration.shape))
                stub.count += 1
                return concentration / rate + concentration.sqrt() / rate * n
        return _Draw()


def reference_noise(k_cum, theta_t, alphas, shape, L, prefix, t_min=-1, per_step=True):
    """(warm-start z or None, per-step noise list) the reference ``ddpm_sampler`` (``per_step``) or ``ddim_sampler``
    forms from ``GammaStub(prefix)`` draws with L subsampled steps (models/__init__.py:125-153, 228-328), in the
    order it draws them; entries of steps the sampler skips are None."""
    skip = len(alphas) // L
    steps = torch.tensor(range(0, len(alphas), skip))
    alphas = alphas.index_select(0, steps)
    ks_cum, thetas = k_cum.index_select(0, steps), theta_t.index_select(0, steps)
    gamma = GammaStub(prefix)
    warm, noise = None, [None] * (len(steps) - 1)
    started = False
    for i, step in enumerate(steps):
        if step < t_min * len(alphas):
            continue
        if not started and t_min > 0:
            z = gamma(torch.full(shape[1:], ks_cum[i]), torch.full(shape[1:], 1 / thetas[i])).sample((shape[0],))
            warm = (z - ks_cum[i] * thetas[i]) / (1 - alphas[i]).sqrt()
        started = True
        if per_step and i + 1 < len(steps):
            z = gamma(torch.full(shape[1:], ks_cum[i]), torch.full(shape[1:], 1 / thetas[i])).sample((shape[0],))
            noise[i] = (z - ks_cum[i] * thetas[i]) / ((1 - alphas[i]).sqrt())
    return warm, noise


def reference_init(k_cum, theta_t, shape, i):
    """x_T of AR block i (runners/ncsn_runner.py:1471-1474, 1546-1549) from ``GammaStub(f"ar_init{i}_")``."""
    used_k, used_theta = k_cum[0], theta_t[0]
    z = GammaStub(f"ar_init{i}_")(torch.full(shape, used_k), torch.full(shape, 1 / used_theta)).sample()
    return z - used_k * used_theta


def gen():
    cfg = configs.workload(NAME)
    net = ref_import.build_reference_net(cfg)
    ddpm, ddim = ref_import.ref_models()[1:3]
    import models as M
    B, L = cfg.bench_batch, cfg.sampling.subsample
    x, cond = detfill.synthetic_inputs(cfg, B)
    kw = dict(cond=cond, final_only=True, denoise=True, subsample_steps=L, clip_before=True, log=False, verbose=False,
              gamma=True)
    out = {"k": net.k.numpy(), "k_cum": net.k_cum.numpy(), "theta_t": net.theta_t.numpy(),
           "keys": np.array(list(net.state_dict().keys()))}
    with torch.no_grad():
        with mock.patch.object(M, "Gamma", GammaStub("ddpm_g")):
            out["ddpm"] = ddpm(x.clone(), net, **kw)[0].numpy()
        with mock.patch.object(M, "Gamma", GammaStub("tmin_g")):
            out["ddpm_tmin"] = ddpm(x.clone(), net, t_min=T_MIN, **kw)[0].numpy()
        with mock.patch.object(M, "Gamma", GammaStub("ddim_g")):
            out["ddim_tmin"] = ddim(x.clone(), net, t_min=T_MIN, **kw)[0].numpy()
        inits = [reference_init(net.k_cum, net.theta_t, x.shape, i) for i in range(-(-NUM_FRAMES_PRED //
                                                                                       cfg.data.num_frames))]

        def sampler(x_T, c, i):
            with mock.patch.object(M, "Gamma", GammaStub(f"ar{i}_g")):
                return ddpm(x_T.clone(), net, **dict(kw, cond=c))
        out["video"] = O.video_gen_loop(cfg, sampler, cond, inits, NUM_FRAMES_PRED).numpy()
    path = os.path.join(OUT, f"{NAME}.npz")
    np.savez_compressed(path, **out)
    print(NAME, {k: v.shape for k, v in out.items()}, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    gen()
