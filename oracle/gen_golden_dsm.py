"""Generate tests/golden/dsm.npz from the UNMODIFIED reference.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden_dsm

Calls the reference ``losses.dsm.anneal_dsm_score_estimation`` on ``tiny`` (L2 and ``L1=True``), ``tiny_spade`` and
``tiny_gamma`` (``gamma=True``), with the labels ``LABELS`` spread over the schedule and the clean frames ``clean``.
For the duration of each call ``torch.randn_like`` returns ``detfill.normal(NOISE_TAG)`` and ``losses.dsm.Gamma`` is
``gen_golden_gamma.GammaStub(GAMMA_TAG)``, so ``reference_noise`` regenerates exactly the z the reference used.  The
network is wrapped in a module that records the ``x_t`` it receives.  Recorded per case: the per-clip losses from
the reference's ``hook``, the returned mean and the recorded ``x_t`` (once per workload: L1 perturbs alike).
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
from oracle import ref_import                                 # noqa: E402
from oracle.gen_golden import OUT                             # noqa: E402
from oracle.gen_golden_gamma import GammaStub                 # noqa: E402

LABELS = (0, 250, 640, 999)
NOISE_TAG = "dsm_z"
GAMMA_TAG = "dsm_g"
CASES = (("tiny", "tiny", False), ("tiny_l1", "tiny", True), ("tiny_spade", "tiny_spade", False),
         ("tiny_gamma", "tiny_gamma", False))                 # (key, workload, L1)


def clean(cfg, B):
    """(clean frames x in [-1, 1] [B, C*F, S, S], cond [B, C*Fc, S, S])"""
    C, F, S = cfg.data.channels, cfg.data.num_frames, cfg.data.image_size
    return detfill.uniform("dsm_x", (B, C * F, S, S), -1.0, 1.0), detfill.synthetic_inputs(cfg, B)[1]


def reference_noise(net, labels, shape, gamma):
    """The z losses/dsm.py forms under the golden's patches: ``detfill.normal(NOISE_TAG)``, or for a Gamma model
    ``(G - k theta) / sqrt(1 - a)`` from the ``GammaStub(GAMMA_TAG)`` draw, in the reference's fp32 operations."""
    if not gamma:
        return detfill.normal(NOISE_TAG, shape)
    B = shape[0]
    used_alphas = net.alphas[labels].reshape(B, 1, 1, 1)
    used_k = net.k_cum[labels].reshape(B, 1, 1, 1).repeat(1, *shape[1:])
    used_theta = net.theta_t[labels].reshape(B, 1, 1, 1).repeat(1, *shape[1:])
    z = GammaStub(GAMMA_TAG)(used_k, 1 / used_theta).sample()
    return (z - used_k * used_theta) / (1 - used_alphas).sqrt()


class Recorder(torch.nn.Module):
    """The reference network behind a module that keeps the x_t it is called with (``.module`` is what
    anneal_dsm_score_estimation unwraps for the schedule)."""

    def __init__(self, net):
        super().__init__()
        self.module = net
        self.x_t = None

    def forward(self, x, y, cond=None, cond_mask=None):
        self.x_t = x.clone()
        return self.module(x, y, cond=cond, cond_mask=cond_mask)


def gen():
    ref_import.ref_models()
    import losses.dsm as LD
    out = {"labels": np.array(LABELS, dtype=np.int64)}
    labels = torch.tensor(LABELS)
    for key, name, l1 in CASES:
        cfg = configs.workload(name)
        net = ref_import.build_reference_net(cfg)
        gamma = bool(cfg.model.gamma)
        x, cond = clean(cfg, len(LABELS))
        rec = Recorder(net)
        hooked = {}
        with torch.no_grad(), \
                mock.patch.object(torch, "randn_like", lambda t: detfill.normal(NOISE_TAG, tuple(t.shape))), \
                mock.patch.object(LD, "Gamma", GammaStub(GAMMA_TAG)):
            mean = LD.anneal_dsm_score_estimation(rec, x.clone(), labels=labels.clone(), cond=cond, gamma=gamma, L1=l1,
                                                  hook=lambda loss, lab: hooked.update(loss=loss.clone()))
        z = reference_noise(net, labels, x.shape, gamma)
        used = net.alphas[labels].reshape(-1, 1, 1, 1)
        want = used.sqrt() * x + (1 - used).sqrt() * z
        assert torch.equal(rec.x_t, want), f"{key}: reference_noise does not reproduce the reference's z"
        out[f"{key}_loss"] = hooked["loss"].numpy()
        out[f"{key}_mean"] = np.float32(mean.item())
        if key == "tiny_l1":
            assert np.array_equal(out["tiny_xt"], rec.x_t.numpy())
        else:
            out[f"{key}_xt"] = rec.x_t.numpy()
    path = os.path.join(OUT, "dsm.npz")
    np.savez_compressed(path, **out)
    print("dsm", {k: v.shape for k, v in out.items()}, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    gen()
