"""Generate the golden fixtures in tests/golden/ from the UNMODIFIED reference.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden

For each small workload it instantiates the reference ``UNetMore_DDPM`` on CPU, re-randomises the
weights with the deterministic hash fill (``mcvd_b200.detfill``; seed 1234), and records
  * the forward output eps for t in {0, 37, 990} on the synthetic (x_T, cond),
  * the output of the reference ``ddpm_sampler`` / ``ddim_sampler`` / ``FPNDM_sampler`` (L = the
    workload's subsample) with per-step noise injected by patching ``torch.randn_like`` around the
    unmodified reference call,
  * the autoregressive video_gen block loop (restated; the reference's loop is entangled with
    dataset / metric code) driven by the reference sampler.
Inputs and weights are NOT stored (they regenerate bit-identically from the hash); only outputs are.

``reference_pins.npz`` pins what the tests otherwise read from the live reference tree: per workload the
reference module's state_dict names, shapes and SHA-256 of the re-randomised values, its named parameters and its
forward output on mixed timesteps; and, per masking setting, the outputs of the reference ``conditioning_fn``
(SHA-256 of the clip tensors' bytes, which are too large to store; masks verbatim).
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mcvd_b200 import configs, detfill          # noqa: E402
from oracle import ref_import, mcvd_oracle as O  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
T_VALUES = (0, 37, 990)


def step_noise(shape, L, tag="z"):
    return [detfill.normal(f"{tag}{i}", shape) for i in range(L - 1)]


PIN_WORKLOADS = ("tiny", "tiny_spade", "cfg1")
MASK_CASES = ((0.0, 0.0, False), (0.5, 0.0, False), (0.5, 0.5, False), (0.5, 0.5, True), (0.0, 1.0, False),
              (0.3, 1.0, False))


def sha(t) -> str:
    import hashlib
    a = np.ascontiguousarray(t.detach().cpu().numpy())
    return hashlib.sha256(a.tobytes()).hexdigest() + f"|{a.dtype}|{a.shape}"


def pin_forward_t(B):
    return torch.tensor([3, 640][:B] + [77] * max(0, B - 2))


def mask_setup(p_cond, p_fut, sync):
    cfg = configs.workload("tiny")
    cfg.data.num_frames_future = 2
    cfg.data.prob_mask_sync = sync
    n = cfg.data.num_frames_cond + cfg.data.num_frames + cfg.data.num_frames_future
    return cfg, detfill.normal("clips", (6, n, cfg.data.channels, 32, 32))


def mask_key(p_cond, p_fut, sync):
    return f"mask_{p_cond}_{p_fut}_{int(sync)}"


def gen_pins():
    out = {}
    for name in PIN_WORKLOADS:
        cfg = configs.workload(name)
        ref = ref_import.build_reference_net(cfg)
        rsd = ref.state_dict()
        out[f"{name}_keys"] = np.array(list(rsd.keys()))
        out[f"{name}_sha"] = np.array([sha(v) for v in rsd.values()])
        out[f"{name}_params"] = np.array([n for n, _ in ref.named_parameters()])
        B = cfg.bench_batch
        x, cond = detfill.synthetic_inputs(cfg, B)
        with torch.no_grad():
            out[f"{name}_forward"] = ref(x, pin_forward_t(B), cond=cond).numpy()
    R = ref_import.ref_runner()
    for case in MASK_CASES:
        cfg, X = mask_setup(*case)
        torch.manual_seed(7)
        p, c, m = R.conditioning_fn(cfg, X, num_frames_pred=cfg.data.num_frames, prob_mask_cond=case[0],
                                    prob_mask_future=case[1])
        k = mask_key(*case)
        out[f"{k}_pred"], out[f"{k}_cond"] = np.array(sha(p)), np.array(sha(c))
        if m is not None:
            out[f"{k}_mask"] = m.numpy()
        out[f"{k}_uncond"] = np.array(sha(R.conditioning_fn(cfg, X, conditional=False)[0]))
    path = os.path.join(OUT, "reference_pins.npz")
    np.savez_compressed(path, **out)
    print("reference_pins", os.path.getsize(path) // 1024, "KiB")


def gen(name):
    cfg = configs.workload(name)
    net = ref_import.build_reference_net(cfg)
    _, ddpm, ddim, fpndm = ref_import.ref_models()
    B = cfg.bench_batch
    x, cond = detfill.synthetic_inputs(cfg, B)
    L = cfg.sampling.subsample
    out = {}
    with torch.no_grad():
        for t in T_VALUES:
            out[f"eps_t{t}"] = net(x, torch.full((B,), t, dtype=torch.long), cond=cond).numpy()
        zs = step_noise(x.shape, L)
        it = iter(zs)
        with mock.patch("torch.randn_like", lambda _x: next(it)):
            out["ddpm"] = ddpm(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                               clip_before=True, log=False, verbose=False)[0].numpy()
        # init_prev_t warm start (t_min > 0): first randn_like call is the re-noising, then the per-step noise
        it2 = iter([detfill.normal("warm", x.shape)] + zs)
        with mock.patch("torch.randn_like", lambda _x: next(it2)):
            out["ddpm_tmin"] = ddpm(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                                    clip_before=True, log=False, verbose=False, t_min=0.35)[0].numpy()
        out["ddim"] = ddim(x.clone(), net, cond=cond, final_only=True, denoise=True, subsample_steps=L,
                           clip_before=True, log=False, verbose=False)[0].numpy()
        out["fpndm"] = fpndm(x.clone(), net, cond=cond, final_only=True, subsample_steps=L,
                             clip_before=True, log=False, verbose=False)[0].numpy()
        # AR loop (runner:1501-1570 restated in the oracle) around the reference sampler
        nfp = cfg.sampling.num_frames_pred
        n_iter = -(-nfp // cfg.data.num_frames)
        inits = [detfill.normal(f"ar_init{i}", x.shape) for i in range(n_iter)]

        def sampler(x_T, c, i):
            zi = iter(step_noise(x.shape, L, tag=f"ar{i}_z"))
            with mock.patch("torch.randn_like", lambda _x: next(zi)):
                return ddpm(x_T.clone(), net, cond=c, final_only=True, denoise=True, subsample_steps=L,
                            clip_before=True, log=False, verbose=False)
        out["video"] = O.video_gen_loop(cfg, sampler, cond, inits, nfp).numpy()
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(name, {k: v.shape for k, v in out.items()}, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    for n in (sys.argv[1:] or ["tiny", "tiny_spade", "tiny_rgb", "cfg1", "reference_pins"]):
        gen_pins() if n == "reference_pins" else gen(n)
