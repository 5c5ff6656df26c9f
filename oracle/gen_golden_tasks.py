"""Generate the task goldens tests/golden/tiny_general.npz and tiny_spade_general.npz from the UNMODIFIED
reference.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden_tasks

For each "general" workload (past and future frames masked in training) and each task its mode table gives
(``tasks_oracle.tasks_in_order``), the reference's ``conditioning_fn`` splits the synthetic test batch
(``tasks_oracle.golden_clips``) with the task's masking probabilities, and the restated AR loop
(``tasks_oracle.video_gen_loop``) drives the reference ``ddpm_sampler`` over the reference network with
injected noise: x_T of block i is ``detfill.normal(f"{task}_ar_init{i}")`` and its per-step noise
``detfill.normal(f"{task}_ar{i}_z{k}")``, the tag scheme of ``gen_golden.py``'s ``video`` with the task as prefix.
Each task's frames are stored as ``video_{task}``; inputs and weights regenerate from the hash.
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mcvd_b200 import configs, detfill                        # noqa: E402
from oracle import ref_import, tasks_oracle as T              # noqa: E402
from oracle.gen_golden import OUT, step_noise                 # noqa: E402

WORKLOADS = ("tiny_general", "tiny_spade_general")


def task_noise(config, task, n_clips):
    """(init_fn(i, shape), noise_fn(i)) of the goldens: block i's x_T and its L - 1 per-step noise tensors."""
    C, F, S, L = config.data.channels, config.data.num_frames, config.data.image_size, config.sampling.subsample
    shape = (n_clips, C * F, S, S)

    def init_fn(i, _shape=None):
        return detfill.normal(f"{task}_ar_init{i}", shape)

    def noise_fn(i):
        return step_noise(shape, L, tag=f"{task}_ar{i}_z")
    return init_fn, noise_fn


def gen(name):
    cfg = configs.workload(name)
    net = ref_import.build_reference_net(cfg)
    ddpm = ref_import.ref_models()[1]
    R = ref_import.ref_runner()
    X = T.golden_clips(cfg)
    L = cfg.sampling.subsample
    out = {}
    with torch.no_grad():
        for task in T.tasks_in_order(cfg):
            nfp, p_cond, p_fut = T.task_setup(cfg, task)
            _, cond, _ = R.conditioning_fn(cfg, 2 * X - 1, num_frames_pred=nfp, prob_mask_cond=p_cond,
                                           prob_mask_future=p_fut)
            init_fn, noise_fn = task_noise(cfg, task, len(X))
            n_iter = -(-nfp // cfg.data.num_frames)

            def sampler(x_T, c, i):
                zi = iter(noise_fn(i))
                with mock.patch("torch.randn_like", lambda _x: next(zi)):
                    return ddpm(x_T.clone(), net, cond=c, final_only=True, denoise=True, subsample_steps=L,
                                clip_before=True, log=False, verbose=False)
            inits = [init_fn(i) for i in range(n_iter)]
            out[f"video_{task}"] = T.video_gen_loop(cfg, sampler, cond, inits, nfp).numpy()
    path = os.path.join(OUT, f"{name}.npz")
    np.savez_compressed(path, **out)
    print(name, {k: v.shape for k, v in out.items()}, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    for n in (sys.argv[1:] or WORKLOADS):
        gen(n)
