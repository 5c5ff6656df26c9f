"""Generate tests/golden/fvd.npz from the UNMODIFIED reference FVD code.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden_fvd

Drives the reference's ``models.fvd.fvd.preprocess_single``, ``models.fvd.pytorch_i3d.InceptionI3d`` (400 classes,
eval mode) and ``models.fvd.fvd.frechet_distance`` on the CPU, with ``i3d_oracle.synthetic_weights()`` loaded strictly.
The videos go through ``to_i3d`` (runners/ncsn_runner.py:1918-1923) and ``get_feats``' batching of 10 videos stacked
as float64 (models/fvd/fvd.py:41-49), restated here because ``get_feats`` always moves its input to ``cuda:0``.
SciPy 1.16 removed ``sqrtm``'s ``disp`` argument, which ``frechet_distance`` passes; with a newer SciPy the module's
``sqrtm`` is wrapped to accept it and return ``(sqrtm(A), None)``, the same matrix.

The weights and videos regenerate anywhere from the hash (``i3d_oracle.golden_cases``), so the fixture stores only
a checksum of the videos, their features and the distances, per case:
  ``{case}_real_sha`` / ``{case}_fake_sha`` (sha256 of the float32 videos), ``{case}_channels``, ``{case}_p``,
  ``{case}_real_feats`` [B, 400], ``{case}_fake_feats`` [B*p, 400] (float64), ``{case}_fvd`` (all fake videos),
  ``{case}_traj_fvd`` [p] (``fake[j::p]`` against the real set, as ``fvd_stuff`` forms them).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import i3d_oracle as IO, ref_import                # noqa: E402
from oracle.gen_golden import OUT                             # noqa: E402


def reference_feats(model, preprocess_single, videos: torch.Tensor, channels: int, bs: int = 10) -> np.ndarray:
    B, CT, S, _ = videos.shape
    x = videos.reshape(B, CT // channels, channels, S, S)
    if channels == 1:
        x = x.repeat(1, 1, 3, 1, 1)
    x = x.permute(0, 2, 1, 3, 4)                              # to_i3d: BTCHW -> BCTHW
    feats = np.empty((0, 400))
    with torch.no_grad():
        for i in range((len(x) - 1) // bs + 1):
            batch = torch.stack([preprocess_single(v) for v in x[i * bs:(i + 1) * bs]])
            feats = np.vstack([feats, model(batch).detach().cpu().numpy()])
    return feats


def gen():
    ref_import._ensure_path()
    import inspect
    import scipy.linalg
    import models.fvd.fvd as ref_fvd
    if "disp" not in inspect.signature(scipy.linalg.sqrtm).parameters:
        ref_fvd.sqrtm = lambda A, disp=True: (scipy.linalg.sqrtm(A), None)
    frechet_distance, preprocess_single = ref_fvd.frechet_distance, ref_fvd.preprocess_single
    from models.fvd.pytorch_i3d import InceptionI3d
    torch.set_num_threads(os.cpu_count() or 1)
    model = InceptionI3d(400, in_channels=3)
    model.load_state_dict(IO.synthetic_weights(), strict=True)
    model.eval()
    out = {}
    for name, (real, fake, C, p) in IO.golden_cases().items():
        rf = reference_feats(model, preprocess_single, torch.from_numpy(real), C)
        ff = reference_feats(model, preprocess_single, torch.from_numpy(fake), C)
        out.update({f"{name}_real_sha": IO.checksum(real), f"{name}_fake_sha": IO.checksum(fake),
                    f"{name}_channels": np.int64(C), f"{name}_p": np.int64(p),
                    f"{name}_real_feats": rf, f"{name}_fake_feats": ff,
                    f"{name}_fvd": np.float64(frechet_distance(ff, rf)),
                    f"{name}_traj_fvd": np.array([frechet_distance(ff[j::p], rf) for j in range(p)])})
        print(name, real.shape, fake.shape, "feature scale", np.abs(rf).max(), "fvd", out[f"{name}_fvd"], flush=True)
    path = os.path.join(OUT, "fvd.npz")
    np.savez_compressed(path, **out)
    print("fvd", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    gen()
