"""Generate tests/golden/fid.npz from the UNMODIFIED reference FID code.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden_fid

Drives the reference's ``evaluation.inception.InceptionV3([3])`` and ``evaluation.fid_PR`` on the CPU with
``inception_oracle.synthetic_weights()``: ``evaluation.inception.load_state_dict_from_url`` is patched to return them
(``fid_inception_v3`` loads them strictly), so nothing is downloaded.  The reference takes RGB frames only, so a grey
case is given its frames repeated to RGB (the native path accepts the grey frames and must give the same features).
SciPy 1.16 removed ``sqrtm``'s ``disp`` argument, which ``calculate_frechet_distance`` passes; with a newer SciPy
the module's ``linalg`` is wrapped to accept it and return ``(sqrtm(A), None)``, the same matrix.

The weights and frames regenerate anywhere from the hash (``inception_oracle.golden_cases``), so the fixture stores
only a checksum of the frames, their features and the results, per case:
  ``{case}_real_sha`` / ``{case}_fake_sha`` (sha256 of the float32 frames), ``{case}_real_feats`` /
  ``{case}_fake_feats`` (``calculate_activations``, float32 [N, 2048]), ``{case}_fid``, ``{case}_precision``,
  ``{case}_recall`` (``get_fid_PR`` with k = 3) and ``{case}_margin`` (``inception_oracle.cover_margin`` of the
  features: how far every precision / recall comparison is from its radius);
and per ``inception_oracle.frechet_cases`` entry ``fd_{name}`` (``calculate_frechet_distance``).
"""
from __future__ import annotations

import inspect
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import inception_oracle as NO, ref_import          # noqa: E402
from oracle.gen_golden import OUT                             # noqa: E402


def rgb(frames: np.ndarray) -> torch.Tensor:
    x = torch.from_numpy(frames)
    return x.repeat(1, 3, 1, 1) if x.shape[1] == 1 else x


def gen():
    ref_import._ensure_path()
    import scipy.linalg
    import evaluation.inception as ref_inception
    import evaluation.fid_PR as ref_fid
    if "disp" not in inspect.signature(scipy.linalg.sqrtm).parameters:
        def sqrtm(A, disp=True):
            root = scipy.linalg.sqrtm(A)
            return root if disp else (root, None)
        ref_fid.linalg = types.SimpleNamespace(sqrtm=sqrtm)
    sd = NO.synthetic_weights()
    ref_inception.load_state_dict_from_url = lambda *a, **kw: {k: v.clone() for k, v in sd.items()}
    torch.set_num_threads(os.cpu_count() or 1)
    cpu = torch.device("cpu")
    model = ref_inception.InceptionV3([ref_inception.InceptionV3.BLOCK_INDEX_BY_DIM[2048]]).to(cpu)
    out = {}
    with torch.no_grad():
        for name, (real, fake) in NO.golden_cases().items():
            rf = ref_fid.calculate_activations(rgb(real), model, 50, 2048, cpu).numpy()
            ff = ref_fid.calculate_activations(rgb(fake), model, 50, 2048, cpu).numpy()
            fid, precision, recall = ref_fid.get_fid_PR(rgb(real), rgb(fake), device=cpu, k=3)
            out.update({f"{name}_real_sha": NO.checksum(real), f"{name}_fake_sha": NO.checksum(fake),
                        f"{name}_real_feats": rf, f"{name}_fake_feats": ff, f"{name}_fid": np.float64(fid),
                        f"{name}_precision": np.float64(precision), f"{name}_recall": np.float64(recall),
                        f"{name}_margin": np.float64(NO.cover_margin(rf, ff))})
            print(name, real.shape, fake.shape, "feature scale", np.abs(rf).max(), "fid", fid, "P/R", precision,
                  recall, "margin", out[f"{name}_margin"], flush=True)
    for name, (m1, s1, m2, s2) in NO.frechet_cases().items():
        out[f"fd_{name}"] = np.float64(ref_fid.calculate_frechet_distance(m1, s1, m2, s2))
        print("fd", name, out[f"fd_{name}"])
    path = os.path.join(OUT, "fid.npz")
    np.savez_compressed(path, **out)
    print("fid", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    gen()
