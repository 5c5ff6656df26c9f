"""Generate tests/golden/lpips.npz from the UNMODIFIED reference ``PerceptualLoss``.  TEST INFRASTRUCTURE.

Run where the reference tree is available (MCVD_REFERENCE_ROOT):   python -m oracle.gen_golden_lpips

Drives ``models.eval_models.PerceptualLoss(model='net-lin', net='alex')`` on the CPU through the reference loop's own
calls (runners/ncsn_runner.py:1427-1430, 1590-1609): ``ToPILImage()(frame).convert("RGB")``, the ``T2`` transform,
``model_lpips.forward(real, pred)``, the per-clip ``avg_distance`` summed in fp32 and divided by the frame count.

Nothing can be downloaded: ``models.pretrained_networks.tv.alexnet`` is patched to build with ``weights=None``,
``torch.hub.load_state_dict_from_url`` raises, and ``skimage`` (imported at module scope, unused here) is stubbed.
The weights, loaded over the network's after construction, are ``lpips_oracle.synthetic_weights()``; they regenerate
anywhere from the hash, so the fixture stores only the frames and the distances:
  ``{case}_pred``, ``{case}_real`` [B, C*F, S, S], ``{case}_channels``, ``{case}_frame`` [B, F] (per-frame distance),
  ``{case}_clip`` [B] (``avg_distance.item() / F``).
"""
from __future__ import annotations

import os
import sys
from unittest import mock

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import lpips_oracle as LO, ref_import             # noqa: E402
from oracle.gen_golden import OUT                             # noqa: E402


def _no_download(*a, **k):
    raise RuntimeError("gen_golden_lpips: a download was attempted")


def reference_model(sd):
    """The reference ``PerceptualLoss`` with ``sd`` (a PNetLin state_dict) loaded, built without network access."""
    import torchvision
    ref_import._ensure_path()
    for name in ("skimage", "skimage.color", "skimage.transform", "skimage.metrics"):
        sys.modules.setdefault(name, mock.MagicMock(name=name))
    with mock.patch("torch.hub.load_state_dict_from_url", _no_download), \
            mock.patch("torchvision.models._api.load_state_dict_from_url", _no_download, create=True):
        import models.pretrained_networks as pn
        from models import eval_models
        alexnet = torchvision.models.alexnet                  # pn.tv is torchvision.models itself
        with mock.patch.object(pn.tv, "alexnet", lambda pretrained=False, **kw: alexnet(weights=None)):
            model = eval_models.PerceptualLoss(model='net-lin', net='alex', device='cpu')
    missing, unexpected = model.model.net.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith("scaling_layer") for k in missing), (missing, unexpected)
    return model.eval()


def reference_loop(model, pred: torch.Tensor, real: torch.Tensor, channels: int):
    """(per-frame distances [B, F], per-clip avg_distance / F [B]) exactly as the reference loop forms them."""
    import torchvision.transforms as Transforms
    T2 = Transforms.Compose([Transforms.Resize((128, 128)), Transforms.ToTensor(),
                             Transforms.Normalize(mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))])
    B, F = pred.shape[0], pred.shape[1] // channels
    frame, clip = np.zeros((B, F)), np.zeros(B)
    for ii in range(B):
        avg_distance = 0
        for jj in range(F):
            pred_ij = pred[ii, channels * jj:channels * jj + channels]
            real_ij = real[ii, channels * jj:channels * jj + channels]
            pred_ij_pil = Transforms.ToPILImage()(pred_ij).convert("RGB")
            real_ij_pil = Transforms.ToPILImage()(real_ij).convert("RGB")
            pred_ij_LPIPS = T2(pred_ij_pil).unsqueeze(0)
            real_ij_LPIPS = T2(real_ij_pil).unsqueeze(0)
            d = model.forward(real_ij_LPIPS, pred_ij_LPIPS)
            frame[ii, jj] = float(d)
            avg_distance += d
        clip[ii] = avg_distance.data.item() / F
    return frame, clip


def gen():
    model = reference_model(LO.synthetic_weights())
    out = {}
    with torch.no_grad():
        for name, (pred, real, C) in LO.golden_cases().items():
            frame, clip = reference_loop(model, torch.from_numpy(pred), torch.from_numpy(real), C)
            out.update({f"{name}_pred": pred, f"{name}_real": real, f"{name}_channels": np.int64(C),
                        f"{name}_frame": frame, f"{name}_clip": clip})
            print(name, pred.shape, frame.min(), frame.max())
    path = os.path.join(OUT, "lpips.npz")
    np.savez_compressed(path, **out)
    print("lpips", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    assert ref_import.available(), "reference tree not found"
    gen()
