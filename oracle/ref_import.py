"""Import the UNMODIFIED reference (voletiv/mcvd-pytorch) in place.  TEST INFRASTRUCTURE ONLY.

Works only where the reference tree exists (``MCVD_REFERENCE_ROOT`` names it).  Used (a) to pin ``oracle/mcvd_oracle.py`` against the real reference and
(b) by ``oracle/gen_golden.py`` to produce the fixtures committed under ``tests/golden/``.
Nothing in the product package imports this.
"""
from __future__ import annotations

import os
import sys
import types
from unittest import mock

REF_ROOT = os.environ.get("MCVD_REFERENCE_ROOT", "")

# optional third-party modules the reference imports at module scope in runners/ncsn_runner.py
# that may be absent -- none is used on the sampling path.
_STUBS = ["imageio", "matplotlib", "matplotlib.pyplot", "skimage", "skimage.metrics",
          "skimage.transform", "h5py", "progressbar", "seaborn", "lpips", "ninja"]


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "models", "better"))


def _ensure_path():
    if not available():
        raise RuntimeError(f"reference tree not found at {REF_ROOT}")
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)


def ref_models():
    """-> (UNetMore_DDPM, ddpm_sampler, ddim_sampler, FPNDM_sampler) from the reference."""
    _ensure_path()
    from models.better.ncsnpp_more import UNetMore_DDPM          # noqa
    from models import ddpm_sampler, ddim_sampler, FPNDM_sampler  # noqa
    return UNetMore_DDPM, ddpm_sampler, ddim_sampler, FPNDM_sampler


def ref_runner():
    """Import runners.ncsn_runner with the missing optional modules stubbed."""
    _ensure_path()
    for name in _STUBS:
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = mock.MagicMock(name=name)
    import runners.ncsn_runner as R  # noqa
    return R


def build_reference_net(config, seed: int = 1234):
    """Reference ``UNetMore_DDPM(config)`` on CPU with deterministic re-randomised weights."""
    import torch
    from mcvd_b200.detfill import randomize_state_dict
    UNetMore_DDPM = ref_models()[0]
    config.device = torch.device("cpu")
    net = UNetMore_DDPM(config).eval()
    sd = net.state_dict()
    randomize_state_dict(sd, seed)
    net.load_state_dict(sd)
    return net
