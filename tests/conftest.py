import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (sm_90a, H100); run with -m gpu")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        # a deadlocked kernel must cost minutes, not the whole GPU session: pytest-timeout's thread method dumps the
        # stacks and exits the process even while the main thread sits in cudaStreamSynchronize
        if config.pluginmanager.hasplugin("timeout"):
            for it in items:
                if "gpu" in it.keywords and it.get_closest_marker("timeout") is None:
                    it.add_marker(pytest.mark.timeout(240, method="thread"))
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
