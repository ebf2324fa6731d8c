import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA GPU (an H100)")


def pytest_collection_modifyitems(config, items):
    import torch
    if torch.cuda.is_available():
        # a kernel that hangs must fail its test, not the whole run (pytest-timeout is part of the image; without it the
        # marker is inert)
        if config.pluginmanager.hasplugin("timeout"):
            for item in items:
                if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                    item.add_marker(pytest.mark.timeout(180, method="thread"))   # "thread": a test blocked inside a CUDA call
                                                                                   # (a hung kernel) cannot be interrupted by a signal
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
