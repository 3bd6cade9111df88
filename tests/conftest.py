import os
import sys

import pytest

# every use of a registered tf32-lo weight twin is verified on the device during the tests (include/sfb200.h)
os.environ.setdefault("SFB200_CHECK_LO", "1")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """GPU tests are skipped (not failed) when no device is visible and -m gpu was not requested explicitly."""
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
