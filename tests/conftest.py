import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a machine without a CUDA device: skip the gpu-marked tests instead of erroring in them."""
    if os.path.exists("/dev/nvidiactl") or os.path.exists("/dev/nvidia0"):
        return
    skip = pytest.mark.skip(reason="no CUDA device on this machine (the -m gpu tests run on an H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return os.path.join(ROOT, "tests", "golden")
