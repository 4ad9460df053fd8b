import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def cuda_lib():
    """Loaded libadflow_b200.so bound to cuda:0 (gpu tests only)."""
    from adflow_b200 import _lib

    L = _lib.load()
    if L.adfb_device_count() < 1:
        pytest.fail("gpu-marked test running without a CUDA device")
    return L
