import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(scope="session")
def lib():
    """The loaded C-ABI library; GPU tests must go through it (no fallback)."""
    from assembled_cnn_b200 import _lib
    return _lib.load()
