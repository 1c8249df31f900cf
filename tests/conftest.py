import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100)")


@pytest.fixture(scope="session")
def lib():
    """The C-ABI library, built on demand (nvcc cross-compiles without a GPU)."""
    from pulser_b200 import build

    build.build()
    from pulser_b200 import _lib

    return _lib.lib
