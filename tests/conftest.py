import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def native():
    """The ctypes binding; building the library first if it is missing (nvcc cross-compiles on CPU)."""
    from distributed_reinforcement_learning_b200 import build
    build.build()
    from distributed_reinforcement_learning_b200 import _native
    return _native
