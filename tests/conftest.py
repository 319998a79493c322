import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def native_lib():
    """Build (if stale) and load the C-ABI library."""
    from fruitnerf_b200 import _build, _lib

    _build.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")
