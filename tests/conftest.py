import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: test needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def built_lib():
    from equiformer_b200 import _lib
    _lib.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda_device():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("CUDA device required")
    from equiformer_b200 import _lib
    if not _lib.LIB_PATH.exists():
        _lib.build()
    return torch.device("cuda:0")
