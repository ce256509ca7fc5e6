import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA sm_90 (H100) device")


@pytest.fixture(scope="session")
def built_lib():
    """libfemasr_b200.so, (re)built from source when stale (nvcc cross-compiles without a GPU)."""
    from femasr_b200 import build
    return build.build()


@pytest.fixture(scope="session")
def cuda(built_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from femasr_b200 import lib
    lib.require_device()
    return torch.device("cuda", 0)
