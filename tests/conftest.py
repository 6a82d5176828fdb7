import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (sm_90a); run with -m gpu")
    config.addinivalue_line("markers", "slow: long-running")


@pytest.fixture(autouse=True)
def _seed():
    import torch
    torch.manual_seed(1)
    yield


@pytest.fixture(scope="session")
def lib():
    """Build (if needed) and load the C-ABI library."""
    from sbi_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.fixture(scope="session")
def cuda_lib(lib):
    import torch
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but torch.cuda.is_available() is False")
    assert lib.sbi_b200_device_ok() == 1, "device 0 is not sm_90 (H100)"
    return lib
