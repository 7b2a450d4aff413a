import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def built_lib():
    """Builds (if stale) and loads libsrcv_b200.so."""
    from simplerecon_b200 import _native
    from simplerecon_b200.build import build
    build()
    return _native.load()


@pytest.fixture(scope="session")
def cuda_device(built_lib):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from simplerecon_b200 import _native
    _native.check(built_lib.srcv_check_device())
    return torch.device("cuda:0")
