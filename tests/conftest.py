import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_lib
    oracle_lib.lib()
    return oracle_lib


@pytest.fixture(scope="session")
def sdb():
    """The native library; GPU tests fail loudly (not skip) if it is missing or no device is present."""
    import sigdigger_b200
    sigdigger_b200.load_library()
    if sigdigger_b200.device_count() < 1:
        pytest.fail("CUDA device required for -m gpu tests (no CPU fallback exists)")
    return sigdigger_b200
