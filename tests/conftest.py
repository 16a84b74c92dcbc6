import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """Builds (if needed) and returns the oracle ctypes module.  Test infrastructure only."""
    from oracle import oracle_lib
    oracle_lib.build()
    return oracle_lib


@pytest.fixture(scope="session")
def oracle_ref(oracle):
    if not oracle.have_ref():
        pytest.skip("oracle/_ref/liborbref.so not built (needs /root/reference)")
    return oracle
