import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (test infrastructure).  Built on demand with g++."""
    from oracle import oracle_py

    oracle_py.lib()
    return oracle_py


@pytest.fixture(scope="session")
def gpu_ok():
    from rpt_b200 import _capi as capi

    n = capi.lib().rptb_device_count()
    if n <= 0:
        pytest.fail("GPU test selected but no CUDA device is visible (rpt_b200 has no CPU fallback)")
    return n
