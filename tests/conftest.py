import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100: pytest -m gpu)")


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (oracle/epp_oracle.c via ctypes).  Test infrastructure only."""
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle
