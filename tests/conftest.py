import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def lib():
    """The CUDA library, initialised on cuda:0.  GPU tests fail loudly if it cannot start."""
    from tinysql_b200 import _lib as L
    l = L.load()
    L.check(l.tq_init(0))
    return l
