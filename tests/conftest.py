import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Make sure the oracle, the harness and libvxs.so exist (cross-compiles without a GPU)."""
    import __graft_entry__ as ge
    ge.build(quiet=True)
    yield
