import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100, sm_90a); run with -m gpu")


@pytest.fixture(scope="session")
def lib():
    """libsa_b200.so, built in-tree if missing (nvcc cross-compiles without a GPU)."""
    from qsa_b200 import capi
    if not os.path.exists(capi.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    return capi.load()
