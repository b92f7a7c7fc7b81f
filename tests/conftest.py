import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the oracle (CPU) and make sure the product library exists before any test."""
    from oracle import oracle
    oracle.lib()
    import mpi_b200
    if not os.path.exists(mpi_b200.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
