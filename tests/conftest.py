import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    """CPU oracle (test infrastructure only)."""
    from oracle import oracle as orc

    orc.build()
    return orc
