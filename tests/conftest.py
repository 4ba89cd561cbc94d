import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _build_checkers():
    """Build oracle/liboracle.so (and oracle/_ref where /root/reference exists)."""
    from oracle import pyoracle
    pyoracle.build()
