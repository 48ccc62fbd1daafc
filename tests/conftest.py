import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def pkg():
    import __graft_entry__ as ge
    return ge.load_package()


@pytest.fixture(scope="session")
def codec(pkg):
    c = pkg.Codec(0)
    yield c
    c.close()
