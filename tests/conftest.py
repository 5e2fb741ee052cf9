import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; select with -m gpu)")


@pytest.fixture(scope="session")
def lib():
    """the product library; building it is part of the fixture so `pytest` alone works from a clean tree"""
    from matrixone_b200 import build, capi
    build.build()
    return capi.load_library()


@pytest.fixture(scope="session")
def gpu(lib):
    from matrixone_b200 import capi
    rc = lib.MoB200_Init(-1)
    if rc != 0:
        pytest.fail("libmo_b200 could not initialise a CUDA device: " + capi.last_error(lib))
    return lib
