import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run with -m gpu on an H100)")


@pytest.fixture(scope="session")
def b200lib():
    from libde265_b200 import build, capi
    build.build_library()  # in-tree nvcc build for sm_90a if missing / stale (cross-compiles without a GPU); raises on failure
    return capi.load()  # raises when the CUDA library is missing: never silently skipped


@pytest.fixture(scope="session")
def oracle_mod():
    import oracle_lib
    oracle_lib.oracle()
    return oracle_lib
