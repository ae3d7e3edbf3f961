import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a)")


GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import ffi
    ffi.lib()
    return ffi


@pytest.fixture(scope="session")
def have_ref():
    from oracle import ffi
    return ffi.have_ref()
