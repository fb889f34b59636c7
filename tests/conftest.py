"""pytest configuration: the `gpu` marker and shared library fixtures."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def port():
    from tests import oracle_lib
    return oracle_lib.load_port()


@pytest.fixture(scope="session")
def ref():
    """The real reference, compiled by oracle/Makefile into oracle/_ref/ (may be absent)."""
    from tests import oracle_lib
    lib = oracle_lib.load_ref()
    if lib is None:
        pytest.skip("oracle/_ref/libdaala_ref.so not built (needs the reference sources)")
    return lib
