import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    import oracle_ffi

    oracle_ffi.lib()
    return oracle_ffi


@pytest.fixture(scope="session")
def gpu():
    """The CUDA library bound to device 0; fails (does not skip) if it cannot run."""
    from poly_b200 import _lib

    _lib.check(_lib.lib().pg_init(int(os.environ.get("LOCAL_RANK", "0"))))  # one process per GPU under torchrun
    return _lib
