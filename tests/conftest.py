import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session")
def built():
    """Make sure the CUDA library and the oracle are compiled (both cross-compile without a GPU)."""
    import __graft_entry__ as g

    g.build()
    return True


@pytest.fixture(scope="session")
def clib(built):
    from pecos_b200 import core

    return core.get_clib()


@pytest.fixture(scope="session")
def gpu_clib(clib):
    if clib.device_count() <= 0:
        pytest.fail("this test is marked gpu but no CUDA device is visible")
    clib.set_device(0)
    return clib


@pytest.fixture(scope="session")
def have_ref():
    import oracle

    return oracle.have_ref()
