import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def gen():
    from oracle import pyoracle
    return pyoracle.Gen()


@pytest.fixture(scope="session")
def port():
    from oracle import pyoracle
    return pyoracle.Port()


@pytest.fixture(scope="session")
def ref():
    """The unmodified reference, if its .so was built (oracle/_ref/); else skip."""
    from oracle import pyoracle
    if not pyoracle.ref_available():
        pytest.skip("oracle/_ref/libbsc_ref.so not built")
    return pyoracle.Ref()


@pytest.fixture(scope="session")
def checker():
    """Strongest oracle on this machine: the real reference when built, else our C port."""
    from oracle import pyoracle
    return pyoracle.best()


@pytest.fixture(scope="session")
def bsc():
    """The product: CUDA library through its host-pointer C ABI.  No fallback."""
    import libbsc_b200
    L = libbsc_b200.lib()                                  # a missing / unloadable library is an ERROR, never a skip
    if L.bsc_init(3) == -8:                                # LIBBSC_GPU_NOT_SUPPORTED: no CUDA device on this machine
        pytest.skip("no CUDA device (gpu-marked tests need an H100)")
    return libbsc_b200.Bsc(features=3)
