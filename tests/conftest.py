import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure): builds liboracle.so on first use."""
    from oracle import oracle as O
    O.lib()
    return O


def _gpu_missing():
    """-> reason why the GPU suite cannot run here, or None.  Only a MISSING library or the absence of a device skips: a library
    that is there but does not load (a symbol the header declares and the build lacks) must fail the tests loudly."""
    from s2p_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        return "%s is not built" % _lib.LIB_PATH
    if _lib.lib().s2pb_device_count() <= 0:
        return "no CUDA device is visible"
    return None


def pytest_collection_modifyitems(config, items):
    """A plain `pytest` on a CPU box skips the GPU suite instead of erroring in every test; set S2PB_REQUIRE_GPU=1
    (the GPU job) to make a missing device or library a failure."""
    if os.environ.get("S2PB_REQUIRE_GPU") == "1":
        return
    gpu_items = [it for it in items if "gpu" in it.keywords]
    if not gpu_items:
        return
    why = _gpu_missing()
    if why:
        skip = pytest.mark.skip(reason=why)
        for it in gpu_items:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def engine():
    from s2p_b200.engine import Engine
    eng = Engine(0)
    yield eng
    eng.close()
