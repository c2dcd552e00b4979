import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")
    config.addinivalue_line("markers", "timeout: per-test time limit (pytest-timeout; a no-op without the plugin)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.lib()
    return O


@pytest.fixture(scope="session")
def qrl():
    import qradiolink_b200 as q
    # QRL_EMULATED_LIB=<path of a libqrl_b200_emu.so built by tools/emu/build_emulated_lib.py> runs the GPU tier's tests against the
    # host-thread build of the library (slow; development aid for a container without a GPU, see tools/emu/).  The package itself has
    # no such switch: the path is patched in here, in the test harness.
    emu = os.environ.get("QRL_EMULATED_LIB")
    if emu:
        from qradiolink_b200 import lib as L
        L._LIB_PATH, L._LIB = emu, None
    q.load_library()
    return q
