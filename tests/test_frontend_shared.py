"""CPU tier: the receive front end fed one wideband stream (qrl_frontend_work with stride 0), through the library's own sources run on
host threads (tools/emu/build_emulated_lib.py): every channel equal to the oracle front end fed the same stream and to a twin handle
fed identical rows; host, device and per-channel calls on one handle; the top rate create accepts; Frontend.work's shape rules."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_frontend(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_fesh")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    assert L.device_count() == 1
    yield q
    L._LIB_PATH, L._LIB = saved


def _host_as_device(x):
    """the emulated library's device memory is host memory: a host array at an odd sample offset stands for a device pointer"""
    buf = np.zeros(len(x) + 1, np.complex64)
    buf[1:] = x
    return buf.ctypes.data + 8, buf


# chunks: 0, 1, fewer than N, fewer than ntaps, and several strips; a retune of all channels, then of one
SIZES = [3000, 0, 1, 3, 40, 1500, 9000]
RETUNES = {0: [(1, 150000.0), (2, -330000.0)], 3: [(-1, 62500.0)], 5: [(2, -125000.0)]}


@pytest.mark.parametrize("samp_rate", [2000000, 5000000])
def test_shared_stream_through_the_emulated_library(emu_frontend, oracle, samp_rate):
    from tests import test_gpu_frontend_shared as TG
    TG.parity(emu_frontend, oracle, samp_rate, 3, SIZES, RETUNES)


def test_host_device_and_per_channel_calls_on_one_handle(emu_frontend, oracle):
    from tests import test_gpu_frontend_shared as TG
    TG.parity(emu_frontend, oracle, 2000000, 3, [2500, 777, 3100, 5, 2000], RETUNES, kinds=("host", "dev", "rows"),
              dev_input=_host_as_device)


def test_top_rate_is_checked_at_create(emu_frontend):
    """107 Msps is the highest rate whose decimating FIR fits its kernel's shared memory: 108 Msps fails at create with the limit named"""
    emu_frontend.Frontend(107000000, n_channels=2, max_in=4096).close()
    for rate in (108000000, 250000000):
        with pytest.raises(emu_frontend.QrlError, match="qrl_frontend_create: samp_rate above 107 Msps"):
            emu_frontend.Frontend(rate, n_channels=2, max_in=4096)


def test_shapes(emu_frontend):
    fe = emu_frontend.Frontend(2000000, n_channels=3, max_in=4096)
    x = np.ones(100, np.complex64)
    assert fe.work(x).shape == (3, 50)                                  # 1-D: one stream for every channel
    for bad in (np.ones((2, 100), np.complex64), np.ones((3, 4, 5), np.complex64), np.ones((1, 100), np.complex64)):
        with pytest.raises(ValueError):
            fe.work(bad)
    assert fe.work(np.ones((3, 100), np.complex64)).shape == (3, 50)
    fe.close()
