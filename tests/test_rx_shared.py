"""CPU tier: one stream feeding every receive channel (qrl_rx_work / _sc16 / _sc8 with stride 0) through the library's own sources run
on host threads (tools/emu/build_emulated_lib.py): 4FSK and NBFM (register-tiled stage 1 with the fused rotator), QPSK-250K (the rotator pass)
at three channels equal a twin handle fed identical rows, bit for bit, with host, device, sc16 and sc8 input and per-row calls on the
same handle; RxBlock.work_shared's shape rules."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.timeout(900)


@pytest.fixture(scope="module")
def emu_rx(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_rxsh")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    assert L.device_count() == 1
    yield q
    L._LIB_PATH, L._LIB = saved


def _host_as_device(a):
    """the emulated library's device memory is host memory: a host array 8 bytes past a 16-byte boundary stands for a device pointer"""
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    buf = np.zeros(len(raw) + 32, np.uint8)
    base = (-buf.ctypes.data) % 16 + 8
    buf[base:base + len(raw)] = raw
    return buf.ctypes.data + base, buf


KINDS = {
    "4fsk": lambda q: (lambda n, m: q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=n, max_samples=m)),
    "nbfm": lambda q: (lambda n, m: q.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=n, max_samples=m)),
    "qpsk": lambda q: (lambda n, m: q.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=n, max_samples=m)),
}


@pytest.mark.parametrize("name", sorted(KINDS))
def test_shared_stream_matches_identical_rows(emu_rx, name):
    from tests import test_gpu_rx_shared as TG
    retunes = {0: [(1, 397100.0), (2, -401900.0)], 3: [(-1, 62500.0)], 4: [(2, -125000.0)]}
    TG.parity(KINDS[name](emu_rx), 3, [6000, 1, 3001, 0, 5000, 4000], retunes,
              kinds=("host", "dev", "sc16", "rows", "sc8", "dev_sc16"), dev_input=_host_as_device, rssi=True, seed=2)


def test_work_shared_shapes(emu_rx):
    blk = KINDS["4fsk"](emu_rx)(3, 4096)
    blk.work_shared(np.ones(100, np.complex64))
    blk.work_shared_sc16(np.ones((100, 2), np.int16))
    blk.work_shared_sc8(np.ones((100, 2), np.int8))
    for bad in (np.ones((3, 100), np.complex64), np.ones((1, 100), np.complex64), np.ones((3, 4, 5), np.complex64)):
        with pytest.raises(ValueError):
            blk.work_shared(bad)
    for bad in (np.ones(100, np.int16), np.ones((100, 3), np.int16), np.ones((3, 100, 2), np.int16)):
        with pytest.raises(ValueError):
            blk.work_shared_sc16(bad)
        with pytest.raises(ValueError):
            blk.work_shared_sc8(bad.astype(np.int8))
    with pytest.raises(emu_rx.QrlError):
        blk.work_shared(np.ones(4097, np.complex64))             # T > max_samples: QRL_ERANGE
    blk.close()
