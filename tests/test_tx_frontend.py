"""CPU tier: the transmit front end's definition (tests/tx_frontend_oracle.c: gr_mod_base's rotator at 1 Msps + x N interpolator) by
known answers, and the library's own sources for it run on host threads (tools/emu/build_emulated_lib.py) against that definition."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tests import tx_frontend_oracle as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NTAPS = {2: (419, 210), 3: (627, 209), 5: (1045, 209), 10: (2091, 210), 20: (4181, 210), 32: (6691, 210)}


def _design(N):
    """low_pass(N, N 1e6, 480000, 20000, BLACKMAN_HARRIS) from the library's host-side firdes"""
    import qradiolink_b200 as q
    L = q.load_library()
    out = np.zeros(16384, np.float32)
    n = L.qrl_firdes_low_pass(float(N), N * 1e6, 480000.0, 20000.0, 5, out.ctypes.data_as(C.c_void_p), len(out))
    assert n > 0
    return out[:n]


@pytest.mark.parametrize("N", sorted(NTAPS))
def test_taps_are_the_library_design(N):
    ntaps, nt = NTAPS[N]
    f = TO.TxFrontend(N * 1000000)
    assert f.ntaps == ntaps and (ntaps + N - 1) // N == nt
    taps = _design(N)
    assert len(taps) == ntaps
    # a unit impulse returns the N arms interleaved: y[N m + p] = arm[p][m] = taps[p + N m], the zero-padded tap array
    y = f.work(np.eye(1, nt, dtype=np.complex64)[0])
    assert len(y) == N * nt
    want = np.zeros(N * nt, np.float32); want[:ntaps] = taps
    assert np.array_equal(y.real.view(np.uint32), want.view(np.uint32)) and not np.any(y.imag)


def test_every_rate_has_about_210_taps_per_arm():
    for N in range(2, 33):
        assert (TO.TxFrontend(N * 1000000).ntaps + N - 1) // N in (209, 210), N


def test_bad_rates_are_refused():
    for fs in (0, 500000, 1500000, 33000000):
        with pytest.raises(ValueError):
            TO.TxFrontend(fs)


def test_one_msps_without_offset_is_the_identity():
    x = (np.random.default_rng(1).standard_normal(5000) + 1j * np.random.default_rng(2).standard_normal(5000)).astype(np.complex64)
    f = TO.TxFrontend(1000000)
    assert f.ntaps == 0
    y = f.work(x)
    assert np.array_equal(y.view(np.uint32), x.view(np.uint32))
    f.set_carrier_offset(0.0)                     # inc = base = 0: still no rotation
    assert np.array_equal(f.work(x).view(np.uint32), x.view(np.uint32))


@pytest.mark.parametrize("N,offset", [(1, 125000.0), (10, 300000.0), (10, -230000.0), (2, -25000.0)])
def test_offset_moves_dc_to_a_tone_at_plus_f(N, offset):
    n = 8192
    f = TO.TxFrontend(N * 1000000)
    f.set_carrier_offset(offset)
    y = f.work(np.full(n, 0.5 + 0j, np.complex64))[N * 400:]           # past the interpolator's start-up
    spec = np.abs(np.fft.fft(y))
    peak = np.fft.fftfreq(len(y), 1.0 / (N * 1e6))[np.argmax(spec)]
    assert abs(peak - offset) <= N * 1e6 / len(y), (peak, offset)


def test_retune_is_phase_continuous():
    f = TO.TxFrontend(1000000)
    n0, n1 = 3000, 4000
    f.set_carrier_offset(10000.0)
    a = f.work(np.ones(n0, np.complex64))
    f.set_carrier_offset(-37000.0)
    b = f.work(np.ones(n1, np.complex64))
    k = np.arange(n0 + n1)
    ph = np.where(k < n0, 2 * np.pi * 10000.0 * k / 1e6, 2 * np.pi * (10000.0 * n0 - 37000.0 * (k - n0)) / 1e6)
    y = np.concatenate([a, b])
    assert np.max(np.abs(y - np.exp(1j * ph))) < 2e-5


@pytest.mark.parametrize("N", [1, 3, 10])
def test_chunking_does_not_change_the_output(N):
    rng = np.random.default_rng(N)
    x = (0.3 * (rng.standard_normal(9000) + 1j * rng.standard_normal(9000))).astype(np.complex64)
    one = TO.TxFrontend(N * 1000000); one.set_carrier_offset(77000.0)
    want = one.work(x)
    f = TO.TxFrontend(N * 1000000); f.set_carrier_offset(77000.0)
    parts, lo = [], 0
    for m in [1, 4000, 0, 13, 2500, 7, 10000]:
        parts.append(f.work(x[lo:lo + m])); lo += m
    got = np.concatenate(parts)
    assert len(got) == len(want) == N * len(x)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------ the library's own sources, on host threads
@pytest.fixture(scope="module")
def emu_tx_frontend(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_txfe")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    assert L.device_count() == 1
    yield q
    L._LIB_PATH, L._LIB = saved


@pytest.mark.parametrize("samp_rate", [2000000, 10000000])
def test_device_parity_through_the_emulated_library(emu_tx_frontend, samp_rate):
    from tests import test_gpu_tx_frontend as TG
    TG.parity(emu_tx_frontend, samp_rate, 2, [700, 1, 333, 0, 90], {1: [(-1, 150000.0)], 2: [(1, -70000.0)]})


def test_one_msps_through_the_emulated_library(emu_tx_frontend):
    from tests import test_gpu_tx_frontend as TG
    TG.parity(emu_tx_frontend, 1000000, 2, [500, 1, 200], {1: [(1, 40000.0)]})
