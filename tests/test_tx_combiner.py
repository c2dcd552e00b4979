"""CPU tier: the transmit combiner's definition (tests/tx_combiner_oracle.c: per channel gr_mod_base's x N interpolator, a rotator at the
device rate, add_cc in blocks of 8, x 1 / C, x bb_gain) by known answers and against an independent float64 statement, and the library's
own sources for it run on host threads (tools/emu/build_emulated_lib.py) against that definition."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
from scipy import signal as sps

from tests import tx_combiner_oracle as TCO
from tests import tx_frontend_oracle as TO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _x(seed, C, n, amp=0.3):
    rng = np.random.default_rng(seed)
    return (amp * (rng.standard_normal((C, n)) + 1j * rng.standard_normal((C, n)))).astype(np.complex64)


def _design(N):
    """low_pass(N, N 1e6, 480000, 20000, BLACKMAN_HARRIS) from the library's host-side firdes"""
    import qradiolink_b200 as q
    L = q.load_library()
    out = np.zeros(16384, np.float32)
    n = L.qrl_firdes_low_pass(float(N), N * 1e6, 480000.0, 20000.0, 5, out.ctypes.data_as(C.c_void_p), len(out))
    assert n > 0
    return out[:n]


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("N", [1, 2, 10])
def test_one_channel_without_offset_is_the_tx_frontend(N):
    x = _x(N, 1, 6000)
    t, f = TCO.TxCombiner(N * 1000000, 1), TO.TxFrontend(N * 1000000)
    assert t.ntaps == f.ntaps
    for lo, m in ((0, 2500), (2500, 1), (2501, 3499)):
        assert _same(t.work(x[:, lo:lo + m]), f.work(x[0, lo:lo + m]))


@pytest.mark.parametrize("fs,f", [(10000000, 4.5e6), (10000000, -4.5e6), (10000000, 1e6), (2000000, 1e6 - 0.5e6)])
def test_dc_row_becomes_a_line_at_plus_f(fs, f):
    """a DC row on channel 2 of 5 at offset f: one line at +f at the device rate, amplitude 1 / C (+1 MHz lies outside what the
    1 Msps rotator of qrl_tx_frontend can place)"""
    Cn, n, N = 5, 4096, fs // 1000000
    x = np.zeros((Cn, n), np.complex64); x[2] = 1.0
    t = TCO.TxCombiner(fs, Cn)
    t.set_carrier_offset(f, 2)
    y = t.work(x)[N * 400:]                                                        # past the interpolator's start-up
    spec = np.fft.fft(y) / len(y)
    k = np.argmax(np.abs(spec))
    assert abs(np.fft.fftfreq(len(y), 1.0 / fs)[k] - f) <= fs / len(y)
    assert abs(np.abs(spec[k]) - 1.0 / Cn) < 0.01 / Cn
    assert np.sort(np.abs(spec))[-2] < 0.02 / Cn                                   # nothing else near that level


def _statement(X, fs, offs_by_sample, gain_by_sample):
    """float64: upfirdn with the library's taps, exp(j 2 pi f n / fs) with the NCO's Q32 frequency and a continuous phase, sum, x 1 / C
    x gain.  offs_by_sample[c]: per output sample frequency (Hz), gain_by_sample: per output sample gain."""
    N = fs // 1000000
    Cn, n = X.shape
    taps = _design(N).astype(np.float64) if N > 1 else np.ones(1)
    S = np.zeros(N * n, np.complex128)
    for c in range(Cn):
        u = sps.upfirdn(taps, X[c].astype(np.complex128), up=N)[:N * n]
        fq = np.rint(offs_by_sample[c] / fs * 2 ** 32) / 2 ** 32                  # cycles per sample
        ph = 2 * np.pi * np.concatenate([[0.0], np.cumsum(fq)[:-1]])
        S += u * np.exp(1j * ph)
    return S / Cn * gain_by_sample


def test_matches_an_independent_float64_statement():
    """C = 11 (two blocks) at 10 Msps, mixed offsets, one channel retuned and the gain changed mid-stream"""
    fs, Cn, N = 10000000, 11, 10
    n0, n1 = 3000, 2500
    X = _x(5, Cn, n0 + n1, 0.2)
    offs = [-4.2e6, -3e6, -1.7e6, -0.6e6, 0.0, 0.35e6, 1e6, 1.9e6, 2.8e6, 3.6e6, 4.4e6]
    t = TCO.TxCombiner(fs, Cn)
    for c, f in enumerate(offs):
        t.set_carrier_offset(f, c)
    a = t.work(X[:, :n0])
    t.set_carrier_offset(-2.2e6, 7); t.set_gain(0.6)
    b = t.work(X[:, n0:])
    y = np.concatenate([a, b])
    per = np.array([np.where(np.arange(N * (n0 + n1)) < N * n0, f, -2.2e6 if c == 7 else f) for c, f in enumerate(offs)])
    g = np.where(np.arange(N * (n0 + n1)) < N * n0, 1.0, 0.6)
    want = _statement(X, fs, per, g)
    err = np.sqrt(np.mean(np.abs(y - want) ** 2)) / np.sqrt(np.mean(np.abs(want) ** 2))
    assert err < 1e-5, err


@pytest.mark.parametrize("N", [1, 3, 10])
def test_chunking_does_not_change_the_output(N):
    Cn = 9
    x = _x(N, Cn, 9000)
    whole = TCO.TxCombiner(N * 1000000, Cn)
    whole.set_carrier_offset(-0.4e6 * N, 1); whole.set_carrier_offset(0.2e6 * N, -1)
    a = whole.work(x[:, :4014])
    whole.set_carrier_offset(0.33e6 * N, 4); whole.set_gain(2.0)
    want = np.concatenate([a, whole.work(x[:, 4014:])])
    t = TCO.TxCombiner(N * 1000000, Cn)
    t.set_carrier_offset(-0.4e6 * N, 1); t.set_carrier_offset(0.2e6 * N, -1)
    parts, lo = [], 0
    for m in [1, 4000, 0, 13, 2500, 7, 2479]:
        if lo == 4014:
            t.set_carrier_offset(0.33e6 * N, 4); t.set_gain(2.0)
        parts.append(t.work(x[:, lo:lo + m])); lo += m
    got = np.concatenate(parts)
    assert len(got) == N * 9000 and _same(got, want)


def test_retune_is_phase_continuous_at_the_device_rate():
    """DC through one channel at 3 Msps: after the start-up the output is e^{j theta(n)} with theta continuous across a retune made
    between calls, its slope 2 pi f / 3e6 per OUTPUT sample"""
    fs, n0, n1 = 3000000, 3000, 4000
    t = TCO.TxCombiner(fs, 1)
    t.set_carrier_offset(400000.0)
    a = t.work(np.ones((1, n0), np.complex64))
    t.set_carrier_offset(-1.1e6)
    b = t.work(np.ones((1, n1), np.complex64))
    k = np.arange(3 * (n0 + n1))
    k0 = 3 * n0
    ph = np.where(k < k0, 2 * np.pi * 400000.0 * k / fs, 2 * np.pi * (400000.0 * k0 - 1.1e6 * (k - k0)) / fs)
    y = np.concatenate([a, b])
    s = slice(3 * 400, None)
    assert np.max(np.abs(y[s] - np.exp(1j * ph[s]))) < 2e-3


def test_zero_offset_channel_is_not_rotated_but_a_retuned_back_one_is():
    """offset 0 since create: the channel passes through bit-exact; retuned away and back to 0, its NCO keeps the phase it reached"""
    x = _x(3, 2, 500)
    t, f = TCO.TxCombiner(2000000, 1), TO.TxFrontend(2000000)
    t.set_carrier_offset(0.0, 0)
    assert _same(t.work(x[:1]), f.work(x[0]))
    t.set_carrier_offset(123456.0, 0); t.work(x[:1, :7]); f.work(x[0, :7])
    t.set_carrier_offset(0.0, 0)
    assert not _same(t.work(x[1:]), f.work(x[1]))


def test_bad_shapes_are_refused():
    for fs, Cn in ((0, 1), (1500000, 1), (33000000, 1), (2000000, 0)):
        with pytest.raises(ValueError):
            TCO.TxCombiner(fs, Cn)


# ------------------------------------------------------------------ the library's own sources, on host threads
@pytest.fixture(scope="module")
def emu_tx_combiner(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_txc")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    assert L.device_count() == 1
    yield q
    L._LIB_PATH, L._LIB = saved


@pytest.mark.parametrize("samp_rate", [2000000, 10000000])
def test_device_parity_through_the_emulated_library(emu_tx_combiner, samp_rate):
    from tests import test_gpu_tx_combiner as TG
    Cn = 9
    off = TG.spread(samp_rate, Cn)
    TG.parity(emu_tx_combiner, samp_rate, Cn, [700, 1, 333, 0, 90],
              {0: [("offset", c, off[c]) for c in range(Cn)], 2: [("offset", 8, 0.4e6), ("gain", 0.8)], 3: [("offset", -1, -0.25e6)]})


def test_one_msps_through_the_emulated_library(emu_tx_combiner):
    from tests import test_gpu_tx_combiner as TG
    TG.parity(emu_tx_combiner, 1000000, 9, [500, 1, 200], {1: [("offset", 1, 400000.0), ("gain", 3.0)]})
