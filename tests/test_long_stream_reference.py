"""CPU tier: the float64 statement that tests/test_gpu_long_stream.py holds the streaming front ends to far past 2^32 samples, pinned here
against the oracle (oracle/qrl_oracle.c's front end, tests/tx_frontend_oracle.c, tests/tx_combiner_oracle.c) at small absolute indices,
where the oracle can run: a zero prefix, offsets set before it, a retune after it, then a burst of signal, at every rate and channel
count the GPU file uses.

The statement: the rotator's phase phi(n) = (base + inc (n - n_base)) mod 2^32 in Python integers, carried across retunes; the angle
phi as a signed 32-bit number times pi / 2^31; the FIR with the library's own taps (qrl_firdes_low_pass, the design its create calls
make); all of it in float64, with zero input before the burst."""
import ctypes as C

import numpy as np
import pytest
from scipy import signal as sps

from tests import tx_combiner_oracle as TCO
from tests import tx_frontend_oracle as TO

TWO32 = 1 << 32
RMS_TOL = 1e-5        # RMS error over the RMS of the statement's output
PEAK_TOL = 1e-4       # largest error of one sample over the RMS of the statement's output


def design(gain, fs, cutoff, tw):
    """low_pass(gain, fs, cutoff, tw, BLACKMAN_HARRIS) from the library's host-side firdes, as float64"""
    import qradiolink_b200 as q
    out = np.zeros(16384, np.float32)
    n = q.load_library().qrl_firdes_low_pass(float(gain), float(fs), float(cutoff), float(tw), 5, out.ctypes.data_as(C.c_void_p), len(out))
    assert n > 0
    return out[:n].astype(np.float64)


def rx_taps(fs):
    """gr_demod_base's decimator: low_pass(1, fs, 480000, 100000, BLACKMAN_HARRIS)"""
    return design(1, fs, 480000, 100000)


def tx_taps(fs):
    """gr_mod_base's interpolator: low_pass(N, fs, 480000, 20000, BLACKMAN_HARRIS)"""
    return design(fs // 1000000, fs, 480000, 20000)


def q32_inc(offset_hz, rate):
    """phase step per sample of a rotator turning by offset_hz at `rate`: rint(offset / rate 2^32) mod 2^32"""
    return int(np.rint(offset_hz / rate * 2.0 ** 32)) % TWO32


class Nco:
    """Q32 phase across retunes: from absolute sample n_base on, phi(n) = base + inc (n - n_base); a retune at n carries the phase
    it reached into base.  Python integers throughout, so no index or phase is truncated however far the stream runs."""

    def __init__(self):
        self.inc = self.base = self.n_base = 0

    def retune(self, n, inc):
        self.base = (self.base + self.inc * (n - self.n_base)) % TWO32
        self.n_base, self.inc = int(n), int(inc)

    def phase(self, n0, count):
        """phi(n0 .. n0 + count - 1) as uint64"""
        p0 = (self.base + self.inc * (int(n0) - self.n_base)) % TWO32
        return (np.uint64(p0) + np.uint64(self.inc) * np.arange(count, dtype=np.uint64)) % np.uint64(TWO32)

    def rotate(self, x, n0):
        """x[i] exp(j theta(n0 + i)), theta = phi as signed 32-bit times pi / 2^31, in float64"""
        ph = self.phase(n0, len(x)).astype(np.int64)
        ph = np.where(ph >= 1 << 31, ph - TWO32, ph)
        return np.asarray(x, np.complex128) * np.exp(1j * (ph * (np.pi / 2 ** 31)))


def rx_frontend(x, n0, D, taps, nco):
    """gr_demod_base's front end for a burst x at absolute input samples n0 .. (n0 a multiple of D, zero input before it):
    rotator at the device rate, then y[k] = sum_j taps[j] r[D k - j] for every k with D k in the burst (outputs from n0 / D on)"""
    assert n0 % D == 0
    return sps.upfirdn(taps, nco.rotate(x, n0), down=D)[:(len(x) + D - 1) // D]


def tx_frontend(x, m0, N, taps, nco):
    """gr_mod_base's front end for a burst x at absolute 1 Msps inputs m0 .. (zero input before it): rotator at 1 Msps, then
    y[N m + p] = sum_i taps[p + N i] r[m - i]; N = 1 is the rotator alone"""
    r = nco.rotate(x, m0)
    return r if N == 1 else sps.upfirdn(taps, r, up=N)[:N * len(x)]


def tx_combiner(X, n0, N, taps, ncos, gain=1.0):
    """the transmit combiner for bursts X [C, m] whose first output is absolute device-rate sample n0 (zero input before them):
    per channel x N, the rotator at the device rate, sum, x 1 / C, x gain"""
    S = np.zeros(N * X.shape[1], np.complex128)
    for c in range(X.shape[0]):
        u = np.asarray(X[c], np.complex128) if N == 1 else sps.upfirdn(taps, X[c].astype(np.complex128), up=N)[:N * X.shape[1]]
        S += ncos[c].rotate(u, n0)
    return S / X.shape[0] * gain


def assert_close(got, want, where):
    """RMS error <= RMS_TOL and every sample's error <= PEAK_TOL, both relative to the RMS of want"""
    got = np.asarray(got)
    assert got.shape == want.shape, (where, got.shape, want.shape)
    scale = np.sqrt(np.mean(np.abs(want) ** 2))
    assert scale > 0, where
    err = np.abs(got.astype(np.complex128) - want)
    rms, peak = np.sqrt(np.mean(err ** 2)) / scale, np.max(err) / scale
    assert rms <= RMS_TOL and peak <= PEAK_TOL, (where, rms, peak)


def burst(seed, shape, amp=0.3):
    rng = np.random.default_rng(seed)
    return (amp * (rng.standard_normal(shape) + 1j * rng.standard_normal(shape))).astype(np.complex64)


def general(rate, k):
    """a general offset within +-rate / 2: its Q32 phase step is odd, so it is no multiple of rate / 2^12, and a phase argument that
    lost its top bit would turn the rotator by pi"""
    step = int((0.1234567 + 0.211 * k) % 0.5 * TWO32) | 1
    return (1 if k % 2 else -1) * step / TWO32 * rate


# ------------------------------------------------------------------ pinned against the oracle
@pytest.mark.parametrize("fs", [32000000, 33000000, 107000000])
def test_rx_frontend_statement_matches_the_oracle(oracle, fs):
    """zero prefix of P samples with the offset set before it, a retune after it, then a burst: the statement at absolute index P"""
    D = fs // 1000000
    taps = rx_taps(fs)
    assert len(taps) == oracle.Frontend(fs).ntaps
    P, T = D * 4096 * 3, D * 1500 + 7
    x = burst(fs, T)
    for k, (f0, f1) in enumerate([(general(fs, 1), None), (general(fs, 2), general(fs, 3)), (3 * fs / 4096, -5 * fs / 4096)]):
        o = oracle.Frontend(fs)
        nco = Nco()
        o.set_carrier_offset(f0); nco.retune(0, q32_inc(-f0, fs))
        for lo in range(0, P, 50000):
            o.work(np.zeros(min(50000, P - lo), np.complex64))
        if f1 is not None:
            o.set_carrier_offset(f1); nco.retune(P, q32_inc(-f1, fs))
        got = np.concatenate([o.work(x[:T // 3]), o.work(x[T // 3:])])
        assert_close(got, rx_frontend(x, P, D, taps, nco), (fs, k))


@pytest.mark.parametrize("fs", [5000000, 32000000])
def test_tx_frontend_statement_matches_the_oracle(fs):
    N = fs // 1000000
    taps = tx_taps(fs)
    assert len(taps) == TO.TxFrontend(fs).ntaps
    P, T = 4096 * 5, 3001
    x = burst(fs + 1, T)
    for k, (f0, f1) in enumerate([(general(1e6, 1), None), (general(1e6, 2), general(1e6, 3)), (7e6 / 4096, -11e6 / 4096)]):
        o = TO.TxFrontend(fs)
        nco = Nco()
        o.set_carrier_offset(f0); nco.retune(0, q32_inc(f0, 1e6))
        o.work(np.zeros(P, np.complex64))
        if f1 is not None:
            o.set_carrier_offset(f1); nco.retune(P, q32_inc(f1, 1e6))
        got = np.concatenate([o.work(x[:1000]), o.work(x[1000:])])
        assert_close(got, tx_frontend(x, P, N, taps, nco), (fs, k))


@pytest.mark.parametrize("Cn", [3, 33])
def test_tx_combiner_statement_matches_the_oracle(Cn):
    """offsets across +-fs/2, some general and some multiples of fs / 2^12; one channel retuned after the prefix; a gain"""
    fs = 32000000
    N = fs // 1000000
    taps = tx_taps(fs)
    P, T = 4096 * 3, 1200
    X = burst(Cn, (Cn, T), 0.2)
    offs = [(-0.5 + (c + 0.5) / Cn) * fs if c % 2 else round((-0.5 + (c + 0.5) / Cn) * 4096) * fs / 4096 for c in range(Cn)]
    o = TCO.TxCombiner(fs, Cn)
    ncos = [Nco() for _ in range(Cn)]
    for c, f in enumerate(offs):
        o.set_carrier_offset(f, c); ncos[c].retune(0, q32_inc(f, fs))
    o.work(np.zeros((Cn, P), np.complex64))
    o.set_carrier_offset(general(fs, 4) / 2, 1); ncos[1].retune(N * P, q32_inc(general(fs, 4) / 2, fs))
    o.set_gain(0.7)
    got = np.concatenate([o.work(X[:, :500]), o.work(X[:, 500:])])
    assert_close(got, tx_combiner(X, N * P, N, taps, ncos, 0.7), Cn)


# ------------------------------------------------------------------ the statement's own arithmetic
def test_nco_phase_is_exact_past_2_64_products():
    """inc (n - n_base) exceeds 2^64 at these indices: the phase must still be the exact residue"""
    nco = Nco()
    nco.retune(0, 0xDEADBEEF)
    n0 = (1 << 33) + 12345
    assert int(nco.phase(n0, 3)[2]) == (0xDEADBEEF * (n0 + 2)) % TWO32
    nco.retune((1 << 40) + 1, 0x12345)
    base = (0xDEADBEEF * ((1 << 40) + 1)) % TWO32
    assert nco.base == base
    assert int(nco.phase((1 << 40) + 11, 1)[0]) == (base + 0x12345 * 10) % TWO32


def test_general_offsets_have_odd_phase_steps():
    """the general offsets above turn by an odd number of Q32 steps: a lost top bit of the index moves their phase by pi"""
    for fs in (32000000, 33000000, 107000000):
        for k in (1, 2, 3):
            assert q32_inc(-general(fs, k), fs) % 2 == 1, (fs, k)
    for k in (1, 2, 3):
        assert q32_inc(general(1e6, k), 1e6) % 2 == 1, k
