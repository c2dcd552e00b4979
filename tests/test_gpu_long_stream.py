"""GPU tier: every streaming handle driven past 2^31 and 2^32 samples.  Each case feeds a zero prefix from one zero-filled device buffer,
reused call after call, then a short burst of signal, and checks the burst's output two ways:
(a) bit-exact (by value: a rotated exact zero may carry the other sign) against a fresh twin with the same settings fed only the burst,
    where the prefix is a multiple of every rate change and frame period and the offsets are multiples of rate / 2^12, so the prefix
    leaves zero history and the phase back at its base;
(b) within the float budget of the float64 statement at the absolute index (tests/test_long_stream_reference.py, pinned there against
    the oracle), for general offsets too, set before the prefix (a phase argument that lost a high bit turns them by pi) or retuned
    after it (n_base above 2^32).
The host-thread build cannot run 2^32 samples: skipped under QRL_EMULATED_LIB."""
import math
import os
import time

import numpy as np
import pytest

from tests import siggen
from tests import test_long_stream_reference as R
from tests.test_gpu_dispatch import free_device

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(bool(os.environ.get("QRL_EMULATED_LIB")), reason="2^32 samples are out of reach of the host-thread build")]

TWO31, TWO32 = 1 << 31, 1 << 32
PAST_2_32 = TWO32 + TWO31   # past 2^32 with bit 31 of the index set: a phase argument cut to 31 bits moves an odd step's phase by pi
CALL = 1 << 26              # device-rate samples per zero-prefix call


def past(threshold, period, at_least=0):
    """the smallest multiple of period above threshold and not below at_least"""
    return max(threshold // period + 1, -(-at_least // period)) * period


def device_zeros(shape):
    import torch
    z = torch.zeros(shape, dtype=torch.complex64, device="cuda")
    torch.cuda.synchronize()
    return z


def feed_zeros(work, n, upto, per_call):
    """work(m) consumes m zero samples; from absolute position n up to `upto`; returns upto"""
    while n < upto:
        m = min(per_call, upto - n)
        work(m)
        n += m
    return n


def timed(fn):
    t0 = time.perf_counter()
    fn()
    print("%s: %.1f s" % (fn.__name__, time.perf_counter() - t0))


# ------------------------------------------------------------------ receive front end (rotator + /N)
@pytest.mark.parametrize("fs,shared", [(32000000, True), (33000000, True), (107000000, True), (107000000, False)])
def test_frontend_past_2_31_and_2_32(qrl, fs, shared):
    """3 channels: channel 0 at multiples of fs / 2^12 (a), channels 1 and 2 at general offsets (b); a burst past 2^31, then one past
    2^32 after channel 0 and channel 2 retune there.  Stride 0 runs frontend_shared_kernel up to 32 Msps and frontend_fir_kernel
    above; per-channel rows run frontend_fir_kernel."""
    D, Cn = fs // 1000000, 3
    taps = R.rx_taps(fs)
    step = math.lcm(D, 4096)
    T = D * 2048 + 5
    offs = [3 * fs / 4096, R.general(fs, 1), R.general(fs, 2)]
    retunes = {0: -5 * fs / 4096, 2: R.general(fs, 3)}

    def case():
        fe = qrl.Frontend(fs, n_channels=Cn, max_in=CALL)
        ncos = [R.Nco() for _ in range(Cn)]
        for c, f in enumerate(offs):
            fe.set_carrier_offset(f, channel=c); ncos[c].retune(0, R.q32_inc(-f, fs))
        z = device_zeros(CALL if shared else (Cn, CALL))
        n = 0
        for stage, thresh in enumerate((TWO31, PAST_2_32)):
            B = past(thresh, step, n + 4 * len(taps))
            n = feed_zeros(lambda m: fe.work_device(z.data_ptr(), m, 0 if shared else CALL), n, B, CALL)
            assert n == B > thresh
            cur = list(offs)
            if stage == 1:
                for c, f in retunes.items():
                    fe.set_carrier_offset(f, channel=c); ncos[c].retune(B, R.q32_inc(-f, fs)); cur[c] = f
            x = R.burst(fs + stage, T if shared else (Cn, T))
            got = fe.work(x)
            twin = qrl.Frontend(fs, n_channels=Cn, max_in=T)
            for c, f in enumerate(cur):
                twin.set_carrier_offset(f, channel=c)
            want = twin.work(x)
            twin.close()
            assert np.array_equal(got[0], want[0]), (fs, shared, B)
            for c in range(Cn):
                R.assert_close(got[c], R.rx_frontend(x if shared else x[c], B, D, taps, ncos[c]), (fs, shared, B, c))
            n += T
        fe.close()
        del z
        free_device()
    timed(case)


# ------------------------------------------------------------------ transmit front end (rotator at 1 Msps + xN)
@pytest.mark.parametrize("N", [32, 5])
def test_tx_frontend_past_2_32_outputs(qrl, N):
    """2^32 device-rate outputs are 2^32 / N inputs: the rotator's index runs at 1 Msps.  Channel 0 at multiples of 1e6 / 2^12 (a),
    channels 1 and 2 general (b), channels 0 and 2 retuned after the prefix."""
    fs, Cn = N * 1000000, 3
    taps = R.tx_taps(fs)
    per_call = CALL // N
    T = 2048 + 3
    offs = [7e6 / 4096, R.general(1e6, 1), R.general(1e6, 2)]
    retunes = {0: -11e6 / 4096, 2: R.general(1e6, 3)}

    def case():
        fe = qrl.TxFrontend(fs, n_channels=Cn, max_in=per_call)
        ncos = [R.Nco() for _ in range(Cn)]
        for c, f in enumerate(offs):
            fe.set_carrier_offset(f, channel=c); ncos[c].retune(0, R.q32_inc(f, 1e6))
        z = device_zeros((Cn, per_call))
        B = past(TWO32 // N, 4096)
        feed_zeros(lambda m: fe.work_device(z.data_ptr(), m, per_call), 0, B, per_call)
        assert N * B > TWO32
        cur = list(offs)
        for c, f in retunes.items():
            fe.set_carrier_offset(f, channel=c); ncos[c].retune(B, R.q32_inc(f, 1e6)); cur[c] = f
        x = R.burst(N, (Cn, T))
        got = fe.work(x)
        twin = qrl.TxFrontend(fs, n_channels=Cn, max_in=T)
        for c, f in enumerate(cur):
            twin.set_carrier_offset(f, channel=c)
        want = twin.work(x)
        twin.close()
        assert np.array_equal(got[0], want[0]), (N, B)
        for c in range(Cn):
            R.assert_close(got[c], R.tx_frontend(x[c], B, N, taps, ncos[c]), (N, B, c))
        fe.close()
        del z
        free_device()
    timed(case)


# ------------------------------------------------------------------ transmit combiner (xN, rotator at the device rate, sum)
@pytest.mark.parametrize("Cn", [3, 33])
def test_tx_combiner_past_2_32_outputs(qrl, Cn):
    """offsets across +-fs / 2: even channels at multiples of fs / 2^12, odd channels general; channels 0 and 1 retuned after the
    prefix, so channel 1's n_base is above 2^32.  Burst A drives the even channels only and must equal a fresh twin's output (a);
    after a zero gap, burst B drives every channel and is held to the statement (b)."""
    fs, N = 32000000, 32
    taps = R.tx_taps(fs)
    per_call = CALL // N
    T, gap = 2048 + 3, 4096
    offs = [round((-0.5 + (c + 0.5) / Cn) * 4096) * fs / 4096 if c % 2 == 0 else R.general(fs, c) for c in range(Cn)]
    retunes = {0: -(5 * fs) / 4096, 1: R.general(fs, Cn + 1)}

    def case():
        t = qrl.TxCombiner(fs, n_channels=Cn, max_in=per_call)
        t.set_gain(0.7)
        ncos = [R.Nco() for _ in range(Cn)]
        for c, f in enumerate(offs):
            t.set_carrier_offset(f, channel=c); ncos[c].retune(0, R.q32_inc(f, fs))
        z = device_zeros((Cn, per_call))
        rows = [z.data_ptr() + 8 * per_call * c for c in range(Cn)]
        B = past(PAST_2_32 // N, 4096)
        feed_zeros(lambda m: t.work_device(rows, m), 0, B, per_call)
        assert N * B > PAST_2_32
        cur = list(offs)
        for c, f in retunes.items():
            t.set_carrier_offset(f, channel=c); ncos[c].retune(N * B, R.q32_inc(f, fs)); cur[c] = f
        xa = R.burst(Cn, (Cn, T), 0.2)
        xa[1::2] = 0
        got = t.work(xa)
        twin = qrl.TxCombiner(fs, n_channels=Cn, max_in=T)
        twin.set_gain(0.7)
        for c, f in enumerate(cur):
            twin.set_carrier_offset(f, channel=c)
        want = twin.work(xa)
        twin.close()
        assert np.array_equal(got, want), (Cn, B)
        t.work(np.zeros((Cn, gap), np.complex64))
        xb = R.burst(Cn + 1, (Cn, T), 0.2)
        R.assert_close(t.work(xb), R.tx_combiner(xb, N * (B + T + gap), N, taps, ncos, 0.7), (Cn, B))
        t.close()
        del z
        free_device()
    timed(case)


# ------------------------------------------------------------------ polyphase channelizer / synthesizer
@pytest.mark.parametrize("M", [400, 4096])
def test_pfb_past_2_32_wideband_samples(qrl, M):
    """the channelizer after a zero prefix of P > 2^32 wideband samples (P a multiple of M), the synthesizer after P / M zero columns:
    the burst's output equals a fresh twin's"""
    taps = (0.05 * np.random.default_rng(M).standard_normal(6 * M - 5)).astype(np.float32)
    P = past(TWO32, M)

    def case():
        ch = qrl.PfbChannelizer(M, taps, max_in=CALL)
        z = device_zeros(CALL)
        assert feed_zeros(lambda m: ch.work_device(z.data_ptr(), m), 0, P, CALL) == P > TWO32
        x = R.burst(M, 64 * M + 17)
        got = ch.work(x)
        want = qrl.PfbChannelizer(M, taps, max_in=len(x)).work(x)
        assert got.shape == want.shape and np.array_equal(got, want), M
        ch.close()
        del z
        cols = CALL // M
        sy = qrl.PfbSynthesizer(M, taps, max_in=cols)
        z = device_zeros((M, cols))
        assert M * feed_zeros(lambda m: sy.work_device(z.data_ptr(), m, cols), 0, P // M, cols) > TWO32
        x = R.burst(M + 1, (M, 64))
        got = sy.work(x)
        want = qrl.PfbSynthesizer(M, taps, max_in=64).work(x)
        assert got.shape == want.shape and np.array_equal(got, want), M
        sy.close()
        del z
        free_device()
    timed(case)


# ------------------------------------------------------------------ receive chains at 1 Msps, one channel, the rotator on
RX_STEP = 4096 * 125    # a multiple of 4096 (the offsets below) and of every decimation and resampler period of the two chains


def _rx_case(qrl, make, x):
    """the carrier offset (a multiple of 1e6 / 2^12) set before a zero prefix of P > 2^32 samples and retuned after it, RSSI on; then
    the burst x, moved to the retuned offset.  Port 0 (feed-forward) and the RSSI value must equal a fresh twin's fed the burst alone.  Returns the handle, for
    the caller's checks of what the loops made of the burst (their state is carried across the prefix, so not compared bit for
    bit)."""
    blk = make(CALL)
    blk.enable_rssi(True)
    blk.set_carrier_offset(3e6 / 4096)
    z = device_zeros(CALL)
    P = past(TWO32, RX_STEP)
    assert feed_zeros(lambda m: blk.work_device(z.data_ptr(), m, CALL), 0, P, CALL) == P > TWO32
    blk.set_carrier_offset(-7e6 / 4096)
    x = (x * np.exp(2j * np.pi * (-7e6 / 4096) * np.arange(len(x)) / 1e6)).astype(np.complex64)     # the signal sits at the offset
    blk.work(x[None, :])
    twin = make(len(x))
    twin.enable_rssi(True)
    twin.set_carrier_offset(-7e6 / 4096)
    twin.work(x[None, :])
    got, want = blk.read_port(0)[0], twin.read_port(0)[0]
    assert len(got) == len(want) > 0 and np.array_equal(got, want)
    assert np.array_equal(blk.rssi(), twin.rssi())
    twin.close()
    del z
    free_device()
    return blk


def test_4fsk_fm_past_2_32_samples(qrl):
    """the headline chain (QRL_DEMOD_4FSK, FM, the fused front end): the burst's decoded frames are the planted payloads"""
    from tests.test_gpu_dispatch import F4
    X, payloads = siggen.gen_4fsk_channels(1, 1 << 20, seed0=4321)

    def case():
        blk = _rx_case(qrl, lambda m: qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=1, max_samples=m), X[0])
        good, found = siggen.count_good_frames(blk.read_port(2)[0], *F4, payloads[0])
        assert good >= 1 and good >= len(payloads[0]) - 6, (good, found, len(payloads[0]))
        blk.close()
    timed(case)


def test_nbfm_past_2_32_samples(qrl):
    """QRL_DEMOD_NBFM: the burst's audio carries its 1 kHz tone, within the NBFM parity test's 12 Hz"""
    x = siggen.gen_nbfm_channels(1, 1 << 19, seed0=1)[0]

    def case():
        blk = _rx_case(qrl, lambda m: qrl.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=1, max_samples=m), x)
        seg = blk.read_port(1)[0][2000:4000].astype(np.float64)
        assert len(seg) == 2000
        f = np.fft.rfftfreq(len(seg), 1 / 8000.0)
        pk = f[np.argmax(np.abs(np.fft.rfft(seg * np.hanning(len(seg)))))]
        assert abs(pk - 1000.0) < 12.0, pk
        blk.close()
    timed(case)
