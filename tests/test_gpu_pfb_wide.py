"""GPU tier: the polyphase channelizer / synthesizer past 64 channels (pfb_fir_kernel + pfb_dft_kernel), bit-identical to the CPU
oracle at M up to 4096: ragged host chunks, device input 8 bytes past a 16-byte boundary, synthesizer device input with a row stride
larger than the column count; synthesizer -> channelizer loop-back at M = 400; and the MMDVM bank, 400 channels of 25 kHz at 10 Msps
through qrl_mmdvm_tx -> synthesizer -> channelizer -> qrl_mmdvm_rx."""
import numpy as np
import pytest

from tests.test_gpu_pfb import device_copy, noise, pfb_read

pytestmark = pytest.mark.gpu


def rand_taps(seed, n):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32) / n


def chan_parity(q, oracle, M, taps, sizes, kinds, dev_input):
    """channelizer fed `sizes` wideband samples per call, host ("host") or device ("dev") input by turns; every call bit-identical
    to the oracle fed the same chunks"""
    x = noise(np.random.default_rng(M + len(taps)), sum(sizes))
    ch = q.PfbChannelizer(M, taps, max_in=max(sizes))
    och = oracle.PfbChannelizer(M, taps)
    lo = 0
    for i, m in enumerate(sizes):
        xi = x[lo:lo + m]
        want = och.work(xi)
        if kinds[i % len(kinds)] == "dev":
            ptr, keep = dev_input(xi)
            n = ch.work_device(ptr, m)
            got = pfb_read(q, ch, (M, max(1, n)), max(1, n))[:, :n]
            del keep
        else:
            got = ch.work(xi)
        assert got.shape == want.shape and np.array_equal(got, want), (M, len(taps), i)
        lo += m
    ch.close()


def synth_parity(q, oracle, M, taps, sizes, kinds, dev_input):
    """synthesizer fed `sizes` columns per call; device calls pass [M][stride] rows with stride > n and NaN past n"""
    rng = np.random.default_rng(7 * M + len(taps))
    z = (rng.standard_normal((M, sum(sizes))) + 1j * rng.standard_normal((M, sum(sizes)))).astype(np.complex64)
    sy = q.PfbSynthesizer(M, taps, max_in=max(sizes))
    osy = oracle.PfbSynthesizer(M, taps)
    lo = 0
    for i, m in enumerate(sizes):
        zi = z[:, lo:lo + m]
        want = osy.work(zi)
        if kinds[i % len(kinds)] == "dev":
            stride = m + 3 + 2 * i
            rows = np.full((M, stride), np.nan, np.complex64)
            rows[:, :m] = zi
            ptr, keep = dev_input(rows)
            n = sy.work_device(ptr, m, stride)
            got = pfb_read(q, sy, max(1, n), 0)[:n]
            del keep
        else:
            got = sy.work(zi)
        assert len(got) == len(want) == m * M and np.array_equal(got, want), (M, len(taps), i)
        lo += m
    sy.close()


def _dev8(x):
    return device_copy(x, 8)


# (M, taps per branch, channelizer chunk sizes, synthesizer column counts): chunks of 1, M - 3, not multiples of M, and more than
# one CTA tile (72 FIR / 64 DFT times) except at M = 4096, where the oracle's O(M^2) DFT limits the test to a few dozen columns
WIDE = [
    (65, 34, [1, 62, 65 * 150 + 7, 3, 65 * 200 + 64], [1, 5, 150, 17, 70]),
    (128, 2, [1, 125, 128 * 140 + 1, 1000, 128 * 75], [1, 3, 140, 66, 9]),
    (400, 34, [1, 397, 400 * 130 + 13, 401, 400 * 20], [1, 4, 130, 8, 65]),
    (1000, 17, [1, 997, 1000 * 70 + 999, 77], [1, 2, 70, 5]),
    (1024, 128, [1, 1021, 1024 * 66 + 5, 4099], [1, 2, 66, 3]),
    (4096, 34, [1, 4093, 4096 * 24 + 5, 4097 * 3], [1, 2, 17, 6]),
]


@pytest.mark.parametrize("M,tpf,csizes,ssizes", WIDE, ids=[str(w[0]) for w in WIDE])
def test_wide_channelizer_bit_identical(qrl, oracle, M, tpf, csizes, ssizes):
    chan_parity(qrl, oracle, M, rand_taps(M, tpf * M - 5), csizes, ("host", "dev", "host"), _dev8)


@pytest.mark.parametrize("M,tpf,csizes,ssizes", WIDE, ids=[str(w[0]) for w in WIDE])
def test_wide_synthesizer_bit_identical(qrl, oracle, M, tpf, csizes, ssizes):
    synth_parity(qrl, oracle, M, rand_taps(M + 1, tpf * M - 3), ssizes, ("dev", "host"), _dev8)


def test_create_limits(qrl):
    qrl.PfbChannelizer(4096, np.ones(4096 * 128, np.float32), max_in=8192).close()
    with pytest.raises(qrl.QrlError, match="M above 4096"):
        qrl.PfbChannelizer(4097, np.ones(4097, np.float32), max_in=8192)
    with pytest.raises(qrl.QrlError, match="bad argument"):
        qrl.PfbSynthesizer(4096, np.ones(4096 * 128 + 1, np.float32), max_in=16)


def test_wide_loop_back(qrl, oracle):
    """synthesizer(400) -> channelizer(400) at 10 Msps: channel c of the synthesizer input comes back on port c"""
    M, n, fs = 400, 3000, 10e6
    rng = np.random.default_rng(4000)
    on = {0: 1.0, 1: 0.7, 199: 0.5, 200: 0.9, 201: 0.6, 333: 0.8, 399: 0.4}
    z = (rng.standard_normal((M, n)) + 1j * rng.standard_normal((M, n))).astype(np.complex64) * 0.01
    for c, a in on.items():
        z[c] += (a * np.exp(2j * np.pi * (0.003 + 0.0001 * (c % 7)) * np.arange(n))).astype(np.complex64)
    wide = qrl.PfbSynthesizer(M, oracle.low_pass_2(M, fs, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS), max_in=n).work(z)
    back = qrl.PfbChannelizer(M, oracle.low_pass_2(1, fs, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS), max_in=len(wide)).work(wide)
    p = np.sqrt(np.mean(np.abs(back[:, 500:]) ** 2, axis=1))
    for c, a in on.items():
        assert abs(p[c] - a) < 0.05, (c, p[c])
    assert np.all(np.delete(p, list(on)) < 0.05)


BANK_ROWS = [0, 1, 37, 99, 150, 199, 200, 201, 256, 311, 398, 399]


def mmdvm_bank(q, oracle, chunks):
    """FM tones on 12 of 400 rows -> qrl_mmdvm_tx -> synthesizer(400) at 10 Msps -> + noise -> channelizer(400) in `chunks`
    -> qrl_mmdvm_rx on the same rows: int16 equal to oracle channelizer + oracle MmdvmRx per row, each tone at its frequency"""
    M, fs, n24 = 400, 10e6, 7200
    rows = BANK_ROWS
    t = np.arange(n24)
    S = np.stack([(6000 * np.sin(2 * np.pi * (300 + 130 * i) * t / 24000)).astype(np.int16) for i in range(len(rows))])
    tx = q.MmdvmChannelsTx(len(rows), rows=rows, n_rows=M, max_in=n24)
    slab = tx.work(S)
    assert slab.shape[0] == M
    sy = q.PfbSynthesizer(M, oracle.low_pass_2(M, fs, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS), max_in=slab.shape[1])
    wide = sy.work(slab)
    rng = np.random.default_rng(9601)
    wide = (wide + 0.002 * (rng.standard_normal(len(wide)) + 1j * rng.standard_normal(len(wide)))).astype(np.complex64)
    ctaps = oracle.low_pass_2(1, fs, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS)
    ch = q.PfbChannelizer(M, ctaps, max_in=max(chunks))
    parts, lo, i = [], 0, 0
    while lo < len(wide):
        m = min(chunks[i % len(chunks)], len(wide) - lo); i += 1
        parts.append(ch.work(wide[lo:lo + m])); lo += m
    chan = np.concatenate(parts, 1)
    want_chan = oracle.PfbChannelizer(M, ctaps).work(wide)
    assert np.array_equal(chan, want_chan)
    rx = q.MmdvmChannelsRx(len(rows), rows=rows, n_rows=M, max_in=chan.shape[1])
    got = rx.work(chan)[0]
    for i, r in enumerate(rows):
        want = oracle.MmdvmRx(5000).work(want_chan[r])[0]
        m = min(got.shape[1], len(want))
        assert m > 6000 and abs(got.shape[1] - len(want)) <= 1
        assert np.array_equal(got[i, :m], want[:m]), r
        seg = got[i, 1500:m].astype(np.float64)
        spec = np.abs(np.fft.rfft(seg * np.hanning(len(seg))))
        assert abs(np.argmax(spec[5:]) + 5 - (300 + 130 * i) * len(seg) / 24000) < 2, r


def test_mmdvm_bank_400_channels(qrl, oracle):
    mmdvm_bank(qrl, oracle, [1000003, 397, 1, 400 * 777 + 5, 2000000])
