"""GPU tier: polyphase channelizer / synthesizer (SURVEY 8f row 1) against the CPU oracle: bit-identical float
streams, chunk invariance (ragged chunk sizes, not multiples of M), generic (M, taps) shapes, the reference's
M = 10 / 341-tap configuration, synthesizer -> channelizer loop-back, and channelizer -> 4FSK demod chaining."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def rel_rms(a, b):
    return float(np.sqrt(np.mean(np.abs(a - b) ** 2)) / max(1e-30, np.sqrt(np.mean(np.abs(b) ** 2))))


def noise(rng, n):
    return ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.3).astype(np.complex64)


def test_channelizer_reference_config_bit_identical_and_chunked(qrl, oracle):
    taps = oracle.low_pass_2(1, 250000, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS)      # gr_demod_mmdvm_multi2.cpp:56-57
    assert len(taps) == 341
    rng = np.random.default_rng(11)
    x = noise(rng, 200003)
    x[:50000] += np.exp(2j * np.pi * (3 * 25000 + 800) * np.arange(50000) / 250000).astype(np.complex64)
    want = oracle.PfbChannelizer(10, taps).work(x)
    ch = qrl.PfbChannelizer(10, taps, max_in=len(x))
    got = ch.work(x)
    assert got.shape == want.shape == (10, 20000)
    assert rel_rms(got, want) <= 1e-5
    assert np.array_equal(got, want)
    # ragged chunks: sizes that are not multiples of M, odd, tiny, larger than one tile
    ch2 = qrl.PfbChannelizer(10, taps, max_in=70001)
    parts, lo, i = [], 0, 0
    sizes = [1, 9, 10, 11, 70001, 2881, 3, 12345, 7]
    while lo < len(x):
        n = min(sizes[i % len(sizes)], len(x) - lo); i += 1
        parts.append(ch2.work(x[lo:lo + n])); lo += n
    got2 = np.concatenate(parts, axis=1)
    assert np.array_equal(got2, want)
    assert ch.launches >= 2


# Shapes the generic kernels serve, up to the largest qrl_pfb_create accepts (M = 64, 128 taps per branch): M = 64 on either side of
# 65 taps per branch (4160 taps), where the synthesizer's window passes 48 KiB of shared memory, and M = 48 / 63 / 33 beyond it; odd
# M; M = 2; and M = 10 with 34 and 36 taps per branch, next to the register-tiled M = 10 / 35 shape.
GENERIC_SHAPES = [(64, 8192), (64, 4160), (64, 4161), (48, 88 * 48), (63, 8001), (33, 1000), (2, 256), (10, 340), (10, 351)]


@pytest.mark.parametrize("M,ntaps", [(4, 33), (7, 50), (16, 161), (10, 101), (1, 9)] + GENERIC_SHAPES)
def test_channelizer_generic_shapes(qrl, oracle, M, ntaps):
    rng = np.random.default_rng(100 + M)
    taps = rng.standard_normal(ntaps).astype(np.float32) / ntaps
    n1 = max(4096, 2 * ntaps)                   # the last call's filters reach back into the first call, not into the initial zeros
    x = noise(rng, n1 + 904 + M + 3)
    want = oracle.PfbChannelizer(M, taps).work(x)
    ch = qrl.PfbChannelizer(M, taps, max_in=n1)
    got = np.concatenate([ch.work(x[:n1]), ch.work(x[n1:n1 + 1]), ch.work(x[n1 + 1:])], axis=1)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_synthesizer_matches_oracle_and_loops_back(qrl, oracle):
    taps = oracle.low_pass_2(10, 250000, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS)     # gr_mod_mmdvm_multi2.cpp:88-89
    rng = np.random.default_rng(12)
    n = 4000
    z = np.zeros((10, n), np.complex64)
    z[3] = np.exp(2j * np.pi * 0.01 * np.arange(n)); z[9] = 0.5 * np.exp(-2j * np.pi * 0.02 * np.arange(n))
    z += (rng.standard_normal((10, n)) + 1j * rng.standard_normal((10, n))).astype(np.complex64) * 0.01
    want = oracle.PfbSynthesizer(10, taps).work(z)
    sy = qrl.PfbSynthesizer(10, taps, max_in=n)
    got = np.concatenate([sy.work(z[:, :17]), sy.work(z[:, 17:1000]), sy.work(z[:, 1000:])])
    assert len(got) == len(want) == n * 10 and np.array_equal(got, want)
    # loop-back: channel c of the synthesizer input comes back on port c of the channelizer
    ctaps = oracle.low_pass_2(1, 250000, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS)
    back = qrl.PfbChannelizer(10, ctaps, max_in=len(got)).work(got)
    p = np.sqrt(np.mean(np.abs(back[:, 500:]) ** 2, axis=1))
    assert abs(p[3] - 1.0) < 0.05 and abs(p[9] - 0.5) < 0.05 and np.all(np.delete(p, [3, 9]) < 0.05)
    assert qrl.mmdvm_port_map(7) == [0, 1, 2, 3, 9, 8, 7]


@pytest.mark.parametrize("M,ntaps", [(4, 33), (7, 50), (16, 161), (1, 9)] + GENERIC_SHAPES)
def test_synthesizer_generic_shapes(qrl, oracle, M, ntaps):
    rng = np.random.default_rng(200 + M)
    taps = rng.standard_normal(ntaps).astype(np.float32) / ntaps
    z = (rng.standard_normal((M, 700)) + 1j * rng.standard_normal((M, 700))).astype(np.complex64)
    want = oracle.PfbSynthesizer(M, taps).work(z)
    sy = qrl.PfbSynthesizer(M, taps, max_in=512)
    got = np.concatenate([sy.work(z[:, :512]), sy.work(z[:, 512:513]), sy.work(z[:, 513:])])
    assert np.array_equal(got, want)


def device_copy(x, offset):
    """x (any shape) copied to a fresh GPU buffer starting `offset` bytes (0 or 8) past a 16-byte boundary: (device pointer, owner)"""
    import torch
    k = offset // 8
    buf = torch.zeros(x.size + 2, dtype=torch.complex64, device="cuda")        # torch's allocations are 512-byte aligned
    buf[k:k + x.size] = torch.from_numpy(np.ascontiguousarray(x).reshape(-1))
    torch.cuda.synchronize()
    ptr = buf.data_ptr() + offset
    assert ptr % 16 == offset
    return ptr, buf


def pfb_read(qrl, h, shape, dst_stride):
    import ctypes as C
    out = np.zeros(shape, np.complex64)
    assert qrl.load_library().qrl_pfb_read(h._h, out.ctypes.data_as(C.c_void_p), dst_stride) == 0
    return out


def _chan_taps(oracle, M):
    if M == 10:
        return oracle.low_pass_2(1, 250000, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS)         # 341 taps: the tiled kernel
    return np.random.default_rng(300 + M).standard_normal(50).astype(np.float32) / 50


@pytest.mark.parametrize("offset", [0, 8])
@pytest.mark.parametrize("M", [10, 7])
def test_channelizer_device_input(qrl, oracle, M, offset):
    """Wideband input already on the device, at a 16-byte boundary (M = 10: the tiled kernel's cp.async.bulk window fetch) and 8 bytes
    past one (its plain-load fetch), alternating with host calls on one handle: chunks of 1, fewer than M, odd, and several CTA tiles
    (288 outputs at M = 10, 292 at M = 7); every call bit-identical to the oracle fed the same chunks."""
    taps = _chan_taps(oracle, M)
    big = 3 * 300 * M + 5
    sizes = [1, M - 3, 1001, big, 1, M - 3, 1001, big, 4000]
    kinds = ("dev", "host", "dev")
    x = noise(np.random.default_rng(400 + M), sum(sizes))
    ch = qrl.PfbChannelizer(M, taps, max_in=big)
    och = oracle.PfbChannelizer(M, taps)
    lo = 0
    for i, m in enumerate(sizes):
        xi = x[lo:lo + m]
        want = och.work(xi)
        if kinds[i % len(kinds)] == "dev":
            ptr, keep = device_copy(xi, offset)
            n = ch.work_device(ptr, m)
            got = pfb_read(qrl, ch, (M, max(1, n)), max(1, n))[:, :n]            # waits for the handle's stream: keep may go
            del keep
        else:
            got = ch.work(xi)
        assert got.shape == want.shape and np.array_equal(got, want), (M, offset, i)
        lo += m


@pytest.mark.parametrize("M,ntaps", [(10, 341), (7, 50)])
def test_synthesizer_device_input(qrl, oracle, M, ntaps):
    """[M][stride] input on the device with stride > n_in, 8 bytes past a 16-byte boundary, alternating with host calls: ragged column
    counts (1, 5, more than one 320-column CTA of the tiled kernel, 17, the rest); every call bit-identical to the oracle."""
    taps = (oracle.low_pass_2(M, 250000, 5000, 2000, 60, oracle.WIN_BLACKMAN_HARRIS) if M == 10
            else np.random.default_rng(500 + M).standard_normal(ntaps).astype(np.float32) / ntaps)
    assert len(taps) == ntaps
    rng = np.random.default_rng(600 + M)
    sizes = [1, 5, 700, 17, 1, 333, 250]
    kinds = ("dev", "host")
    z = (rng.standard_normal((M, sum(sizes))) + 1j * rng.standard_normal((M, sum(sizes)))).astype(np.complex64)
    sy = qrl.PfbSynthesizer(M, taps, max_in=max(sizes))
    osy = oracle.PfbSynthesizer(M, taps)
    lo = 0
    for i, m in enumerate(sizes):
        zi = z[:, lo:lo + m]
        want = osy.work(zi)
        if kinds[i % len(kinds)] == "dev":
            stride = m + 3 + 2 * i
            rows = np.zeros((M, stride), np.complex64)
            rows[:, :m] = zi
            rows[:, m:] = np.nan                # the columns past n_in must not be read
            ptr, keep = device_copy(rows, 8)
            n = sy.work_device(ptr, m, stride)
            got = pfb_read(qrl, sy, max(1, n), 0)[:n]
            del keep
        else:
            got = sy.work(zi)
        assert len(got) == len(want) == m * M and np.array_equal(got, want), (M, i)
        lo += m


def test_channelizer_feeds_the_demodulator_on_device(qrl, oracle):
    """The channelizer's [M][stride] device output is the demodulator's device-resident input: wideband 10 Msps ->
    10 channels at 1 Msps -> make_gr_demod_4fsk, bits bit-exact against oracle channelizer + oracle demodulator."""
    from tests import siggen
    M, T = 10, 1 << 17
    X, _ = siggen.gen_4fsk_channels(4, T, seed0=7700)
    z = np.zeros((M, T), np.complex64)
    ports = qrl.mmdvm_port_map(4)
    for i, p in enumerate(ports):
        z[p] = X[i]
    st = oracle.low_pass(M, 1e7, 300e3, 150e3, oracle.WIN_BLACKMAN_HARRIS)
    ct = oracle.low_pass(1, 1e7, 300e3, 150e3, oracle.WIN_BLACKMAN_HARRIS)
    wide = qrl.PfbSynthesizer(M, st, max_in=T).work(z)
    assert len(wide) == M * T
    want_ch = oracle.PfbChannelizer(M, ct).work(wide)
    ch = qrl.PfbChannelizer(M, ct, max_in=len(wide))
    import ctypes as C
    n = C.c_long()
    L = qrl.load_library()
    assert L.qrl_pfb_work(ch._h, wide.ctypes.data_as(C.c_void_p), len(wide), 0, 0, C.byref(n)) == 0
    ch.sync()
    ptr, stride, items = ch.out_device()
    assert items == T == n.value
    rx = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=M, max_samples=T)
    rx.work_device(ptr, T, stride)
    bits = rx.read_port(2)
    for i, p in enumerate(ports):
        o = oracle.Rx(oracle.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1)
        o.work(want_ch[p])
        assert np.array_equal(bits[p], o.port(2)), p
        assert len(bits[p]) > 100
