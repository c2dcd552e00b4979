"""GPU tier: the display spectrum (rx_fft_c, rx_fft.cpp:44-129) through the C ABI against the CPU oracle's restatement (pinned to the
compiled reference block in tests/test_oracle_ref.py): same ready / not-ready sequence for ragged calls, dB points within 2e-4 dB on
bins above the noise floor (float FFT against the oracle's double-precision definition)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def signal(rng, S, n):
    t = np.arange(n)
    X = np.zeros((S, n), np.complex64)
    for s in range(S):
        x = 0.3 * np.exp(2j * np.pi * (0.05 + 0.11 * s) * t) + 0.02 * np.exp(-2j * np.pi * 0.31 * t)
        X[s] = (x + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    return X


def check(got, want, where):
    """A float FFT's error scales with the strongest line, not with the bin: dB within 2e-4 on bins less than 40 dB below the peak,
    and every bin's amplitude within 2e-6 of the peak amplitude (north_star's float tolerance is 1e-5 RMS)."""
    strong = want > want.max() - 40.0
    assert np.max(np.abs(got[strong] - want[strong])) < 2e-4, where
    ag, aw = 10.0 ** (got.astype(np.float64) / 20), 10.0 ** (want.astype(np.float64) / 20)
    assert np.max(np.abs(ag - aw)) < 2e-6 * aw.max(), where
    assert np.sqrt(np.mean((ag - aw) ** 2)) < 1e-5 * np.sqrt(np.mean(aw ** 2)), where


def ragged_parity(qrl, oracle, n_fft, window, S, seed, oracle_window=None):
    """S streams through one handle and through S oracle blocks in the same ragged calls (the first while disabled); every other call
    fetches the spectra: the same ready / not-ready sequence, each stream within check() and its strongest line on the right bin.
    Returns the fetched spectra."""
    rng = np.random.default_rng(seed)
    n = 7 * n_fft + 1234
    X = signal(rng, S, n)
    g = qrl.Spectrum(n_fft, window, n_streams=S, max_samples=3 * n_fft + 64)
    os_ = [oracle.Spectrum(n_fft, window if oracle_window is None else oracle_window) for _ in range(S)]
    sizes = [n_fft // 3, 17, n_fft, n_fft // 2 + 5, 2 * n_fft + 9, 100, n_fft - 1, 3 * n_fft]
    g.work(X[:, :50])                                   # disabled: dropped on both sides
    for o, x in zip(os_, X):
        o.work(x[:50])
    g.set_enabled(True)
    for o in os_:
        o.set_enabled(True)
    lo, spectra = 0, []
    for step, m in enumerate(sizes):
        m = min(m, n - lo)
        g.work(X[:, lo:lo + m])
        for o, x in zip(os_, X):
            o.work(x[lo:lo + m])
        lo += m
        if step % 2 == 1:
            got = g.get_fft_data()
            want = [o.get() for o in os_]
            assert (got is None) == (want[0] is None), step
            if got is not None:
                spectra.append(got)
                for s in range(S):
                    check(got[s], want[s], (step, s))
                    f = (0.05 + 0.11 * s + 0.5) % 1.0 - 0.5                    # stream s's strong line, aliased into [-fs/2, fs/2)
                    assert abs(int(np.argmax(got[s])) - (n_fft // 2 + round(f * n_fft))) <= 1, (step, s)
    assert len(spectra) >= 3
    g.close()
    return spectra


@pytest.mark.parametrize("n_fft", [256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536])
def test_spectrum_matches_the_oracle(qrl, oracle, n_fft):
    """every size the handle accepts: each is its own (N1, N2) split of the four-step FFT"""
    ragged_parity(qrl, oracle, n_fft, oracle.WIN_BLACKMAN_HARRIS, 3, 8100 + n_fft)


@pytest.mark.parametrize("window", [0, 1, 2, 3, 5])
def test_spectrum_windows(qrl, oracle, window):
    """Hamming, Hann, Blackman, rectangular and Blackman-Harris against the oracle's window of the same type"""
    ragged_parity(qrl, oracle, 4096, window, 3, 8300 + window)


def test_spectrum_out_of_range_window_is_hamming(qrl, oracle):
    """a window type outside 0..7 is Hamming (rx_fft.cpp:176-179): bit for bit what type 0 gives, and the oracle's Hamming"""
    ham = ragged_parity(qrl, oracle, 4096, 0, 3, 8400)
    for window in (-1, 8, 9):
        got = ragged_parity(qrl, oracle, 4096, window, 3, 8400, oracle_window=oracle.WIN_HAMMING)
        assert len(got) == len(ham) and all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, ham)), window


@pytest.mark.parametrize("window", [4, 6, 7])
def test_spectrum_refuses_the_windows_it_does_not_build(qrl, window):
    """Kaiser, Bartlett and flat-top are valid types that this handle does not build: create fails instead of using another window"""
    with pytest.raises(qrl.QrlError, match="window type not built"):
        qrl.Spectrum(4096, window)


def test_spectrum_many_streams(qrl, oracle):
    """37 streams from host input (a stream per channel of a batch): every stream against its own oracle block"""
    ragged_parity(qrl, oracle, 1024, oracle.WIN_BLACKMAN_HARRIS, 37, 8500)


def test_spectrum_set_fft_size_and_device_input(qrl, oracle):
    import torch
    rng = np.random.default_rng(8200)
    X = signal(rng, 2, 40000)
    g = qrl.Spectrum(4096, 5, n_streams=2, max_samples=40000)
    o = oracle.Spectrum(4096, oracle.WIN_BLACKMAN_HARRIS)
    g.set_enabled(True); o.set_enabled(True)
    Xd = torch.from_numpy(X).cuda()
    g.work_device(Xd.data_ptr(), 5000, Xd.shape[1]); o.work(X[0, :5000])
    a, b = g.get_fft_data(), o.get()
    assert a is not None
    check(a[0], b, 0)
    g.set_fft_size(1024); o.set_fft_size(1024)
    assert g.get_fft_data() is None and o.get() is None
    g.work_device(Xd[:, 5000:].data_ptr(), 3000, Xd.shape[1]); o.work(X[0, 5000:8000])
    a, b = g.get_fft_data(), o.get()
    assert a.shape == (2, 1024)
    check(a[0], b, 1)
    with pytest.raises(qrl.QrlError):
        qrl.Spectrum(3000, 5)
