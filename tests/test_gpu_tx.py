"""GPU tier: CUDA TX chains (make_gr_mod_4fsk / make_gr_mod_qpsk) against the CPU oracle: 1 Msps IQ within 1e-5 RMS
(bit-identical in practice), state carried across calls, and a GPU TX -> GPU RX loop-back recovering the frames."""
import numpy as np
import pytest

from tests import siggen

pytestmark = pytest.mark.gpu


def rel_rms(a, b):
    return float(np.sqrt(np.mean(np.abs(a - b) ** 2)) / max(1e-30, np.sqrt(np.mean(np.abs(b) ** 2))))


def test_tx_4fsk_matches_oracle_and_streams(qrl, oracle):
    C, n = 3, 200
    rng = np.random.default_rng(5000)
    data = rng.integers(0, 256, (C, n), dtype=np.uint8)
    tx = qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=C, max_items=n)
    got = tx.work(data)
    assert got.shape == (C, n * 4000)
    for c in range(C):
        o = oracle.Tx(oracle.MOD_4FSK, 25, 1000000, 1700, 3500, 1)
        want = o.work(data[c])
        assert len(want) == got.shape[1]
        assert rel_rms(got[c], want) <= 1e-5
        assert np.array_equal(got[c], want)
    # same bytes in three uneven calls: identical stream (filter history, phase accumulator, LFSR, encoder carried)
    tx2 = qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=C, max_items=n)
    parts = [tx2.work(data[:, a:b]) for a, b in ((0, 1), (1, 77), (77, n))]
    assert np.array_equal(np.concatenate(parts, axis=1), got)
    assert np.max(np.abs(got)) <= 1.0


def test_tx_qpsk_matches_oracle(qrl, oracle):
    C, n = 2, 3000
    rng = np.random.default_rng(5100)
    data = rng.integers(0, 256, (C, n), dtype=np.uint8)
    tx = qrl.make_gr_mod_qpsk(4, 1000000, 1700, 160000, n_channels=C, max_items=n)
    got = tx.work(data)
    assert got.shape == (C, n * 32)
    for c in range(C):
        want = oracle.Tx(oracle.MOD_QPSK, 4, 1000000, 1700, 160000, 0).work(data[c])
        assert np.array_equal(got[c], want)


def test_gpu_tx_to_gpu_rx_loopback(qrl):
    """config-5 TX chain feeding the config-2 RX chain, everything on the GPU: every frame comes back."""
    C = 4
    streams, payloads = [], []
    for c in range(C):
        d, pl = siggen.frames_4fsk(np.random.default_rng(7000 + c), 60)
        streams.append(d); payloads.append(pl)
    n = max(len(d) for d in streams)
    data = np.full((C, n), 0xAA, np.uint8)
    for c, d in enumerate(streams):
        data[c, :len(d)] = d
    tx = qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=C, max_items=n)
    iq = tx.work(data)
    rng = np.random.default_rng(1)
    iq = (0.8 * iq + 0.02 * (rng.standard_normal(iq.shape) + 1j * rng.standard_normal(iq.shape))).astype(np.complex64)
    rx = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=C, max_samples=iq.shape[1])
    rx.work(iq)
    bits = rx.read_port(2)
    for c in range(C):
        good, found = siggen.count_good_frames(bits[c], 0xED89AA, 24, 7, payloads[c])
        assert good >= len(payloads[c]) - 4 and found - good <= 1, (c, good, found)


TX_CASES = [
    # name, python factory name, args (reference instances gr_mod_base.cpp:155-177), oracle kind, oracle args, bytes
    ("4fsk1kfm", "make_gr_mod_4fsk", (50, 1000000, 1700, 2000, True), "MOD_4FSK", (50, 1000000, 1700, 2000, 1), 60),
    ("4fsk10kfm", "make_gr_mod_4fsk", (5, 1000000, 1700, 20000, True), "MOD_4FSK", (5, 1000000, 1700, 20000, 1), 600),
    ("4fsk2k", "make_gr_mod_4fsk", (25, 1000000, 1700, 4000, False), "MOD_4FSK", (25, 1000000, 1700, 4000, 0), 100),
    ("4fsk100k", "make_gr_mod_4fsk", (2, 1000000, 1700, 125000, True), "MOD_4FSK", (2, 1000000, 1700, 125000, 1), 3000),
    ("qpsk20k", "make_gr_mod_qpsk", (100, 1000000, 1700, 6500), "MOD_QPSK", (100, 1000000, 1700, 6500, 0), 300),
    ("qpsk2k", "make_gr_mod_qpsk", (500, 1000000, 1700, 1300), "MOD_QPSK", (500, 1000000, 1700, 1300, 0), 60),
    ("bpsk2k", "make_gr_mod_bpsk", (250, 1000000, 1700, 2800), "MOD_BPSK", (250, 1000000, 1700, 2800, 0), 60),
    ("bpsk1k", "make_gr_mod_bpsk", (500, 1000000, 1700, 1500), "MOD_BPSK", (500, 1000000, 1700, 1500, 0), 40),
    ("2fsk2kfm", "make_gr_mod_2fsk", (25, 1000000, 1700, 4000, True), "MOD_2FSK", (25, 1000000, 1700, 4000, 1), 100),
    ("2fsk1kfm", "make_gr_mod_2fsk", (50, 1000000, 1700, 2500, True), "MOD_2FSK", (50, 1000000, 1700, 2500, 1), 60),
    ("2fsk2k", "make_gr_mod_2fsk", (25, 1000000, 1700, 4000, False), "MOD_2FSK", (25, 1000000, 1700, 4000, 0), 100),
    ("2fsk10kfm", "make_gr_mod_2fsk", (5, 1000000, 1700, 25000, True), "MOD_2FSK", (5, 1000000, 1700, 25000, 1), 600),
]


@pytest.mark.parametrize("name,factory,args,okind,oargs,nbytes", TX_CASES)
def test_tx_all_digital_modes(qrl, oracle, name, factory, args, okind, oargs, nbytes):
    C = 2
    rng = np.random.default_rng(5200)
    data = rng.integers(0, 256, (C, nbytes), dtype=np.uint8)
    tx = getattr(qrl, factory)(*args, n_channels=C, max_items=nbytes)
    cut = nbytes // 3
    got = np.concatenate([tx.work(data[:, :cut]), tx.work(data[:, cut:])], axis=1)      # two calls: state carried
    for c in range(C):
        want = getattr(oracle, "Tx")(getattr(oracle, okind), *oargs).work(data[c])
        assert got.shape[1] == len(want), (got.shape, len(want))
        assert rel_rms(got[c], want) <= 1e-5
        assert np.array_equal(got[c], want), name


@pytest.mark.parametrize("kind", ["nbfm2500", "nbfm5000", "usb", "lsb"])
def test_tx_analog_modulators(qrl, oracle, kind):
    """NBFM / SSB modulators (8 ksps float audio in) against the oracle, streamed in three uneven calls."""
    C, n = 2, 4000
    t = np.arange(n)
    audio = np.stack([(0.5 * np.sin(2 * np.pi * (700 + 300 * c) * t / 8000) + 0.3 * np.sin(2 * np.pi * 1900 * t / 8000 + c)).astype(np.float32)
                      for c in range(C)])
    if kind.startswith("nbfm"):
        fw = int(kind[4:])
        tx = qrl.make_gr_mod_nbfm(20, 1000000, 1700, fw, n_channels=C, max_items=n)
        okind, oargs = oracle.MOD_NBFM, (20, 1000000, 1700, fw, 0)
    else:
        sb = 1 if kind == "lsb" else 0
        tx = qrl.make_gr_mod_ssb(125, 1000000, 1700, 2700, sb, n_channels=C, max_items=n)
        okind, oargs = oracle.MOD_SSB, (125, 1000000, 1700, 2700, sb)
    got = np.concatenate([tx.work_audio(audio[:, a:b]) for a, b in ((0, 1), (1, 1501), (1501, n))], axis=1)
    for c in range(C):
        want = oracle.Tx(okind, *oargs).work(audio[c])
        assert got.shape[1] == len(want), (got.shape, len(want))
        assert rel_rms(got[c], want) <= 1e-5
        assert np.array_equal(got[c], want), kind


@pytest.mark.parametrize("sps,fw,nbytes", [(50, 4000, 40), (100, 2000, 24), (10, 20000, 120)])
def test_tx_gmsk_matches_oracle_and_loops_back(qrl, oracle, sps, fw, nbytes):
    """gr_mod_gmsk (GMSK2K / 1K / 10K instances): bit-identical to the oracle with the state carried across calls; the
    GMSK2K output is demodulated by the CUDA GMSK receiver."""
    C = 2
    rng = np.random.default_rng(5300 + sps)
    data = rng.integers(0, 256, (C, nbytes), dtype=np.uint8)
    tx = qrl.make_gr_mod_gmsk(sps, 1000000, 1700, fw, n_channels=C, max_items=nbytes)
    cut = nbytes // 3
    got = np.concatenate([tx.work(data[:, :cut]), tx.work(data[:, cut:])], axis=1)
    for c in range(C):
        want = oracle.Tx(oracle.MOD_GMSK, sps, 1000000, 1700, fw, 0).work(data[c])
        assert got.shape[1] == len(want), (got.shape, len(want))
        assert np.array_equal(got[c], want), (sps, c)
    if sps == 50:
        frames, pl = siggen.frames_4fsk(np.random.default_rng(9), 6)
        tx2 = qrl.make_gr_mod_gmsk(50, 1000000, 1700, 4000, n_channels=1, max_items=len(frames))
        iq = tx2.work(frames[None, :])[0]
        x = siggen.channel(iq, np.random.default_rng(10), fo_hz=20, phase=0.2, delay=50, snr_db=25, amp=0.5, total=len(iq) + 20000)
        rx = qrl.make_gr_demod_gmsk(5, 1000000, 1700, 4000, n_channels=1, max_samples=len(x))
        rx.work(x[None, :])
        good = max(siggen.count_good_frames(rx.read_port(p)[0], 0xED89AA, 24, 7, pl)[0] for p in (2, 3))
        assert good == len(pl)


def test_tx_am_modulator(qrl, oracle):
    """gr_mod_am (gr_mod_am.cpp:25-72: agc2_ff, rail, band-pass, carrier, x125, 4545-tap output filter at 1 Msps) against the oracle,
    streamed in uneven calls, audio loud enough to drive the AGC and the rail; then CUDA TX -> CUDA AM RX recovers the tone."""
    C, n = 2, 1200
    t = np.arange(n)
    audio = np.stack([((0.9 + 0.8 * c) * np.sin(2 * np.pi * (700 + 300 * c) * t / 8000) + 0.3 * np.sin(2 * np.pi * 1900 * t / 8000 + c)).astype(np.float32)
                      for c in range(C)])
    tx = qrl.make_gr_mod_am(125, 1000000, 1700, 5000, n_channels=C, max_items=n)
    tx.set_bb_gain(0.9)
    got = np.concatenate([tx.work_audio(audio[:, a:b]) for a, b in ((0, 1), (1, 403), (403, n))], axis=1)
    for c in range(C):
        o = oracle.Tx(oracle.MOD_AM, 125, 1000000, 1700, 5000, 0)
        o.set_bb_gain(0.9)
        want = o.work(audio[c])
        assert got.shape[1] == len(want) == n * 125
        assert rel_rms(got[c], want) <= 1e-5
        assert np.array_equal(got[c], want), c
    rx = qrl.make_gr_demod_am(125, 1000000, 1700, 5000, n_channels=C, max_samples=got.shape[1])
    rx.work(got)
    a = rx.read_port(1)[0][500:]
    spec = np.abs(np.fft.rfft(a * np.hanning(len(a))))
    assert abs(np.argmax(spec[3:]) + 3 - 700 * len(a) / 8000) < 2


def test_tx_nbfm_set_filter_width_mid_stream(qrl, oracle):
    """gr_mod_nbfm::set_filter_width (gr_mod_nbfm.cpp:78-93) between calls: new resampler / IF / interpolator taps (longer than the ones the
    block was made with) and a new sensitivity meet the true history of the stream; IQ bit-identical to the oracle's restatement."""
    C, n = 2, 3000
    t = np.arange(n)
    audio = np.stack([(0.5 * np.sin(2 * np.pi * (600 + 250 * c) * t / 8000) + 0.2 * np.sin(2 * np.pi * 2100 * t / 8000 + c)).astype(np.float32)
                      for c in range(C)])
    tx = qrl.make_gr_mod_nbfm(20, 1000000, 1700, 5000, n_channels=C, max_items=n)
    os_ = [oracle.Tx(oracle.MOD_NBFM, 20, 1000000, 1700, 5000, 0) for _ in range(C)]
    got, want = [], [[] for _ in range(C)]
    for a, b, fw in ((0, 1000, None), (1000, 1003, 2500), (1003, 2200, None), (2200, n, 4000)):
        if fw is not None:
            tx.set_filter_width(fw)
            for o in os_:
                o.set_param(3, fw)
        got.append(tx.work_audio(audio[:, a:b]))
        for c in range(C):
            want[c].append(os_[c].work(audio[c, a:b]))
    got = np.concatenate(got, axis=1)
    for c in range(C):
        w = np.concatenate(want[c])
        assert got.shape[1] == len(w) and np.array_equal(got[c], w), c
    with pytest.raises(qrl.QrlError):
        qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=1, max_items=16).set_filter_width(3000)


@pytest.mark.parametrize("kind", ["usb", "lsb", "am"])
def test_tx_ssb_am_set_filter_width_mid_stream(qrl, oracle, kind):
    """gr_mod_ssb::set_filter_width (gr_mod_ssb.cpp:85-100; the new side-band filter is 300 .. fw / 250 Hz, not the constructor's 200 .. fw /
    200 Hz) and gr_mod_am::set_filter_width (gr_mod_am.cpp:75-85) between calls, against the oracle's restatement."""
    C, n = 2, 900 if kind == "am" else 3000
    t = np.arange(n)
    audio = np.stack([(0.5 * np.sin(2 * np.pi * (600 + 250 * c) * t / 8000) + 0.2 * np.sin(2 * np.pi * 2100 * t / 8000 + c)).astype(np.float32)
                      for c in range(C)])
    if kind == "am":
        tx = qrl.make_gr_mod_am(125, 1000000, 1700, 5000, n_channels=C, max_items=n)
        okind, oargs = oracle.MOD_AM, (125, 1000000, 1700, 5000, 0)
        steps = ((0, 300, None), (300, 302, 3500), (302, n, None))
    else:
        sb = 1 if kind == "lsb" else 0
        tx = qrl.make_gr_mod_ssb(125, 1000000, 1700, 2700, sb, n_channels=C, max_items=n)
        okind, oargs = oracle.MOD_SSB, (125, 1000000, 1700, 2700, sb)
        steps = ((0, 1000, None), (1000, 1003, 2200), (1003, 2200, None), (2200, n, 3000))
    os_ = [oracle.Tx(okind, *oargs) for _ in range(C)]
    got, want = [], [[] for _ in range(C)]
    for a, b, fw in steps:
        if fw is not None:
            tx.set_filter_width(fw)
            for o in os_:
                o.set_param(3, fw)
        got.append(tx.work_audio(audio[:, a:b]))
        for c in range(C):
            want[c].append(os_[c].work(audio[c, a:b]))
    got = np.concatenate(got, axis=1)
    for c in range(C):
        w = np.concatenate(want[c])
        assert got.shape[1] == len(w) and np.array_equal(got[c], w), c


def nbfm_ctcss_case(qrl, oracle):
    """gr_mod_nbfm::set_ctcss (gr_mod_nbfm.cpp:101-139) mid-stream: tone on (88.5 Hz, then 123 Hz: the tone source keeps its phase), tone
    off (gain 0.98, not the constructor's 0.99), IQ bit-identical to the oracle; returns the IQ."""
    C, n = 2, 6000
    t = np.arange(n)
    audio = np.stack([(0.4 * np.sin(2 * np.pi * (900 + 250 * c) * t / 8000)).astype(np.float32) for c in range(C)])
    tx = qrl.make_gr_mod_nbfm(20, 1000000, 1700, 2500, n_channels=C, max_items=n)
    os_ = [oracle.Tx(oracle.MOD_NBFM, 20, 1000000, 1700, 2500, 0) for _ in range(C)]
    got, want = [], [[] for _ in range(C)]
    for a, b, f in ((0, 700, None), (700, 3200, 88.5), (3200, 3201, 123.0), (3201, 5000, None), (5000, n, 0.0)):
        if f is not None:
            tx.set_ctcss(f)
            for o in os_:
                o.set_param(7, f)
        got.append(tx.work_audio(audio[:, a:b]))
        for c in range(C):
            want[c].append(os_[c].work(audio[c, a:b]))
    got = np.concatenate(got, axis=1)
    for c in range(C):
        w = np.concatenate(want[c])
        assert got.shape[1] == len(w) and np.array_equal(got[c], w), c
    return got


def test_tx_nbfm_set_ctcss(qrl, oracle):
    """nbfm_ctcss_case against the oracle; the tone is in the demodulated audio of the CUDA receiver."""
    got = nbfm_ctcss_case(qrl, oracle)
    rx = qrl.make_gr_demod_nbfm(125, 1000000, 1700, 2500, n_channels=1, max_samples=got.shape[1])
    rx.work(got[:1])
    a = rx.read_port(1)[0]
    seg = a[1200:3000]                                            # tone at 88.5 Hz on, 8 ksps audio
    spec = np.abs(np.fft.rfft(seg * np.hanning(len(seg))))
    fb = np.fft.rfftfreq(len(seg), 1 / 8000.0)
    assert spec[np.argmin(np.abs(fb - 88.5))] > 20 * np.median(spec[(fb > 200) & (fb < 700)])
