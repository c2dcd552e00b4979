"""GPU tier: one 1 Msps stream feeding every receive channel (qrl_rx_work / _sc16 / _sc8 with stride 0; one SDR source -> rotator_cc
per channel -> demodulator, gr_demod_mmdvm_multi.cpp:68-123's wiring at the demodulators' own rate).  Every port, port count and RSSI
value of every channel equals a twin handle fed the same chunks as n_channels identical rows, bit for bit: every receive kind, host,
device, sc16 and sc8 input, 1 / 33 / 97 channels, ragged chunks with retunes, shared and per-row calls on one handle, overlapped calls,
the rotator pass; three 4FSK signals in one capture decode like the oracle receiver; the error codes."""
import ctypes as C

import numpy as np
import pytest

from tests import siggen

pytestmark = pytest.mark.gpu


def stream(T, seed):
    """one 1 Msps capture: a 4FSK-2k-FM signal at 0 Hz, tones across the band (one near each of the +-400 kHz channels) and noise"""
    rng = np.random.default_rng(seed)
    x = siggen.gen_4fsk_channels(1, T, seed0=seed)[0][0].astype(np.complex128)
    n = np.arange(T)
    for f, a in ((0.3971, 0.3), (-0.4019, 0.3), (0.13, 0.1), (-0.21, 0.1)):
        x = x + a * np.exp(2j * np.pi * f * n)
    x = x + 0.02 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))
    return (0.5 * x).astype(np.complex64)


def wire(x, kind):
    """the int pair stream an sc16 / sc8 SDR would deliver for x: [T][2]"""
    scale, top, dt = (16000.0, 32767, np.int16) if kind.endswith("16") else (90.0, 127, np.int8)
    v = np.stack([x.real, x.imag], axis=-1) * scale
    return np.clip(np.rint(v), -top, top).astype(dt)


def torch_device_input(a):
    """a copied to the GPU 8 bytes past a 16-byte boundary (the stage-1 window then takes its plain-load fetch): (pointer, owner)"""
    import torch
    raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    buf = torch.zeros(len(raw) + 16, dtype=torch.uint8, device="cuda")
    buf[8:8 + len(raw)] = torch.from_numpy(raw)
    torch.cuda.synchronize()
    return buf.data_ptr() + 8, buf


def _ports_equal(a, b, tag):
    for p in range(a.nports):
        pa, pb = a.read_port(p), b.read_port(p)
        for c in range(a.n_channels):
            assert len(pa[c]) == len(pb[c]) and pa[c].tobytes() == pb[c].tobytes(), tag + (p, c)


def parity(make, Cn, sizes, retunes, kinds=("host",), dev_input=None, seed=0, rssi=False, overlap=False):
    """Feed one stream in the given chunks to a handle with stride 0 and, as [Cn, m] identical rows, to a twin handle; kinds[i % len]
    says how chunk i reaches the first handle: "host", "dev" (device pointer from dev_input), "sc16", "sc8", "dev_sc16" (stride 0)
    or "rows" (a per-row call).  After every chunk each port of each channel, the counts and (rssi) qrl_rx_rssi equal the twin's.
    retunes: {chunk index: [(channel, hz), ...]} before that chunk; channel -1 = all."""
    X = stream(sum(sizes), seed)
    m_max = max(max(sizes), 1)
    blk, twin = make(Cn, m_max), make(Cn, m_max)
    for b in (blk, twin):
        if rssi:
            b.enable_rssi()
        if overlap:
            b.set_overlap()
    lo = 0
    for i, m in enumerate(sizes):
        for ch, hz in retunes.get(i, []):
            blk.set_carrier_offset(hz, channel=ch); twin.set_carrier_offset(hz, channel=ch)
        x = X[lo:lo + m]
        kind = kinds[i % len(kinds)]
        if kind in ("sc16", "sc8", "dev_sc16"):
            w = wire(x, kind)
            if kind == "sc16":
                blk.work_shared_sc16(w)
            elif kind == "sc8":
                blk.work_shared_sc8(w)
            else:
                ptr, keep = dev_input(w)
                blk.work_sc16_device(ptr, m, 0)
                blk.sync()
                del keep
            rows = np.repeat(w[None], Cn, axis=0)
            (twin.work_sc8 if kind == "sc8" else twin.work_sc16)(rows)
        else:
            if kind == "dev":
                ptr, keep = dev_input(x)
                blk.work_device(ptr, m, 0)
                blk.sync()
                del keep
            elif kind == "rows":
                blk.work(np.repeat(x[None], Cn, axis=0))
            else:
                blk.work_shared(x)
            twin.work(np.repeat(x[None], Cn, axis=0))
        _ports_equal(blk, twin, (Cn, i, kind))
        if rssi:
            assert blk.rssi().tobytes() == twin.rssi().tobytes(), (Cn, i, kind)
        lo += m
    blk.close(); twin.close()


def factory(name):
    import qradiolink_b200 as q
    if name == "qpsk2k":        # /100 with 28 taps per branch (2727 taps): the stage-1 shape test_gpu_dispatch's table does not run
        return lambda n, m: q.make_gr_demod_qpsk(125, 1000000, 1700, 1300, n_channels=n, max_samples=m)
    from tests.test_gpu_dispatch import RX
    mk = RX[name][0]
    return lambda n, m: mk(q, n, m)


# channel 0 at 0 Hz, the others near +-400 kHz (set before the first chunk)
NEAR_EDGES = {0: [(1, 397100.0), (2, -401900.0)]}
ALL_KINDS = ["nbfm", "am", "usb", "lsb", "wbfm", "freedv_usb", "freedv_lsb", "4fsk", "4fsk_disc", "4fsk1k", "4fsk10k", "4fsk100k",
             "qpsk", "qpsk20k", "qpsk2k", "bpsk", "2fsk", "2fsk_band", "gmsk", "m17", "dmr", "dsss"]


@pytest.mark.parametrize("name", ALL_KINDS)
def test_every_kind_matches_identical_rows(qrl, name):
    """3 channels at 0 Hz and near +-400 kHz; host, device (odd offset), sc16, sc8 and device sc16 input, each against identical rows"""
    parity(factory(name), 3, [40000, 1, 20003, 60000, 31000], NEAR_EDGES, kinds=("host", "dev", "sc16", "sc8", "dev_sc16"),
           dev_input=torch_device_input, seed=11)


@pytest.mark.parametrize("name", ["4fsk", "nbfm", "4fsk1k", "2fsk", "qpsk20k", "qpsk2k"])
def test_every_register_tiled_shape(qrl, name):
    """every register-tiled stage-1 shape (/50, /125, /100 with 9 and 28 taps per branch, /25 with 9 and 28) with the carrier offset
    fused into the window, at 4 channels: host, device (plain-load fetch), sc16 and sc8 input with a retune of one channel"""
    r = {0: [(1, 397100.0), (2, -401900.0), (3, 123456.0)], 2: [(2, -125000.0)]}
    parity(factory(name), 4, [40000, 1, 20003, 60000], r, kinds=("host", "dev", "sc16", "sc8"), dev_input=torch_device_input, seed=13)


@pytest.mark.parametrize("name", ["4fsk", "nbfm", "qpsk"])
@pytest.mark.parametrize("Cn", [1, 33, 97])
def test_channel_counts(qrl, name, Cn):
    """one channel, a partial last 32-channel group and the many-channel loop geometry"""
    r = {0: [(c, (c * 0.61 % 1.0 - 0.5) * 0.9e6) for c in range(1, Cn)], 2: [(Cn // 2, 31250.0)]}
    parity(factory(name), Cn, [30000, 1, 4999, 70000], r, kinds=("host", "dev"), dev_input=torch_device_input, seed=Cn)


RETUNES = {0: [(1, 150000.0), (2, -330000.0)], 3: [(-1, 62500.0)], 5: [(2, -125000.0)], 7: [(0, 250000.0)]}


@pytest.mark.parametrize("name", ["4fsk", "nbfm", "qpsk20k", "usb"])
def test_ragged_chunks_retunes_and_per_row_calls(qrl, name):
    """chunks of 0, 1 and 3 samples among long ones, retunes of every channel and of one mid-stream, shared and per-row calls
    alternating on one handle (each channel's stream continues across the switch), RSSI after every call"""
    parity(factory(name), 3, [30000, 0, 1, 3, 50, 7777, 2501, 60000, 12345], RETUNES, kinds=("host", "rows", "dev", "rows", "sc16"),
           dev_input=torch_device_input, rssi=True, seed=3)


def test_overlapped_4fsk_calls(qrl):
    """QRL_PARAM_OVERLAP_CALLS with stride 0: the staging of call k+1 is rewritten while call k's tail still runs, and the call
    length changes twice"""
    parity(factory("4fsk"), 5, [1 << 17, 1 << 17, 70000, 70000, 1 << 17, 1 << 17], {0: [(c, 90000.0 * c - 180000.0) for c in range(5)]},
           kinds=("host", "host", "dev", "sc16", "host", "rows"), dev_input=torch_device_input, overlap=True, seed=5)


@pytest.mark.parametrize("name", ["4fsk", "usb"])
def test_rotator_pass_equals_fused(qrl, monkeypatch, name):
    """QRL_ROTATOR_PASS (DESIGN section 10): the separate rotator pass fed the one stream equals the fused stage 1"""
    make = factory(name)
    X = stream(150000, 7)
    a, b = make(3, 60000), make(3, 60000)
    for h in (a, b):
        for ch, hz in NEAR_EDGES[0]:
            h.set_carrier_offset(hz, channel=ch)
    for lo, m in ((0, 60000), (60000, 1), (60001, 59999), (120000, 30000)):
        monkeypatch.setenv("QRL_ROTATOR_PASS", "1")
        a.work_shared(X[lo:lo + m]); a.sync()
        monkeypatch.delenv("QRL_ROTATOR_PASS")
        b.work_shared(X[lo:lo + m])
        _ports_equal(a, b, (lo,))
    a.close(); b.close()


def test_three_4fsk_signals_in_one_capture(qrl, oracle):
    """Three 4FSK-2k-FM signals at -300, +120 and +380 kHz in one 1 Msps capture, a 4-channel receiver (the fourth on an empty
    frequency) fed it by one shared call: each channel's port 2 equals the oracle receiver with the same carrier offset, and the
    frames come back on the three occupied channels"""
    offs = [-300000.0, 120000.0, 380000.0, -150000.0]
    T = 1 << 19
    n = np.arange(T)
    cap = np.zeros(T, np.complex128)
    payloads = []
    for c in range(3):
        x, pl = siggen.gen_4fsk_channels(1, T, seed0=8200 + 17 * c, snr_db=30.0)
        payloads.append(pl[0])
        cap += x[0] * np.exp(2j * np.pi * offs[c] * n / 1e6)
    cap = (cap / 3).astype(np.complex64)
    rx = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=4, max_samples=T)
    for c, f in enumerate(offs):
        rx.set_carrier_offset(f, channel=c)
    rx.work_shared(cap)
    bits = rx.read_port(2)
    for c in range(4):
        o = oracle.Rx(oracle.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1)
        o.set_carrier_offset(offs[c])
        o.work(cap)
        assert np.array_equal(bits[c], o.port(2)), c
        if c < 3:
            good, found = siggen.count_good_frames(bits[c], 0xED89AA, 24, 7, payloads[c])
            assert good >= len(payloads[c]) - 4, (c, good, found)
    rx.close()


def test_error_codes(qrl):
    L = qrl.load_library()
    rx = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=3, max_samples=1000)
    x = np.zeros(1001, np.complex64)
    w = np.zeros((1001, 2), np.int16)
    p = x.ctypes.data_as(C.c_void_p)
    assert L.qrl_rx_work(rx._h, p, 1001, 0, 0) == -34                                           # QRL_ERANGE
    assert L.qrl_rx_work_sc16(rx._h, w.ctypes.data_as(C.c_void_p), 1001, 0, C.c_float(1.0), 0) == -34
    assert L.qrl_rx_work_sc8(rx._h, w.ctypes.data_as(C.c_void_p), 1001, 0, C.c_float(1.0), 0) == -34
    assert L.qrl_rx_work(rx._h, p, 0, 0, 0) == 0
    assert L.qrl_rx_work(rx._h, p, 1000, 0, 0) == 0
    with pytest.raises(ValueError):
        rx.work_shared(np.zeros((3, 10), np.complex64))
    import torch
    if torch.cuda.device_count() > 1:
        other = torch.zeros(2000, dtype=torch.complex64, device="cuda:1")
        assert L.qrl_rx_work(rx._h, C.c_void_p(other.data_ptr()), 1000, 0, 1) == -22            # QRL_EINVAL
    rx.close()
