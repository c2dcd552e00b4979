"""GPU tier: the transmit front end (qrl_tx_frontend_*, gr_mod_base.cpp:38,211-293,799-805: carrier-offset rotator at 1 Msps + x N
interpolator to the device rate) bit-identical to its oracle (tests/tx_frontend_oracle.c) at every supported shape, with ragged chunks,
host and device input and mid-stream retunes; a wideband modulator behind it; a whole TX -> front end -> RX front end -> RX chain on
one caller stream; and the handle's lifecycle."""
import ctypes as C

import numpy as np
import pytest

from tests import siggen
from tests import tx_frontend_oracle as TO

pytestmark = pytest.mark.gpu

SIZES = [20000, 1, 7777, 13, 3000, 0, 4096]


def _signal(rng, C, T):
    """[C, T] complex64 at 1 Msps: a tone per channel plus noise, amplitude about 0.5."""
    n = np.arange(T)
    return np.stack([(0.4 * np.exp(2j * np.pi * (-90000.0 + 37000.0 * c) * n / 1e6)
                      + 0.05 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))).astype(np.complex64) for c in range(C)])


def _same(got, want):
    return got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def parity(q, samp_rate, C, sizes, retunes=None, device=False, pad=0, classes=None, seed=0):
    """Feed [C, sum(sizes)] through one library handle in the given chunks and through one oracle per class of channels; every output
    must equal the oracle bit for bit.  retunes: {chunk index: [(channel, hz), ...]} applied before that chunk (channel -1 = all).
    classes: channel c carries base signal classes[c] (all channels of a class must then retune alike); None = each its own.
    device: the input is a device tensor with channel stride T + pad (torch), else a host array."""
    retunes = retunes or {}
    classes = list(range(C)) if classes is None else list(classes)
    K = max(classes) + 1
    T = sum(sizes)
    base = _signal(np.random.default_rng(seed + samp_rate // 1000000), K, T)
    X = base[classes]
    fe = q.TxFrontend(samp_rate, n_channels=C, max_in=max(max(sizes), 1))
    rep = {k: classes.index(k) for k in range(K)}                      # class -> its first channel, the one the oracle runs
    reps = sorted(rep.values())
    ofe = {c: TO.TxFrontend(samp_rate) for c in reps}
    N = samp_rate // 1000000
    if device:
        import torch
        Xd = torch.zeros((C, T + pad), dtype=torch.complex64, device="cuda")
        Xd[:, :T] = torch.from_numpy(X)
        stride = T + pad
    lo = 0
    for i, m in enumerate(sizes):
        for ch, hz in retunes.get(i, []):
            fe.set_carrier_offset(hz, channel=ch)
            for c in reps:
                if ch < 0 or ch == c:
                    ofe[c].set_carrier_offset(hz)
        if device:
            nout = fe.work_device(Xd[:, lo:].data_ptr(), m, stride)
            got = fe.read()
        else:
            got = fe.work(X[:, lo:lo + m])
            nout = got.shape[1]
        assert nout == N * m and got.shape == (C, N * m), (samp_rate, i, got.shape)
        want = {c: ofe[c].work(X[c, lo:lo + m]) for c in reps}
        for c in range(C):
            w = want[rep[classes[c]]]
            assert len(w) == N * m and _same(got[c], w), (samp_rate, i, c)
        lo += m
    fe.close()


RETUNES = {1: [(-1, 150000.0)], 3: [(1, -70000.0)], 5: [(-1, 0.0)], 6: [(0, 312500.0)]}


@pytest.mark.parametrize("samp_rate", [1000000, 2000000, 3000000, 5000000, 10000000, 20000000, 32000000])
def test_tx_frontend_matches_oracle(qrl, samp_rate):
    parity(qrl, samp_rate, 3, SIZES, RETUNES)


@pytest.mark.parametrize("C", [33, 97])
def test_tx_frontend_many_channels(qrl, C):
    """33 and 97 channels at 10 Msps: five base signals; every channel must equal its class's oracle; retunes of all channels."""
    classes = [c % 5 for c in range(C)]
    parity(qrl, 10000000, C, [9000, 1, 4000], {1: [(-1, -200000.0)]}, classes=classes)


@pytest.mark.parametrize("samp_rate", [1000000, 10000000])
def test_tx_frontend_device_input_with_stride(qrl, samp_rate):
    parity(qrl, samp_rate, 3, SIZES, RETUNES, device=True, pad=37)


def test_tx_frontend_wideband_qpsk(qrl):
    """QPSK 250 ksym/s modulator (make_gr_mod_qpsk(4, ...)) at 10 Msps, +300 kHz, fed from the modulator's device output."""
    import torch
    from oracle import oracle as O
    Cn, n = 2, 3000
    data = np.random.default_rng(5200).integers(0, 256, (Cn, n), dtype=np.uint8)
    s = torch.cuda.Stream()
    tx = qrl.make_gr_mod_qpsk(4, 1000000, 1700, 160000, n_channels=Cn, max_items=n)
    fe = qrl.TxFrontend(10000000, n_channels=Cn, max_in=n * 32)
    tx.set_stream(s.cuda_stream); fe.set_stream(s.cuda_stream)
    fe.set_carrier_offset(300000.0)
    d = torch.from_numpy(data).cuda()
    torch.cuda.synchronize()
    tx.work_device(d.data_ptr(), n, n)
    L = qrl.load_library()
    p, st, items = C.c_void_p(), C.c_long(), C.c_long()
    assert L.qrl_tx_out_device(tx._h, C.byref(p), C.byref(st), C.byref(items)) == 0 and items.value == n * 32
    assert fe.work_device(p.value, items.value, st.value) == 10 * n * 32
    got = fe.read()
    for c in range(Cn):
        o = TO.TxFrontend(10000000); o.set_carrier_offset(300000.0)
        want = o.work(O.Tx(O.MOD_QPSK, 4, 1000000, 1700, 160000, 0).work(data[c]))
        assert _same(got[c], want), c
        spec = np.abs(np.fft.fftshift(np.fft.fft(got[c]))) ** 2
        f = np.fft.fftshift(np.fft.fftfreq(len(got[c]), 1 / 10e6))
        assert abs(np.sum(f * spec) / np.sum(spec) - 300000.0) < 20000.0           # the signal's centroid moved to +300 kHz
    tx.close(); fe.close()


def test_tx_to_rx_chain_on_one_stream(qrl, oracle):
    """4FSK-2k-FM modulator -> transmit front end (2 Msps, +25 kHz) -> receive front end (2 Msps, 25 kHz) -> 4FSK receiver, all on
    one caller stream with no host copy in between: the decoded bits equal the same chain of oracle blocks and the frames come back."""
    import torch
    Cn = 2
    streams, payloads = [], []
    for c in range(Cn):
        d, pl = siggen.frames_4fsk(np.random.default_rng(7300 + c), 30)
        streams.append(d); payloads.append(pl)
    n = max(len(d) for d in streams)
    data = np.full((Cn, n), 0xAA, np.uint8)
    for c, d in enumerate(streams):
        data[c, :len(d)] = d
    s = torch.cuda.Stream()
    tx = qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=Cn, max_items=n)
    L = qrl.load_library()
    d = torch.from_numpy(data).cuda()
    torch.cuda.synchronize()
    tx.set_stream(s.cuda_stream)
    tx.work_device(d.data_ptr(), n, n)
    p, st, items = C.c_void_p(), C.c_long(), C.c_long()
    assert L.qrl_tx_out_device(tx._h, C.byref(p), C.byref(st), C.byref(items)) == 0
    m = items.value
    assert m > 0
    fe_tx = qrl.TxFrontend(2000000, n_channels=Cn, max_in=m)
    fe_rx = qrl.Frontend(2000000, n_channels=Cn, max_in=2 * m)
    rx = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=Cn, max_samples=m + 8)
    for h in (fe_tx, fe_rx, rx):
        h.set_stream(s.cuda_stream)
    fe_tx.set_carrier_offset(25000.0); fe_rx.set_carrier_offset(25000.0)
    assert fe_tx.work_device(p.value, m, st.value) == 2 * m
    p2, st2, n2 = fe_tx.out_device()
    k = fe_rx.work_device(p2, n2, st2)
    p3, st3, n3 = fe_rx.out_device()
    assert k == n3 == m
    rx.work_device(p3, n3, st3)
    bits = rx.read_port(2)
    s.synchronize()
    for c in range(Cn):
        y = oracle.Tx(oracle.MOD_4FSK, 25, 1000000, 1700, 3500, 1).work(data[c])
        assert len(y) == m
        o1 = TO.TxFrontend(2000000); o1.set_carrier_offset(25000.0)
        o2 = oracle.Frontend(2000000); o2.set_carrier_offset(25000.0)
        r = oracle.Rx(oracle.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1)
        r.work(o2.work(o1.work(y)))
        assert np.array_equal(bits[c], r.port(2)), c
        good, found = siggen.count_good_frames(bits[c], 0xED89AA, 24, 7, payloads[c])
        assert good >= len(payloads[c]) - 2, (c, good, found)
    for h in (tx, fe_tx, fe_rx, rx):
        h.close()


def _run(h, k):
    x = _signal(np.random.default_rng(3300 + k), 2, 3000)
    return h.work(x)


def test_tx_frontend_set_stream_and_back(qrl):
    """a handle moved to a caller's stream and back to its own gives bit-identical output to a twin that never moved"""
    import torch
    s = torch.cuda.Stream()
    h, twin = qrl.TxFrontend(5000000, n_channels=2, max_in=4096), qrl.TxFrontend(5000000, n_channels=2, max_in=4096)
    h.set_carrier_offset(40000.0); twin.set_carrier_offset(40000.0)
    assert _same(_run(h, 0), _run(twin, 0))
    for k, st in enumerate([s.cuda_stream, None, None], 1):
        h.set_stream(st)
        assert _same(_run(h, k), _run(twin, k)), k
    s.synchronize()
    h.close(); twin.close()


def test_tx_frontend_null_handles_and_errors(qrl):
    L = qrl.load_library()
    assert L.qrl_tx_frontend_destroy(None) == 0                                     # QRL_OK, like qrl_frontend_destroy
    assert L.qrl_tx_frontend_set_stream(None, None) == -22
    assert L.qrl_tx_frontend_launch_count(None) == 0
    for bad in ((0, 1, 16), (1500000, 1, 16), (33000000, 1, 16), (2000000, 0, 16), (2000000, 1, 0)):
        assert L.qrl_tx_frontend_create(bad[0], bad[1], bad[2], 0, C.byref(C.c_void_p())) == -22, bad
        assert L.qrl_last_error(None).decode().startswith("qrl_tx_frontend_create: "), L.qrl_last_error(None)
    assert L.qrl_tx_frontend_create(2000000, 1, 16, L.qrl_device_count(), C.byref(C.c_void_p())) == -19
    assert L.qrl_last_error(None).decode().startswith("qrl_tx_frontend_create: "), L.qrl_last_error(None)
    fe = qrl.TxFrontend(2000000, n_channels=1, max_in=16)
    x = np.zeros(17, np.complex64)
    n = C.c_long()
    assert L.qrl_tx_frontend_work(fe._h, x.ctypes.data_as(C.c_void_p), 17, 17, 0, C.byref(n)) == -34    # QRL_ERANGE
    assert L.qrl_tx_frontend_work(fe._h, x.ctypes.data_as(C.c_void_p), 0, 0, 0, C.byref(n)) == 0 and n.value == 0
    assert fe.launches == 0
    fe.work(x[:16])
    assert fe.launches == 2                                                         # interpolator + history tail
    fe.close()
