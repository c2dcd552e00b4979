"""GPU tier: the transmit combiner (qrl_tx_combiner_*: per channel x N interpolation, a rotator at the device rate, add_cc, x 1 / C,
x bb_gain -- gr_mod_mmdvm_multi.cpp:53-125 with gr_mod_base's interpolator) bit-identical to its oracle (tests/tx_combiner_oracle.c)
at every supported rate and around the 8-channel block size, with ragged chunks, retunes and gain changes; host rows, device rows of
separate allocations at odd 8-byte offsets and a strided slab; several modulators -> one SDR stream -> the receive front end -> the
receivers on one caller stream; and the handle's lifecycle."""
import ctypes as C

import numpy as np
import pytest

from tests import siggen
from tests import tx_combiner_oracle as TCO

pytestmark = pytest.mark.gpu

SIZES = [20000, 1, 7777, 13, 3000, 0, 4096]


def _signal(rng, C, T):
    """[C, T] complex64 at 1 Msps: a tone per channel plus noise, amplitude about 0.5."""
    n = np.arange(T)
    return np.stack([(0.4 * np.exp(2j * np.pi * (-90000.0 + 37000.0 * (c % 7)) * n / 1e6)
                      + 0.05 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))).astype(np.complex64) for c in range(C)])


def _same(got, want):
    return got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def spread(samp_rate, C):
    """C carrier offsets across the band, inside +-(samp_rate / 2 - 0.5 MHz) where the interpolator's image-free band allows"""
    half = max(samp_rate / 2 - 500000.0, 0.0)
    return [0.0 if C == 1 else -half + 2 * half * c / (C - 1) + 1234.5 * (c % 3) for c in range(C)]


def parity(q, samp_rate, C, sizes, events=None, device=None, seed=0):
    """Feed [C, sum(sizes)] through one library handle and the oracle in the given chunks; every chunk's output must be bit-identical.
    events: {chunk index: [("offset", channel, hz) | ("gain", g), ...]} applied to both before that chunk (channel -1 = all).
    device: None = host rows; "slab" = one torch tensor [C, T + 37] (row c at c stride); "separate" = one allocation per row, row c
    starting (c % 3) samples past a 16-byte boundary (odd 8-byte offsets included)."""
    events = events or {}
    T = sum(sizes)
    X = _signal(np.random.default_rng(seed + samp_rate // 1000000 + 7 * C), C, T)
    fe = q.TxCombiner(samp_rate, n_channels=C, max_in=max(max(sizes), 1))
    o = TCO.TxCombiner(samp_rate, C)
    N = samp_rate // 1000000
    if device:
        import torch
        if device == "slab":
            Xd = torch.zeros((C, T + 37), dtype=torch.complex64, device="cuda")
            Xd[:, :T] = torch.from_numpy(X)
            base = [Xd[c].data_ptr() for c in range(C)]
        else:
            Xd = [torch.zeros(T + 3, dtype=torch.complex64, device="cuda") for _ in range(C)]
            for c in range(C):
                Xd[c][c % 3:c % 3 + T] = torch.from_numpy(X[c])
            base = [Xd[c].data_ptr() + 8 * (c % 3) for c in range(C)]
        torch.cuda.synchronize()
    lo = 0
    for i, m in enumerate(sizes):
        for ev in events.get(i, []):
            if ev[0] == "offset":
                fe.set_carrier_offset(ev[2], channel=ev[1]); o.set_carrier_offset(ev[2], ev[1])
            else:
                fe.set_gain(ev[1]); o.set_gain(ev[1])
        if device:
            nout = fe.work_device([b + 8 * lo for b in base], m)
            got = fe.read()
        else:
            got = fe.work(X[:, lo:lo + m])
            nout = len(got)
        want = o.work(X[:, lo:lo + m])
        assert nout == N * m == len(want), (samp_rate, C, i, nout)
        assert _same(got, want), (samp_rate, C, i, np.flatnonzero(got != want)[:5])
        lo += m
    fe.close()


def events_for(samp_rate, C):
    off = spread(samp_rate, C)
    ev = {0: [("offset", c, off[c]) for c in range(C) if off[c] != 0.0]}
    ev[2] = [("offset", C // 2, -off[C // 2] * 0.5 + 10000.0)]                   # one channel retunes
    ev[4] = [("gain", 0.7)]
    ev[6] = [("offset", -1, 0.3 * min(samp_rate / 2, 1e6)), ("gain", 1.25)]      # every channel retunes
    return ev


@pytest.mark.parametrize("samp_rate", [1000000, 2000000, 3000000, 5000000, 10000000, 20000000, 32000000])
def test_tx_combiner_matches_oracle(qrl, samp_rate):
    parity(qrl, samp_rate, 3, SIZES, events_for(samp_rate, 3))


@pytest.mark.parametrize("C", [1, 8, 9, 33, 97])
def test_tx_combiner_channel_counts(qrl, C):
    """around the 8-channel block and past several blocks, at 10 Msps"""
    parity(qrl, 10000000, C, [3000, 1, 1700, 0, 900], {0: events_for(10000000, C)[0], 1: [("gain", 0.5)],
                                                       3: [("offset", -1, -2.5e6)]})


@pytest.mark.parametrize("device", ["slab", "separate"])
@pytest.mark.parametrize("samp_rate", [1000000, 10000000])
def test_tx_combiner_device_rows(qrl, samp_rate, device):
    parity(qrl, samp_rate, 9, SIZES, events_for(samp_rate, 9), device=device)


def test_tx_combiner_scratch_ranges(qrl):
    """at 32 Msps with 97 channels a 65 536-sample call is cut into several launch ranges of block partials; it equals a twin fed in
    4096-sample calls (one range each, the path the oracle tests cover), and its start equals the oracle"""
    C, n, k = 97, 1 << 16, 4096
    X = _signal(np.random.default_rng(11), C, n)
    fe, twin = qrl.TxCombiner(32000000, n_channels=C, max_in=n), qrl.TxCombiner(32000000, n_channels=C, max_in=k)
    for h in (fe, twin):
        h.set_carrier_offset(-7.5e6, channel=3); h.set_carrier_offset(11e6, channel=90)
    got = fe.work(X)
    assert fe.launches // 2 >= 3                                                    # kernel + block sum per range
    want = np.concatenate([twin.work(X[:, lo:lo + k]) for lo in range(0, n, k)])
    assert _same(got, want)
    o = TCO.TxCombiner(32000000, C)
    o.set_carrier_offset(-7.5e6, 3); o.set_carrier_offset(11e6, 90)
    assert _same(got[:32 * 1000], o.work(X[:, :1000]))
    fe.close(); twin.close()


def test_modulators_to_one_sdr_and_back(qrl, oracle):
    """4FSK-2k-FM (2 channels), NBFM and QPSK-250k modulators on one caller stream -> the combiner at 10 Msps (-3.0 / -1.2 / +1.5 /
    +3.5 MHz) -> the receive front end on that one stream (stride 0) at the same offsets -> the three receivers.  The decoded bits and
    the NBFM audio equal the same chain of oracle blocks, and the 4FSK frames come back."""
    import torch
    FS, OFF = 10000000, [-3.0e6, -1.2e6, 1.5e6, 3.5e6]
    payloads, streams = [], []
    for c in range(2):
        d, pl = siggen.frames_4fsk(np.random.default_rng(7400 + c), 12)
        streams.append(d); payloads.append(pl)
    nb = max(len(d) for d in streams) + 32                   # 16 idle bytes before (receiver lock) and after (the chain's delay)
    d4 = np.full((2, nb), 0xAA, np.uint8)
    for c, d in enumerate(streams):
        d4[c, 16:16 + len(d)] = d
    s = torch.cuda.Stream()
    L = qrl.load_library()

    def out_of(tx):
        p, st, items = C.c_void_p(), C.c_long(), C.c_long()
        assert L.qrl_tx_out_device(tx._h, C.byref(p), C.byref(st), C.byref(items)) == 0
        return p.value, st.value, items.value

    tx4 = qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=2, max_items=nb)
    tx4.set_stream(s.cuda_stream)
    g4 = torch.from_numpy(d4).cuda()
    torch.cuda.synchronize()
    tx4.work_device(g4.data_ptr(), nb, nb)
    p4, st4, m = out_of(tx4)
    na, nq = m // 125 + 2, m // 32 + 2
    t = np.arange(na) / 8000.0
    audio = (0.5 * np.sin(2 * np.pi * 700 * t) + 0.3 * np.sin(2 * np.pi * 1900 * t)).astype(np.float32)[None, :]
    dq = np.random.default_rng(7402).integers(0, 256, (1, nq), dtype=np.uint8)
    txn = qrl.make_gr_mod_nbfm(20, 1000000, 1700, 5000, n_channels=1, max_items=na)
    txq = qrl.make_gr_mod_qpsk(4, 1000000, 1700, 160000, n_channels=1, max_items=nq)
    ga, gq = torch.from_numpy(audio).cuda(), torch.from_numpy(dq).cuda()
    torch.cuda.synchronize()
    for tx, g, n in ((txn, ga, na), (txq, gq, nq)):
        tx.set_stream(s.cuda_stream)
        tx.work_device(g.data_ptr(), n, n)
    pn, _, mn = out_of(txn)
    pq, _, mq = out_of(txq)
    assert mn >= m and mq >= m, (m, mn, mq)
    comb = qrl.TxCombiner(FS, n_channels=4, max_in=m)
    fe = qrl.Frontend(FS, n_channels=4, max_in=10 * m)
    rx4 = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=2, max_samples=m + 8)
    rxn = qrl.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=1, max_samples=m + 8)
    rxq = qrl.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=1, max_samples=m + 8)
    for h in (comb, fe, rx4, rxn, rxq):
        h.set_stream(s.cuda_stream)
    for c, f in enumerate(OFF):
        comb.set_carrier_offset(f, channel=c)
        fe.set_carrier_offset(f, channel=c)
    assert comb.work_device([p4, p4 + 8 * st4, pn, pq], m) == 10 * m
    py, ny = comb.out_device()
    assert fe.work_device(py, ny, 0) == m
    pf, stf, nf = fe.out_device()
    assert nf == m
    rx4.work_device(pf, m, stf)
    rxn.work_device(pf + 2 * 8 * stf, m, stf)
    rxq.work_device(pf + 3 * 8 * stf, m, stf)
    bits4, audio_rx, bitsq = rx4.read_port(2), rxn.read_port(1), rxq.read_port(2)
    s.synchronize()
    # the same chain of oracle blocks
    rows = [oracle.Tx(oracle.MOD_4FSK, 25, 1000000, 1700, 3500, 1).work(d4[c])[:m] for c in range(2)]
    rows.append(oracle.Tx(oracle.MOD_NBFM, 20, 1000000, 1700, 5000, 0).work(audio[0])[:m])
    rows.append(oracle.Tx(oracle.MOD_QPSK, 4, 1000000, 1700, 160000, 0).work(dq[0])[:m])
    oc = TCO.TxCombiner(FS, 4)
    for c, f in enumerate(OFF):
        oc.set_carrier_offset(f, c)
    y = oc.work(np.stack(rows))
    assert _same(comb.read(), y)
    rxs = [oracle.Rx(oracle.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1) for _ in range(2)]
    rxs += [oracle.Rx(oracle.DEMOD_NBFM, 125, 1000000, 1700, 5000, 0), oracle.Rx(oracle.DEMOD_QPSK, 2, 1000000, 1700, 160000, 0)]
    for c, f in enumerate(OFF):
        of = oracle.Frontend(FS); of.set_carrier_offset(f)
        rxs[c].work(of.work(y))
    for c in range(2):
        assert np.array_equal(bits4[c], rxs[c].port(2)), c
        good, found = siggen.count_good_frames(bits4[c], 0xED89AA, 24, 7, payloads[c])
        assert good >= len(payloads[c]) - 2, (c, good, found)
    want_audio = rxs[2].port(1)
    assert len(want_audio) > 1000 and _same(audio_rx[0], want_audio)
    want_q = rxs[3].port(2)
    assert len(want_q) > 1000 and np.array_equal(bitsq[0], want_q)
    for h in (tx4, txn, txq, comb, fe, rx4, rxn, rxq):
        h.close()


def _run(h, k):
    return h.work(_signal(np.random.default_rng(3300 + k), 3, 3000))


def test_tx_combiner_set_stream_and_back(qrl):
    """a handle moved to a caller's stream and back to its own gives bit-identical output to a twin that never moved"""
    import torch
    s = torch.cuda.Stream()
    h, twin = qrl.TxCombiner(5000000, n_channels=3, max_in=4096), qrl.TxCombiner(5000000, n_channels=3, max_in=4096)
    for x in (h, twin):
        x.set_carrier_offset(1.1e6, channel=1)
    assert _same(_run(h, 0), _run(twin, 0))
    for k, st in enumerate([s.cuda_stream, None, None], 1):
        h.set_stream(st)
        assert _same(_run(h, k), _run(twin, k)), k
    s.synchronize()
    h.close(); twin.close()


def test_tx_combiner_null_handles_and_errors(qrl):
    L = qrl.load_library()
    assert L.qrl_tx_combiner_destroy(None) == 0                                     # QRL_OK
    assert L.qrl_tx_combiner_set_stream(None, None) == -22
    assert L.qrl_tx_combiner_set_gain(None, 1.0) == -22
    assert L.qrl_tx_combiner_set_carrier_offset(None, -1, 0.0) == -22
    assert L.qrl_tx_combiner_work(None, None, 0, 0, None) == -22
    assert L.qrl_tx_combiner_out_device(None, None, None) == -22
    assert L.qrl_tx_combiner_read(None, None, 0) == -22
    assert L.qrl_tx_combiner_launch_count(None) == 0
    for bad in ((0, 1, 16), (1500000, 1, 16), (33000000, 1, 16), (2000000, 0, 16), (2000000, 1, 0)):
        assert L.qrl_tx_combiner_create(bad[0], bad[1], bad[2], 0, C.byref(C.c_void_p())) == -22, bad
        assert L.qrl_last_error(None).decode().startswith("qrl_tx_combiner_create: "), L.qrl_last_error(None)
    assert L.qrl_tx_combiner_create(2000000, 1, 16, L.qrl_device_count(), C.byref(C.c_void_p())) == -19
    h = qrl.TxCombiner(2000000, n_channels=2, max_in=16)
    for ch, hz in ((2, 0.0), (-2, 0.0), (0, 1000001.0), (-1, -1000001.0), (0, float("nan"))):
        assert L.qrl_tx_combiner_set_carrier_offset(h._h, ch, hz) == -22, (ch, hz)
    assert L.qrl_tx_combiner_set_carrier_offset(h._h, 1, 1000000.0) == 0           # +samp_rate / 2 itself is accepted
    x = np.zeros((2, 17), np.complex64)
    n = C.c_long()
    rows = (C.c_void_p * 2)(x.ctypes.data, x.ctypes.data + x.strides[0])
    assert L.qrl_tx_combiner_work(h._h, rows, 17, 0, C.byref(n)) == -34             # QRL_ERANGE
    assert L.qrl_tx_combiner_work(h._h, (C.c_void_p * 2)(x.ctypes.data, None), 16, 0, C.byref(n)) == -22
    assert L.qrl_tx_combiner_work(h._h, None, 16, 0, C.byref(n)) == -22
    assert L.qrl_tx_combiner_work(h._h, (C.c_void_p * 2)(x.ctypes.data + 4, x.ctypes.data), 16, 0, C.byref(n)) == -22
    assert L.qrl_tx_combiner_work(h._h, rows, 0, 0, C.byref(n)) == 0 and n.value == 0
    assert h.launches == 0 and len(h.read()) == 0
    h.work(x[:, :16])
    assert h.launches == 1                                                           # one channel block: one kernel
    h.close()
