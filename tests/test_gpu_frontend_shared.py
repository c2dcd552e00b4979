"""GPU tier: one wideband stream feeding every channel of the receive front end (qrl_frontend_work with stride 0; gr_demod_mmdvm_multi's
one source -> rotator + /N resampler per channel): every channel bit-identical to a twin handle fed C identical rows and to the oracle
front end fed the same stream, at the register-tiled rates and one rate above them, with ragged chunks, retunes, host and device
input; three 4FSK signals in one 10 Msps capture decoded through one shared call; the error codes."""
import ctypes as C

import numpy as np
import pytest

from tests import siggen

pytestmark = pytest.mark.gpu

SIZES = [20000, 0, 1, 3, 50, 7777, 2501, 60000]  # at 107 Msps the last chunk alone is 560 outputs: five 128-output CTAs per channel
TOP_TILED = 32                                  # frontend_shared_kernel serves N <= 32; above, frontend_fir_kernel reads the one stream
TOP_RATE = 107000000                            # the highest rate qrl_frontend_create accepts (frontend_fir_kernel's shared memory)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _stream(samp_rate, T, seed):
    """one wideband capture: tones spread over the band plus noise, amplitude about 0.8"""
    rng = np.random.default_rng(seed)
    n = np.arange(T)
    x = 0.05 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))
    for f in (-0.37, -0.11, 0.02, 0.23, 0.41):
        x = x + 0.15 * np.exp(2j * np.pi * f * n)
    return x.astype(np.complex64)


def _read(q, fe):
    n = fe.out_device()[2]
    out = np.zeros((fe.n_channels, max(1, n)), np.complex64)
    assert q.load_library().qrl_frontend_read(fe._h, out.ctypes.data_as(C.c_void_p), out.shape[1]) == 0
    return out[:, :n]


def torch_device_input(x):
    """x copied to the GPU at an odd sample offset (8 bytes past a 16-byte boundary): (device pointer, owner)"""
    import torch
    buf = torch.zeros(len(x) + 1, dtype=torch.complex64, device="cuda")
    buf[1:] = torch.from_numpy(x)
    torch.cuda.synchronize()
    return buf.data_ptr() + 8, buf


def parity(q, oracle, samp_rate, Cn, sizes, retunes, kinds=("host",), dev_input=None, seed=0):
    """Feed one stream in the given chunks through a handle with stride 0 and, as [Cn, m] identical rows, through a twin handle;
    kinds[i % len(kinds)] says how chunk i reaches the first handle: "host" (stride 0), "dev" (stride 0, dev_input(x) gives the
    device pointer) or "rows" (a per-channel call with Cn identical rows).  Every chunk's output must equal the twin's bit for bit,
    and each channel must equal an oracle front end fed the stream: bit for bit, except that a channel at zero offset (never tuned)
    while others rotate may differ in the sign of an exact zero component (DESIGN §8 row a1).
    retunes: {chunk index: [(channel, hz), ...]} before that chunk; channel -1 = all."""
    T = sum(sizes)
    X = _stream(samp_rate, T, seed + samp_rate // 1000000)
    m_max = max(max(sizes), 1)
    fe = q.Frontend(samp_rate, n_channels=Cn, max_in=m_max)
    twin = q.Frontend(samp_rate, n_channels=Cn, max_in=m_max)
    ofe = [oracle.Frontend(samp_rate) for _ in range(Cn)]
    tuned = [False] * Cn
    lo = 0
    for i, m in enumerate(sizes):
        for ch, hz in retunes.get(i, []):
            fe.set_carrier_offset(hz, channel=ch); twin.set_carrier_offset(hz, channel=ch)
            for c in range(Cn):
                if ch < 0 or ch == c:
                    ofe[c].set_carrier_offset(hz); tuned[c] = True
        x = X[lo:lo + m]
        kind = kinds[i % len(kinds)]
        if kind == "dev":
            ptr, keep = dev_input(x)
            fe.work_device(ptr, m, 0)
            got = _read(q, fe)
            del keep
        elif kind == "rows":
            got = fe.work(np.repeat(x[None, :], Cn, axis=0))
        else:
            got = fe.work(x)
        ref = twin.work(np.repeat(x[None, :], Cn, axis=0))
        assert _same(got, ref), (samp_rate, Cn, i, kind)
        for c in range(Cn):
            want = ofe[c].work(x)
            assert len(want) == got.shape[1], (samp_rate, i, c)
            if tuned[c] or not any(tuned):
                assert _same(got[c], want), (samp_rate, Cn, i, c)
            else:
                assert np.array_equal(got[c], want), (samp_rate, Cn, i, c)
        lo += m
    fe.close(); twin.close()


def _offsets(samp_rate, Cn):
    """Cn distinct offsets across the band, channel 0 left at zero"""
    return {0: [(c, (c * 0.61 % 1.0 - 0.5) * 0.9 * samp_rate) for c in range(1, Cn)]}


RETUNES_ALL = {3: [(-1, 137500.0)], 5: [(1, -250000.0)]}


@pytest.mark.parametrize("samp_rate", [2000000, 5000000, 10000000, 20000000, TOP_TILED * 1000000, (TOP_TILED + 1) * 1000000, TOP_RATE])
def test_shared_stream_matches_twin_and_oracle(qrl, oracle, samp_rate):
    """3 channels at their own offsets (channel 0 at zero until all retune), then a retune of all and of one; host and device input
    at an odd sample offset, and per-channel calls, on one handle; up to the top rate (4475 taps, 162 416 B of shared memory)"""
    r = _offsets(samp_rate, 3)
    r.update(RETUNES_ALL)
    parity(qrl, oracle, samp_rate, 3, SIZES, r, kinds=("host", "dev", "rows", "host", "dev"), dev_input=torch_device_input)


@pytest.mark.parametrize("samp_rate,Cn", [(2000000, 1), (10000000, 33), (10000000, 97), (2000000, 97), (TOP_TILED * 1000000, 33),
                                          ((TOP_TILED + 1) * 1000000, 33)])
def test_shared_stream_channel_counts(qrl, oracle, samp_rate, Cn):
    """1, 33 and 97 channels: partial channel groups and (short chunks) one channel per group"""
    r = _offsets(samp_rate, Cn)
    r.update({2: [(-1, -62500.0)], 3: [(Cn // 2, 31250.0)]})
    parity(qrl, oracle, samp_rate, Cn, [30000, 1, 4999, 250000], r, kinds=("dev", "host"), dev_input=torch_device_input)


def test_one_capture_several_4fsk_signals(qrl, oracle):
    """Three 4FSK-2k-FM signals, each taken to 10 Msps by the transmit front end's oracle and moved to -3, +1 and +3.5 MHz, summed
    into one capture; one stride-0 call of a 4-channel front end (the fourth on an empty frequency) feeds the 4FSK receiver on the
    device.  Port 2 equals the oracle chain's and the frames come back on the three occupied channels: the oracle chain itself
    recovers 27 of the 30 frames on the -3 MHz channel of this capture (30 with that signal alone), so the bound is 4 short."""
    import torch
    from tests import tx_frontend_oracle as TO
    fs = 10000000
    offs = [-3000000.0, 1000000.0, 3500000.0, -1500000.0]
    datas, payloads = [], []
    for c in range(3):
        d, pl = siggen.frames_4fsk(np.random.default_rng(8100 + c), 30)
        datas.append(d); payloads.append(pl)
    sigs = []
    for c in range(3):
        y = oracle.Tx(oracle.MOD_4FSK, 25, 1000000, 1700, 3500, 1).work(datas[c])
        sigs.append(TO.TxFrontend(fs).work(y))
    T = max(len(s) for s in sigs)
    n = np.arange(T)
    cap = np.zeros(T, np.complex128)
    for c in range(3):
        cap[:len(sigs[c])] += sigs[c] * np.exp(2j * np.pi * offs[c] * n[:len(sigs[c])] / fs)
    cap = cap.astype(np.complex64)
    Cn = 4
    s = torch.cuda.Stream()
    fe = qrl.Frontend(fs, n_channels=Cn, max_in=T)
    rx = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=Cn, max_samples=T // 10 + 8)
    fe.set_stream(s.cuda_stream); rx.set_stream(s.cuda_stream)
    for c, f in enumerate(offs):
        fe.set_carrier_offset(f, channel=c)
    xd = torch.from_numpy(cap).cuda()
    torch.cuda.synchronize()
    k = fe.work_device(xd.data_ptr(), T, 0)
    p, st, items = fe.out_device()
    assert k == items == (T + 9) // 10
    rx.work_device(p, items, st)
    bits = rx.read_port(2)
    s.synchronize()
    for c in range(Cn):
        o = oracle.Frontend(fs); o.set_carrier_offset(offs[c])
        r = oracle.Rx(oracle.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1)
        r.work(o.work(cap))
        assert np.array_equal(bits[c], r.port(2)), c
        if c < 3:
            good, found = siggen.count_good_frames(bits[c], 0xED89AA, 24, 7, payloads[c])
            assert good >= len(payloads[c]) - 4, (c, good, found)
    fe.close(); rx.close()


def test_shared_stream_error_codes(qrl):
    L = qrl.load_library()
    fe = qrl.Frontend(2000000, n_channels=3, max_in=16)
    x = np.zeros(17, np.complex64)
    n = C.c_long(7)
    assert L.qrl_frontend_work(fe._h, x.ctypes.data_as(C.c_void_p), 17, 0, 0, C.byref(n)) == -34       # QRL_ERANGE
    assert L.qrl_frontend_work(fe._h, x.ctypes.data_as(C.c_void_p), 0, 0, 0, C.byref(n)) == 0 and n.value == 0
    assert fe.out_device()[2] == 0
    fe.close()
    # above the top rate the decimating FIR does not fit its kernel's shared memory: refused at create, not at every work call
    h = C.c_void_p()
    assert L.qrl_frontend_create(TOP_RATE + 1000000, 3, 4096, 0, C.byref(h)) == -22 and not h.value        # QRL_EINVAL
    msg = L.qrl_last_error(None).decode()
    assert msg.startswith("qrl_frontend_create: ") and "107 Msps" in msg, msg
    with pytest.raises(qrl.QrlError, match="107 Msps"):
        qrl.Frontend(108000000, n_channels=3, max_in=4096)
    fe = qrl.Frontend(TOP_RATE, n_channels=3, max_in=4096)
    assert fe.work(np.zeros(4096, np.complex64)).shape == (3, 39)
    fe.close()
