"""GPU tier: the M17 frame codec on the device (qrl_m17.cu) against tests/m17_model.py, the numpy restatement the CPU tier pins to
the reference's own M17 code (tests/test_m17_codec.py), and against the compiled reference itself where oracle/_ref holds it."""
import ctypes as C

import numpy as np
import pytest

from qradiolink_b200 import m17 as Q
from tests import m17_model as M
from tests import test_m17_codec as T

pytestmark = [pytest.mark.gpu]


def _bits_of_records(recs, rng):
    """a bit stream (one bit per byte) that carries the records, each behind its sync word, with a little filler in between"""
    parts = []
    for t, p in recs:
        sync = t.to_bytes(4 if t == M.EOT else 2, "big")
        parts.append(np.zeros(int(rng.integers(0, 24)), np.uint8))
        parts.append(np.unpackbits(np.frombuffer(sync + bytes(p), np.uint8)))
    parts.append(np.zeros(16, np.uint8))
    return np.concatenate(parts)


@pytest.mark.parametrize("C_", [1, 33, 97, 4096])
def test_decoder_fed_by_the_deframer(qrl, C_):
    n_rec = 24 if C_ < 1000 else 6
    chans = T.rx_case(2000 + C_, C_, n_rec)
    rng = np.random.default_rng(C_)
    bits = [_bits_of_records(r, rng) for r in chans]
    dfr = qrl.Deframer.for_mode("M17", n_channels=C_, max_bits=max(len(b) for b in bits), max_frames=2 * n_rec)
    dec = Q.M17Decoder(C_, 2 * n_rec)
    recs = dfr.work(bits)
    got = dec.work_from_deframer(dfr)
    want = M.decode_channels([[(t, p) for t, p in r] for r in recs])
    R = T.ref_m17()
    for c in range(C_):
        assert len(recs[c]) >= len([r for r in chans[c] if r[0] in (M.LSF, M.STREAM, M.EOT)]), c
        mine = T.snapshots(got[c])
        assert mine == want[c], c
        if R is not None and c < 40:
            assert mine == T.ref_decode(R, recs[c]), c


def test_golay_every_error_pattern_up_to_weight_4(qrl):
    """all 12 951 error patterns of weight <= 4 on a 24-bit LICH word, each in a channel of six stream records (segments 0-5): the
    pattern sits in word (p mod 4) of segment (p mod 6); whether and how the LSF reassembles shows the Golay decoder's verdict"""
    pats = [0]
    for w in range(1, 5):
        from itertools import combinations
        pats += [sum(1 << b for b in comb) for comb in combinations(range(24), w)]
    assert len(pats) == 12951
    tx = M.Transmitter()
    tx.set_lsf(Q.m17_lsf("AB1CD", "W1AW", 5, 0))
    frames = [tx.step(2, bytes([k] * 16))[2:48] for k in range(6)]
    chans = []
    for p, e in enumerate(pats):
        seg, word = p % 6, p % 4
        recs = [(M.STREAM, f) for f in frames]
        flips = [24 * word + (23 - b) for b in range(24) if e >> b & 1]
        recs[seg] = (M.STREAM, T._scrambled_flip(frames[seg], flips))
        chans.append(recs)
    dec = Q.M17Decoder(len(chans), 6)
    got = dec.work(chans)
    want = M.decode_channels(chans)
    n_valid = 0
    for c in range(len(chans)):
        mine = T.snapshots(got[c])
        assert mine == want[c], c
        n_valid += got[c][-1][2]
        if bin(pats[c]).count("1") <= 3:
            assert got[c][-1][2] and got[c][-1][1] == tx.lsf30, c
    assert n_valid >= 2325                  # every pattern of weight <= 3 corrects


def test_encoder_is_the_reference(qrl):
    C_, K, calls = 9, 12, 4
    args, ops, pl = T.tx_case(2100, C_, K, calls)
    enc = Q.M17Encoder(C_, K)
    for c in range(C_):
        enc.set_lsf(c, Q.m17_lsf(*args[c]))
    out = [b""] * C_
    for k in range(calls):
        got = enc.work(ops[:, k * K:(k + 1) * K], pl[:, k * K:(k + 1) * K])
        out = [o + g.tobytes() for o, g in zip(out, got)]
    R = T.ref_m17()
    for c in range(C_):
        assert out[c] == T.model_tx(args[c], ops[c], pl[c]), c
        if R is not None:
            assert out[c] == b"".join(T.ref_transmit(R, args[c], ops[c], pl[c])), c
    T.test_encoder_counters_wrap_across_calls(qrl, None)


def test_round_trip_on_the_device(qrl):
    """encoder -> QRL_MOD_M17 -> AWGN at 30 dB -> QRL_DEMOD_M17 -> deframer (sync class 4) -> decoder, every buffer in HBM until the
    decoder's records are read: every channel recovers its LSF with a valid CRC and every payload"""
    torch = pytest.importorskip("torch")
    L = qrl.load_library()
    C_, n_frames = 8, 30
    K = n_frames + 2
    ops = np.array([[1] + [2] * n_frames + [3]] * C_, np.uint8)
    rng = np.random.default_rng(2200)
    pl = rng.integers(0, 256, (C_, K, 16), dtype=np.uint8)
    enc = Q.M17Encoder(C_, K)
    lsfs = [Q.m17_lsf("CH%d" % c, "W1AW", c % 16, 0) for c in range(C_)]
    for c in range(C_):
        enc.set_lsf(c, lsfs[c])
    enc.work(ops, pl, collect=False)
    optr, ostride, _ = enc.out_device()
    n = 96 + 48 * n_frames + 64
    enc.sync()
    tx = qrl.make_gr_mod_m17(n_channels=C_, max_items=n)
    tx.work_device(optr.value, n, ostride)
    nout = C.c_long()
    assert L.qrl_tx_out_device(tx._h, None, None, C.byref(nout)) == 0
    y = torch.zeros((C_, nout.value), dtype=torch.complex64, device="cuda")
    n2 = C.c_long()
    assert L.qrl_tx_read(tx._h, C.c_void_p(y.data_ptr()), nout.value, C.byref(n2), 1) == 0
    torch.cuda.synchronize()
    g = torch.Generator(device="cuda").manual_seed(2201)
    lead, tail = 2000, 60000
    x = torch.zeros((C_, lead + n2.value + tail), dtype=torch.complex64, device="cuda")
    x[:, lead:lead + n2.value] = 0.5 * y[:, :n2.value]
    p = (x[:, lead:lead + n2.value].abs() ** 2).mean()
    sigma = torch.sqrt(p / 1000.0 / 2.0)                      # 30 dB SNR, complex AWGN
    x += torch.complex(torch.randn(x.shape, generator=g, device="cuda"), torch.randn(x.shape, generator=g, device="cuda")) * sigma
    x = x.contiguous()
    torch.cuda.synchronize()
    rx = qrl.make_gr_demod_m17(n_channels=C_, max_samples=x.shape[1])
    rx.work_device(x.data_ptr(), x.shape[1], x.shape[1])
    data, cap, cnts = C.c_void_p(), C.c_long(), C.c_void_p()
    assert L.qrl_rx_port_device(rx._h, 2, C.byref(data), C.byref(cap), C.byref(cnts)) == 0
    rx.sync()
    dfr = qrl.Deframer.for_mode("M17", n_channels=C_, max_bits=cap.value, max_frames=K + 8)
    assert L.qrl_deframer_work(dfr._h, data, cnts, cap.value, 1) == 0
    dec = Q.M17Decoder(C_, K + 8)
    got = dec.work_from_deframer(dfr)                           # the first copy to the host
    for c in range(C_):
        lsf30 = lsfs[c] + Q.m17_crc16(lsfs[c]).to_bytes(2, "big")
        assert any(v and lsf == lsf30 for t, lsf, v, sf in got[c]), c          # from the LSF frame or reassembled from the LICH
        seen = {}
        for t, lsf, v, sf in got[c]:
            if t == M.STREAM:
                seen[int.from_bytes(sf[:2], "big") & 0x7FFF] = sf[2:]
        for k in range(n_frames + 1):
            assert seen.get(k) == pl[c, k + 1].tobytes(), (c, k)
        assert any(t == M.EOT for t, _, _, _ in got[c]), c


def test_handles_streams_and_errors(qrl):
    L = qrl.load_library()
    assert L.qrl_m17_rx_destroy(None) != 0 and L.qrl_m17_tx_destroy(None) != 0
    h = C.c_void_p()
    assert L.qrl_m17_rx_create(0, 4, 0, C.byref(h)) != 0
    assert b"bad argument" in L.qrl_last_error(None)
    dec = Q.M17Decoder(2, 4)
    with pytest.raises(qrl.QrlError):
        dec.reset(2)
    with pytest.raises(ValueError):
        dec.work([[(M.STREAM, bytes(46))] * 5, []])             # more records than max_frames
    buf = np.zeros((2, 8, 56), np.uint8); cnt = np.zeros(2, np.int32)
    assert L.qrl_m17_rx_work(dec._h, buf.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), 56, 8, 0) != 0   # > max_frames
    assert b"max_frames" in L.qrl_last_error(dec._h)
    enc = Q.M17Encoder(2, 4)
    with pytest.raises(qrl.QrlError):
        enc.set_lsf(5, bytes(28))
    assert L.qrl_m17_tx_work(enc._h, buf.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), 5, 0) != 0
    # a caller's stream: the same results
    s = pytest.importorskip("torch").cuda.Stream()
    tx = M.Transmitter(); tx.set_lsf(Q.m17_lsf("N0CALL"))
    recs = [[(M.LSF, tx.step(1, None)[50:])], [(M.STREAM, tx.step(2, bytes(16))[2:48])]]
    want = [T.snapshots(g) for g in dec.work(recs)]
    dec2 = Q.M17Decoder(2, 4)
    dec2.set_stream(s.cuda_stream)
    assert [T.snapshots(g) for g in dec2.work(recs)] == want
    dec2.set_stream(0)
    enc.set_stream(s.cuda_stream)
    enc.set_lsf(0, Q.m17_lsf("N0CALL")); enc.set_lsf(1, Q.m17_lsf("N0CALL"))
    o = enc.work(np.array([[1, 2, 0, 3]] * 2, np.uint8))
    assert o[0].tobytes() == o[1].tobytes() and len(o[0]) == 96 + 48 + 64
    assert dec.launches == 3 and enc.launches == 2      # reset at create + frame + state kernels; scan + encode
    for x in (dec, dec2, enc):
        x.close()
