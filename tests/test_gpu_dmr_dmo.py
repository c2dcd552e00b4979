"""GPU tier of the DMR direct-mode (DMO) burst decoder (qrl_dmr.cu's dmr_dmo_sink_kernel): the device against the restatement in
tests/dmr_dmo_model.py at 1, 33, 97 and 4096 channels with ragged per-channel counts, from host and device input; the overflow /
dropped path; reset(channel) equal to a fresh handle; a caller's stream; argument errors; port 3 of QRL_DEMOD_DMR read in place; and
the round trip DmrBurstEncoder -> QRL_MOD_DMR -> 30 dB AWGN -> QRL_DEMOD_DMR -> DmrDmoBurstDecoder, with and without the
zero_samples tags."""
import numpy as np
import pytest

from tests import dmr_dmo_model as D
from tests import dmr_model as M

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def q():
    import qradiolink_b200 as q
    if q.device_count() < 1:
        pytest.skip("no CUDA device")
    return q


_POOL = []


def pool():
    """8 distinct streams of the CPU tier's cases, each with the model's records over its whole length"""
    if not _POOL:
        from tests.test_dmr_dmo_codec import CASES
        n = max(len(x) for _, x, _ in CASES)
        rng = np.random.default_rng(9)
        for k in range(8):
            x = CASES[k][1]
            x = np.concatenate([x, D.to_samples(D.random_symbols(rng, (n - len(x)) // 5 + 1))])[:n].astype(np.float32)
            _POOL.append((x, D.DmoDecoder(1, True).work([x])[0]))
    return _POOL


def between(recs, a, b):
    return [r for r in recs if a <= r["position"] < b]


@pytest.mark.parametrize("C", [1, 33, 97, 4096])
@pytest.mark.parametrize("device_input", [False, True])
def test_device_equals_model_ragged(q, C, device_input):
    import torch
    P = pool()
    n = len(P[0][0])
    rng = np.random.default_rng(C + device_input)
    mid = np.sort(rng.integers(0, n + 1, (C, 2)), axis=1)       # two ragged cuts per channel: three calls
    cuts = [np.zeros(C, int), mid[:, 0], mid[:, 1], np.full(C, n)]
    dec = q.DmrDmoBurstDecoder(C, n, ambe_fec=True)
    for a, b in zip(cuts[:-1], cuts[1:]):
        cnt = (b - a).astype(np.int32)
        buf = np.zeros((C, n), np.float32)
        for c in range(C):
            buf[c, :cnt[c]] = P[c % 8][0][a[c]:b[c]]
        if device_input:
            tb, tc = torch.from_numpy(buf).cuda(), torch.from_numpy(cnt).cuda()
            torch.cuda.synchronize()
            dec.work_device(tb.data_ptr(), n, n, tc.data_ptr())
            got = dec.read()
        else:
            got = dec.work(buf, cnt)
        for c in (range(C) if C <= 97 else list(range(0, C, 61)) + [C - 1]):
            want = between(P[c % 8][1], a[c], b[c])
            assert M.records_equal(got[c], want) is None, (C, c, M.records_equal(got[c], want))
    assert not dec.dropped().any()
    dec.close()


def test_dropped_and_reset_equals_fresh(q):
    x, recs = pool()[2]
    dec = q.DmrDmoBurstDecoder(2, len(x), 3, True)
    got = dec.work(np.stack([x, x]))
    assert len(recs) > 3 and all(M.records_equal(g, recs[:3]) is None for g in got)
    assert list(dec.dropped()) == [len(recs) - 3] * 2
    dec.reset(1)
    assert list(dec.dropped()) == [len(recs) - 3, 0]
    got = dec.work(np.stack([x, x]))
    fresh = q.DmrDmoBurstDecoder(1, len(x), 3, True)
    assert np.array_equal(got[1], fresh.work(x[None, :])[0])
    dec.close(); fresh.close()


def test_caller_stream_and_errors(q):
    import torch
    with pytest.raises(q.QrlError):
        q.DmrDmoBurstDecoder(0, 100)
    with pytest.raises(q.QrlError):
        q.DmrDmoBurstDecoder(1, 0)
    dec = q.DmrDmoBurstDecoder(2, 1000)
    with pytest.raises(q.QrlError):
        dec.work(np.zeros((2, 2000), np.float32))          # n > max_samples
    with pytest.raises(q.QrlError):
        dec.work(np.zeros((2, 100), np.float32), np.array([5, 101], np.int32))
    with pytest.raises(q.QrlError):
        dec.reset(2)
    L = q.load_library()
    assert L.qrl_dmr_dmo_rx_work(None, None, 0, None, 0, 0) != 0
    assert L.qrl_dmr_dmo_rx_record_bytes(None) == 0 and L.qrl_dmr_dmo_rx_record_bytes(dec._h) == 72
    dec.close()
    P = pool()
    xs = np.stack([P[0][0], P[5][0]])
    a = q.DmrDmoBurstDecoder(2, xs.shape[1], ambe_fec=True)
    b = q.DmrDmoBurstDecoder(2, xs.shape[1], ambe_fec=True)
    s = torch.cuda.Stream()
    b.set_stream(s.cuda_stream)
    ga, gb = a.work(xs), b.work(xs)
    for c in range(2):
        assert np.array_equal(ga[c], gb[c]) and len(ga[c]) > 3
    a.close(); b.close()


def demod_port3(q, iq, rng):
    from tests import siggen
    x = siggen.channel(iq, rng, fo_hz=30, phase=0.2, delay=97, snr_db=30, amp=0.5, total=len(iq) + 30000)
    rx = q.make_gr_demod_dmr(n_channels=1, max_samples=len(x))
    rx.work(x[None, :])
    return rx, x


def test_work_from_demod_equals_model_on_oracle_port3(q):
    from oracle import oracle as O
    from tests.test_dmr_dmo_codec import oracle_port3
    rng = np.random.default_rng(31)
    y = oracle_port3()
    # the oracle's port 3 fed through the decoder's own input, and the device demodulator's port 3 read in place
    dec = q.DmrDmoBurstDecoder(1, len(y), ambe_fec=True)
    assert M.records_equal(dec.work(y[None, :])[0], D.DmoDecoder(1, True).work([y])[0]) is None
    enc = q.DmrBurstEncoder(1, 64)
    ops = np.array([[2] + [3] * 45 + [4] + [3] * 6], np.uint8)
    enc.work(ops, rng.integers(0, 256, (1, ops.shape[1], 9)).astype(np.uint8))
    tx = q.make_gr_mod_dmr(n_channels=1, max_items=1 << 16)
    iq = enc.feed(tx)[0]
    rx, x = demod_port3(q, iq, rng)
    p3 = rx.read_port(3)[0]
    ref = O.Rx(O.DEMOD_DMR, 5, 1000000, 0, 0, 0)
    ref.work(x)
    assert np.array_equal(p3, ref.port(3))
    dec2 = q.DmrDmoBurstDecoder(1, len(p3), ambe_fec=True)
    got = dec2.work_from_demod(rx)[0]
    assert len(got) > 10 and M.records_equal(got, D.DmoDecoder(1, True).work([p3])[0]) is None
    dec.close(); dec2.close(); enc.close()


@pytest.mark.parametrize("tags", [False, True])
def test_round_trip_through_the_dmr_modem(q, tags):
    """DmrBurstEncoder's voice call (LC header x2, 7 superframes, terminator x2) -> QRL_MOD_DMR -> 30 dB AWGN -> QRL_DEMOD_DMR ->
    DmrDmoBurstDecoder.  The model says what comes back: both LC headers, every voice burst with FN 0..5, the first terminator
    (which resets the sink, so the second and the empty frames are not written), all with the encoder's colour code.  Without the
    tags every burst's bytes are the encoder's but for its last symbol (the sink slices it from the ring slot after the end pointer,
    which holds the sample of 1439 samples before).  With them the modulator clears the last 3.1 bytes of each burst (INTEGRATION
    §3h) and the transmit and receive filters spread that edge over a few more symbols, so bytes 0-25 of every voice burst match (a
    header or terminator whose cleared bits validate() fails to correct keeps no promise about its bytes)."""
    rng = np.random.default_rng(41 + tags)
    enc = q.DmrBurstEncoder(1, 160)
    enc.set_config(color_code=9, src_id=4242, dst_id=77)
    K = 1 + 7 * 6 * 3 + 1 + 3
    ops = np.array([[2] + [3] * (K - 5) + [4] + [3] * 3], np.uint8)
    audio = rng.integers(0, 256, (1, K, 9)).astype(np.uint8)
    sent, recs = enc.work(ops, audio)
    sent, recs = sent[0], recs[0]
    tx = q.make_gr_mod_dmr(n_channels=1, max_items=len(sent) + 64)
    if tags:
        iq = enc.feed(tx)[0]
    else:
        iq = tx.work(sent[None, :])[0]
    rx, _ = demod_port3(q, iq, rng)
    p3 = rx.read_port(3)[0]
    dec = q.DmrDmoBurstDecoder(1, len(p3), ambe_fec=False)
    got = dec.work_from_demod(rx)[0]
    want = D.DmoDecoder(1, False).work([p3])[0]
    assert M.records_equal(got, want) is None
    kinds = [int(r["kind"]) for r in recs]
    bursts = [sent[72 * i:72 * i + 33] for i in range(len(recs))]
    exp = [i for i, k in enumerate(kinds) if k in (2, 3, 4)] + [kinds.index(5)]
    assert len(got) == len(exp), (len(got), len(exp))
    m = 26 if tags else 32
    for r, i in zip(got, exp):
        if not tags or kinds[i] in (3, 4):
            assert bytes(r["frame"][:m]) == bytes(bursts[i][:m])
        assert tags or (r["frame"][32] ^ bursts[i][32]) & 0xFC == 0
        assert r["color_code"] == 9 and r["slot_no"] == 2
        assert int(r["fn"]) == (int(recs[i]["fn"]) if kinds[i] in (3, 4) else 0)
        assert int(r["frame_type"]) == {2: 0, 3: 2, 4: 1, 5: 0}[kinds[i]]
    lc = [r for r in got if r["frame_type"] == 0]
    assert [int(r["data_type"]) for r in lc] == [1, 1, 2]
    if not tags:
        assert all(r["valid"] for r in lc)
    dec.close(); enc.close()
