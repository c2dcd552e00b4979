"""GPU tier of the DMR burst decoder (qrl_dmr.cu): the device against the restatement in tests/dmr_model.py at 1, 33, 97 and 4096
channels with ragged chunks, the overflow / dropped path, reset(channel) equal to a fresh handle, every slot-type word, the EMB of
voice bursts (all 2^16 EMB words), every Golay(24,12) error pattern of weight <= 4 on AMBE frames, a round trip through the DMR
modulator and demodulator with port 2 read in place, handle errors and caller streams."""
import numpy as np
import pytest

from tests import dmr_model as M

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def q():
    import qradiolink_b200 as q
    if q.device_count() < 1:
        pytest.skip("no CUDA device")
    return q


_STREAMS = {}


def streams(C, seed):
    """C channels: a pool of 8 distinct mixed streams, each channel starting at its own offset"""
    if seed not in _STREAMS:
        rng = np.random.default_rng(seed)
        _STREAMS[seed] = [M.mixed_stream(rng, 12) for _ in range(8)]
    pool = _STREAMS[seed]
    return [np.roll(pool[c % 8], 37 * c) for c in range(C)]


def model_records(chans, cuts, ambe_fec):
    md = M.Decoder(len(chans), ambe_fec)
    out = [[] for _ in chans]
    for a, b in zip(cuts[:-1], cuts[1:]):
        for c, r in enumerate(md.work([ch[a[i]:b[i]] for i, ch in enumerate(chans)])):
            out[c] += r
    return out


@pytest.mark.parametrize("C", [1, 33, 97, 4096])
def test_device_equals_model_ragged(q, C):
    chans = streams(C, 5)
    lens = np.array([len(ch) for ch in chans])
    n = int(lens.max())
    rng = np.random.default_rng(C)
    mid = np.sort(rng.integers(0, lens[:, None] + 1, (C, 2)), axis=1)      # two ragged cuts per channel: three calls
    cuts = [np.zeros(C, int), mid[:, 0], mid[:, 1], lens]
    dec = q.DmrBurstDecoder(C, n, 64, ambe_fec=True)
    got = [[] for _ in range(C)]
    for a, b in zip(cuts[:-1], cuts[1:]):
        buf = np.zeros((C, n), np.uint8)
        cnt = (b - a).astype(np.int32)
        for c in range(C):
            buf[c, :cnt[c]] = chans[c][a[c]:b[c]]
        for c, g in enumerate(dec.work(buf, cnt)):
            got[c] += list(g)
    check = range(C) if C <= 97 else list(range(0, C, 97)) + [C - 1]
    want = model_records([chans[c] for c in check], [x[list(check)] for x in cuts], True)
    for i, c in enumerate(check):
        assert M.records_equal(got[c], want[i]) is None, (c, M.records_equal(got[c], want[i]))
    dec.close()


def test_dropped_and_reset_channel(q):
    chans = streams(4, 7)
    dec = q.DmrBurstDecoder(4, len(chans[0]), 4, ambe_fec=False)
    want = M.Decoder(4, False).work(chans)
    got = dec.work(chans)
    for c in range(4):
        assert M.records_equal(got[c], want[c][:4]) is None
    assert list(dec.dropped()) == [max(len(w) - 4, 0) for w in want]
    dec.work([c[:500] for c in chans])
    dec.reset(2)
    fresh = q.DmrBurstDecoder(4, len(chans[0]), 4, ambe_fec=False)
    a, b = dec.work(chans), fresh.work(chans)
    assert M.records_equal(a[2], M.Decoder(1).work([chans[2]])[0][:4]) is None
    assert [int(x) for x in a[2]["position"]] == [int(x) for x in b[2]["position"]]
    dec.close(); fresh.close()


def np_poly_mod(r, top, g, deg):
    for b in range(top, deg - 1, -1):
        r = np.where((r >> b) & 1, r ^ (g << (b - deg)), r)
    return r


def test_every_slot_type_word(q):
    """all 2^20 slot-type words, as data bursts of 4096 channels x 256 bursts, every one against the model's decoder"""
    C, per = 4096, 256
    base = M.data_burst(0, 9)
    words = np.arange(1 << 20, dtype=np.int64).reshape(C, per)
    burst = np.array(M.cach_bits(0, 1, 0) + base, np.uint8)
    bits = np.tile(burst, (C, per))
    pos = list(range(122, 132)) + list(range(180, 190))
    v = bits.reshape(C, per, 288)
    for j, p in enumerate(pos):
        v[:, :, p] = (words >> (19 - j)) & 1
    dec = q.DmrBurstDecoder(C, bits.shape[1], per)
    got = dec.work(bits)
    assert all(len(g) == per for g in got)
    code = words >> 1
    st = ((code ^ np.array(M.GOLAY19)[np_poly_mod(code, 18, 0xC75, 11)]) >> 11) & 0xFF
    cc = np.stack([g["color_code"] for g in got]).astype(np.int64)
    dt = np.stack([g["data_type"] for g in got]).astype(np.int64)
    assert np.array_equal((cc << 4) | dt, st)
    for c in (0, 1, 2047, 4095):
        assert M.records_equal(got[c], M.Decoder(1).work([bits[c]])[0]) is None
    dec.close()


def test_every_emb_word_and_ambe_error_pattern(q):
    """all 2^16 EMB words on voice bursts B-F, and every error pattern of weight <= 4 on the Golay(24,12) A word of AMBE frames"""
    C, SF = 4096, 2         # per channel 2 x (two superframes interleaved burst by burst, one per time slot)
    rng = np.random.default_rng(4)
    templates = []
    for t in range(16):
        sf = []
        for k in range(6):
            for slot in (1, 2):
                fb = M.voice_burst(rng, sync="bs_voice") if k == 0 else M.voice_burst(rng, emb=(0, 0, 0))
                sf += M.cach_bits(0, slot, 0) + fb
        templates.append(sf)
    T = np.array(templates, np.uint8)                                   # [16][12 * 288]
    bits = T[np.arange(C * SF) % 16].reshape(C, SF, 12, 288).copy()
    voice = bits[:, :, 2:, :].reshape(C, SF, 10, 288)                   # bursts B-F of both slots (a view: writes land in bits)
    n_b = C * SF * 10
    e = (np.arange(n_b) % 65536).reshape(C, SF, 10)
    for j in range(16):
        voice[..., 24 + (108 + j if j < 8 else 140 + j)] = (e >> (15 - j)) & 1
    pats = np.array([sum(1 << p for p in pos) for w in range(5) for pos in __import__("itertools").combinations(range(24), w)])
    assert len(pats) == 12951
    pat = pats[(np.arange(n_b * 3) % len(pats))].reshape(C, SF, 10, 3)
    for f in range(3):
        for t in range(24):
            voice[..., 24 + M.ambe_bit(f, t)] ^= ((pat[..., f] >> (23 - t)) & 1).astype(np.uint8)
    bits = bits.reshape(C, -1)
    dec = q.DmrBurstDecoder(C, bits.shape[1], SF * 12, ambe_fec=True)
    got = dec.work(bits)
    assert all(len(g) == SF * 12 for g in got)
    recs = np.stack(got).reshape(C, SF, 12)[:, :, 2:]
    code = e >> 1
    e8 = ((code ^ np.array(M.QR15)[np_poly_mod(code, 14, 0x139, 8)]) >> 7) & 0xFF
    assert np.array_equal(recs["emb_cc"], e8 >> 4) and np.array_equal(recs["emb_pi"], (e8 >> 3) & 1)
    assert np.array_equal(recs["emb_lcss"], (e8 >> 1) & 3)
    # AMBE error counts and regenerated bytes against the model, burst by burst (each distinct burst once)
    vb = voice.reshape(n_b, 288)
    want = np.zeros(n_b, np.int64)
    for i in range(n_b):
        fb = [int(x) for x in vb[i, 24:]]
        errs = 0
        for f in range(3):
            a = int("".join(str(fb[M.ambe_bit(f, t)]) for t in range(24)), 2)
            b = int("".join(str(fb[M.ambe_bit(f, t)]) for t in range(24, 47)), 2)
            errs += M.ambe_regenerate(a, b, 0)[3]
        want[i] = errs
    assert np.array_equal(recs["ambe_errors"].reshape(-1), want)
    for c in (0, 1, 4095):
        assert M.records_equal(got[c], M.Decoder(1, True).work([bits[c]])[0]) is None
    dec.close()


def test_round_trip_through_the_dmr_modem(q):
    """bursts built by the model -> QRL_MOD_DMR -> 30 dB AWGN -> QRL_DEMOD_DMR -> port 2 read in place (work_from_demod): every sent
    burst comes back with validate() true and the sent IDs"""
    from tests import siggen
    rng = np.random.default_rng(77)
    sent, stream = [], []
    filler = M.data_burst(1, 7, payload12=bytes(12))
    for k in range(40):
        slot = 1 + (k & 1)
        if k < 4 or k >= 34:
            fb = filler
        else:
            dst, src = int(rng.integers(1, 1 << 24)), int(rng.integers(1, 1 << 24))
            if k % 2:
                fb = M.data_burst(k % 16, 3, payload12=M.csbk_payload(0x04, 0, dst, src))
            else:
                fb = M.data_burst(k % 16, 1, payload12=M.lc_payload(0, 0, dst, src, 1))
            sent.append((src, dst))
        stream += M.cach_bits(0, slot, 0) + fb
    data = np.frombuffer(M.to_bytes(stream), np.uint8)
    iq = q.make_gr_mod_dmr(n_channels=1, max_items=len(data)).work(data[None, :])[0]
    x = siggen.channel(iq, rng, fo_hz=30, phase=0.2, delay=97, snr_db=30, amp=0.5, total=len(iq) + 30000)
    rx = q.make_gr_demod_dmr(n_channels=1, max_samples=len(x))
    rx.work(x[None, :])
    dec = q.DmrBurstDecoder(1, 1 << 20, 128)
    got = dec.work_from_demod(rx)[0]
    ids = {(int(r["src_id"]), int(r["dst_id"])) for r in got if r["valid"] and r["data_type"] in (1, 3)}
    assert set(sent) <= ids, (len(sent), len(ids))
    assert all(r["downlink"] for r in got)
    dec.close()


def test_handle_errors_and_caller_stream(q):
    import torch
    with pytest.raises(q.QrlError):
        q.DmrBurstDecoder(0, 100, 4)
    dec = q.DmrBurstDecoder(2, 1000, 4)
    with pytest.raises(q.QrlError):
        dec.work(np.zeros((2, 2000), np.uint8))
    with pytest.raises(q.QrlError):
        dec.reset(5)
    s = torch.cuda.Stream()
    dec.set_stream(s.cuda_stream)
    chans = streams(2, 5)
    dec2 = q.DmrBurstDecoder(2, len(chans[0]), 64)
    dec2.set_stream(s.cuda_stream)
    want = M.Decoder(2).work(chans)
    got = dec2.work(chans)
    for c in range(2):
        assert M.records_equal(got[c], want[c]) is None
    dec.close(); dec2.close()
