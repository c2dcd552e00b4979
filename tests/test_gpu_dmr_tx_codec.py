"""GPU tier of the DMR burst encoder (qrl_dmr.cu's qrl_dmr_tx_*): the device against the restatement in tests/dmr_tx_model.py at 1, 33,
97 and 4096 channels with per-channel settings, ragged calls, reset(channel) mid-stream and calls at max_ops; device input on a
caller's stream; handle errors; and round trips encoder -> QRL_MOD_DMR -> 30 dB AWGN -> QRL_DEMOD_DMR -> qrl_dmr_rx reading port 2
in place, with the zero tags registered by DmrBurstEncoder.feed (the cleared spans placed to the output item) and without them (every
burst that comes back is one the encoder sent)."""
import numpy as np
import pytest

from tests import dmr_model as M
from tests import dmr_tx_model as T
from tests.test_dmr_tx_codec import random_cfgs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def q():
    import qradiolink_b200 as q
    if q.device_count() < 1:
        pytest.skip("no CUDA device")
    return q


def configure(q, enc, cfgs):
    for c, cfg in enumerate(cfgs):
        enc.set_config(q.dmr_tx_config(cfg.color_code, cfg.timeslot, cfg.src_id, cfg.dst_id, cfg.private_call, cfg.codec2,
                                       cfg.talker_alias), channel=c)
    enc.reset()


def check_call(got, model, ops, audio, chans):
    got_b, got_r = got
    for c in chans:
        wb, wr = model[c].work(ops[c], audio[c])
        assert bytes(got_b[c]) == wb, c
        assert [tuple(int(x) for x in r) for r in got_r[c]] == [tuple(x) for x in wr], c


@pytest.mark.parametrize("C_", [1, 33, 97, 4096])
def test_device_equals_model(q, C_):
    rng = np.random.default_rng(C_)
    cfgs = random_cfgs(rng, C_)
    max_ops = 48
    enc = q.DmrBurstEncoder(C_, max_ops)
    configure(q, enc, cfgs)
    # the model runs on every channel up to 97, on a spread of channels at 4096
    chans = list(range(C_)) if C_ <= 97 else sorted(set(range(0, C_, 127)) | {C_ - 1})
    model = {c: T.Channel(cfgs[c]) for c in chans}
    for call, K in enumerate([5, 48, 1, 0, 17, 48, 30]):
        ops = np.stack([T.random_ops(rng, K) for _ in range(C_)]) if K else np.zeros((C_, 0), np.uint8)
        if call == 0:
            ops[:, 0] = T.OP_HEADER
        if call == 5:
            ops[::2] = T.OP_CSBK                                  # max_ops reached: 3 * max_ops bursts
        audio = rng.integers(0, 256, (C_, K, 9)).astype(np.uint8)
        got = enc.work(ops, audio)
        check_call(got, model, ops, audio, chans)
        if call == 5:
            assert len(got[1][0]) == 3 * max_ops
        if call == 3:                                             # reset(channel) mid-stream
            enc.reset(chans[-1])
            model[chans[-1]].reset(cfgs[chans[-1]])
    enc.close()


def test_device_input_on_a_caller_stream(q):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(4)
    C_, K = 64, 40
    cfgs = random_cfgs(rng, C_)
    enc = q.DmrBurstEncoder(C_, K)
    configure(q, enc, cfgs)
    s = torch.cuda.Stream()
    enc.set_stream(s.cuda_stream)
    model = [T.Channel(cfg) for cfg in cfgs]
    for call in range(3):
        ops = np.stack([T.random_ops(rng, K) for _ in range(C_)])
        ops[:, 0] = T.OP_HEADER if call == 0 else ops[:, 0]
        audio = rng.integers(0, 256, (C_, K, 9)).astype(np.uint8)
        with torch.cuda.stream(s):
            d_ops = torch.from_numpy(ops).cuda()
            d_audio = torch.from_numpy(audio).cuda()
        enc.work_device(d_ops.data_ptr(), d_audio.data_ptr(), K)
        check_call(enc.read(), model, ops, audio, range(C_))
    enc.close()


def test_op_indices_past_int16(q):
    """vocoder frames addressed by op indices above 32767, one of them carried into the next call"""
    K = 32800
    enc = q.DmrBurstEncoder(1, K)
    model = T.Channel()
    rng = np.random.default_rng(6)
    for call in range(2):
        ops = np.zeros((1, K), np.uint8)
        ops[0, 0] = T.OP_HEADER if call == 0 else T.OP_NONE
        ops[0, [32770, 32780, 32790, 32799] if call == 0 else [3, 4]] = T.OP_AUDIO
        audio = rng.integers(0, 256, (1, K, 9)).astype(np.uint8)
        got = enc.work(ops, audio)
        check_call(got, {0: model}, ops, audio, [0])
        assert len(got[1][0]) == (3 if call == 0 else 1)
    enc.close()


def test_handle_errors(q):
    L = q.load_library()
    with pytest.raises(q.QrlError):
        q.DmrBurstEncoder(0, 4)
    enc = q.DmrBurstEncoder(2, 4)
    with pytest.raises(q.QrlError):
        enc.work(np.zeros((2, 5), np.uint8))                       # K > max_ops
    for bad in (dict(color_code=16), dict(timeslot=0), dict(timeslot=3), dict(src_id=1 << 24), dict(dst_id=1 << 24)):
        with pytest.raises(q.QrlError):
            enc.set_config(**bad)
    cfg = q.dmr_tx_config()
    cfg.talker_alias_len = 28
    with pytest.raises(q.QrlError):
        enc.set_config(cfg)
    cfg.talker_alias_len, cfg.private_call = 0, 2
    with pytest.raises(q.QrlError):
        enc.set_config(cfg)
    with pytest.raises(q.QrlError):
        enc.set_config(channel=2)
    with pytest.raises(q.QrlError):
        enc.reset(2)
    assert L.qrl_dmr_tx_work(None, None, None, 0, 0) == -22
    assert L.qrl_dmr_tx_reset(None, 0) == -22 and L.qrl_dmr_tx_sync(None) == -22 and L.qrl_dmr_tx_launch_count(None) == 0
    enc.close()


# ---------------------------------------------------------------- round trips through the DMR modem
UP_NUM, UP_DEN = 125, 3           # gr_mod_dmr's final interpolator: 125 / 3 output items per 24 ksps item
ITEMS_PER_BYTE = 20               # 4 symbols per byte, 5 items per symbol
ZERO_LEAD = 62                    # gr_zero_idle_bursts loads its counter `delay` items before the tagged item
HISTORY = 1439                    # gr_zero_idle_bursts' history: 2 * 720 - 1 silent items in front of the stream
RT_OPS = [T.OP_CSBK, T.OP_HEADER] + [T.OP_AUDIO] * 54 + [T.OP_STOP] + [T.OP_AUDIO] * 3


def zero_runs(iq):
    """[start, end) of every run of output items that are exactly zero"""
    d = np.diff(np.concatenate([[0], (iq == 0).astype(np.int8), [0]]))
    return list(zip(np.flatnonzero(d == 1).tolist(), np.flatnonzero(d == -1).tolist()))


def check_cleared_spans(iq, recs):
    """every burst's zero_samples tag (byte position + 33, 780 items) as a run of exact zeros in the modulator's output: it ends on the
    output item where the 780 cleared 24 ksps items end, and starts once the interpolator's window holds only cleared items, the same
    number of items after the cleared span's start for every burst.  Burst 0's span falls inside the silence of the history."""
    runs = zero_runs(iq)
    assert runs[0] == (0, -(-HISTORY * UP_NUM // UP_DEN))
    spans = []                                                                # (first cleared item x 125, end output item)
    for r in recs:
        s = (int(r["position"]) + 33) * ITEMS_PER_BYTE - ZERO_LEAD            # first cleared 24 ksps item
        spans.append((s * UP_NUM, -(-(s + T.ZERO_SAMPLES) * UP_NUM // UP_DEN)))
    assert spans[0][1] <= runs[0][1]
    assert len(runs) == len(recs), (len(runs), len(recs))
    lead = runs[1][0] * UP_DEN - spans[1][0]                                  # in 1/3 output items
    assert 0 < lead <= 33 * UP_NUM                                            # the interpolator's arms: 33 taps
    for (start, end), (s125, e0) in zip(runs[1:], spans[1:]):
        assert end == e0 and start * UP_DEN - s125 == lead, (start, end, s125, e0)


def through_the_modem(q, enc, ops, audio, rng, tagged):
    """encoder -> QRL_MOD_DMR (through feed with the zero tags, or the bytes alone) -> 30 dB AWGN -> QRL_DEMOD_DMR -> qrl_dmr_rx on port
    2 in place: (sent bytes, records, modulator output, decoder records, port-2 bits)"""
    sent_b, sent_r = enc.work(ops, audio)
    mod = q.make_gr_mod_dmr(n_channels=1, max_items=len(sent_b[0]))
    iq = enc.feed(mod)[0] if tagged else mod.work(sent_b[0][None, :])[0]
    x = siggen_channel(iq, rng)
    rx = q.make_gr_demod_dmr(n_channels=1, max_samples=len(x))
    rx.work(x[None, :])
    bits = rx.read_port(2)[0]
    dec = q.DmrBurstDecoder(1, 1 << 20, 256)
    got = dec.work_from_demod(rx)[0]
    dec.close()
    return bytes(sent_b[0]), sent_r[0], iq, got, bits


def siggen_channel(iq, rng):
    from tests import siggen
    return siggen.channel(iq, rng, fo_hz=30, phase=0.2, delay=97, snr_db=30, amp=0.5, total=len(iq) + 30000)


DATA_TYPES = [3, 3, 3, 1, 1, 2, 2]      # the cut data bursts: 3 CSBK, 2 LC headers, 2 terminators


def check_tagged(sent, recs, got):
    """with the zero tags: every data burst is cut and keeps its slot type (colour code 5), none is one of the sent bursts -- the
    clear starts 62 items (3.1 bytes) before the tagged byte 33, on the burst's own last bytes, as gr_zero_idle_bursts' lead does"""
    data = [r for r in got if r["frame_type"] == 0]
    assert [int(r["data_type"]) for r in data] == DATA_TYPES
    assert all(r["color_code"] == 5 for r in data)
    bursts = {sent[r["position"]:r["position"] + 33] for r in recs}
    for r in data:
        assert (bytes(r["frame"]) in bursts) == bool(r["valid"])


def check_untagged(sent, recs, got):
    """without the tags the 39 zero bytes are modulated: every cut burst is one the encoder sent, bytes for bytes.  Data bursts
    validate (the first may fall in the receiver's pull-in) with colour code 5 and the sent IDs; voice sync bursts come back whole;
    gr_dmr_sink cuts voice bursts B-F by count, 288 bits each, so in the 576-bit period of this layout every other cut is a sent
    voice burst (EMB colour code 5, the sent LCSS) and the others are the 264 zero bits after one (EMB 0)."""
    by_bytes = {sent[r["position"]:r["position"] + 33]: r for r in recs}
    data = [r for r in got if r["frame_type"] == 0]
    assert [int(r["data_type"]) for r in data] == DATA_TYPES
    assert all(r["valid"] for r in data[1:]) and all(r["color_code"] == 5 for r in data)
    for r in data:
        if r["valid"]:
            sr = by_bytes[bytes(r["frame"])]
            assert sr["kind"] in (T.KIND_CSBK, T.KIND_LC_HEADER, T.KIND_TERMINATOR) and r["src_id"] == 0x12345
    sync = [r for r in got if r["frame_type"] == 2]
    assert len(sync) == 3 and all(by_bytes[bytes(r["frame"])]["kind"] == T.KIND_VOICE_SYNC for r in sync)
    voice = [r for r in got if r["frame_type"] == 1]
    assert len(voice) >= 10
    n_sent = 0
    for r in voice:
        if r["emb_cc"] == 5:
            sr = by_bytes[bytes(r["frame"])]
            assert sr["kind"] == T.KIND_VOICE and sr["lcss"] == r["emb_lcss"]
            n_sent += 1
        else:
            assert bytes(r["frame"]) == bytes(33) and r["emb_cc"] == 0
    assert n_sent >= 5


def round_trip_encoder(q):
    enc = q.DmrBurstEncoder(1, len(RT_OPS))
    enc.set_config(color_code=5, timeslot=2, src_id=0x12345, dst_id=0x777, talker_alias="N0CALL")
    enc.reset()
    return enc


def test_round_trip_with_zero_tags(q):
    """DmrBurstEncoder.feed registers every burst's zero_samples tag: the cleared spans sit where the records put them, to the output
    item; the decoder's records are the receive restatement's on the same bits; and what comes back is check_tagged's"""
    rng = np.random.default_rng(78)
    ops = np.array(RT_OPS, np.uint8)[None, :]
    audio = rng.integers(0, 256, (1, ops.shape[1], 9)).astype(np.uint8)
    enc = round_trip_encoder(q)
    sent, recs, iq, got, bits = through_the_modem(q, enc, ops, audio, rng, True)
    enc.close()
    check_cleared_spans(iq, recs)
    assert M.records_equal(got, M.Decoder(1).work([bits])[0]) is None
    check_tagged(sent, recs, got)


def test_round_trip_without_zero_tags(q):
    """the encoder's bytes through the modem with no tags: the decoder's records are the receive restatement's on the same bits, and
    every burst it cuts is one the encoder sent (check_untagged)"""
    rng = np.random.default_rng(79)
    ops = np.array(RT_OPS, np.uint8)[None, :]
    audio = rng.integers(0, 256, (1, ops.shape[1], 9)).astype(np.uint8)
    enc = round_trip_encoder(q)
    sent, recs, iq, got, bits = through_the_modem(q, enc, ops, audio, rng, False)
    enc.close()
    assert zero_runs(iq) == [(0, -(-HISTORY * UP_NUM // UP_DEN))]
    assert M.records_equal(got, M.Decoder(1).work([bits])[0]) is None
    check_untagged(sent, recs, got)
