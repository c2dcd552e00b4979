"""CPU tier of the DMR burst encoder (qrl_dmr.cu's qrl_dmr_tx_*, qradiolink_b200/dmr.py's DmrBurstEncoder), pinned to the reference's
own DMRFrame and src/MMDVM encoders compiled behind oracle/ref_dmr_tx_shim.cpp (oracle/_ref/libqrl_ref_dmr_tx.so, built by
oracle/ref_dmr_tx.mk), or to the digests of their results in tests/golden/ref_dmr_tx.json where the reference is absent
(`python -m tests.test_dmr_tx_codec` regenerates them):
  * the restatement tests/dmr_tx_model.py, burst for burst: CSBK, header and terminator over all 16 colour codes x both slots, group
    and private calls, AMBE and codec2 FID; voice at every FN of every superframe position with talker aliases of 0, 1, 6, 7, 26 and 27
    bytes;
  * every burst it encodes decodes through the receive restatement (tests/dmr_model.decode_burst) to the same fields and bytes;
  * DMRControl's state machine against expectations read off its lines;
  * the library's own kernels, compiled for host threads (tools/emu/build_emulated_lib.py), through the real C ABI, against the
    restatement for random op streams cut into ragged calls."""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from tests import dmr_model as M
from tests import dmr_tx_model as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_dmr_tx.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_dmr_tx.json")
TA_LENGTHS = (0, 1, 6, 7, 26, 27)


def digest(b):
    return hashlib.sha256(bytes(b)).hexdigest()


class Ref:
    """the compiled reference encoders"""

    def __init__(self):
        self.L = C.CDLL(REF_LIB)
        self.o = np.zeros(33, np.uint8)

    def _p(self, a):
        return a.ctypes.data_as(C.c_void_p)

    def csbk(self, cc, slot, src, dst):
        self.L.ref_dmr_tx_csbk(cc, slot, C.c_uint(src), C.c_uint(dst), self._p(self.o))
        return self.o.tobytes()

    def lc(self, dt, cc, slot, flco, fid, src, dst):
        self.L.ref_dmr_tx_lc(dt, cc, slot, flco, fid, C.c_uint(src), C.c_uint(dst), self._p(self.o))
        return self.o.tobytes()

    def voice(self, audio27, fn, cc, lc9):
        a = np.frombuffer(bytes(audio27), np.uint8).copy()
        src, dst = int.from_bytes(lc9[6:9], "big"), int.from_bytes(lc9[3:6], "big")
        self.L.ref_dmr_tx_voice(self._p(a), fn, cc, lc9[0] & 0x3F, lc9[1], lc9[2], C.c_uint(src), C.c_uint(dst), self._p(self.o))
        return self.o.tobytes()


@pytest.fixture(scope="module")
def R():
    return Ref() if os.path.exists(REF_LIB) else None


# ---------------------------------------------------------------- burst cases: (what the reference call is, the model's bytes)
def control_cases():
    """CSBK, header and terminator for every colour code x slot, group / private, AMBE / codec2: [(ref call args, model bytes)]"""
    rng = np.random.default_rng(21)
    out = []
    for cc in range(16):
        for slot in (1, 2):
            src, dst = int(rng.integers(0, 1 << 24)), int(rng.integers(0, 1 << 24))
            out.append((("csbk", cc, slot, src, dst), T.csbk_burst(cc, src, dst)))
            for private in (False, True):
                flco = T.FLCO_USER_USER if private else T.FLCO_GROUP
                for fid in (0, 0xC2):
                    out.append((("lc", T.DT_VOICE_LC_HEADER, cc, slot, flco, fid, src, dst),
                                T.lc_burst(T.lc_bytes(flco, fid, 0, src, dst), T.DT_VOICE_LC_HEADER, cc)))
                out.append((("lc", T.DT_TERMINATOR_WITH_LC, cc, slot, flco, 0, src, dst),
                            T.lc_burst(T.lc_bytes(flco, 0, 0, src, dst), T.DT_TERMINATOR_WITH_LC, cc)))
    return out


def voice_cases(ta_len):
    """one channel through a header and 5 superframes (every FN at every superframe position, the talker-alias LCs among them):
    [(fn, cc, audio27, embedded LC, model bytes)]"""
    rng = np.random.default_rng(100 + ta_len)
    cfg = T.Config(color_code=int(rng.integers(0, 16)), timeslot=2, src_id=int(rng.integers(0, 1 << 24)),
                   dst_id=int(rng.integers(0, 1 << 24)), private_call=bool(ta_len & 1), codec2=ta_len % 3 == 0,
                   talker_alias=bytes(int(x) for x in rng.integers(32, 127, ta_len)))
    ch = T.Channel(cfg)
    ch.op(T.OP_HEADER)
    out = []
    for _ in range(3 * 6 * 6):
        a = bytes(int(x) for x in rng.integers(0, 256, 9))
        fn, lc, pending = ch.fn, ch.emb_lc, list(ch.pending)
        for kind, slot, bfn, lcss, b in ch.op(T.OP_AUDIO, a):
            assert bfn == fn
            out.append((fn, cfg.color_code, b"".join(pending) + a, lc, b))
    assert len(out) == 36 and [o[0] for o in out] == list(range(6)) * 6
    return out


def ref_bytes(R, case):
    kind, *args = case
    return R.csbk(*args) if kind == "csbk" else R.lc(*args)


def test_control_bursts_are_the_reference(R):
    cases = control_cases()
    model = b"".join(b for _, b in cases)
    if R is not None:
        for args, b in cases:
            assert ref_bytes(R, args) == b, args
    assert digest(model) == json.load(open(GOLDEN))["control"]


@pytest.mark.parametrize("ta_len", TA_LENGTHS)
def test_voice_bursts_are_the_reference(R, ta_len):
    cases = voice_cases(ta_len)
    if R is not None:
        for fn, cc, audio, lc, b in cases:
            assert R.voice(audio, fn, cc, lc) == b, (fn, lc.hex())
    assert digest(b"".join(c[-1] for c in cases)) == json.load(open(GOLDEN))["voice_ta%d" % ta_len]


# ---------------------------------------------------------------- through the receive restatement
def decode(b, frame_type, fn=0):
    return M.decode_burst(dict(bits=[0] * 24 + M.to_bits(b), frame_type=frame_type, fn=fn, downlink=0, position=0, ts_index=0), False)


def test_control_bursts_decode():
    for args, b in control_cases():
        o = decode(b, 0)
        cc, src, dst = args[1 if args[0] == "csbk" else 2], args[-2], args[-1]
        assert o["valid"] == 1 and o["color_code"] == cc and o["frame"] == b
        assert (o["src_id"], o["dst_id"]) == ((src, 0) if args[0] == "csbk" else (src, dst))     # BSDWNACT carries the BS ID
        if args[0] == "csbk":
            assert o["data_type"] == T.DT_CSBK and o["flco"] == T.CSBKO_BSDWNACT and o["fid"] == 0
        else:
            assert (o["data_type"], o["flco"], o["fid"]) == (args[1], args[4], args[5])


@pytest.mark.parametrize("ta_len", TA_LENGTHS)
def test_voice_bursts_decode(ta_len):
    raw = {}
    for fn, cc, audio, lc, b in voice_cases(ta_len):
        o = decode(b, 2 if fn == 0 else 1, fn)
        assert o["frame"] == b
        fb = M.to_bits(b)
        assert M.to_bytes(fb[:108] + fb[156:]) == audio                  # setVoice: 216 vocoder bits around the middle 48
        if fn == 0:
            assert o["data_type"] == M.DT_VOICE_SYNC and M.to_bytes(fb[108:156]) == M.SYNC_BYTES["ms_voice"]
        else:
            assert (o["emb_cc"], o["emb_pi"], o["emb_lcss"]) == (cc, 0, T.LCSS_OF_FN[fn])
            raw.setdefault(lc, []).append(fb[116:148])
    # the four fragments of an embedded LC de-interleave to the LC and its checksum
    for lc, frags in raw.items():
        bits = sum(frags[:4], [])
        data = [0] * 128
        b = 0
        for a in range(128):
            data[b] = bits[a]
            b += 16
            if b > 127:
                b -= 127
        pos = list(range(0, 11)) + list(range(16, 27)) + [a for r in range(2, 7) for a in range(16 * r, 16 * r + 10)]
        assert M.to_bytes([data[p] for p in pos]) == lc
        assert sum((data[16 * r + 10] << (6 - r)) for r in range(2, 7)) == sum(lc) % 31


def test_talker_alias_lcs():
    ta = bytes(range(0x41, 0x41 + 27))
    ch = T.Channel(T.Config(talker_alias=ta, src_id=0x123456, dst_id=0x654321, codec2=True))
    ch.op(T.OP_HEADER)
    lcs = []
    for _ in range(5 * 6 * 3 + 6):
        lc = ch.emb_lc
        if [b[2] for b in ch.op(T.OP_AUDIO)] == [1]:
            lcs.append(lc)
    assert lcs[0] == bytes([0, 0xC2, 0, 0x65, 0x43, 0x21, 0x12, 0x34, 0x56])          # superframe 0: the voice LC
    assert lcs[1] == bytes([4, 0, 0x76]) + ta[0:6]                                       # header: format 1, length 0x1B
    assert lcs[2] == bytes([5, 0]) + ta[6:13] and lcs[3] == bytes([6, 0]) + ta[12:19] and lcs[4] == bytes([7, 0]) + ta[18:25]
    assert lcs[5] == lcs[0]                                                              # the superframe wraps after 5


# ---------------------------------------------------------------- the state machine, from DMRControl's lines
def kinds(bursts):
    return [b[0] for b in bursts]


def test_audio_before_a_header_is_dropped():
    ch = T.Channel()
    assert all(ch.op(T.OP_AUDIO) == [] for _ in range(7)) and ch.pending == []
    assert kinds(ch.op(T.OP_CSBK)) == [T.KIND_CSBK] * 3 and ch.state == T.IDLE
    assert kinds(ch.op(T.OP_HEADER)) == [T.KIND_LC_HEADER] * 2 and ch.state == T.ACTIVE
    assert [kinds(ch.op(T.OP_AUDIO)) for _ in range(3)] == [[], [], [T.KIND_VOICE_SYNC]]


@pytest.mark.parametrize("stop_fn", range(6))
def test_stop_at_every_fn(stop_fn):
    ch = T.Channel()
    ch.op(T.OP_HEADER)
    for _ in range(3 * stop_fn):
        ch.op(T.OP_AUDIO)
    assert ch.fn == stop_fn
    ch.op(T.OP_AUDIO)                                  # one frame pending across the stop
    assert ch.op(T.OP_STOP) == [] and ch.state == T.ENDING
    got = []
    for _ in range(3 * 7):
        got += ch.op(T.OP_AUDIO)
        if ch.state == T.IDLE:
            break
    want = [T.KIND_VOICE_SYNC if f == 0 else T.KIND_VOICE for f in range(stop_fn, 6)] if stop_fn else []
    want += [T.KIND_TERMINATOR, T.KIND_TERMINATOR, T.KIND_EMPTY, T.KIND_EMPTY]
    assert kinds(got) == want
    assert [b[2] for b in got[:-4]] == list(range(stop_fn, 6)) if stop_fn else True
    assert got[-1][1] == 0 and got[-1][4] == bytes(33) and got[-4][1] == 1
    assert ch.pending == [] and ch.sf == 0 and ch.fn == 0
    assert all(ch.op(T.OP_AUDIO) == [] for _ in range(4))          # idle again: audio dropped


def test_terminator_needs_three_frames_at_fn0():
    ch = T.Channel()
    ch.op(T.OP_HEADER)
    ch.op(T.OP_STOP)
    assert ch.op(T.OP_AUDIO) == [] and ch.op(T.OP_AUDIO) == []
    assert kinds(ch.op(T.OP_AUDIO)) == [T.KIND_TERMINATOR] * 2 + [T.KIND_EMPTY] * 2


def test_stop_from_idle():
    ch = T.Channel(T.Config(private_call=True, codec2=True))
    assert ch.op(T.OP_STOP) == [] and ch.state == T.ENDING
    ch.op(T.OP_AUDIO), ch.op(T.OP_AUDIO)
    got = ch.op(T.OP_AUDIO)
    assert kinds(got) == [T.KIND_TERMINATOR] * 2 + [T.KIND_EMPTY] * 2
    o = decode(got[0][4], 0)                                       # the constructor's FLCO, no codec2 FID on a terminator
    assert (o["data_type"], o["flco"], o["fid"], o["valid"]) == (T.DT_TERMINATOR_WITH_LC, T.FLCO_USER_USER, 0, 1)


def test_header_keeps_pending_frames():
    ch = T.Channel()
    ch.op(T.OP_HEADER)
    ch.op(T.OP_AUDIO, b"\x01" * 9), ch.op(T.OP_AUDIO, b"\x02" * 9)
    ch.op(T.OP_HEADER)
    got = ch.op(T.OP_AUDIO, b"\x03" * 9)
    assert kinds(got) == [T.KIND_VOICE_SYNC]
    fb = M.to_bits(got[0][4])
    assert M.to_bytes(fb[:108] + fb[156:]) == b"\x01" * 9 + b"\x02" * 9 + b"\x03" * 9


def test_settings_change_mid_transmission():
    ch = T.Channel(T.Config(color_code=3, src_id=10, dst_id=20))
    ch.op(T.OP_HEADER)
    for _ in range(3):
        ch.op(T.OP_AUDIO)
    ch.cfg = T.Config(color_code=9, src_id=11, dst_id=21, private_call=True, codec2=False, timeslot=2)
    got = []
    for _ in range(3):
        got += ch.op(T.OP_AUDIO)
    assert got[0][1] == 2 and decode(got[0][4], 1, 1)["emb_cc"] == 9            # colour code and slot: the next burst
    assert ch.emb_lc == T.lc_bytes(0, 0xC2, 0, 10, 20) == ch.lc_tx               # the LC: not before the next header
    ch.op(T.OP_HEADER)
    assert ch.lc_tx == T.lc_bytes(3, 0, 0, 11, 21)


def test_superframe_wraps_after_five():
    ch = T.Channel()
    ch.op(T.OP_HEADER)
    sfs = []
    for _ in range(3 * 6 * 11):
        if ch.op(T.OP_AUDIO) and ch.fn == 1:
            sfs.append(ch.sf)
    assert sfs == [0, 1, 2, 3, 4, 0, 1, 2, 3, 4, 0]


def test_record_positions_and_tags():
    ch = T.Channel()
    ops = [T.OP_CSBK, T.OP_HEADER] + [T.OP_AUDIO] * 6 + [T.OP_STOP] + [T.OP_AUDIO] * 15
    b, recs = ch.work(ops, [bytes(9)] * len(ops))
    assert len(b) == 72 * len(recs) and [r[0] for r in recs] == list(range(0, len(b), 72))
    assert all(b[r[0] + 33:r[0] + 72] == bytes(39) for r in recs)
    assert T.tags(recs)[:2] == [("tx_time", 0, 1), ("zero_samples", 33, 780)]
    assert [r[5] for r in recs[:5]] == [0, 0, 0, 1, 1]


# ---------------------------------------------------------------- the kernels, on host threads
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_dmr_tx")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    yield q
    L._LIB_PATH, L._LIB = saved


def run_cuts(q, cfgs, ops, audio, cuts, max_ops):
    """feed [C][N] ops in calls cut at `cuts`; compare bytes and records with the model call by call"""
    C_, N = ops.shape
    enc = q.DmrBurstEncoder(C_, max_ops)
    model = [T.Channel(cfg) for cfg in cfgs]
    for c, cfg in enumerate(cfgs):
        enc.set_config(q.dmr_tx_config(cfg.color_code, cfg.timeslot, cfg.src_id, cfg.dst_id, cfg.private_call, cfg.codec2,
                                       cfg.talker_alias), channel=c)
    enc.reset()
    edges = [0] + list(cuts) + [N]
    nb = 0
    for a, b in zip(edges[:-1], edges[1:]):
        got_b, got_r = enc.work(ops[:, a:b], audio[:, a:b])
        for c in range(C_):
            wb, wr = model[c].work(ops[c, a:b], audio[c, a:b])
            assert bytes(got_b[c]) == wb, (a, b, c)
            assert [tuple(int(x) for x in r) for r in got_r[c]] == [tuple(x) for x in wr], (a, b, c)
            nb += len(wr)
    enc.close()
    return nb


def random_cfgs(rng, n):
    return [T.Config(int(rng.integers(0, 16)), int(rng.integers(1, 3)), int(rng.integers(0, 1 << 24)), int(rng.integers(0, 1 << 24)),
                     bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), bytes(int(x) for x in rng.integers(0, 256, int(rng.integers(0, 28)))))
            for _ in range(n)]


def test_kernels_equal_the_model_in_ragged_calls(emu):
    rng = np.random.default_rng(8)
    C_, N = 5, 400
    ops = np.stack([T.random_ops(rng, N) for _ in range(C_)])
    ops[:, 0] = T.OP_HEADER
    ops[0, ::37] = 7                                           # values above 4 count as none
    audio = rng.integers(0, 256, (C_, N, 9)).astype(np.uint8)
    # one cut at every op position within a 4-op window, then ragged calls, empty ones included
    cuts = [10, 11, 12, 13, 14, 14, 30, 31, 97, 98, 99, 150, 233, 234, 300, 301, 302, 303]
    assert run_cuts(emu, random_cfgs(rng, C_), ops, audio, cuts, 120) > 100


def test_kernels_at_max_ops_and_reset(emu):
    rng = np.random.default_rng(9)
    C_, K = 3, 16
    cfgs = random_cfgs(rng, C_)
    ops = np.full((C_, K), T.OP_AUDIO, np.uint8)
    ops[:, 0] = T.OP_HEADER
    ops[1, 5:] = T.OP_STOP                                     # a terminator every third audio op: 4 bursts per op at most
    ops[1, 6::3] = T.OP_AUDIO
    ops[2, :] = T.OP_CSBK                                      # 3 bursts per op, the full K
    audio = rng.integers(0, 256, (C_, K, 9)).astype(np.uint8)
    enc = emu.DmrBurstEncoder(C_, K)
    for c, cfg in enumerate(cfgs):
        enc.set_config(emu.dmr_tx_config(cfg.color_code, cfg.timeslot, cfg.src_id, cfg.dst_id, cfg.private_call, cfg.codec2,
                                         cfg.talker_alias), channel=c)
    enc.reset()
    model = [T.Channel(cfg) for cfg in cfgs]
    for rep in range(3):
        got_b, got_r = enc.work(ops, audio)
        for c in range(C_):
            wb, wr = model[c].work(ops[c], audio[c])
            assert bytes(got_b[c]) == wb and len(got_r[c]) == len(wr), (rep, c)
        if rep == 1:                                           # reset(channel): the constructor state, position 0
            enc.reset(1)
            model[1].reset(cfgs[1])
    assert len(got_r[2]) == 3 * K
    with pytest.raises(Exception):
        enc.work(np.zeros((C_, K + 1), np.uint8))
    enc.close()


def regenerate_golden():
    R = Ref()
    golden = {"control": digest(b"".join(ref_bytes(R, args) for args, _ in control_cases()))}
    for n in TA_LENGTHS:
        golden["voice_ta%d" % n] = digest(b"".join(R.voice(audio, fn, cc, lc) for fn, cc, audio, lc, _ in voice_cases(n)))
    json.dump(golden, open(GOLDEN, "w"), indent=1, sort_keys=True)
    open(GOLDEN, "a").write("\n")


if __name__ == "__main__":
    regenerate_golden()
