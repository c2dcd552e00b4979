"""CPU tier of the DMR burst decoder (qrl_dmr.cu, qradiolink_b200/dmr.py), pinned to the reference's own gr_dmr_sink, DMRFrame and
src/MMDVM code compiled behind oracle/ref_dmr_shim.cpp (oracle/_ref/libqrl_ref_dmr.so, built by oracle/ref_dmr.mk), or to the digests of
its results in tests/golden/ref_dmr.json where the reference is absent (`python -m tests.test_dmr_codec` regenerates them):
  * the decoders the restatement's generated tables drive, exhaustively: Golay(20,8) over 2^20 words, QR(16,7) over 2^16, Golay(24,12)
    over 2^24, Golay(23,12) over 2^23, and (as bursts) the CACH check over its 2^7 bit patterns;
  * the restatement tests/dmr_model.py, record for record, one bit per call (exact positions and slots), and the same streams in ragged
    calls, long enough for the trim at the start of gr_dmr_sink::work to run, where every record but its position and slot must hold;
  * the library's own kernels, compiled for host threads (tools/emu/build_emulated_lib.py), through the real C ABI, record for record
    against the restatement in tests/dmr_model.py: BS and MS syncs in both slots, voice superframes, every data type with 0-3 bit
    errors, rate 3/4 with errors, a sync arriving with fewer than 180 bits buffered, overlapping sync words, ambe_fec on and off, and
    the same stream cut into calls at every bit phase of a burst."""
import hashlib
import json
import ctypes as C
import os
import sys

import numpy as np
import pytest

from tests import dmr_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_dmr.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_dmr.json")
RAGGED = [37, 1100, 5, 2900, 288, 1, 977]


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Ref:
    """the compiled reference, or None"""

    def __init__(self):
        L = C.CDLL(REF_LIB)
        L.ref_dmr_create.restype = C.c_void_p
        for f in ("ref_golay24128_decode", "ref_golay23127_decode"):
            getattr(L, f).restype = C.c_uint32
        self.L = L

    def work(self, bits, chunks, ambe_fec):
        from qradiolink_b200.dmr import DMR_RECORD
        L = self.L
        h = C.c_void_p(L.ref_dmr_create())
        bits = np.ascontiguousarray(bits, np.uint8)
        ch = np.array(chunks, np.int32)
        out = np.zeros((8192, 72), np.uint8)
        n = L.ref_dmr_work(h, bits.ctypes.data_as(C.c_void_p), C.c_long(len(bits)), ch.ctypes.data_as(C.c_void_p), len(ch), int(ambe_fec),
                           out.ctypes.data_as(C.c_void_p), len(out))
        L.ref_dmr_destroy(h)
        return out[:n].copy().view(DMR_RECORD).reshape(-1)


@pytest.fixture(scope="module")
def R():
    return Ref() if os.path.exists(REF_LIB) else None


def model_array(recs):
    """Decoder.work's records of one channel -> a DMR_RECORD array"""
    from qradiolink_b200.dmr import DMR_RECORD
    a = np.zeros(len(recs), DMR_RECORD)
    for i, r in enumerate(recs):
        for k in M.REC_FIELDS:
            a[i][k] = r[k]
        a[i]["cach"] = np.frombuffer(r["cach"], np.uint8)
        a[i]["frame"] = np.frombuffer(r["frame"], np.uint8)
    return a


def without_position(a):
    a = a.copy()
    a["position"] = 0
    a["ts_index"] = 0
    return a


def pinned(R, key, want_array):
    """the reference's result for `key` (computed by fn) or its committed digest"""
    golden = json.load(open(GOLDEN))
    assert digest(want_array) == golden[key], key


# ---------------------------------------------------------------- generated tables, exhaustively, through the model's decoders (numpy)
def np_poly_mod(r, top, g, deg):
    r = r.astype(np.int64)
    for b in range(top, deg - 1, -1):
        r = np.where((r >> b) & 1, r ^ (g << (b - deg)), r)
    return r


def model_slot_type(w20):
    code = w20 >> 1
    return ((code ^ np.array(M.GOLAY19)[np_poly_mod(code, 18, 0xC75, 11)]) >> 11) & 0xFF


def model_emb(w16):
    code = w16 >> 1
    return ((code ^ np.array(M.QR15)[np_poly_mod(code, 14, 0x139, 8)]) >> 7) & 0xFF


def model_golay24(w24):
    syn = np_poly_mod(w24 >> 1, 22, 0xC75, 11)
    out = w24 ^ (np.array(M.GOLAY23)[syn] << 1)
    pc = lambda v: np.array([bin(x).count("1") for x in range(1 << 12)])[v & 0xFFF] + np.array([bin(x).count("1") for x in range(1 << 12)])[(v >> 12) & 0xFFF]
    valid = (pc(syn) < 3) | ((pc(out) & 1) == 0)
    return (out >> 12) | (valid.astype(np.int64) << 12)


def model_golay23(w23):
    return (w23 ^ np.array(M.GOLAY23)[np_poly_mod(w23, 22, 0xC75, 11)]) >> 11


TABLE_CASES = {"golay2087": (20, model_slot_type), "qr1676": (16, model_emb), "golay24128": (24, model_golay24), "golay23127": (23, model_golay23)}


def ref_table(R, name):
    n = TABLE_CASES[name][0]
    L = R.L
    f = {"golay2087": L.ref_golay2087_decode, "qr1676": L.ref_qr1676_decode, "golay23127": L.ref_golay23127_decode}.get(name)
    if f is not None:
        return np.array([f(w) for w in range(1 << n)], np.int64)
    out = np.zeros(1 << n, np.int64)
    o = C.c_uint32()
    for w in range(1 << n):
        v = L.ref_golay24128_decode(w, C.byref(o))
        out[w] = o.value | (v << 12)
    return out


@pytest.mark.parametrize("name", sorted(TABLE_CASES))
def test_generated_tables_are_the_reference(R, name):
    n, fn = TABLE_CASES[name]
    got = fn(np.arange(1 << n, dtype=np.int64))
    if R is not None and n <= 20:
        assert np.array_equal(got, ref_table(R, name))
    pinned(R, "table_" + name, got)


def test_golden_tables_match_the_reference(R):
    if R is None:
        pytest.skip("reference tree absent")
    golden = json.load(open(GOLDEN))
    for name in sorted(TABLE_CASES):
        if TABLE_CASES[name][0] > 20:
            assert digest(ref_table(R, name)) == golden["table_" + name], name


def test_golay23_table_corrects_every_pattern_of_weight_3():
    assert len(set(M.GOLAY23)) == 2048
    for w in range(4):
        for e in [sum(1 << p for p in pos) for pos in __import__("itertools").combinations(range(23), w)][:400]:
            assert M.GOLAY23[M.poly_mod(e, 22, 0xC75, 11)] == e


def test_table_leaders_have_least_weight():
    for tab, n, g, deg in ((M.GOLAY19, 19, 0xC75, 11), (M.QR15, 15, 0x139, 8)):
        for s, e in enumerate(tab):
            if e:
                assert M.poly_mod(e, n - 1, g, deg) == s
    # the (19,8) code has 4 syndromes whose leaders weigh 6: they stay 0
    assert sum(1 for s, e in enumerate(M.GOLAY19) if s and not e) == 4
    assert all(M.QR15[s] or s == 0 for s in range(256))


def test_codes_round_trip():
    rng = np.random.default_rng(3)
    for _ in range(50):
        d = int(rng.integers(0, 4096))
        ok, got = M.golay24_decode(M.golay24_encode(d) ^ (1 << int(rng.integers(0, 24))))
        assert ok and got == d
        pl = bytes(int(x) for x in rng.integers(0, 256, 12))
        fb = [0] * 264
        M.bptc_encode(pl, fb)
        for i in rng.choice(196, 2, replace=False):
            fb[M.info_bit(int(i))] ^= 1
        assert M.bptc_decode(fb) == pl
        pts = M.trellis_encode(bytes(int(x) for x in rng.integers(0, 256, 18)))
        assert M.trellis_check(pts)[0] == 999


def cases():
    """(name, per-channel bit streams, ambe_fec)"""
    rng = np.random.default_rng(11)
    out = [("mixed", [M.mixed_stream(rng, 10), M.mixed_stream(rng, 10, errors=(0,))], True),
           ("mixed_no_fec", [M.mixed_stream(rng, 10)], False)]
    # MS syncs, a sync with fewer than 180 bits buffered, overlapping sync words, rate 3/4 with errors
    fb = M.data_burst(3, 3, payload12=M.csbk_payload(0x04, 0, 12345, 678))
    ms = M.data_burst(5, 1, payload12=M.lc_payload(0, 0, 99, 4242, 1), sync="ms_data")
    r34 = M.flip(M.data_burst(7, 8, points=M.trellis_encode(bytes(range(18)))), rng, 3)
    short = [0] * 50 + fb[108:156] + [0] * 200           # sync 98 bits into the stream
    overlap = M.to_bits(M.SYNC_BYTES["bs_data"] + M.SYNC_BYTES["bs_voice"])
    s = M.cach_bits(0, 1, 0) + fb + M.cach_bits(1, 2, 3) + ms + short + overlap + [1, 0] * 300 + M.cach_bits(0, 1, 1) + r34
    s += M.cach_bits(0, 2, 0) + M.voice_burst(rng, sync="ms_voice") + sum((M.voice_burst(rng, emb=(2, 1, 1)) for _ in range(5)), [])
    s += [int(x) for x in rng.integers(0, 2, 2600)]         # a long search: the sink's buffer passes 864 bits
    s += sum((M.cach_bits(0, 1, 0) + M.data_burst(1, 3, payload12=M.csbk_payload(0x3D, 0, 5, 6)) for _ in range(2)), [])
    out.append(("edges", [np.array(s, np.uint8)], True))
    # the CACH check over all 2^7 patterns of its 7 bits, each in front of a valid burst
    cach = []
    for v in range(128):
        cb = [0] * 24
        for j, p in enumerate((0, 4, 8, 12, 14, 18, 22)):
            cb[p] = (v >> (6 - j)) & 1
        cach += cb + M.data_burst(2, 7, payload12=bytes(12))
    out.append(("cach", [np.array(cach, np.uint8)], False))
    return out


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_dmr")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    yield q
    L._LIB_PATH, L._LIB = saved


def run(q, streams, ambe_fec, cuts, max_bursts=256):
    """feed each stream in calls cut at the given bit offsets; returns the records per channel and the model's"""
    dec = q.DmrBurstDecoder(len(streams), max(len(s) for s in streams), max_bursts, ambe_fec)
    model = M.Decoder(len(streams), ambe_fec)
    got, want = [[] for _ in streams], [[] for _ in streams]
    edges = [0] + list(cuts) + [max(len(s) for s in streams)]
    for a, b in zip(edges[:-1], edges[1:]):
        part = [s[a:b] for s in streams]
        for c, g in enumerate(dec.work(part)):
            got[c] += list(g)
        for c, w in enumerate(model.work(part)):
            want[c] += w
    dec.close()
    return got, want


@pytest.mark.parametrize("name,streams,ambe_fec", cases(), ids=[c[0] for c in cases()])
def test_model_is_the_reference(R, name, streams, ambe_fec):
    for c, s in enumerate(streams):
        want = model_array(M.Decoder(1, ambe_fec).work([s])[0])
        assert len(want) >= 4
        if R is not None:
            ref = R.work(s, [1], ambe_fec)
            assert M.records_equal(ref, M.Decoder(1, ambe_fec).work([s])[0]) is None, M.records_equal(ref, M.Decoder(1, ambe_fec).work([s])[0])
            # ragged calls: the trim at the start of work() changes no burst
            assert np.array_equal(without_position(R.work(s, RAGGED, ambe_fec)), without_position(want))
        pinned(R, "rec_%s_%d" % (name, c), want)


@pytest.mark.parametrize("name,streams,ambe_fec", cases(), ids=[c[0] for c in cases()])
def test_kernels_equal_the_model(emu, R, name, streams, ambe_fec):
    got, want = run(emu, streams, ambe_fec, ())
    assert sum(len(w) for w in want) >= 4
    for c in range(len(streams)):
        assert M.records_equal(got[c], want[c]) is None, (c, M.records_equal(got[c], want[c]))
        if R is not None:
            assert np.array_equal(np.array(got[c]), R.work(streams[c], [1], ambe_fec))
        pinned(R, "rec_%s_%d" % (name, c), np.array(got[c]))


def test_chunk_cuts_at_every_bit_phase(emu):
    streams = cases()[2][1]
    n = len(streams[0])
    assert n > 5000
    for phase in range(0, 288, 13):
        cuts = list(range(100 + phase, n, 288 + 7))
        got, want = run(emu, streams, True, cuts)
        assert M.records_equal(got[0], want[0]) is None, (phase, M.records_equal(got[0], want[0]))


def test_dropped_and_reset(emu):
    streams = cases()[0][1][:1]
    dec = emu.DmrBurstDecoder(1, len(streams[0]), 3, True)
    want = M.Decoder(1, True).work(streams)[0]
    got = dec.work(streams)[0]
    assert len(want) > 3 and M.records_equal(got, want[:3]) is None
    assert dec.dropped()[0] == len(want) - 3
    dec.reset(0)
    assert dec.dropped()[0] == 0
    assert M.records_equal(dec.work(streams)[0], want[:3]) is None
    dec.close()


def regenerate_golden():
    R = Ref()
    golden = {}
    for name in sorted(TABLE_CASES):
        golden["table_" + name] = digest(ref_table(R, name))
    for name, streams, ambe_fec in cases():
        for c, s in enumerate(streams):
            golden["rec_%s_%d" % (name, c)] = digest(R.work(s, [1], ambe_fec))
    json.dump(golden, open(GOLDEN, "w"), indent=1, sort_keys=True)
    open(GOLDEN, "a").write("\n")


if __name__ == "__main__":
    regenerate_golden()


ASAN_SCRIPT = r"""
import sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tools/emu")
from build_emulated_lib import build
lib, _ = build(sys.argv[2])
import qradiolink_b200 as q
from qradiolink_b200 import lib as L
L._LIB_PATH, L._LIB = lib, None
from tests import test_dmr_codec as T, dmr_model as M
streams = T.cases()[2][1]
got, want = T.run(q, streams, True, list(range(300, len(streams[0]), 1500)))
assert M.records_equal(got[0], want[0]) is None
print("asan ok")
"""


def test_emulated_build_under_address_sanitizer(tmp_path):
    import subprocess
    libasan = subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip()
    if not os.path.isabs(libasan):
        pytest.skip("no libasan")
    env = dict(os.environ, QRL_EMU_ASAN="1", LD_PRELOAD=libasan, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", ASAN_SCRIPT, ROOT, str(tmp_path)], env=env, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0 and "asan ok" in r.stdout, r.stderr[-3000:]
