"""CPU tier: the M17 frame codec (qrl_m17.cu, qradiolink_b200/m17.py) against the reference's own M17 code.

oracle/_ref/libqrl_ref_m17.so is src/M17/M17 of the reference compiled unmodified behind oracle/ref_m17_shim.cpp (oracle/ref_m17.mk,
which __graft_entry__.build() runs).  Where it was not built, the reference's results on the same seeded cases stand in as SHA-256 digests in
tests/golden/ref_m17.json; `python -m tests.test_m17_codec` rewrites that file from the compiled reference.

  * the numpy restatement tests/m17_model.py (the GPU tier's expected values) and the LSF / callsign helpers of m17.py are pinned to
    the reference (or its digests) case by case;
  * the library's own kernels, compiled for host threads (tools/emu/build_emulated_lib.py), are run through the real C ABI and the
    real Python wrappers and must give the reference's bytes, record for record."""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from qradiolink_b200 import m17 as Q
from tests import m17_model as M

pytestmark = pytest.mark.timeout(900)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_m17.json")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_m17.so")


def ref_m17():
    """the compiled reference codec, or None where oracle/_ref was not built"""
    if not os.path.exists(REF_SO):
        return None
    R = C.CDLL(REF_SO)
    vp = C.c_void_p
    R.ref_m17_dec_create.restype = vp
    R.ref_m17_dec_destroy.argtypes = [vp]
    R.ref_m17_dec_record.argtypes = [vp, C.c_uint32, vp, vp]
    R.ref_m17_tx_create.restype = vp
    R.ref_m17_tx_destroy.argtypes = [vp]
    R.ref_m17_tx_start.argtypes = [vp, C.c_char_p, C.c_char_p, C.c_int, C.c_int, vp]
    R.ref_m17_tx_send.argtypes = [vp, vp, C.c_int, vp]
    R.ref_m17_lsf.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_int, vp]
    R.ref_m17_encode_callsign.argtypes = [C.c_char_p, vp]
    R.ref_m17_decode_callsign.argtypes = [vp, C.c_char_p, C.c_int]
    return R


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------ reference runs
def ref_decode(R, records):
    """records: list of (type, 46 bytes) of one channel -> list of 56-byte snapshots from M17FrameDecoder behind gr_modem"""
    h = R.ref_m17_dec_create()
    out, o = [], np.zeros(56, np.uint8)
    for t, p in records:
        a = np.frombuffer(bytes(p)[:46].ljust(46, b"\0"), np.uint8).copy()
        R.ref_m17_dec_record(h, t, _p(a), _p(o))
        out.append(o.tobytes())
    R.ref_m17_dec_destroy(h)
    return out


def ref_transmit(R, lsf_args, ops, payloads):
    """one channel: M17Transmitter::start(src, dst, can, destination_type) for op 1, send() for 2, send(last) + EOT tail for 3"""
    h = R.ref_m17_tx_create()
    out, buf = [], np.zeros(256, np.uint8)
    src, dst, can, dt = lsf_args
    for op, pl in zip(ops, payloads):
        if op == 1:
            n = R.ref_m17_tx_start(h, src.encode(), dst.encode(), can, dt, _p(buf))
        elif op in (2, 3):
            a = np.ascontiguousarray(pl, np.uint8)
            n = R.ref_m17_tx_send(h, _p(a), int(op == 3), _p(buf))
        else:
            n = 0
        out.append(buf[:n].tobytes())
    R.ref_m17_tx_destroy(h)
    return out


def ref_lsf(R, args):
    o = np.zeros(30, np.uint8)
    R.ref_m17_lsf(args[0].encode(), args[1].encode(), args[2], args[3], _p(o))
    return o.tobytes()


# ------------------------------------------------------------------------------------------------ seeded cases
LSF_ARGS = [("N0CALL", "", 0, 0), ("AB1CD", "W1AW", 5, 0), ("XX9XYZ/P", "ECHO", 15, 2), ("M17-TEST", "", 3, 1), ("a.b", "Q", 7, 3),
            ("VERYLONGCALL", "UNLINKME", 9, 4), ("K1", "LONGDESTINATION", 1, 0)]
CALLSIGNS = ["N0CALL", "AB1CD", "M17-A/B.", "", "123456789", "TOOLONGCALL", "lower", "A B", "ZZZZZZZZZ"]


def tx_case(seed, C, K, calls):
    """per channel: LSF args, ops [calls * K], payloads; the first op of a channel is a start"""
    rng = np.random.default_rng(seed)
    ops = rng.choice([0, 1, 2, 2, 2, 2, 3], size=(C, calls * K)).astype(np.uint8)
    ops[:, 0] = 1
    pl = rng.integers(0, 256, (C, calls * K, 16), dtype=np.uint8)
    return [LSF_ARGS[c % len(LSF_ARGS)] for c in range(C)], ops, pl


def _flip(b, positions):
    b = bytearray(b)
    for q in positions:
        b[q >> 3] ^= 0x80 >> (q & 7)
    return bytes(b)


def _scrambled_flip(rec, deint_positions):
    """flip bits of a record's 46 payload bytes at positions of the deinterleaved frame (0-95: LICH, 96-: punctured stream data)"""
    return _flip(rec, [int(M.QPP[q]) for q in deint_positions])


def _lich_with(lsf30, n, seg_num):
    ch = lsf30[5 * n:5 * n + 5]
    blocks = [ch[0] << 4 | ch[1] >> 4, (ch[1] & 15) << 8 | ch[2], ch[3] << 4 | ch[4] >> 4, (ch[4] & 15) << 8 | (seg_num << 5)]
    return b"".join(M.golay_encode(int(b)).to_bytes(3, "big") for b in blocks)


def rx_case(seed, C, n_rec):
    """per channel a record list: a transmission (preamble skipped) with LSF / stream / EOT records, corrupted at random: 1-4 bit
    flips in LICH words and payloads, uncorrectable LICHs, crafted segment numbers 6 / 7, corrupted LSFs, EOT records with valid and
    invalid LSFs, unknown types; the lengths are ragged"""
    rng = np.random.default_rng(seed)
    chans = []
    for c in range(C):
        tx = M.Transmitter()
        tx.set_lsf(Q.m17_lsf(*LSF_ARGS[(c + seed) % len(LSF_ARGS)]))
        recs = []
        n = int(rng.integers(max(1, n_rec // 2), n_rec + 1))
        fresh = True
        while len(recs) < n:
            r = rng.random()
            if fresh or r < 0.06:
                f = tx.step(1, None)[48:]
                p = f[2:]
                if rng.random() < 0.3:
                    p = _flip(p, rng.integers(0, 368, int(rng.integers(1, 12))))
                recs.append((M.LSF, p)); fresh = False
                continue
            if r < 0.12:
                lsf = bytes(tx.lsf30) if rng.random() < 0.5 else _flip(tx.lsf30, [int(rng.integers(0, 240))])
                n_seg = int(rng.integers(6, 8))
                f = M.stream_frame(_lich_with(np.frombuffer(lsf, np.uint8).astype(int), 0, n_seg), tx.fn, False, rng.bytes(16))
                recs.append((M.STREAM, f[2:]))
                continue
            if r < 0.18:
                recs.append((M.EOT, rng.bytes(46)))
                if rng.random() < 0.5:
                    fresh = True
                continue
            if r < 0.21:
                recs.append((int(rng.choice([0x1234, 0x55F6, 0xED89])), rng.bytes(46)))
                continue
            f = tx.step(2, rng.bytes(16))
            p = f[2:48]
            k = rng.random()
            if k < 0.2:           # 1-4 bit errors spread over the LICH words
                p = _scrambled_flip(p, rng.choice(96, int(rng.integers(1, 5)), replace=False))
            elif k < 0.3:         # 4-7 errors in one Golay word: often uncorrectable, sometimes miscorrected
                w = int(rng.integers(0, 4))
                p = _scrambled_flip(p, 24 * w + rng.choice(24, int(rng.integers(4, 8)), replace=False))
            elif k < 0.45:        # 1-4 errors in the convolutional part
                p = _scrambled_flip(p, 96 + rng.choice(272, int(rng.integers(1, 5)), replace=False))
            elif k < 0.5:         # a burst the Viterbi decoder cannot fix
                p = _scrambled_flip(p, 96 + np.arange(int(rng.integers(0, 200)), 0, -1)[:30] % 272)
            recs.append((M.STREAM, p))
        chans.append(recs)
    return chans


RX_CASES = {"rx_a": (1701, 3, 40), "rx_b": (1702, 2, 30)}
TX_CASES = {"tx_a": (1801, 4, 6, 3)}


def _digest(blobs):
    return hashlib.sha256(b"".join(hashlib.sha256(b).digest() for b in blobs)).hexdigest()


def reference_results(R):
    """every seeded case through the compiled reference: name -> list of byte strings"""
    res = {}
    for name, (seed, C_, n) in RX_CASES.items():
        res[name] = [s for recs in rx_case(seed, C_, n) for s in ref_decode(R, recs)]
    for name, (seed, C_, K, calls) in TX_CASES.items():
        args, ops, pl = tx_case(seed, C_, K, calls)
        res[name] = [b"".join(ref_transmit(R, args[c], ops[c], pl[c])) for c in range(C_)]
    res["wrap"] = [b"".join(ref_transmit(R, LSF_ARGS[1], *_wrap_ops()))]
    res["lsf"] = [ref_lsf(R, a) for a in LSF_ARGS]
    cs = []
    for s in CALLSIGNS:
        o = np.zeros(6, np.uint8)
        R.ref_m17_encode_callsign(s.encode(), _p(o))
        buf = C.create_string_buffer(64)
        R.ref_m17_decode_callsign(_p(o), buf, 64)
        cs += [o.tobytes(), buf.value]
    res["callsign"] = cs
    return res


def _wrap_ops():
    """a start, 2100 stream frames (the frame number wraps at 0x7FF), a last frame, a stream frame after it"""
    ops = np.array([1] + [2] * 2100 + [3, 2], np.uint8)
    pl = np.random.default_rng(1900).integers(0, 256, (len(ops), 16), dtype=np.uint8)
    return ops, pl


@pytest.fixture(scope="module")
def R():
    return ref_m17()


def check(R, name, mine):
    """mine: the results of case `name`, in order, against the compiled reference's (or their committed digest)"""
    if R is None:
        assert _digest(mine) == json.load(open(GOLDEN))[name], name
        return
    want = reference_results_cached(R)[name]
    assert len(mine) == len(want), name
    for i, (g, w) in enumerate(zip(mine, want)):
        assert g == w, (name, i, g.hex(), w.hex())


_CACHE = {}


def reference_results_cached(R):
    if "r" not in _CACHE:
        _CACHE["r"] = reference_results(R)
    return _CACHE["r"]


# ------------------------------------------------------------------------------------------------ the restatements
def model_rx(name):
    seed, C_, n = RX_CASES[name]
    return [s for recs in rx_case(seed, C_, n) for s in M.Decoder().work(recs)]


def model_tx(args, ops, pl):
    t = M.Transmitter()
    t.set_lsf(Q.m17_lsf(*args))
    return b"".join(t.step(int(o), bytes(p)) for o, p in zip(ops, pl))


@pytest.mark.parametrize("name", sorted(RX_CASES))
def test_model_decoder_is_the_reference(R, name):
    check(R, name, model_rx(name))


def test_model_transmitter_is_the_reference(R):
    for name, (seed, C_, K, calls) in TX_CASES.items():
        args, ops, pl = tx_case(seed, C_, K, calls)
        check(R, name, [model_tx(args[c], ops[c], pl[c]) for c in range(C_)])
    check(R, "wrap", [model_tx(LSF_ARGS[1], *_wrap_ops())])


def test_lsf_and_callsign_helpers_are_the_reference(R):
    check(R, "lsf", [Q.m17_lsf(*a) + Q.m17_crc16(Q.m17_lsf(*a)).to_bytes(2, "big") for a in LSF_ARGS])
    cs = []
    for s in CALLSIGNS:
        e = Q.m17_encode_callsign(s)
        cs += [e, Q.m17_callsign(e).encode()]
    check(R, "callsign", cs)


def test_generated_constants():
    """the Golay rows from g(x) = 0xC75 form a self-dual code (rows x transpose = identity) of minimum distance 8, and every
    error of weight <= 3 is corrected; the interleaver is a permutation"""
    for d in range(4096):
        assert M._mul(M._mul(d, M.GOLAY_ENC), M.GOLAY_DEC) == d
    assert min(bin(M.golay_encode(d)).count("1") for d in range(1, 4096)) == 8
    rng = np.random.default_rng(5)
    for _ in range(300):
        d = int(rng.integers(0, 4096))
        e = sum(1 << int(b) for b in rng.choice(24, int(rng.integers(0, 4)), replace=False))
        assert M.golay_decode(M.golay_encode(d) ^ e) == d
    assert sorted(M.QPP) == list(range(368))
    assert M.P1.sum() == 46 and len(M.P1) == 61 and M.P2.sum() == 11


# ------------------------------------------------------------------------------------------------ the library on host threads
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_m17")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    yield q
    L._LIB_PATH, L._LIB = saved


def snapshots(got):
    """M17Decoder.read() tuples -> the 56-byte layout"""
    return [int(t).to_bytes(4, "little") + lsf + bytes([v, 0]) + sf + b"\0\0" for t, lsf, v, sf in got]


def run_decoder(q, chans, splits, max_frames=32):
    """feed each channel's records in calls cut at `splits` (fractions of its length): ragged counts per call"""
    dec = Q.M17Decoder(len(chans), max_frames)
    out = [[] for _ in chans]
    edges = [[0] + [int(round(s * len(r))) for s in splits] + [len(r)] for r in chans]
    for k in range(len(splits) + 1):
        got = dec.work([r[e[k]:e[k + 1]] for r, e in zip(chans, edges)])
        for c, g in enumerate(got):
            out[c] += snapshots(g)
    dec.close()
    return out


@pytest.mark.parametrize("name,splits", [("rx_a", (0.37, 0.5, 0.81)), ("rx_b", ())])
def test_decoder_kernels_are_the_reference(emu, R, name, splits):
    seed, C_, n = RX_CASES[name]
    chans = rx_case(seed, C_, n)
    got = run_decoder(emu, chans, splits)
    check(R, name, [s for ch in got for s in ch])


def test_decoder_reset_and_segments_6_7(emu):
    """a crafted segment number 6 / 7 leaves only its map bit: reassembly stalls until reset(channel), then completes"""
    tx = M.Transmitter()
    tx.set_lsf(Q.m17_lsf("AB1CD", "W1AW", 5, 0))
    lsf = np.frombuffer(tx.lsf30, np.uint8).astype(int)
    six = (M.STREAM, M.stream_frame(_lich_with(lsf, 0, 6), 0, False, bytes(16))[2:])
    segs = [(M.STREAM, tx.step(2, bytes([k] * 16))[2:48]) for k in range(6)]
    dec = Q.M17Decoder(2, 8)
    r = dec.work([[six] + segs, segs])
    assert not r[0][-1][2] and r[1][-1][2] and r[1][-1][1] == tx.lsf30
    assert r[0][-1][3] == r[1][-1][3]                  # the stray segment never shows in the stream frame
    dec.reset(0)
    r = dec.work([segs, []])
    assert r[0][-1][2] and r[0][-1][1] == tx.lsf30 and r[1] == []
    dec.close()


def test_encoder_kernels_are_the_reference(emu, R):
    for name, (seed, C_, K, calls) in TX_CASES.items():
        args, ops, pl = tx_case(seed, C_, K, calls)
        enc = Q.M17Encoder(C_, K)
        for c in range(C_):
            enc.set_lsf(c, Q.m17_lsf(*args[c]))
        out = [b""] * C_
        for k in range(calls):
            got = enc.work(ops[:, k * K:(k + 1) * K], pl[:, k * K:(k + 1) * K])
            out = [o + g.tobytes() for o, g in zip(out, got)]
        enc.close()
        check(R, name, out)


def test_encoder_counters_wrap_across_calls(emu, R):
    ops, pl = _wrap_ops()
    K = 128
    enc = Q.M17Encoder(1, K)
    enc.set_lsf(0, Q.m17_lsf(*LSF_ARGS[1]))
    out = b""
    for k in range(0, len(ops), K):
        o = np.zeros((1, K), np.uint8); p = np.zeros((1, K, 16), np.uint8)
        n = min(K, len(ops) - k)
        o[0, :n] = ops[k:k + n]; p[0, :n] = pl[k:k + n]
        out += enc.work(o, p)[0].tobytes()
    enc.close()
    check(R, "wrap", [out])


if __name__ == "__main__":
    R_ = ref_m17()
    if R_ is None:
        raise SystemExit("oracle/_ref/libqrl_ref_m17.so missing: run `make -C oracle -f ref_m17.mk` where the reference tree exists")
    with open(GOLDEN, "w") as f:
        json.dump({name: _digest(v) for name, v in sorted(reference_results(R_).items())}, f, indent=1)
    print("wrote", GOLDEN)
