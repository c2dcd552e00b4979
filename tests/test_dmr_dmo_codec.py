"""CPU tier of the DMR direct-mode (DMO) burst decoder (qrl_dmr.cu's dmr_dmo_sink_kernel, qradiolink_b200.DmrDmoBurstDecoder), pinned to
the reference's own gr_dmr_dmo_sink, CDMRSlotType2 and DMRFrame compiled behind oracle/ref_dmr_dmo_shim.cpp
(oracle/_ref/libqrl_ref_dmr_dmo.so, built by oracle/ref_dmr_dmo.mk), or to digests of its results in tests/golden/ref_dmr_dmo.json where
the reference is absent (`python -m tests.test_dmr_dmo_codec` regenerates them):
  * CDMRSlotType2's decoder, generated from its definition, over all 2^19 inputs decode2087 reads;
  * the restatement tests/dmr_dmo_model.py, record for record, on constructed float streams: voice superframes, a data header with
    rate 1/2, 3/4 and 1 data, a CSBK and a terminator (each ending in the sink's reset), rate data while searching (a stale end
    pointer), BS syncs, 13 bursts without sync, +-1 sample of timing drift per burst, a run of rising correlations that walks the
    window, DC and level changes per burst, prefilter hits that fail the byte check, NaN, -0 and denormal samples, and the
    end-to-end path of the oracle's DMR modulator and demodulator (port 3) behind tests/dmr_tx_model.py's bursts;
  * the library's own kernels compiled for host threads (tools/emu), against the restatement, in ragged calls, with the dropped path,
    reset(channel) and one pass under AddressSanitizer."""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import pytest

from tests import dmr_dmo_model as D
from tests import dmr_model as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libqrl_ref_dmr_dmo.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_dmr_dmo.json")


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Ref:
    def __init__(self):
        self.L = C.CDLL(REF_LIB)
        self.L.ref_dmo_create.restype = C.c_void_p

    def work(self, x, ambe_fec):
        from qradiolink_b200.dmr import DMR_RECORD
        L = self.L
        h = C.c_void_p(L.ref_dmo_create())
        x = np.ascontiguousarray(x, np.float32)
        out = np.zeros((8192, 72), np.uint8)
        n = L.ref_dmo_work(h, x.ctypes.data_as(C.c_void_p), C.c_long(len(x)), int(ambe_fec), out.ctypes.data_as(C.c_void_p), len(out))
        L.ref_dmo_destroy(h)
        return out[:n].copy().view(DMR_RECORD).reshape(-1)


@pytest.fixture(scope="module")
def R():
    return Ref() if os.path.exists(REF_LIB) else None


def model_array(recs):
    from qradiolink_b200.dmr import DMR_RECORD
    a = np.zeros(len(recs), DMR_RECORD)
    for i, r in enumerate(recs):
        for k in M.REC_FIELDS:
            a[i][k] = r[k]
        a[i]["cach"] = np.frombuffer(r["cach"], np.uint8)
        a[i]["frame"] = np.frombuffer(r["frame"], np.uint8)
    return a


def pinned(key, got):
    golden = json.load(open(GOLDEN))
    assert digest(got) == golden[key], key


# ---------------------------------------------------------------- streams
def ms_data(cc, dt, **kw):
    return M.data_burst(cc, dt, sync="ms_data", **kw)


def bursts_to_samples(rng, fbs, lead=300, **kw):
    syms = D.random_symbols(rng, lead)
    for fb in fbs:
        syms += D.dmo_burst(fb, rng)
    syms += D.random_symbols(rng, 400)
    return D.to_samples(syms, rng=rng, noise=kw.pop("noise", 0.01), **kw)


def drift(rng, fbs, steps):
    """one burst per 288 symbols, each shifted by steps[i] samples against the last"""
    x = list(D.to_samples(D.random_symbols(rng, 300), rng=rng, noise=0.01))
    for fb, s in zip(fbs, steps):
        seg = list(D.to_samples(D.dmo_burst(fb, rng), rng=rng, noise=0.01))
        x += seg[:len(seg) + s] if s < 0 else seg + seg[-s:] if s else seg
    return np.array(x + list(D.to_samples(D.random_symbols(rng, 400))), np.float32)


def cases():
    rng = np.random.default_rng(21)
    out = []
    sf = D.random_symbols(rng, 500)
    for cc in (1, 7, 15):
        sf += D.voice_superframe(rng, cc=cc)
    out.append(("voice", D.to_samples(sf, rng=rng, noise=0.02), True))
    lc = ms_data(3, 1, payload12=M.lc_payload(0, 0, 99, 4242, 1))
    term = ms_data(3, 2, payload12=M.lc_payload(0, 0, 99, 4242, 2))
    csbk = ms_data(4, 3, payload12=M.csbk_payload(0x04, 0, 12345, 678))
    hdr = ms_data(2, 6, payload12=M.data_header_payload(0, 5, 6))
    r12 = ms_data(2, 7, payload12=bytes(range(12)))
    r34 = ms_data(2, 8, points=M.trellis_encode(bytes(range(18))))
    r1 = ms_data(2, 10, payload12=bytes(12))
    out.append(("data", bursts_to_samples(rng, [hdr, r12, r34, r1, r12]), False))
    vs = [M.voice_burst(rng, sync="ms_voice")] + [M.voice_burst(rng, emb=(3, 0, 1)) for _ in range(5)]
    out.append(("csbk_terminator", bursts_to_samples(rng, [lc] + vs + [term, term, csbk, lc, csbk]), True))
    out.append(("stale_end", bursts_to_samples(rng, [r12, r34, r1, r12, hdr, r1]), False))
    bs = M.data_burst(1, 3, payload12=M.csbk_payload(0x04, 0, 1, 2), sync="bs_data")
    bsv = M.voice_burst(rng, sync="bs_voice")
    out.append(("bs_syncs", bursts_to_samples(rng, [bs, bsv, bs, csbk]), True))
    noise = [[int(v) for v in rng.integers(0, 2, 264)] for _ in range(16)]
    out.append(("sync_lost", bursts_to_samples(rng, [hdr] + noise + [lc] + vs[:1] + noise), True))
    out.append(("drift", drift(rng, [lc] + vs + vs + [term], [0, 1, -1, 1, 1, -1, 0, 1, -1, -1, 1, 1, 0, -1]), True))
    # rising correlations: the sync's amplitude grows over the samples of each symbol, so the best correlation walks forward
    x = bursts_to_samples(rng, [lc] + vs + vs + [term], noise=0.0)
    ramp = np.tile(np.float32([0.9, 0.95, 1.0, 1.05, 1.1]), len(x) // 5 + 1)[:len(x)].astype(np.float32)
    out.append(("walk", (x * ramp).astype(np.float32), True))
    # DC and level per burst
    syms = D.random_symbols(rng, 300)
    x = [D.to_samples(syms)]
    for k, fb in enumerate([lc] + vs + vs + [term]):
        x.append(D.to_samples(D.dmo_burst(fb, rng), scale=0.2 + 0.05 * (k % 5), dc=0.03 * ((k % 7) - 3), rng=rng, noise=0.01))
    out.append(("dc_level", np.concatenate(x + [D.to_samples(D.random_symbols(rng, 300))]).astype(np.float32), True))
    # prefilter hits that fail the byte check: the sync's symbols right in sign, +-1 in level
    sync_fb = list(csbk)
    for k in range(54, 78, 2):            # symbols 54..77 of 132 carry the sync; swap +3 <-> +1 and -3 <-> -1 on every other one
        sync_fb[2 * k + 1] ^= 1
    out.append(("byte_check", bursts_to_samples(rng, [sync_fb, sync_fb, csbk, sync_fb]), False))
    # NaN, -0 and denormal samples inside syncs and payloads
    x = bursts_to_samples(rng, [lc] + vs + [term], noise=0.0)
    idx = rng.choice(len(x), 300, replace=False)
    x[idx[:100]] = np.nan
    x[idx[100:200]] = np.float32(-0.0)
    x[idx[200:]] = np.float32(1e-41) * np.sign(rng.standard_normal(100)).astype(np.float32)
    x[1500 + 5 * 54: 1500 + 5 * 78: 7] = np.float32(-0.0)
    out.append(("special", x, True))
    return out


CASES = cases()


@pytest.mark.parametrize("name,x,ambe_fec", CASES, ids=[c[0] for c in CASES])
def test_model_is_the_reference(R, name, x, ambe_fec):
    want = model_array(D.DmoDecoder(1, ambe_fec).work([x])[0])
    if name not in ("bs_syncs", "byte_check"):
        assert len(want) >= 3, name
    if R is not None:
        ref = R.work(x, ambe_fec)
        assert np.array_equal(ref, want), M.records_equal(ref, D.DmoDecoder(1, ambe_fec).work([x])[0])
    pinned("rec_" + name, want)


def test_cases_cover_the_state_machine(R):
    by = {name: model_array(D.DmoDecoder(1, f).work([x])[0]) for name, x, f in CASES}
    assert len(by["bs_syncs"]) == 1 and by["bs_syncs"][0]["data_type"] == 3            # only the MS CSBK
    assert len(by["byte_check"]) == 1 and by["byte_check"][0]["data_type"] == 3     # only the clean CSBK
    assert list(by["data"]["data_type"][:5]) == [6, 7, 8, 10, 7]      # then the bursts without sync of RECV_DATA
    assert list(by["voice"]["fn"][:6]) == [0, 1, 2, 3, 4, 5] and set(by["voice"]["color_code"]) == {0}     # only data syncs set it
    assert set(by["csbk_terminator"]["color_code"][:7]) == {3}
    assert len(by["sync_lost"]) >= 13 + 6
    assert any(r["data_type"] == 2 for r in by["csbk_terminator"])


def test_slot_type2_is_the_reference(R):
    got = np.array([D.slot_type2(w) for w in range(1 << 19)], np.int64)
    # the same decoder as DMRFrame's CDMRSlotType on the same 19 bits
    code = np.arange(1 << 19, dtype=np.int64)
    from tests.test_dmr_codec import np_poly_mod
    assert np.array_equal(got, ((code ^ np.array(M.GOLAY19)[np_poly_mod(code, 18, 0xC75, 11)]) >> 11) & 0xFF)
    if R is not None:
        R.L.ref_slot_type2_decode.restype = C.c_int
        ref = np.array([R.L.ref_slot_type2_decode(w) for w in range(1 << 19)], np.int64)
        assert np.array_equal(got, ref)
    pinned("slot_type2", got)


def test_end_to_end_through_the_oracle_modem(R):
    """tests/dmr_tx_model.py's bursts -> the oracle's DMR modulator -> its demodulator's port 3 -> model == reference"""
    x = oracle_port3()
    want = model_array(D.DmoDecoder(1, True).work([x])[0])
    assert len(want) >= 10
    assert set(want["frame_type"]) >= {0, 1, 2}
    if R is not None:
        assert np.array_equal(R.work(x, True), want)
    pinned("rec_oracle_modem", want)


def oracle_port3():
    from oracle import oracle as O
    from tests import dmr_tx_model as T
    ch = T.Channel(T.Config(color_code=6, src_id=1234, dst_id=9))
    rng = np.random.default_rng(5)
    ops = [T.OP_HEADER] + [T.OP_AUDIO] * 60 + [T.OP_STOP] + [T.OP_AUDIO] * 6
    stream, _ = ch.work(np.array(ops, np.uint8), rng.integers(0, 256, (len(ops), 9)).astype(np.uint8))
    iq = O.Tx(O.MOD_DMR, 125, 1000000, 1700, 5000, 0).work(np.frombuffer(stream, np.uint8))
    rx = O.Rx(O.DEMOD_DMR, 5, 1000000, 0, 0, 0)
    rx.work(np.concatenate([np.zeros(5000, np.complex64), iq, np.zeros(20000, np.complex64)]))
    return np.asarray(rx.port(3), np.float32)


# ---------------------------------------------------------------- the library on host threads
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, _ = build(str(tmp_path_factory.mktemp("qrl_emu_dmo")))
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    yield q
    L._LIB_PATH, L._LIB = saved


def run(q, streams, ambe_fec, cuts, max_bursts=None):
    """feed each stream in calls cut at the given sample offsets (ragged: per-channel counts); records per channel, and the model's"""
    n = max(len(s) for s in streams)
    dec = q.DmrDmoBurstDecoder(len(streams), n, max_bursts, ambe_fec)
    model = D.DmoDecoder(len(streams), ambe_fec)
    got, want = [[] for _ in streams], [[] for _ in streams]
    edges = [0] + list(cuts) + [n]
    for a, b in zip(edges[:-1], edges[1:]):
        part = [s[a:b] for s in streams]
        for c, g in enumerate(dec.work(part)):
            got[c] += list(g)
        for c, w in enumerate(model.work(part)):
            want[c] += w
    dec.close()
    return got, want


@pytest.mark.parametrize("name,x,ambe_fec", CASES, ids=[c[0] for c in CASES])
def test_kernels_equal_the_model(emu, name, x, ambe_fec):
    got, want = run(emu, [x], ambe_fec, ())
    assert M.records_equal(got[0], want[0]) is None, M.records_equal(got[0], want[0])


def test_ragged_calls_at_every_phase(emu):
    x = dict((c[0], c[1]) for c in CASES)["csbk_terminator"]
    y = dict((c[0], c[1]) for c in CASES)["drift"]
    streams = [x, y[:len(x)]]
    for phase in list(range(0, 1440, 97)) + [1439]:
        cuts = list(range(phase + 1, len(x), 1440 + 37))
        got, want = run(emu, streams, True, cuts)
        for c in range(2):
            assert M.records_equal(got[c], want[c]) is None, (phase, c, M.records_equal(got[c], want[c]))
    got, want = run(emu, streams, True, list(range(37, len(x), 37)))
    assert all(M.records_equal(got[c], want[c]) is None for c in range(2))


def test_dropped_and_reset(emu):
    x = dict((c[0], c[1]) for c in CASES)["voice"]
    dec = emu.DmrDmoBurstDecoder(1, len(x), 3, True)
    want = D.DmoDecoder(1, True).work([x])[0]
    got = dec.work([x])[0]
    assert len(want) > 3 and M.records_equal(got, want[:3]) is None
    assert dec.dropped()[0] == len(want) - 3
    dec.reset(0)
    assert dec.dropped()[0] == 0
    assert M.records_equal(dec.work([x])[0], want[:3]) is None
    dec.close()


def regenerate_golden():
    R = Ref()
    golden = {"slot_type2": digest(np.array([D.slot_type2(w) for w in range(1 << 19)], np.int64))}
    for name, x, f in CASES:
        golden["rec_" + name] = digest(R.work(x, f))
    golden["rec_oracle_modem"] = digest(R.work(oracle_port3(), True))
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
from tests import test_dmr_dmo_codec as T, dmr_model as M
x = dict((c[0], c[1]) for c in T.CASES)["csbk_terminator"]
got, want = T.run(q, [x], True, list(range(300, len(x), 1500)))
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
