"""Pins the oracle (and the host-side sink restatements) to REFERENCE CODE: oracle/_ref/libqrl_ref_blocks.so is the reference's
src/gr/{gr_4fsk_discriminator, gr_deframer_bb, gr_bit_sink, gr_audio_sink, gr_const_sink, dsss_encoder_bb_impl,
dsss_decoder_cc_impl, cessb/clipper_cc_impl, cessb/stretcher_cc_impl} compiled UNMODIFIED against the runtime stand-in in
oracle/gr_stub/ (oracle/Makefile target `ref`; oracle/ref_blocks_shim.cpp plays the scheduler).  CPU tier.

oracle/_ref is built only where the reference tree is.  Everywhere else the reference blocks' results on the same seeded inputs,
committed under tests/golden/ (per test, a SHA-256 over the SHA-256 of each result's bytes, and the clipper's output itself,
which is compared with a tolerance), stand in for them; `python -m tests.test_oracle_ref` rewrites those files from the compiled blocks."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import oracle as O

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLDEN = os.path.join(GOLDEN_DIR, "ref_blocks.json")
CLIPPER_NPY = os.path.join(GOLDEN_DIR, "ref_cessb_clipper.npy")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _digest(v):
    """dtype, shape and SHA-256 of the bytes: two results have the same digest only if they are bitwise equal."""
    if v is None:
        return "None"
    a = np.ascontiguousarray(np.int64(v) if isinstance(v, (int, np.integer)) else v)
    return "%s%s:%s" % (a.dtype.str, list(a.shape), hashlib.sha256(a.tobytes()).hexdigest())


def _as(v, dtype):
    """v itself, after checking that it has the reference buffer's dtype (no conversion may hide a difference)."""
    assert v.dtype == dtype, (v.dtype, dtype)
    return v


@pytest.fixture(scope="module")
def R():
    return O.ref_blocks()        # None without oracle/_ref: the committed results stand in


def _sequence_digest(digests):
    return hashlib.sha256("\n".join(digests).encode()).hexdigest()


def check(R, name, mine):
    """mine: digests of the restatement's results, in order; against those of the compiled reference block (REF_RUNS[name])."""
    if R is None:
        assert _sequence_digest(mine) == json.load(open(GOLDEN))[name], name
        return
    want = REF_RUNS[name](R)
    assert len(mine) == len(want), name
    for i, (g, w) in enumerate(zip(mine, want)):
        assert g == w, (name, i)


# ------------------------------------------------------------------------------------------------ 4FSK discriminator
def _disc_inputs():
    rng = np.random.default_rng(11)
    n = 20000
    m = rng.random((4, n)).astype(np.float32)
    m[:, :2000] = np.round(m[:, :2000] * 4) / 4          # many exact ties: the strict-greater rule decides
    m[:, 2000:2100] = 0.0
    return m, n


def _ref_disc(R):
    m, n = _disc_inputs()
    ref = np.zeros(2 * n, np.float32)
    R.ref_disc4(_p(m[0]), _p(m[1]), _p(m[2]), _p(m[3]), n, _p(ref))
    return [_digest(ref)]


def test_discriminator_is_the_reference_block(R):
    m, n = _disc_inputs()
    got = np.zeros(2 * n, np.float32)
    O.lib().qo_disc4(_p(m[0]), _p(m[1]), _p(m[2]), _p(m[3]), n, _p(got))
    check(R, "disc4", [_digest(got)])
    assert np.any(got == 0.0) and len(np.unique(got)) == 3      # -0.707107, 0, +0.707107 all occur


# ------------------------------------------------------------------------------------------------ CESSB clipper / stretcher
def _clipper_inputs():
    rng = np.random.default_rng(12)
    n = 8 * 1024
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * rng.choice([0.05, 0.5, 1.5], n)).astype(np.complex64)
    x[:16] = 0
    return x, n


def _ref_clipper_output(R):
    x, n = _clipper_inputs()
    ref = np.zeros(n, np.complex64)
    assert R.ref_cessb_clipper(_p(x), n, 0.95, _p(ref)) == n
    return ref


def test_cessb_clipper_against_the_reference_block(R):
    x, n = _clipper_inputs()
    ref = _ref_clipper_output(R) if R is not None else np.load(CLIPPER_NPY)
    got = np.zeros(n, np.complex64)
    O.lib().qo_cessb_clipper(_p(x), n, C.c_float(0.95), _p(got))
    # magnitude path (sqrt, min) is IEEE on both sides; the phase goes through cos / sin, libm (VOLK generic) in the compiled
    # reference vs the oracle's fixed polynomial: 3e-7 each (tests/test_oracle.py::test_sincos_and_atan)
    assert np.max(np.abs(ref - got)) < 5e-7
    assert np.max(np.abs(np.abs(ref) - np.abs(got))) < 2e-7 and np.max(np.abs(got)) <= 0.95 + 1e-6
    small = np.abs(x) < 0.9
    assert np.max(np.abs(np.abs(got[small]) - np.abs(x[small]))) < 3e-7      # below the clip level only the rounding of cos/sin


STRETCHER_CHUNKS = [1024, 3072]


def _stretcher_inputs():
    rng = np.random.default_rng(13)
    n = 9 * 1024 + 2
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * rng.choice([0.1, 0.6, 1.2], n)).astype(np.complex64)
    return x, n


def _ref_stretcher(R, chunk):
    x, n = _stretcher_inputs()
    ref = np.zeros(n, np.complex64)
    n_ref = R.ref_cessb_stretcher(_p(x), n, chunk, _p(ref))
    return [_digest(n_ref), _digest(ref[:n_ref].view(np.float32))]


@pytest.mark.parametrize("chunk", STRETCHER_CHUNKS)
def test_cessb_stretcher_is_the_reference_block_bit_for_bit(R, chunk):
    x, n = _stretcher_inputs()
    got = np.zeros(n, np.complex64)
    n_got = O.lib().qo_cessb_stretcher(_p(x), n, _p(got))
    assert n_got == n - 2
    # the reference block emits 9 * 1024 items; chunking of the reference block is invisible
    check(R, "cessb_stretcher_%d" % chunk, [_digest(9 * 1024), _digest(got[:9 * 1024].view(np.float32))])
    assert np.any(np.abs(got[:9 * 1024]) < np.abs(x[:9 * 1024]) * 0.9)                  # the stretcher did act


# ------------------------------------------------------------------------------------------------ gr_deframer_bb
def _planted_bits(rng, n, words):
    bits = rng.integers(0, 2, n, dtype=np.uint8)
    pos = 50
    while pos + 500 < n:
        w, nb = words[int(rng.integers(0, len(words)))]
        bits[pos:pos + nb] = [(w >> (nb - 1 - k)) & 1 for k in range(nb)]
        pos += int(rng.integers(100, 700))
    return bits


DEFRAMER_MODEMS = [1, 2, 3]


def _deframer_chunks(modem_type):
    rng = np.random.default_rng(20 + modem_type)
    words = [(0xED89, 16), (0x89ED, 16), (0x98DE, 16), (0xED77, 16), (0x8CC8, 16), (0x4C8A2B, 24), (0xB5, 8)]
    bits = _planted_bits(rng, 60000, words)
    chunks, pos = [], 0
    while pos < len(bits):
        m = int(rng.integers(1, 3000))
        chunks.append(np.ascontiguousarray(bits[pos:pos + m])); pos += m
    return chunks


def _ref_deframer(R, modem_type):
    h = R.ref_dfbb_create(modem_type)
    ref = []
    for chunk in _deframer_chunks(modem_type):
        out = np.zeros(4 * len(chunk) + 64, np.uint8)
        k = R.ref_dfbb_work(h, _p(chunk), len(chunk), _p(out), len(out))
        ref.append(out[:k].copy())
    R.ref_block_destroy(h)
    return [_digest(np.concatenate(ref))]


@pytest.mark.parametrize("modem_type", DEFRAMER_MODEMS)
def test_gr_deframer_bb_is_the_reference_block(R, modem_type):
    d = O.DeframerBB(modem_type)
    got = np.concatenate([_as(d.work(chunk), np.uint8) for chunk in _deframer_chunks(modem_type)])
    check(R, "deframer_%d" % modem_type, [_digest(got)])
    assert len(got) > 1000


# ------------------------------------------------------------------------------------------------ sinks
SINK_KINDS = ["bit", "audio", "const"]
_SINK_DT = {"bit": np.uint8, "audio": np.float32, "const": np.complex64}


def _sink_schedule(kind):
    """400 steps: ("work", x) or ("get", None), random sizes."""
    rng = np.random.default_rng({"bit": 31, "audio": 32, "const": 33}[kind])
    big = {"bit": 400000, "audio": 3000, "const": 120}[kind]
    for step in range(400):
        if rng.random() < 0.6:
            n = int(rng.integers(0, big))
            if kind == "bit":
                x = rng.integers(0, 2, n, dtype=np.uint8)
            elif kind == "audio":
                x = rng.standard_normal(n).astype(np.float32)
            else:
                x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
            yield "work", x
        else:
            yield "get", None


def _ref_sink(R, kind):
    h = getattr(R, "ref_%s_sink_create" % kind)()
    work, get = getattr(R, "ref_%s_sink_work" % kind), getattr(R, "ref_%s_sink_get" % kind)
    res = []
    for op, x in _sink_schedule(kind):
        if op == "work":
            res.append(_digest(work(h, _p(x), len(x))))
        else:
            out = np.zeros(1 << 21 if kind == "bit" else 1 << 14, _SINK_DT[kind])
            k = get(h, _p(out), len(out))
            res.append(_digest(None if k < 0 else out[:k]))
    R.ref_block_destroy(h)
    return res


@pytest.mark.parametrize("kind", SINK_KINDS)
def test_sink_restatements_follow_the_reference_sinks(R, kind):
    """qradiolink_b200.demod.gr_*_sink (what the Python host side polls) against the compiled gr_*_sink.cpp, random schedules."""
    import importlib
    demod = importlib.import_module("qradiolink_b200.demod")
    mine = getattr(demod, "gr_%s_sink" % kind)()
    res = []
    for op, x in _sink_schedule(kind):
        if op == "work":
            res.append(_digest(mine.work(x)))
        else:
            m = mine.get_data()
            res.append(_digest(None if m is None else _as(m, _SINK_DT[kind])))
    check(R, "sink_%s" % kind, res)


def _sample_sink_schedule():
    rng = np.random.default_rng(34)
    for step in range(300):
        r = rng.random()
        if step == 5:
            yield "enable", None
        if r < 0.55:
            n = int(rng.integers(0, 200000))
            yield "work", (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        elif r < 0.65:
            yield "window", int(rng.integers(1, 30000))
        else:
            yield "get", None


def _ref_sample_sink(R):
    h = R.ref_sample_sink_create()
    out = np.zeros(1 << 20, np.complex64)
    res = []
    for op, a in _sample_sink_schedule():
        if op == "enable":
            R.ref_sample_sink_set_enabled(h, 1)
        elif op == "work":
            res.append(_digest(R.ref_sample_sink_work(h, _p(a), len(a))))
        elif op == "window":
            R.ref_sample_sink_set_window(h, a)
        else:
            k = R.ref_sample_sink_get(h, _p(out), len(out))
            res.append(_digest(None if k < 0 else out[:k]))
    R.ref_block_destroy(h)
    return res


def test_sample_sink_restatement_follows_the_reference_sink(R):
    """qradiolink_b200.demod.gr_sample_sink against the compiled gr_sample_sink.cpp: enable, window changes (odd sizes), the 524288-item
    drop rule, random schedules."""
    import importlib
    demod = importlib.import_module("qradiolink_b200.demod")
    mine = demod.gr_sample_sink()
    res = []
    for op, a in _sample_sink_schedule():
        if op == "enable":
            mine.set_enabled(True)
        elif op == "work":
            res.append(_digest(mine.work(a)))
        elif op == "window":
            mine.set_sample_window(a)
        else:
            m = mine.get_data()
            res.append(_digest(None if m is None else _as(m, np.complex64)))
    check(R, "sample_sink", res)


# ------------------------------------------------------------------------------------------------ gr_zero_idle_bursts
def _zero_idle_inputs():
    rng = np.random.default_rng(31)
    n, delay = 30000, 62
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    chunks = np.array([4096, 1000, 8192, 5000, 20000], np.int64)
    edges = np.concatenate([[0], np.cumsum(chunks)])
    tag_items, tag_vals = [], []
    for k in range(len(chunks)):
        lo, hi = edges[k], min(edges[k + 1], n)
        if hi - lo < 400:
            continue
        for j in range(3):
            tag_items.append(int(lo + delay + rng.integers(0, hi - lo - delay)))
            tag_vals.append(int(rng.integers(1, 900)))
    tag_items.append(tag_items[0] + 5); tag_vals.append(3)           # overrides a running count with a short one
    tag_items.append(30); tag_vals.append(500)                        # item < delay: never matches
    return x, n, delay, np.array(tag_items, np.int64), np.array(tag_vals, np.int64), chunks.astype(np.dtype("l"))


def _ref_zero_idle(R):
    x, n, delay, to, tv, ch = _zero_idle_inputs()
    res = []
    for d in (delay, 0):
        ref = np.zeros(n, np.complex64)
        done = R.ref_zero_idle(_p(x), n, d, _p(to), _p(tv), len(to), _p(ch), len(ch), _p(ref))
        res += [_digest(done), _digest(ref.view(np.uint32))]
    return res


def test_zero_idle_bursts_is_the_reference_block(R):
    """gr_zero_idle_bursts.cpp compiled unmodified (stream tags through the stand-in's get_tags_in_window): delay of history-1 items,
    a counter loaded `delay` items before the tagged one, later tags overriding a running count.  Tags are kept at least `delay`
    items inside their work() window -- the only place the restatement deviates (it also honours the ones the reference drops).
    The second run, delay = 0: no history, pure pass-through + tags at their own item."""
    x, n, delay, to, tv, ch = _zero_idle_inputs()
    got = O.zero_idle(x, delay, to, tv)
    got0 = O.zero_idle(x, 0, to, tv)
    check(R, "zero_idle", [_digest(n), _digest(got.view(np.uint32)), _digest(n), _digest(got0.view(np.uint32))])
    assert np.count_nonzero(got == 0) > 1439 + 500 and np.all(got[:1439] == 0)
    nz = got[1439:] != 0
    assert np.array_equal(got[1439:][nz], x[:n - 1439][nz])              # what is not zeroed is the input, 1439 items late


# ------------------------------------------------------------------------------------------------ rx_fft
RX_FFT_SIZES = [1024, 32768]


def _rx_fft_schedule(n_fft):
    """("work", x) / ("get", step) / ("enable", None) / ("size", n) / ("flush", None) operations of the test, in order ("flush": a get
    whose result is not compared)."""
    rng = np.random.default_rng(61)
    n = n_fft * 9 + 777
    t = np.arange(n)
    x = (0.3 * np.exp(2j * np.pi * 0.1234 * t) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    x[5000:5050] = 0
    sizes = [n_fft // 3, 17, n_fft, n_fft // 2 + 5, 2 * n_fft + 9, 100, n_fft - 1, 3 * n_fft]
    lo = 0
    for step, m in enumerate(sizes):
        if step == 0:
            yield "work", x[lo:lo + 50]                 # not enabled yet: dropped
            yield "enable", None
        m = min(m, n - lo)
        yield "work", x[lo:lo + m]; lo += m
        if step % 2 == 1:
            yield "get", step
    yield "size", n_fft // 2
    yield "flush", None
    yield "work", x[:n_fft]
    yield "get", None


def _ref_rx_fft(R, n_fft):
    h = R.ref_rx_fft_create(n_fft, O.WIN_BLACKMAN_HARRIS)
    pts = np.empty(n_fft, np.float32)
    res = []
    for op, a in _rx_fft_schedule(n_fft):
        if op == "work":
            a = np.ascontiguousarray(a)
            R.ref_rx_fft_work(h, _p(a), len(a))
        elif op == "enable":
            R.ref_rx_fft_set_enabled(h, 1)
        elif op == "size":
            R.ref_rx_fft_set_fft_size(h, a)
        elif op == "flush":
            R.ref_rx_fft_get(h, _p(pts))
        else:
            nr = R.ref_rx_fft_get(h, _p(pts))
            res.append(_digest(None if nr == 0 else pts[:nr].view(np.uint32)))
    R.ref_block_destroy(h)
    return res


@pytest.mark.parametrize("n_fft", RX_FFT_SIZES)
def test_rx_fft_restatement_follows_the_reference_block(R, n_fft):
    """rx_fft.cpp compiled unmodified (FFTW replaced by the oracle's own DFT in the stand-in, so this pins the buffering, windowing,
    d_push drop rule, power-spectrum kernel and fft-shift, not FFTW's rounding): same points after every get, for ragged work()
    sizes incl. calls longer than the FFT, calls while a spectrum is pending, disable / enable and a change of size."""
    s = O.Spectrum(n_fft, O.WIN_BLACKMAN_HARRIS)
    res, got_any, last = [], 0, None
    for op, a in _rx_fft_schedule(n_fft):
        if op == "work":
            s.work(a)
        elif op == "enable":
            s.set_enabled(True)
        elif op == "size":
            s.set_fft_size(a)
        elif op == "flush":
            s.get()
        else:
            g = s.get()
            res.append(_digest(None if g is None else _as(g, np.float32).view(np.uint32)))
            if g is not None and a is not None:
                got_any += 1
                assert len(g) == n_fft
                peak = int(np.argmax(g))
                assert abs(peak - (n_fft // 2 + round(0.1234 * n_fft))) <= 1
            last = g
    check(R, "rx_fft_%d" % n_fft, res)
    assert got_any >= 3
    assert last is not None and len(last) == n_fft // 2


# ------------------------------------------------------------------------------------------------ DSSS decoder
BARKER_13 = np.array([1, 1, 1, 1, 1, 0, 0, 1, 1, 0, 1, 0, 1], np.int32)
DSSS_SPS, DSSS_N = 25, 325


def _dsss_input():
    rng = np.random.default_rng(71)
    n_sym = 40
    # a spread BPSK stream + noise so that the maximum is well defined, plus a stretch of exact zeros
    chips = np.repeat(np.where(BARKER_13 > 0, 1.0, -1.0), DSSS_SPS)
    bits = rng.integers(0, 2, n_sym) * 2 - 1
    x = np.concatenate([b * chips for b in bits]).astype(np.complex64) * np.exp(0.4j).astype(np.complex64)
    x = (x + 0.3 * (rng.standard_normal(len(x)) + 1j * rng.standard_normal(len(x)))).astype(np.complex64)
    x[3000:3400] = 0
    return x, n_sym


def _dsss_n_out():
    """Symbols the restatement emits for _dsss_input(): how many the reference is asked for."""
    x, n_sym = _dsss_input()
    got = np.zeros(n_sym + 4, np.complex64)
    return O.lib().qo_dsss_decoder_run(_p(BARKER_13), 13, DSSS_SPS, _p(x), len(x), len(x), _p(got), len(got))


def _ref_dsss(R):
    N, nt = DSSS_N, DSSS_N + 11 * DSSS_SPS
    h = R.ref_dsss_decoder_create(_p(BARKER_13), 13, C.c_float(DSSS_SPS))
    res = [_digest(R.ref_dsss_decoder_history(h))]
    tr = np.zeros(2 * nt, np.float32)
    res.append(_digest(R.ref_dsss_decoder_taps(h, _p(tr), nt)))
    res.append(_digest(tr.view(np.uint32)))
    x, _ = _dsss_input()
    m0 = _dsss_n_out()
    # reference: buffer = [2N - 1 zeros][x][slack]; output m is called with `in` = item m N - (N - 1) (history N), one or more per call
    buf = np.concatenate([np.zeros(2 * N - 1, np.complex64), x, np.zeros(2 * N, np.complex64)])
    for per_call in (1, 3, m0):
        ref = np.zeros(m0, np.complex64)
        done = 0
        while done < m0:
            k = min(per_call, m0 - done)
            cons = C.c_long()
            in_ptr = buf[(2 * N - 1) + done * N - (N - 1):]
            out = np.zeros(k, np.complex64)
            assert R.ref_dsss_decoder_work(h, _p(in_ptr), k, _p(out), C.byref(cons)) == k and cons.value == k * N
            ref[done:done + k] = out; done += k
        res.append(_digest(ref.view(np.uint32)))
    R.ref_block_destroy(h)
    return res


def test_dsss_decoder_restatement_is_the_reference_block(R):
    """dsss_decoder_cc_impl.cc compiled unmodified: the matched-filter taps its constructor builds, and general_work over a buffer laid
    out the way the restatement DEFINES the region in front of the declared history (the stream's own older items, zeros at the
    start): same symbols bit for bit, for several scheduler chunkings of the reference and several of the restatement."""
    N, nt = DSSS_N, DSSS_N + 11 * DSSS_SPS
    tq = np.zeros(2 * nt, np.float32)
    O.lib().qo_dsss_decoder_taps(_p(BARKER_13), 13, DSSS_SPS, _p(tq))
    x, n_sym = _dsss_input()
    n = len(x)
    got = np.zeros(n_sym + 4, np.complex64)
    for chunk in (n, 1000, 77):
        m = O.lib().qo_dsss_decoder_run(_p(BARKER_13), 13, DSSS_SPS, _p(x), n, chunk, _p(got), len(got))
        if chunk == n:
            first, m0 = got[:m].copy(), m
        assert m == m0 and np.array_equal(got[:m].view(np.uint32), first.view(np.uint32)), chunk
    assert m0 >= n_sym - 2
    check(R, "dsss_decoder", [_digest(N), _digest(nt), _digest(tq.view(np.uint32))] + [_digest(first.view(np.uint32))] * 3)


# ------------------------------------------------------------------------------------------------ RSSI tags
RSSI_CHUNKINGS = (lambda n: [n], lambda n: [299, 1, 300, 301, 5000, 2000], lambda n: [7] * 1001)


def _rssi_input():
    rng = np.random.default_rng(81)
    n = 7000
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * np.repeat(rng.uniform(1e-4, 2.0, n // 100), 100)).astype(np.complex64)
    return x, n


def _ref_rssi(R):
    x, n = _rssi_input()
    res = []
    for chunking in RSSI_CHUNKINGS:
        ch = np.array(chunking(n), np.dtype("l"))
        db_r = np.zeros(64, np.float32); at_r = np.zeros(64, np.int64)
        kr = R.ref_rssi_tags(_p(x), n, C.c_float(-3.5), _p(ch), len(ch), _p(db_r), _p(at_r), 64)
        res += [_digest(kr), _digest(at_r[:kr]), _digest(db_r[:kr].view(np.uint32))]
    return res


def test_rssi_tag_rule_is_the_reference_block(R):
    """rssi_tag_block.cpp compiled unmodified (add_item_tag through the stand-in): an "RSSI" tag every 300 items, value and offset, for
    several scheduler chunkings; the float accumulation order is the block's (sequential)."""
    x, n = _rssi_input()
    db_o = np.zeros(64, np.float32); at_o = np.zeros(64, np.int64)
    k = O.lib().qo_rssi_tags_run(_p(x), n, -3.5, _p(db_o), _p(at_o), 64)
    assert k == n // 300
    check(R, "rssi_tags", [_digest(k), _digest(at_o[:k]), _digest(db_o[:k].view(np.uint32))] * len(RSSI_CHUNKINGS))
    assert np.array_equal(at_o[:k], np.arange(k) * 300 + 299)


REF_RUNS = {"disc4": _ref_disc, "zero_idle": _ref_zero_idle, "sample_sink": _ref_sample_sink, "dsss_decoder": _ref_dsss,
            "rssi_tags": _ref_rssi}
REF_RUNS.update({"cessb_stretcher_%d" % c: (lambda R, c=c: _ref_stretcher(R, c)) for c in STRETCHER_CHUNKS})
REF_RUNS.update({"deframer_%d" % m: (lambda R, m=m: _ref_deframer(R, m)) for m in DEFRAMER_MODEMS})
REF_RUNS.update({"sink_%s" % k: (lambda R, k=k: _ref_sink(R, k)) for k in SINK_KINDS})
REF_RUNS.update({"rx_fft_%d" % n: (lambda R, n=n: _ref_rx_fft(R, n)) for n in RX_FFT_SIZES})


if __name__ == "__main__":
    R_ = O.ref_blocks()
    if R_ is None:
        raise SystemExit("oracle/_ref/libqrl_ref_blocks.so missing: run `make -C oracle` where the reference tree exists")
    with open(GOLDEN, "w") as f:
        json.dump({name: _sequence_digest(run(R_)) for name, run in sorted(REF_RUNS.items())}, f, indent=1)
    np.save(CLIPPER_NPY, _ref_clipper_output(R_))
    print("wrote", GOLDEN, "and", CLIPPER_NPY)
