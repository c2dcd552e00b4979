"""CPU tier: the FreeDV chains up to the codec2 modem boundary in the oracle (tests/freedv_oracle.c: gr_demod_freedv.cpp:31-81,
gr_mod_freedv.cpp:27-85) -- the
filter designs, feedforward_agc_cc against an independent numpy statement, chunk invariance, the host-side speech helpers, and the
committed known answers (tests/golden/golden_freedv.json).  The functions at the bottom run the same known answers and the argument
checks through a library build (CUDA on the GPU tier, host threads in tests/test_emulated_freedv.py)."""
import json
import os

import numpy as np
import pytest
from numpy.lib.stride_tricks import sliding_window_view

from tests import freedv_oracle as FO
from tests.golden import freedv_cases as F
from tests.test_golden import check_stream, sha

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_freedv.json")))


def test_filter_designs():
    """RX: /125 low-pass of 1045 taps with a DC gain of 125 (port 0 is 125x the input level), 163-tap side-band and audio filters;
    TX: 131-tap side-band filter, 2007-tap x125 interpolator (17 per arm) with a DC gain of 125."""
    for sb in (0, 1):
        rx = FO.FreedvRx(125, 1000000, 2500, 200, sb)
        t0, t1, t2 = rx.taps(0), rx.taps(1), rx.taps(2)
        assert len(t0) == 1045 and abs(float(np.sum(t0.astype(np.float64))) - 125.0) < 1e-3
        assert len(t1) == 163 and len(t2) == 163
        tx = FO.FreedvTx(125, 1000000, 2500, 200, sb)
        assert len(tx.taps(0)) == 131
        ti = tx.taps(1)
        assert len(ti) == 2007 and (len(ti) + 124) // 125 == 17 and abs(float(np.sum(ti.astype(np.float64))) - 125.0) < 1e-3
    # LSB is the mirror image of USB: conjugate taps
    u = FO.FreedvRx(125, 1000000, 2400, 600, 0).taps(1)
    lsb = FO.FreedvRx(125, 1000000, 2400, 600, 1).taps(1)
    assert np.allclose(lsb, np.conj(u), atol=1e-6)


def ffagc_numpy(x, N, ref):
    """y[n] = (ref / max(1e-4, max_{k=n-N+1..n} env(x[k]))) x[n-N+1], env = max(|re|, |im|), zero history; float32 throughout"""
    x = np.asarray(x, np.complex64)
    xp = np.concatenate([np.zeros(N - 1, np.complex64), x])
    env = np.maximum(np.abs(xp.real), np.abs(xp.imag))
    mx = np.maximum(sliding_window_view(env, N).max(axis=1), np.float32(1e-4))
    g = np.float32(ref) / mx
    return (xp.real[:len(x)] * g + 1j * (xp.imag[:len(x)] * g)).astype(np.complex64), g


def test_feedforward_agc_matches_numpy():
    rng = np.random.default_rng(81)
    n = 6000
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * np.linspace(0.01, 2.0, n)).astype(np.complex64)
    x[2000:2900] = 0                                                   # silence inside the stream: the 1e-4 floor
    want, g = ffagc_numpy(x, 512, 1.0)
    for chunk in (0, 1, 7, 511, 512, 1000):
        got = FO.feedforward_agc(x, 512, 1.0, chunk)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), chunk
    assert np.all(g[2511:2900] == np.float32(1.0) / np.float32(1e-4))  # windows that see only silence: the floor
    # the 511-sample delay: an impulse comes out N - 1 items later, scaled to ref / its own envelope
    imp = np.zeros(1200, np.complex64); imp[100] = 0.25 - 0.5j
    y = FO.feedforward_agc(imp, 512, 1.0)
    assert np.flatnonzero(y).tolist() == [611] and y[611] == np.complex64(0.5 - 1.0j)
    assert not np.any(FO.feedforward_agc(np.zeros(700, np.complex64), 512, 1.0))


@pytest.mark.parametrize("sb", [0, 1])
def test_chains_chunk_invariant(sb):
    X = F.rx_signal("freedv_rx_lsb" if sb else "freedv_rx_usb", C=1, T=90000)[0]
    w0, w1 = FO.FreedvRx(125, 1000000, 2500, 200, sb).work(X)
    rx = FO.FreedvRx(125, 1000000, 2500, 200, sb)
    parts, lo = [], 0
    for m in (1, 124, 125, 40000, 3, 49747):
        parts.append(rx.work(X[lo:lo + m])); lo += m
    assert lo == len(X)
    assert np.array_equal(np.concatenate([p[0] for p in parts]), w0) and np.array_equal(np.concatenate([p[1] for p in parts]), w1)
    assert len(w0) == len(w1) == len(X) // 125
    s = F.tx_input(2500)
    want = FO.FreedvTx(125, 1000000, 2500, 200, sb).work(s)
    tx = FO.FreedvTx(125, 1000000, 2500, 200, sb)
    got, lo = [], 0
    for m in (1, 2, 511, 512, 1474):
        got.append(tx.work(s[lo:lo + m])); lo += m
        assert len(got[-1]) == 125 * m
    assert np.array_equal(np.concatenate(got), want)


def test_speech_side_closed_forms(oracle):
    s = np.array([-32768, -32767, -1, 0, 1, 12345, 32767], np.int16)
    assert np.array_equal(FO.freedv_speech_out(s), (s.astype(np.float64) / 16384.0).astype(np.float32))
    rng = np.random.default_rng(82)
    a = (0.3 * rng.standard_normal(4000)).astype(np.float32)
    a[1000:1010] = 5.0                                                  # drives the converter into its clip
    got = FO.freedv_speech_in(a)
    taps = oracle.band_pass(1, 8000, 200, 3500, 350, oracle.WIN_BLACKMAN_HARRIS)
    y = np.convolve(a.astype(np.float64), taps.astype(np.float64))[:len(a)] * 32765.0
    want = np.rint(np.clip(y, -32768, 32767))
    assert len(got) == len(a) and np.max(np.abs(got.astype(np.float64) - want)) <= 1.0
    assert got.max() == 32767 and got.min() == -32768


def test_golden_freedv_oracle():
    for name, (sps, fs, _cf, fw, lo, sb) in F.RX_CASES.items():
        X = F.rx_signal(name)
        assert sha(X) == G["rx"][name]["input_sha256"], "signal generator drifted"
        for c in range(X.shape[0]):
            p = FO.FreedvRx(sps, fs, fw, lo, sb).work(X[c])
            for k in range(2):
                check_stream(p[k], G["rx"][name]["channels"][c][k], (name, c, k))
    for name, (sps, fs, _cf, fw, lo, sb) in F.TX_CASES.items():
        s = F.tx_input()
        assert sha(s) == G["tx"][name]["input_sha256"]
        check_stream(FO.FreedvTx(sps, fs, fw, lo, sb).work(s), G["tx"][name]["out"], name)


# ------------------------------------------------------------------ run through a library build (GPU tier / host-thread emulation)
def golden_rx_through(q, name):
    sps, fs, cf, fw, lo, sb = F.RX_CASES[name]
    X = F.rx_signal(name)
    blk = q.make_gr_demod_freedv(sps, fs, cf, fw, lo, 0, sb, n_channels=X.shape[0], max_samples=80000)
    assert blk.nports == 2 and blk._itemsize == [8, 2]
    acc = [[[] for _ in range(X.shape[0])] for _ in range(2)]
    a = 0
    for m in (1, 79999, 124, 69876):
        blk.work(X[:, a:a + m]); a += m
        for p in range(2):
            for c, v in enumerate(blk.read_port(p)):
                acc[p][c].append(v)
    assert a == X.shape[1]
    for c in range(X.shape[0]):
        for p in range(2):
            check_stream(np.concatenate(acc[p][c]), G["rx"][name]["channels"][c][p], (name, c, p))


def golden_tx_through(q, name):
    sps, fs, cf, fw, lo, sb = F.TX_CASES[name]
    s = F.tx_input()
    tx = q.make_gr_mod_freedv(sps, fs, cf, fw, lo, 0, sb, n_channels=1, max_items=2000)
    parts, a = [], 0
    for m in (1, 1999, 1000):
        parts.append(tx.work_modem(s[None, a:a + m])[0]); a += m
        assert len(parts[-1]) == 125 * m
    check_stream(np.concatenate(parts), G["tx"][name]["out"], name)


def einval_paths(q):
    """The factory arguments the chain cannot hold and the setters gr_demod_freedv does not have are refused with QRL_EINVAL."""
    import ctypes as C
    L = q.load_library()
    h = C.c_void_p()
    for args in ((125, 1000000, 1700, 2500, 200, 0), (100, 1000000, 1700, 2500, 200, 0), (125, 1000000, 1700, 2500, 2500, 0),
                 (125, 1000000, 1700, 2500, -1, 0), (125, 1000000, 1700, 4001, 200, 0), (0, 1000000, 1700, 2500, 200, 0)):
        bad = args[0] != 125 or not (0 <= args[4] < args[3] <= 4000)
        for fn in (L.qrl_rx_create_freedv, L.qrl_tx_create_freedv):
            rc = fn(*args, 2, 1000, 0, C.byref(h))
            if bad:
                assert rc == -22 and h.value is None, (fn, args)
                assert b"qrl_" in L.qrl_last_error(None)
            else:
                assert rc == 0, (fn, args, L.qrl_last_error(None))
                (L.qrl_rx_destroy if fn is L.qrl_rx_create_freedv else L.qrl_tx_destroy)(h)
                h = C.c_void_p()
    assert L.qrl_rx_create(q.KIND.DEMOD_FREEDV, 125, 1000000, 1700, 2500, 0, 1, 1000, 0, C.byref(h)) == -22
    assert L.qrl_tx_create(q.KIND.MOD_FREEDV, 125, 1000000, 1700, 2500, 0, 1, 1000, 0, C.byref(h)) == -22
    rx = q.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, max_samples=1000)
    for key in (q.PARAM.SQUELCH_DB, q.PARAM.FILTER_WIDTH, q.PARAM.OVERLAP_CALLS, q.PARAM.GAIN):
        assert L.qrl_rx_set_param(rx._h, -1, key, 1.0) == -22, key
    for key in (q.PARAM.AGC_ATTACK, q.PARAM.AGC_DECAY, q.PARAM.CARRIER_OFFSET_HZ):
        assert L.qrl_rx_set_param(rx._h, -1, key, 0.05) == 0, key
    tx = q.make_gr_mod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, max_items=100)
    assert L.qrl_tx_set_param(tx._h, -1, q.PARAM.FILTER_WIDTH, 2000.0) == -22
    assert L.qrl_tx_set_param(tx._h, -1, q.PARAM.BB_GAIN, 0.5) == 0


def test_cpp_freedv_adapter_compiles(tmp_path):
    """The FreeDV factories of the header-only C++ mirror and their loop-back program compile and link against the C ABI (the GPU tier
    runs the program: tests/test_gpu_freedv.py)."""
    import subprocess
    from tests.test_gpu_cpp_adapter import ROOT
    exe = os.path.join(str(tmp_path), "test_freedv_adapter")
    libdir = os.path.join(ROOT, "qradiolink_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "test_freedv_adapter.cpp"), "-o", exe,
                           "-L" + libdir, "-lqrl_b200", "-Wl,-rpath," + libdir])
    assert os.path.exists(exe)
