"""CPU tier: the exact rewrites that shorten the loop-carried chain of the lean real-symbol recurrence in symsync_kernel
(qrl_kernels.cuh, VAR 1 / 2: the 4FSK-FM and M17 receivers).  Each rewrite must give the same bits as the form it replaced."""
import ctypes as C

import numpy as np

M = np.float32(12582912.0)                     # 1.5 * 2^23: fmaf(v, 128, M) holds rint(128 v) in its low mantissa bits
T1, T2, T3 = np.float32(-1.0), np.float32(-5.9604644775390625e-8), np.float32(0.99999988079071044921875)
LEVELS = np.array([-1.5, -0.5, 0.5, 1.5], np.float32)


def _clock_loop_alpha(loop_bw):
    from oracle import oracle as O
    a, b = C.c_float(), C.c_float()
    O.lib().qo_clock_loop_gains(C.c_float(loop_bw), C.c_float(1.0), C.c_float(0.2869), C.byref(a), C.byref(b))
    return np.float32(a.value)


def lean_handle_windows():
    """(name, n0) of every receiver that runs the lean recurrence: the FM branch of make_gr_demod_4fsk (sps 1, 5, 10) and M17, with
    the symbol sync's samples per symbol, period deviation and loop bandwidth as qrl_rx_create sets them; n0 = floor(min_period -
    |alpha|) in float32, and the lean loop is taken when min_period > |alpha| and n0 >= 1."""
    two_pi = 2 * np.pi
    m17_rate = 24000.0 / 5
    handles = [("4fsk_fm_sps1", 8, 0.05, two_pi / 200.0), ("4fsk_fm_sps5", 10, 0.05, two_pi / 200.0),
               ("4fsk_fm_sps10", 10, 0.05, two_pi / 200.0), ("m17", 5, 500.0 / m17_rate, two_pi / (m17_rate / 50))]
    out = []
    for name, sym_sps, dev, loop_bw in handles:
        alpha = _clock_loop_alpha(np.float32(loop_bw))
        min_period = np.float32(np.float32(sym_sps) - np.float32(dev))
        n0 = int(np.floor(np.float32(min_period - abs(alpha))))
        assert min_period > abs(alpha) and n0 >= 1, name
        out.append((name, n0))
    return out


def fmaf(a, b, c):
    """float32 fma: the float64 product and sum are exact for the operands used here, so one rounding to float32 remains."""
    return (a.astype(np.float64) * np.float64(b) + np.float64(c)).astype(np.float32)


def test_tap_row_from_ph_matches_row_from_mu():
    """Rewrite 1: the tap address comes from ph, not from mu = (ph - n0) - s12.  For EVERY float32 ph in [n0, n0 + 3) and every n0 a lean
    handle can have: bits(fmaf(ph, 128, M - 128 n0)) - 128 s12 == bits(fmaf(mu, 128, M)), where s12 = [ph >= n0+1] + [ph >= n0+2] is taken
    from ph directly and equals the old [m0 >= 1] + [m0 >= 2] with m0 = ph - n0."""
    windows = lean_handle_windows()
    assert {n0 for _, n0 in windows} >= {4, 7, 9}
    for name, n0 in sorted(set(windows), key=lambda w: w[1]):
        f0 = np.float32(n0)
        lo, hi = f0.view(np.uint32), np.float32(n0 + 3).view(np.uint32)
        ph = np.arange(lo, hi, dtype=np.uint32).view(np.float32)
        assert ph[0] == f0 and ph[-1] < n0 + 3
        m0 = ph - f0
        s12_old = (m0 >= 1).astype(np.float32) + (m0 >= 2).astype(np.float32)
        mu = m0 - s12_old
        want = fmaf(mu, 128.0, M).view(np.uint32)
        g1, g2 = ph >= np.float32(n0 + 1), ph >= np.float32(n0 + 2)
        assert np.array_equal(g1, m0 >= 1) and np.array_equal(g2, m0 >= 2), name
        q_mph = np.float32(M - np.float32(128.0) * f0)
        assert float(q_mph) == 12582912.0 - 128.0 * n0
        got = fmaf(ph, 128.0, q_mph).view(np.uint32) - np.uint32(128) * (g1.astype(np.uint32) + g2.astype(np.uint32))
        assert np.array_equal(got, want), name
        rows = want - M.view(np.uint32)
        assert rows.min() == 0 and rows.max() == 128, name        # every bank row 0 .. 128 is reached, no other


def _slicer_u_old(yr, h1, h2, dh1, dh2):
    s1 = (yr >= T1).astype(np.float32)
    s23 = (yr >= T2).astype(np.float32) + (yr >= T3).astype(np.float32)
    kd = np.float32(-1.5) - dh2
    br = (s1 + kd) + s23
    return (yr - h2) * dh1 - br * h1


def _slicer_u_new(yr, h1, h2, dh1, dh2):
    pb = [(np.float32(lv) - dh2) * h1 for lv in LEVELS]
    lo = np.where(yr >= T1, pb[1], pb[0])
    hi = np.where(yr >= T3, pb[3], pb[2])
    return (yr - h2) * dh1 - np.where(yr >= T2, hi, lo).astype(np.float32)


def test_slicer_products_picked_by_thresholds_match():
    """Rewrite 2: u = (yr - h2) dh1 - br h1 with br = dn - dh2.  The four products fl(br_k h1) are formed a symbol early and the slicer's
    thresholds pick one; checked over every float32 within 2048 ulps of each threshold (and of 0, +-1, +-2) for every previous
    decision dh2, plus a seeded random sweep of all operands and NaN."""
    rng = np.random.default_rng(20261015)
    near = []
    for c in (T1, T2, T3, np.float32(0.0), np.float32(1.0), np.float32(-2.0), np.float32(2.0)):
        u = c.view(np.uint32).astype(np.int64)
        if c == 0:
            near.append(np.concatenate([np.arange(0, 2049), np.arange(0x80000000, 0x80000000 + 2049)]).astype(np.uint32).view(np.float32))
        else:
            near.append(np.arange(u - 2048, u + 2049).astype(np.uint32).view(np.float32))
    yr_near = np.concatenate(near)
    for dh2 in LEVELS:
        for dh1 in LEVELS:
            n = yr_near.size
            h1 = (rng.standard_normal(n) * 1.5).astype(np.float32)
            h2 = (rng.standard_normal(n) * 1.5).astype(np.float32)
            a = _slicer_u_old(yr_near, h1, h2, dh1, dh2)
            b = _slicer_u_new(yr_near, h1, h2, dh1, dh2)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    n = 2_000_000
    yr = np.concatenate([(rng.standard_normal(n) * 1.5).astype(np.float32), np.array([np.nan, np.inf, -np.inf, -0.0], np.float32)])
    h1 = (rng.standard_normal(yr.size) * 1.5).astype(np.float32)
    h2 = (rng.standard_normal(yr.size) * 1.5).astype(np.float32)
    dh1 = LEVELS[rng.integers(0, 4, yr.size)]
    dh2 = LEVELS[rng.integers(0, 4, yr.size)]
    with np.errstate(invalid="ignore"):
        a = _slicer_u_old(yr, h1, h2, dh1, dh2)
        b = _slicer_u_new(yr, h1, h2, dh1, dh2)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
