"""GPU tier: what a receive handle carries from one stream to the next.  qrl_rx_reset (include/qrl_b200.h) promises that afterwards
every port of every call is bit-identical to a freshly created handle given the settings now in force (carrier offsets, the analog
setters, RSSI, overlapped calls, the caller's stream) before its first call; QRL_PARAM_RSSI promises that every switch-on starts
the tap afresh.  Each case runs a first stream with offsets, a mid-stream retune and the chain's setters, resets, and runs a second
stream next to a fresh twin: every call's ports bit for bit, and the oracle fed the second stream with the same settings.  Then the
paths where a reset has more to undo (many channels, overlapped tails, shared-stream input, a caller's stream), the RSSI tap
switched on mid-stream and off and on again, and overlapped calls switched on and off between calls.

Inputs are host arrays except on the caller-stream case, so the file also runs on the host-thread build of the library
(QRL_EMULATED_LIB, tools/emu)."""
import os

import numpy as np
import pytest

from tests import siggen
from tests.test_gpu_dispatch import (RX, assert_partition, bases, check_rx, concat_calls, default_partition, equal_cuts, free_device,
                                     make_slab, n_sm, ragged, run_rx, spot_shifts, stage_launches)

pytestmark = pytest.mark.gpu

EMULATED = bool(os.environ.get("QRL_EMULATED_LIB"))

OFFSET_HZ, RETUNE_HZ = 40.0, -35.0


def offsets(Cn):
    """carrier offsets of the first stream: every channel before the first call, the last channel (a spot channel of
    test_gpu_dispatch's slabs: its own class) retuned before the third call, so that its rotator has a phase base at a sample other
    than 0; and the settings in force at the reset, as events of the second stream's first call"""
    return [(0, -1, OFFSET_HZ), (2, Cn - 1, RETUNE_HZ)], [(0, -1, OFFSET_HZ), (0, Cn - 1, RETUNE_HZ)]


def setters(qrl, name):
    """(the first stream's setters as (cut index, key, value), the settings in force after them).  NBFM's tone squelch goes in and
    out again: with it in force the audio port of a signal without the tone stays empty."""
    P = qrl.PARAM
    mid = {
        "nbfm": [(1, P.SQUELCH_DB, -20.0), (1, P.FILTER_WIDTH, 4000), (1, P.CTCSS, 88.5), (2, P.CTCSS, 0.0)],
        "am": [(1, P.AGC_ATTACK, 0.5), (1, P.AGC_DECAY, 0.01)],
        "usb": [(1, P.AGC_ATTACK, 0.02), (1, P.AGC_DECAY, 0.3), (1, P.GAIN, 0.5)],
        "lsb": [(1, P.AGC_ATTACK, 0.02), (1, P.AGC_DECAY, 0.3), (1, P.GAIN, 0.5)],
    }.get(name, [])
    in_force = {"nbfm": [(P.SQUELCH_DB, -20.0), (P.FILTER_WIDTH, 4000)]}.get(name, [(k, v) for (_, k, v) in mid])
    return mid, in_force


def feed(blk, X, cuts, offsets=(), sets=()):
    """run_rx with the setters (cut index, key, value) applied before their cut"""
    calls = []
    for k, cut in enumerate(cuts):
        for (sk, key, value) in sets:
            if sk == k:
                blk.set_param(key, value)
        calls += run_rx(blk, X, [cut], [(0, ch, hz) for (ek, ch, hz) in offsets if ek == k])
    return calls


def configure(blk, offsets, in_force):
    for (_, ch, hz) in offsets:
        blk.set_carrier_offset(hz, channel=ch)
    for key, value in in_force:
        blk.set_param(key, value)


def first_stream(X2, T1):
    """different samples from the second stream, at another level (AGC and squelch states away from their start)"""
    T = X2.shape[1]
    return np.ascontiguousarray(X2[:, T // 3:T // 3 + T1] * np.float32(0.7))


def assert_same_calls(got, want, where):
    assert len(got) == len(want), where
    for k, (g, w) in enumerate(zip(got, want)):
        if w is None:
            continue
        for p in range(len(w)):
            for c in range(len(w[p])):
                same = g[p][c].dtype == w[p][c].dtype and np.array_equal(g[p][c].view(np.uint8), w[p][c].view(np.uint8))
                assert same, (where, "call", k, "port", p, "channel", c, len(g[p][c]), len(w[p][c]))


def reset_case(qrl, O, name, Cn, spots, profile=False):
    """handle A: first stream (offsets, retune, setters), reset, second stream; fresh twin B: the settings in force, second stream.
    Returns A (caller closes) after checking A == B call by call and A against the oracle."""
    T = RX[name][3]
    T1 = T // 2
    B, payloads = bases(name, O, T)
    X2 = make_slab(B, Cn, spots)
    X1 = first_stream(X2, T1)
    cuts1, cuts2 = ragged(T1), ragged(T)
    maxs = max(hi - lo for lo, hi in cuts1 + cuts2)
    mid, in_force = setters(qrl, name)
    first, now = offsets(Cn)
    a = RX[name][0](qrl, Cn, maxs)
    try:
        if profile:
            assert a._L.qrl_rx_profile(a._h, 1) == 0
        feed(a, X1, cuts1, first, mid)
        a.reset()
        if profile:                                     # count the launches of the second stream only
            assert a._L.qrl_rx_profile(a._h, 1) == 0
        got = feed(a, X2, cuts2)
        b = RX[name][0](qrl, Cn, maxs)
        try:
            configure(b, now, in_force)
            want = feed(b, X2, cuts2)
        finally:
            b.close()
        assert_same_calls(got, want, name)
        check_rx(name, O, B, payloads, concat_calls(got, a.nports, Cn), spots, cuts2, now, setters=in_force)
    except BaseException:
        a.close()
        raise
    finally:
        del X1, X2
        free_device()
    return a


# ------------------------------------------------------------------ 1. reset on every receive chain
@pytest.mark.parametrize("name", list(RX))
def test_reset_equals_a_fresh_handle(qrl, oracle, name):
    """C = 3 plain channels (each its own base signal).  Every chain has the rotator in front: the retuned channel's phase must
    restart at 0, and every loop, ring and count must be back at its constructor value."""
    reset_case(qrl, oracle, name, 3, {}).close()


# ------------------------------------------------------------------ 2. paths where a reset has more to undo
@pytest.mark.parametrize("Cn", [33, 97])
@pytest.mark.parametrize("name", ["4fsk", "qpsk", "nbfm"])
def test_reset_at_many_channels(qrl, oracle, name, Cn):
    """a one-lane last group; at 97 channels NBFM and QPSK in many mode, 4FSK's Viterbi on the loop partition; NBFM's de-emphasis
    split (C <= SM count) runs as stage 5 before and after the reset"""
    a = reset_case(qrl, oracle, name, Cn, spot_shifts(Cn), profile=name == "nbfm")
    try:
        assert_partition(qrl, a, default_partition(name, Cn))
        if name == "nbfm" and Cn <= n_sm():
            assert stage_launches(a, 5) > 0
    finally:
        a.close()


def _overlapped_reset(qrl, O, cuts1, cuts2):
    name, Cn = "4fsk", 3
    T = RX[name][3]
    B, payloads = bases(name, O, T)
    X2 = make_slab(B, Cn, {})
    X1 = first_stream(X2, cuts1[-1][1])
    maxs = max(hi - lo for lo, hi in cuts1 + cuts2)
    a, b = RX[name][0](qrl, Cn, maxs), RX[name][0](qrl, Cn, maxs)
    try:
        first, now = offsets(Cn)
        a.set_overlap(True)
        for k, (lo, hi) in enumerate(cuts1):           # back to back: no read joins the last call's tail before the reset
            for (ek, ch, hz) in first:
                if ek == k:
                    a.set_carrier_offset(hz, channel=ch)
            a.work(X1[:, lo:hi])
        a.reset()
        got = run_rx(a, X2, cuts2)
        b.set_overlap(True)
        configure(b, now, [])
        want = run_rx(b, X2, cuts2)
        assert_same_calls(got, want, "overlapped 4fsk")
        check_rx(name, O, B, payloads, concat_calls(got, a.nports, Cn), {}, cuts2, now)
    finally:
        a.close(); b.close()


def test_reset_joins_an_overlapped_tail(qrl, oracle):
    """overlapped 4FSK calls issued back to back, reset with the last call's loop / FEC tail still queued"""
    T = RX["4fsk"][3]
    _overlapped_reset(qrl, oracle, equal_cuts(T // 2, 4), equal_cuts(T, 4))


def test_reset_then_an_overlapped_call_of_another_length(qrl, oracle):
    """the first call after the reset is longer than the calls before it: the seam path (a change of length joins the tail)"""
    T = RX["4fsk"][3]
    _overlapped_reset(qrl, oracle, equal_cuts(T // 2, 4), [(0, T // 3), (T // 3, 2 * (T // 3)), (2 * (T // 3), T)])


def _sc16(x):
    return np.stack([np.clip(np.rint(x.real * 20000), -32768, 32767), np.clip(np.rint(x.imag * 20000), -32768, 32767)], -1).astype(np.int16)


@pytest.mark.parametrize("name", ["4fsk", "wbfm"])
def test_reset_with_shared_stream_input(qrl, oracle, name):
    """stride 0 (one stream for every channel), host gr_complex and sc16 calls mixed, before and after the reset; every channel
    applies its own offset to the one stream (4FSK rotates inside stage 1, WBFM in the rotator pass)"""
    Cn = 3
    T = RX[name][3]
    B, _ = bases(name, oracle, T)
    x2 = np.ascontiguousarray(B[0])
    x1 = np.ascontiguousarray(B[1, :T // 2] * np.float32(0.7))
    s1, s2 = _sc16(x1), _sc16(x2)
    cuts1, cuts2 = ragged(T // 2), ragged(T)
    maxs = max(hi - lo for lo, hi in cuts1 + cuts2)

    def run(blk, x, s, cuts, offsets=()):
        calls = []
        for k, (lo, hi) in enumerate(cuts):
            for (ek, ch, hz) in offsets:
                if ek == k:
                    blk.set_carrier_offset(hz, channel=ch)
            if k % 2 == 0:
                blk.work_shared(x[lo:hi])
            else:
                blk.work_shared_sc16(s[lo:hi])
            calls.append([blk.read_port(p) for p in range(blk.nports)])
        return calls

    a, b = RX[name][0](qrl, Cn, maxs), RX[name][0](qrl, Cn, maxs)
    try:
        first, now = offsets(Cn)
        run(a, x1, s1, cuts1, first)
        a.reset()
        got = run(a, x2, s2, cuts2)
        configure(b, now, [])
        want = run(b, x2, s2, cuts2)
        assert_same_calls(got, want, name)
        assert all(len(got[k][0][c]) > 0 for k in (0, 2) for c in range(Cn))
    finally:
        a.close(); b.close()


@pytest.mark.skipif(EMULATED, reason="needs a real CUDA device (a torch stream)")
def test_reset_on_a_caller_stream(qrl, oracle):
    """the handle runs on the caller's stream (qrl_rx_set_stream) when it is reset, and stays on it; the twin runs on its own"""
    import torch
    name, Cn = "4fsk", 3
    T = RX[name][3]
    B, payloads = bases(name, oracle, T)
    X2 = make_slab(B, Cn, {})
    X1 = first_stream(X2, T // 2)
    cuts1, cuts2 = ragged(T // 2), ragged(T)
    maxs = max(hi - lo for lo, hi in cuts1 + cuts2)
    s = torch.cuda.Stream()
    a, b = RX[name][0](qrl, Cn, maxs), RX[name][0](qrl, Cn, maxs)
    try:
        first, now = offsets(Cn)
        a.set_stream(s.cuda_stream)
        feed(a, X1, cuts1, first)
        a.reset()
        got = feed(a, X2, cuts2)
        configure(b, now, [])
        want = feed(b, X2, cuts2)
        assert_same_calls(got, want, "caller stream")
        check_rx(name, oracle, B, payloads, concat_calls(got, a.nports, Cn), {}, cuts2, now)
    finally:
        a.close(); b.close()
        s.synchronize()


@pytest.mark.parametrize("name", ["4fsk", "nbfm"])
def test_reset_twice_and_before_any_work(qrl, oracle, name):
    Cn = 3
    T = RX[name][3]
    B, _ = bases(name, oracle, T)
    X2 = make_slab(B, Cn, {})
    X1 = first_stream(X2, T // 2)
    cuts = ragged(T)
    mk = lambda: RX[name][0](qrl, Cn, T // 2 + 13)
    fresh, early, twice = mk(), mk(), mk()
    try:
        want = feed(fresh, X2, cuts)
        early.reset()
        assert_same_calls(feed(early, X2, cuts), want, (name, "reset before any work"))
        feed(twice, X1, ragged(T // 2))
        twice.reset()
        twice.reset()
        assert_same_calls(feed(twice, X2, cuts), want, (name, "reset twice"))
    finally:
        fresh.close(); early.close(); twice.close()


# ------------------------------------------------------------------ 3. the RSSI tap: switched on mid-stream, off and on, reset
def _rssi_signal(name, T):
    if name == "nbfm":
        return siggen.gen_nbfm_channels(3, T, seed0=700)
    return siggen.gen_4fsk_channels(3, T, seed0=5700)[0]


RSSI_CHAINS = {"4fsk": (lambda q, m: q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=3, max_samples=m), 50),
               "nbfm": (lambda q, m: q.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=3, max_samples=m), 125)}


def _check_rssi(blk, refs, level, where):
    p0 = blk.read_port(0)
    got = blk.rssi(level=level)
    for c in range(len(refs)):
        assert len(p0[c]) > 0, where
        want = refs[c].work(p0[c]) + level
        assert abs(float(got[c]) - want) < 1e-3 or want < -150.0, (where, c, float(got[c]), want)


@pytest.mark.parametrize("name", list(RSSI_CHAINS))
def test_rssi_switched_on_mid_stream(qrl, oracle, name):
    """two calls without the tap, then on: from then on the values of rssi_block constructed at the switch-on"""
    make, dec = RSSI_CHAINS[name]
    n_items = [800, 50, 2600, 1500, 5000]                 # port-0 items per call after the switch-on
    sizes = [dec * 300, dec * 700 + 13] + [dec * n for n in n_items]
    X = _rssi_signal(name, sum(sizes))
    blk = make(qrl, max(sizes))
    try:
        lo = 0
        for k, n in enumerate(sizes):
            if k == 2:
                blk.enable_rssi(True)
                refs = [oracle.Rssi(0.0) for _ in range(3)]
            blk.work(X[:, lo:lo + n]); lo += n
            if k >= 2:
                _check_rssi(blk, refs, -2.5, (name, k))
            else:
                blk.read_port(0)
    finally:
        blk.close()


@pytest.mark.parametrize("name", list(RSSI_CHAINS))
def test_rssi_off_and_on_again(qrl, oracle, name):
    """on for a loud call, off for a call 40 dB quieter, on again: the calls after the re-enable (fewer than 1024 port-0 items,
    then fewer than 3024 in all) must read what an rssi_block constructed at the re-enable reads -- not the window of the first
    switch-on, and not an IIR value carried over it"""
    make, dec = RSSI_CHAINS[name]
    sizes = [dec * 2500, dec * 2500, dec * 800, dec * 2000]
    X = _rssi_signal(name, sum(sizes))
    X[:, sizes[0]:] *= np.float32(0.01)
    blk = make(qrl, max(sizes))
    try:
        blk.enable_rssi(True)
        blk.work(X[:, :sizes[0]])
        loud = blk.rssi()
        blk.enable_rssi(False)
        lo = sizes[0]
        blk.work(X[:, lo:lo + sizes[1]]); lo += sizes[1]
        blk.read_port(0)
        blk.enable_rssi(True)
        refs = [oracle.Rssi(0.0) for _ in range(3)]
        for k, n in enumerate(sizes[2:]):
            blk.work(X[:, lo:lo + n]); lo += n
            _check_rssi(blk, refs, 0.0, (name, "after re-enable", k))
        assert np.all(loud - blk.rssi() > 30.0), (loud, blk.rssi())
    finally:
        blk.close()


@pytest.mark.parametrize("name", list(RSSI_CHAINS))
def test_rssi_across_a_reset(qrl, oracle, name):
    """reset with the tap on: -180 + level until the next call, then bit-identical to a fresh twin's"""
    make, dec = RSSI_CHAINS[name]
    sizes = [dec * 2500, dec * 700, dec * 3000]
    X = _rssi_signal(name, sum(sizes))
    a, b = make(qrl, max(sizes)), make(qrl, max(sizes))
    try:
        a.enable_rssi(True)
        a.work(X[:, :sizes[0]])
        a.reset()
        assert np.array_equal(a.rssi(level=-3.5), np.full(3, np.float32(-180.0) + np.float32(-3.5), np.float32))
        b.enable_rssi(True)
        lo = sizes[0]
        for n in sizes[1:]:
            a.work(X[:, lo:lo + n]); b.work(X[:, lo:lo + n]); lo += n
            ra, rb = a.rssi(level=-3.5), b.rssi(level=-3.5)
            assert np.array_equal(ra.view(np.uint32), rb.view(np.uint32)), (name, n, ra, rb)
            assert_same_calls([[a.read_port(0)]], [[b.read_port(0)]], (name, "rssi reset"))
    finally:
        a.close(); b.close()


# ------------------------------------------------------------------ 4. overlapped calls switched between calls
def test_overlap_switched_mid_stream(qrl, oracle):
    """4FSK-2k-FM: overlapped calls on after two plain calls, off after three more, on again; every call's ports equal a handle that
    never overlapped.  The calls issued overlapped are read only every second call, so their tails really run under the next call."""
    name, Cn = "4fsk", 3
    T = RX[name][3]
    B, _ = bases(name, oracle, T)
    X = make_slab(B, Cn, {})
    cuts = [(0, 40000), (40000, 90001), (90001, 150000), (150000, 210000), (210000, 270000), (270000, 330000), (330000, 330101),
            (330101, 400000), (400000, 460000), (460000, 524288)]
    switches = {2: True, 5: False, 7: True}
    maxs = max(hi - lo for lo, hi in cuts)
    a, ser = RX[name][0](qrl, Cn, maxs), RX[name][0](qrl, Cn, maxs)
    try:
        a.set_carrier_offset(OFFSET_HZ)
        ser.set_carrier_offset(OFFSET_HZ)
        want = run_rx(ser, X, cuts)
        on = False
        for k, (lo, hi) in enumerate(cuts):
            if k in switches:
                on = switches[k]
                a.set_overlap(on)
            a.work(X[:, lo:hi])
            if not on or k % 2 == 1 or k == len(cuts) - 1:
                assert_same_calls([[a.read_port(p) for p in range(a.nports)]], [want[k]], ("overlap switched", k, on))
    finally:
        a.close(); ser.close()
