"""GPU tier: the fused 4FSK-FM receive front end (fsk_fm_frontend_kernel: stage 1, channel filter, discriminator and RRC in one launch
per slice) against a twin created with QRL_FSK_FRONTEND=0, which runs the same arithmetic as three launches through the stage-1 and
channel-filter rings.  Every port and every count of every call must match bit for bit, spot channels must match the oracle, and the
profiler must show the fused path: one stage-1 slot launch per slice, none in the channel-filter and demodulator slots.

Inputs are host arrays except on the caller-stream case, so the file also runs on the host-thread build of the library
(QRL_EMULATED_LIB, tools/emu)."""
import os

import numpy as np
import pytest

from tests.test_gpu_dispatch import RX, bases, check_rx, concat_calls, free_device, make_slab, ragged, spot_shifts, stage_launches
from tests.test_gpu_rx_reset import _sc16, assert_same_calls

pytestmark = pytest.mark.gpu

EMULATED = bool(os.environ.get("QRL_EMULATED_LIB"))
NAME = "4fsk"
T = RX[NAME][3]
OFFSET_HZ, RETUNE_HZ = 40.0, -35.0


def n_slices(T_call, overlap):
    """slices of one call (rx_work_impl): 2 when overlapped, else 12, fewer for a call under 32768 samples per slice"""
    nsub = 2 if overlap else 12
    return nsub if T_call >= 32768 * nsub else max(1, T_call // 32768)


def twins(qrl, monkeypatch, Cn, maxs):
    """(fused handle, QRL_FSK_FRONTEND=0 twin), both profiling"""
    monkeypatch.delenv("QRL_FSK_FRONTEND", raising=False)
    a = RX[NAME][0](qrl, Cn, maxs)
    monkeypatch.setenv("QRL_FSK_FRONTEND", "0")
    try:
        b = RX[NAME][0](qrl, Cn, maxs)
    except BaseException:
        a.close()
        raise
    finally:
        monkeypatch.delenv("QRL_FSK_FRONTEND")
    for h in (a, b):
        assert h._L.qrl_rx_profile(h._h, 1) == 0
    return a, b


def assert_fused(a, b, slices):
    assert [stage_launches(a, s) for s in range(3)] == [slices, 0, 0]
    assert stage_launches(b, 1) == slices and stage_launches(b, 2) == slices


def feed(blk, calls, overlap_at=None):
    """calls: list of (callable(blk), events) -- events (channel or -1, Hz) applied before the call; overlap_at: {call index: on}.
    Returns the ports (and port counts) read after every call"""
    out = []
    for k, (work, events) in enumerate(calls):
        if overlap_at and k in overlap_at:
            blk.set_overlap(overlap_at[k])
        for ch, hz in events:
            blk.set_carrier_offset(hz, channel=ch)
        work(blk)
        out.append([blk.read_port(p) for p in range(blk.nports)] + [blk.read_port_counts(p)[:, None] for p in (1, 2)])
    return out


def slab_calls(X, cuts, events=()):
    ev = {}
    for k, ch, hz in events:
        ev.setdefault(k, []).append((ch, hz))
    return [((lambda blk, lo=lo, hi=hi: blk.work(X[:, lo:hi])), ev.get(k, [])) for k, (lo, hi) in enumerate(cuts)]


def offsets(Cn):
    """every channel offset before the first call, the last channel retuned before the third"""
    return [(0, -1, OFFSET_HZ), (2, Cn - 1, RETUNE_HZ)]


@pytest.mark.parametrize("Cn", [1, 33, 64, 97])
def test_fused_front_end_channel_counts(qrl, oracle, monkeypatch, Cn):
    """serialised ragged calls (one of 101 samples, lengths not a multiple of 2 D), a carrier offset and a mid-stream retune"""
    spots = spot_shifts(Cn) if Cn > 1 else {}
    B, payloads = bases(NAME, oracle, T)
    X = make_slab(B, Cn, spots)
    cuts = [(0, T // 4 + 7), (T // 4 + 7, T // 2 + 13), (T // 2 + 13, T // 2 + 114), (T // 2 + 114, T)]
    ev = offsets(Cn)
    a, b = twins(qrl, monkeypatch, Cn, max(hi - lo for lo, hi in cuts))
    try:
        got, want = feed(a, slab_calls(X, cuts, ev)), feed(b, slab_calls(X, cuts, ev))
        assert_same_calls(got, want, ("channels", Cn))
        assert_fused(a, b, sum(n_slices(hi - lo, False) for lo, hi in cuts))
        check_rx(NAME, oracle, B, payloads, concat_calls([g[:3] for g in got], 3, Cn), spots, cuts, ev)
    finally:
        a.close(); b.close()
        del X
        free_device()


def test_fused_front_end_overlap_switched(qrl, oracle, monkeypatch):
    """overlapped calls switched on, off and on between calls, calls of changing length (one shorter than a strip, one of 101
    samples), the offset retuned mid-stream"""
    Cn = 3
    B, payloads = bases(NAME, oracle, T)
    X = make_slab(B, Cn, {})
    cuts = [(0, 40000), (40000, 90001), (90001, 150000), (150000, 210000), (210000, 270000), (270000, 330000), (330000, 330101),
            (330101, 400000), (400000, 460000), (460000, T)]
    switches = {2: True, 5: False, 7: True}
    ev = [(0, -1, OFFSET_HZ), (4, 1, RETUNE_HZ)]
    a, b = twins(qrl, monkeypatch, Cn, max(hi - lo for lo, hi in cuts))
    try:
        got, want = feed(a, slab_calls(X, cuts, ev), switches), feed(b, slab_calls(X, cuts, ev), switches)
        assert_same_calls(got, want, "overlap switched")
        on, slices = False, 0
        for k, (lo, hi) in enumerate(cuts):
            on = switches.get(k, on)
            slices += n_slices(hi - lo, on)
        assert_fused(a, b, slices)
        check_rx(NAME, oracle, B, payloads, concat_calls([g[:3] for g in got], 3, Cn), {}, cuts, ev)
    finally:
        a.close(); b.close()


def test_fused_front_end_rotator_pass(qrl, oracle, monkeypatch):
    """QRL_ROTATOR_PASS: the offset turns in its own pass over the input, the fused kernel reads the rotated copy"""
    Cn = 3
    B, payloads = bases(NAME, oracle, T)
    X = make_slab(B, Cn, {})
    cuts = ragged(T)
    ev = offsets(Cn)
    a, b = twins(qrl, monkeypatch, Cn, max(hi - lo for lo, hi in cuts))
    monkeypatch.setenv("QRL_ROTATOR_PASS", "1")
    try:
        got, want = feed(a, slab_calls(X, cuts, ev)), feed(b, slab_calls(X, cuts, ev))
        assert_same_calls(got, want, "rotator pass")
        assert_fused(a, b, sum(n_slices(hi - lo, False) for lo, hi in cuts))
        check_rx(NAME, oracle, B, payloads, concat_calls([g[:3] for g in got], 3, Cn), {}, cuts, ev)
    finally:
        a.close(); b.close()


def test_fused_front_end_input_formats(qrl, oracle, monkeypatch):
    """stride 0 (one stream for every channel) as gr_complex, sc16 and sc8, then per-channel host sc16 and sc8, every channel with
    its own offset"""
    Cn = 3
    B, _ = bases(NAME, oracle, T)
    x = np.ascontiguousarray(B[0])
    X = make_slab(B, Cn, {})
    s1, S = _sc16(x), np.stack([_sc16(X[c]) for c in range(Cn)])
    s8, S8 = (s1 // 256).astype(np.int8), (S // 256).astype(np.int8)
    q = T // 5
    calls = [(lambda blk: blk.work_shared(x[:q + 13]), [(-1, OFFSET_HZ), (1, RETUNE_HZ)]),
             (lambda blk: blk.work_shared_sc16(s1[q + 13:2 * q]), []),
             (lambda blk: blk.work_shared_sc8(s8[2 * q:3 * q + 101]), []),
             (lambda blk: blk.work_sc16(S[:, 3 * q + 101:4 * q]), [(2, RETUNE_HZ)]),
             (lambda blk: blk.work_sc8(S8[:, 4 * q:T]), [])]
    lens = [q + 13, q - 13, q + 101, q - 101, T - 4 * q]
    a, b = twins(qrl, monkeypatch, Cn, max(lens))
    try:
        got, want = feed(a, calls), feed(b, calls)
        assert_same_calls(got, want, "input formats")
        assert_fused(a, b, sum(n_slices(n, False) for n in lens))
        assert all(len(got[k][0][c]) > 0 for k in range(len(calls)) for c in range(Cn))
    finally:
        a.close(); b.close()


def test_fused_front_end_rssi_and_reset(qrl, oracle, monkeypatch):
    """the RSSI tap on port 0, and qrl_rx_reset mid-stream: every call and every RSSI value bit for bit"""
    Cn = 3
    B, _ = bases(NAME, oracle, T)
    X = make_slab(B, Cn, {})
    cuts = [(0, 60013), (60013, 200000), (0, 50000), (50000, 170101)]
    a, b = twins(qrl, monkeypatch, Cn, 200000)
    try:
        slices = 0
        for k, (lo, hi) in enumerate(cuts):
            if k == 0:
                a.enable_rssi(True); b.enable_rssi(True)
                a.set_carrier_offset(OFFSET_HZ); b.set_carrier_offset(OFFSET_HZ)
            if k == 2:
                a.reset(); b.reset()
            a.work(X[:, lo:hi]); b.work(X[:, lo:hi])
            slices += n_slices(hi - lo, False)
            assert_same_calls([[a.read_port(p) for p in range(3)]], [[b.read_port(p) for p in range(3)]], ("rssi / reset", k))
            ra, rb = a.rssi(level=-3.5), b.rssi(level=-3.5)
            assert np.array_equal(ra.view(np.uint32), rb.view(np.uint32)), (k, ra, rb)
        assert_fused(a, b, slices)
    finally:
        a.close(); b.close()


# a strip of fsk_fm_frontend_kernel: 2 chunks of 2048 stage-1 outputs less the halo of the 4FSK-2k filters (250 RRC taps of history,
# one discriminator sample, 59 channel-filter taps of history)
STRIP = 2 * 2048 - 310


def slice_outputs(cuts, nsub):
    """stage-1 outputs of every slice of every call (rx_work_impl's cuts: multiples of 2 D inside a call, outputs k with D k below
    the slice's last input)"""
    out, n_in, k = [], 0, 0
    for lo, hi in cuts:
        L = hi - lo
        ns = nsub if L >= 32768 * nsub else max(1, L // 32768)
        for j in range(ns):
            t1 = L if j + 1 >= ns else (L * (j + 1) // ns) // 100 * 100
            k1 = (n_in + t1 + 49) // 50
            out.append(k1 - k)
            k = k1
        n_in += L
    return out


@pytest.mark.parametrize("overlap", [False, True])
def test_fused_front_end_multi_strip_slices(qrl, oracle, monkeypatch, overlap):
    """slices of several strips, so that every strip after the first recomputes its halo from the input (rotated with the offset in
    force): serialised calls of one slice (QRL_NSUB=1) or overlapped calls of two, a ragged partial last strip, a carrier offset and
    a retune of one channel, then the same through stride-0 calls of the one stream"""
    Cn, TL = 33, 1 << 20
    spots = spot_shifts(Cn)
    B, payloads = bases(NAME, oracle, TL)
    X = make_slab(B, Cn, spots)
    if overlap:
        cuts, nsub, switches = [(0, 500013), (500013, 500114), (500114, TL)], 2, {0: True}
    else:
        cuts, nsub, switches = [(0, 450013), (450013, 450114), (450114, TL)], 1, None
        monkeypatch.setenv("QRL_NSUB", "1")
    per_slice = slice_outputs(cuts, nsub)
    assert sum(n > STRIP for n in per_slice) >= 2, per_slice
    ev = [(0, -1, OFFSET_HZ), (2, Cn - 1, RETUNE_HZ)]
    maxs = max(hi - lo for lo, hi in cuts)
    a, b = twins(qrl, monkeypatch, Cn, maxs)
    try:
        got, want = feed(a, slab_calls(X, cuts, ev), switches), feed(b, slab_calls(X, cuts, ev), switches)
        assert_same_calls(got, want, ("multi-strip", overlap))
        assert_fused(a, b, len(per_slice))
        check_rx(NAME, oracle, B, payloads, concat_calls([g[:3] for g in got], 3, Cn), spots, cuts, ev)
    finally:
        a.close(); b.close()
        del X
        free_device()
    x = np.ascontiguousarray(B[3])
    a, b = twins(qrl, monkeypatch, Cn, maxs)
    try:
        calls = [((lambda blk, lo=lo, hi=hi: blk.work_shared(x[lo:hi])), [(ch, hz) for (k2, ch, hz) in ev if k2 == k])
                 for k, (lo, hi) in enumerate(cuts)]
        got, want = feed(a, calls, switches), feed(b, calls, switches)
        assert_same_calls(got, want, ("multi-strip, stride 0", overlap))
        assert_fused(a, b, len(per_slice))
    finally:
        a.close(); b.close()


@pytest.mark.skipif(EMULATED, reason="needs a real CUDA device (a torch stream)")
def test_fused_front_end_on_a_caller_stream(qrl, oracle, monkeypatch):
    """the fused handle on the caller's stream (qrl_rx_set_stream), overlapped calls read every second call, device input"""
    import torch
    Cn = 33
    spots = spot_shifts(Cn)
    B, payloads = bases(NAME, oracle, T)
    X = torch.from_numpy(make_slab(B, Cn, spots)).cuda()
    cuts = [(0, T // 3), (T // 3, 2 * (T // 3)), (2 * (T // 3), T)]
    s = torch.cuda.Stream()
    a, b = twins(qrl, monkeypatch, Cn, T // 3 + 2)
    try:
        a.set_stream(s.cuda_stream)
        calls = [((lambda blk, lo=lo, hi=hi: blk.work_device(X[:, lo:].data_ptr(), hi - lo, X.shape[1])), []) for lo, hi in cuts]
        got, want = feed(a, calls, {0: True}), feed(b, calls, {0: True})
        assert_same_calls(got, want, "caller stream")
        assert_fused(a, b, sum(n_slices(hi - lo, True) for lo, hi in cuts))
        check_rx(NAME, oracle, B, payloads, concat_calls([g[:3] for g in got], 3, Cn), spots, cuts)
    finally:
        a.close(); b.close()
        s.synchronize()
        del X
        free_device()
