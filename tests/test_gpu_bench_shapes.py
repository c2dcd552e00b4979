"""GPU tier: every configuration bench.py times, at its own shape and call pattern, against a serialised twin, the class
representatives and the oracle.

bench.py's numbers come from calls at sizes no other test reaches: 2^22-sample overlapped 4FSK calls (12 strips per fused front-end
slice), 1024-channel handles whose input alone is 2^32 complex samples, 4096-channel QPSK, three handles running at once on their own
streams, 2^27-sample channelizer calls.  Each case here builds its handle as the bench does (same factory and arguments, n_channels
and max_samples = the bench's C and T, the handle on a non-null caller's stream, overlap where the bench sets it, device input) and
runs K calls of it, each on different samples: one slab of [C][S], S = T + (K - 1) DELTA, call k reading columns [k DELTA, k DELTA + T)
at stride S, so a stage that read state one call stale would see different data.  What a channel receives is the concatenation of
its K windows, and that is what the oracle is fed.

Slabs repeat P = 7 base signals with rolled spot channels at the group edges (tests/test_gpu_dispatch.py): every channel equals its
class representative bit for bit (compared on the device, in the handle's own port buffers), and the representatives and spot
channels equal the oracle under check_rx's tail rule.  Overlapped cases run three passes as run_case does (read after every call,
every second call, only after the last): every port read equals a serialised twin's port for that call.  Each case asserts the path
it names: fused front-end launches per slice, the SM partition, QPSK's many mode.

A case that does not fit the free device memory skips with the numbers.  The full-size cases need the device; one reduced instance
of the receive harness (host input) also runs on the host-thread build of the library (QRL_EMULATED_LIB, tools/emu)."""
import ctypes as C
import os
import threading
import time
from contextlib import contextmanager

import numpy as np
import pytest

import bench
from tests.test_gpu_dispatch import (P, RX, SLACK, assert_partition, bases, default_partition, free_device, host_channel,
                                     representatives, spot_shifts, stage_launches, tx_channel)
from tests.test_gpu_fsk_frontend import STRIP, assert_fused, slice_outputs
from tests.test_gpu_spectrum import check

pytestmark = pytest.mark.gpu

EMULATED = bool(os.environ.get("QRL_EMULATED_LIB"))
full_size = pytest.mark.skipif(EMULATED, reason="full size: device input (torch tensors) and hours of host threads")

DELTA = 30002           # columns between calls: even (16-byte aligned rows), not a multiple of the symbol, frame or slice period
GB = float(1 << 30)

# ------------------------------------------------------------------ the shapes, each row citing the bench.py code it mirrors
# receive chains: factory arguments (bench.py) and the oracle's
CHAINS = {
    "4fsk": (lambda q, n, m: q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1)),           # run_ours, cfg2 sweep, mixed_config_block
    "qpsk": (lambda q, n, m: q.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_QPSK, 2, 1000000, 1700, 160000, 0)),         # cfg3 in run_ours, mixed_config_block
    "nbfm": (lambda q, n, m: q.make_gr_demod_nbfm(125, 1000000, 1700, 2500, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_NBFM, 125, 1000000, 1700, 2500, 0)),         # cfg1 in run_ours, mixed_config_block
}
#         id                   chain   C                T              K  overlapped  bench.py
RX_SHAPES = [
    ("headline",              "4fsk", bench.CHANNELS, bench.T_CALL,   6, True),     # run_ours: blk, set_overlap(True), work_device
    ("cfg2_sweep_256",        "4fsk", 256,            bench.T_CALL,   6, True),     # run_ours: cfg2_channel_sweep, Cs = 256
    ("cfg2_sweep_1024",       "4fsk", 1024,           bench.T_CALL,   6, True),     # run_ours: cfg2_channel_sweep, Cs = 1024
    ("cfg3_qpsk_256",         "qpsk", 256,            1 << 20,        4, False),    # run_ours: cfg3_qpsk250k_256ch (rx_config_block)
    ("cfg3_qpsk_sweep_1024",  "qpsk", 1024,           1 << 18,        4, False),    # run_ours: cfg3 channel_sweep, Cq = 1024
    ("cfg3_qpsk_sweep_4096",  "qpsk", 4096,           1 << 18,        4, False),    # run_ours: cfg3 channel_sweep, Cq = 4096
    ("cfg1_nbfm_1ch",         "nbfm", 1,              1 << 22,        6, False),    # run_ours: cfg1_nbfm_1ch (rx_config_block)
    ("cfg1_nbfm_64ch",        "nbfm", 64,             1 << 22,        6, False),    # run_ours: cfg1_nbfm_64ch (rx_config_block)
]
MIXED = ("4fsk", "qpsk", "nbfm"), 128, 1 << 21, 6       # mixed_config_block: 128 channels, c % 3 -> mode, T = 2^21, one rank
TX_SHAPE = 64, 1024, 4, 100                              # tx_config_block: C, bytes per call; K calls, DELTA in bytes
PFB_SHAPE = 10, 341, 1 << 27, 3                          # pfb_config_block: M, taps, wideband samples per call; K
MMDVM_SHAPE = 7, 5000, 1 << 26, 3                        # mmdvm_config_block: MmdvmDemod(7, 5000), samples per call; K
SPECTRUM_SHAPE = 64, 32768, 6, 4098                      # spectrum_config_block: streams, points; K calls, DELTA
REDUCED = ("reduced_33ch", "4fsk", 33, 1 << 17, 4, True)    # the receive harness on a size the host-thread build runs

INT_TORCH = {8: "int64", 4: "int32", 2: "int16", 1: "uint8"}
PORT_NP = {8: np.complex64, 4: np.float32, 2: np.int16, 1: np.uint8}
ROWS = 128              # channels per device comparison (bounds the temporaries)


# ------------------------------------------------------------------ device memory, threads
class Peak:
    """lowest free device memory seen during a case (the library allocates with cudaMalloc, outside torch's accounting)"""

    def __init__(self, name, host):
        self.name, self.host, self.t0 = name, host, time.perf_counter()
        self.low = None
        self.sample()

    def free(self):
        import torch
        return torch.cuda.mem_get_info()

    def sample(self):
        if not self.host:
            f, total = self.free()
            self.total = total
            self.low = f if self.low is None else min(self.low, f)

    def need(self, nbytes, what):
        """skip unless `nbytes` more fit on the device"""
        if self.host:
            return
        f, total = self.free()
        if f < nbytes:
            pytest.skip("%s: %s needs %.1f GB, %.1f GB of %.1f GB free" % (self.name, what, nbytes / GB, f / GB, total / GB))

    def report(self):
        if not self.host:
            print("\n[bench shape %s] peak device memory in use %.1f GB of %.1f GB, %.0f s"
                  % (self.name, (self.total - self.low) / GB, self.total / GB, time.perf_counter() - self.t0))


def parallel(fn, items):
    """fn(item) on one thread each (the oracle's ctypes calls release the GIL); re-raises the first failure"""
    errs = []

    def run(it):
        try:
            fn(it)
        except BaseException as e:          # noqa: BLE001
            errs.append(e)
    th = [threading.Thread(target=run, args=(it,)) for it in items]
    [t.start() for t in th]
    [t.join() for t in th]
    if errs:
        raise errs[0]


class Background:
    """fn(item) for every item on threads that run while the caller drives the GPU; join() returns {item: result}"""

    def __init__(self, fn, items):
        self.out, self.err = {}, []

        def run():
            try:
                parallel(lambda it: self.out.__setitem__(it, fn(it)), items)
            except BaseException as e:      # noqa: BLE001
                self.err.append(e)
        self.th = threading.Thread(target=run)
        self.th.start()

    def join(self):
        self.th.join()
        if self.err:
            raise self.err[0]
        return self.out


@contextmanager
def caller_stream(host):
    """a non-null torch stream, current while the case runs (as run_ours sets it)"""
    if host:
        yield None
        return
    import torch
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        yield s
    s.synchronize()


# ------------------------------------------------------------------ slabs
def window_slab(B, Cn, spots):
    """[Cn][S] complex64 on the device in test_gpu_dispatch.device_slab's layout (class rows, rolled spot channels), gathered ROWS
    channels at a time so that the slab is the only full-size allocation"""
    import torch
    S = B.shape[1]
    Bd = torch.from_numpy(np.ascontiguousarray(B)).cuda()
    X = torch.empty((Cn, S), dtype=torch.complex64, device="cuda")
    for lo in range(0, Cn, ROWS):
        hi = min(Cn, lo + ROWS)
        X[lo:hi] = Bd.index_select(0, torch.arange(lo, hi, device="cuda") % P)
    for c, s in spots.items():
        X[c] = torch.roll(Bd[c % P], s)
    del Bd
    return X


def windows(x, T, K, delta=DELTA):
    return [x[k * delta: k * delta + T] for k in range(K)]


# ------------------------------------------------------------------ ports, read where they are
class _DevArray:
    def __init__(self, ptr, shape, isz):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": np.dtype(INT_TORCH[isz]).str, "data": (ptr, False),
                                         "version": 2, "strides": None}


def port_views(blk, host=False):
    """per port (V, n, itemsize): V [C][cap] the port's buffer as integers (a view of the handle's device buffer, or a host copy on
    the host-thread build), n the per-channel counts.  Valid until the handle's next work() call."""
    import torch
    out = []
    for p in range(blk.nports):
        isz = blk._itemsize[p]
        n = blk.read_port_counts(p).astype(np.int64)            # waits for the call (and joins an overlapped tail)
        ptr, cap, cnt = C.c_void_p(), C.c_long(), C.c_void_p()
        assert blk._L.qrl_rx_port_device(blk._h, p, C.byref(ptr), C.byref(cap), C.byref(cnt)) == 0
        if host:
            buf = np.zeros((blk.n_channels, cap.value), INT_TORCH[isz])
            counts = np.zeros(blk.n_channels, np.int32)
            assert blk._L.qrl_rx_read_port(blk._h, p, buf.ctypes.data_as(C.c_void_p), cap.value,
                                           counts.ctypes.data_as(C.c_void_p), 0) == 0
            assert np.array_equal(counts, n)
            V = torch.from_numpy(buf)
        else:
            V = torch.as_tensor(_DevArray(ptr.value, (blk.n_channels, cap.value), isz), device="cuda")
        out.append((V, n, isz))
    return out


def assert_same_ports(a, b, where):
    """every port of every channel bit for bit, counts included"""
    import torch
    for p, ((Va, na, _), (Vb, nb, _)) in enumerate(zip(a, b)):
        assert np.array_equal(na, nb), (where, p, "counts")
        w = int(na.max(initial=0))
        if w == 0:
            continue
        cols = torch.arange(w, device=Va.device)[None, :]
        for lo in range(0, len(na), ROWS):
            hi = min(len(na), lo + ROWS)
            pad = cols >= torch.from_numpy(na[lo:hi]).to(Va.device)[:, None]
            assert bool(((Va[lo:hi, :w] == Vb[lo:hi, :w]) | pad).all()), (where, p, "channels %d..%d" % (lo, hi - 1))


def assert_classes(ports, reps, spots, where):
    """every plain channel's port equals its class representative's, bit for bit"""
    import torch
    for p, (V, n, _) in enumerate(ports):
        for k, r in reps.items():
            idx = [c for c in range(len(n)) if c % P == k and c not in spots]
            assert np.all(n[idx] == n[r]), (where, p, k, "counts")
            m = int(n[r])
            if m == 0:
                continue
            ii = torch.tensor(idx, device=V.device)
            for lo in range(0, len(idx), ROWS):
                assert bool((V.index_select(0, ii[lo:lo + ROWS])[:, :m] == V[r, :m]).all()), (where, p, "class of channel %d" % r)


def host_rows(ports, chans):
    """{channel: [port arrays]} for the representatives and spot channels"""
    return {c: [V[c, :int(n[c])].cpu().numpy().view(PORT_NP[isz]) for (V, n, isz) in ports] for c in chans}


# ------------------------------------------------------------------ the oracle on the concatenated windows
_ORACLE = {}


def oracle_rx(chain, O, B, spots, T, K):
    """fn(channel) -> the oracle's ports for that channel's K windows, cached per (chain, class or spot roll, windows)"""
    def one(c):
        key = (chain, B.shape[1], c % P, spots.get(c), T, K)
        if key not in _ORACLE:
            rx = CHAINS[chain][1](O)
            for w in windows(host_channel(B, spots, c), T, K):
                rx.work(w)
            _ORACLE[key] = [rx.port(p) for p in range(RX[chain][2])]
        return _ORACLE[key]
    return one


def assert_oracle(chain, got, want, length, where):
    """check_rx's tail rule: lengths within SLACK, at least the chain's minimum for this stream length, equal up to the shorter"""
    mins = [m * length // RX[chain][3] for m in RX[chain][4]]
    for p, (g, w) in enumerate(zip(got, want)):
        n = min(len(g), len(w))
        assert abs(len(g) - len(w)) <= SLACK and n >= mins[p], (where, p, len(g), len(w), mins[p])
        assert np.array_equal(g[:n], w[:n]), "%s: port %d differs from the oracle" % (where, p)


# ------------------------------------------------------------------ the receive harness
class RxShape:
    def __init__(self, qrl, O, tag, chain, Cn, T, K, overlap, host=False):
        self.qrl, self.O, self.tag, self.chain, self.Cn, self.T, self.K, self.overlap, self.host = \
            qrl, O, tag, chain, Cn, T, K, overlap, host
        self.S = T + (K - 1) * DELTA
        self.B = bases(chain, O, self.S)[0]
        self.spots = spot_shifts(Cn)
        self.reps = representatives(Cn, self.spots)
        self.chans = sorted(set(self.reps.values()) | set(self.spots))
        self.X = None

    def make(self, stream, overlap, profile=False, env=None, monkeypatch=None):
        if env:
            for k, v in env.items():
                monkeypatch.setenv(k, v)
        try:
            blk = CHAINS[self.chain][0](self.qrl, self.Cn, self.T)
        finally:
            if env:
                for k in env:
                    monkeypatch.delenv(k)
        if stream is not None:
            blk.set_stream(stream.cuda_stream)
        if overlap:
            blk.set_overlap(True)
        if profile:
            assert blk._L.qrl_rx_profile(blk._h, 1) == 0
        return blk

    def feed(self, blk, k, X=None):
        X = self.X if X is None else X
        if self.host:
            blk.work(X[:, k * DELTA: k * DELTA + self.T])
        else:
            blk.work_device(X[:, k * DELTA:].data_ptr(), self.T, self.S)

    def slab(self):
        if self.host:
            return np.stack([host_channel(self.B, self.spots, c) for c in range(self.Cn)])
        return window_slab(self.B, self.Cn, self.spots)


def lockstep(blk, twin, feed_blk, feed_twin, K, read_every, host, on_read=None, where=""):
    """blk's K calls issued back to back, read after every `read_every`-th and the last; at each read the serialised twin catches up
    call by call and every port of every channel must equal the twin's for that call"""
    t = 0
    for k in range(K):
        feed_blk(blk, k)
        if (k + 1) % read_every and k != K - 1:
            continue
        got = port_views(blk, host)
        while t <= k:
            feed_twin(twin, t)
            t += 1
        assert_same_ports(got, port_views(twin, host), (where, read_every, k))
        if on_read:
            on_read(k, got)


def run_rx_shape(qrl, O, shape, monkeypatch, host=False):
    tag, chain, Cn, T, K, overlap = shape
    sh = RxShape(qrl, O, tag, chain, Cn, T, K, overlap, host)
    peak = Peak(tag, host)
    rows = {c: [[] for _ in range(RX[chain][2])] for c in sh.chans}

    def keep(k, ports):
        assert_classes(ports, sh.reps, sh.spots, (tag, k))
        for c, arrs in host_rows(ports, sh.chans).items():
            for p, a in enumerate(arrs):
                rows[c][p].append(a)

    with caller_stream(host) as s:
        blk = None
        try:
            # the bench's handle first: what it takes sizes the twin; the slab, both handles and the port temporaries must fit
            free0 = None if host else peak.free()[0]
            blk = sh.make(s, overlap, profile=chain == "4fsk")
            if not host:
                handle = free0 - peak.free()[0]
                peak.need(Cn * sh.S * 8 + (handle if overlap else 0) + (1 << 30), "slab %.1f GB + %s%.1f GB handle"
                          % (Cn * sh.S * 8 / GB, "twin of the " if overlap else "", handle / GB))
            sh.X = sh.slab()
            peak.sample()
            oracle = Background(oracle_rx(chain, O, sh.B, sh.spots, T, K), sh.chans)      # runs while the GPU works
            assert_partition(qrl, blk, default_partition(chain, Cn))
            if chain == "qpsk":
                assert_qpsk_many_mode(qrl, Cn, monkeypatch)
            if overlap:
                for read_every in (1, 2, K):
                    if read_every != 1:
                        blk = sh.make(s, True)
                    twin = sh.make(s, False)
                    try:
                        peak.sample()
                        lockstep(blk, twin, sh.feed, sh.feed, K, read_every, host, keep if read_every == 1 else
                                 (lambda k, ports: assert_classes(ports, sh.reps, sh.spots, (tag, k))), tag)
                    finally:
                        twin.close()
                    if read_every == 1 and chain == "4fsk":
                        per_slice = slice_outputs([(0, T)] * K, 2)
                        assert [stage_launches(blk, st) for st in range(3)] == [len(per_slice), 0, 0]
                        if T == bench.T_CALL:           # 2^21 inputs per slice: 12 strips of the fused front end
                            assert min(-(-n // STRIP) for n in per_slice) >= 12, per_slice
                    blk.close()
                    blk = None
            else:
                for k in range(K):
                    sh.feed(blk, k)
                    keep(k, port_views(blk, host))
            free_device()
            want = oracle.join()
            for c in sh.chans:
                got = [np.concatenate(rows[c][p]) for p in range(RX[chain][2])]
                assert_oracle(chain, got, want[c], K * T, (tag, "channel", c))
        finally:
            if blk is not None:
                blk.close()
            sh.X = None
            free_device()
    peak.report()
    return sh


def assert_qpsk_many_mode(qrl, Cn, monkeypatch):
    """QPSK takes no SM partition in either mode; with QRL_QPSK_PARTITION=1 it asks for one, and only many mode (2 ceil(C / 32) loop
    CTAs > 44, C > 704) refuses it: a small probe handle of the same channel count shows which mode C selects"""
    monkeypatch.setenv("QRL_QPSK_PARTITION", "1")
    try:
        probe = CHAINS["qpsk"][0](qrl, Cn, 4096)
    finally:
        monkeypatch.delenv("QRL_QPSK_PARTITION")
    try:
        assert_partition(qrl, probe, not Cn > 704)
    finally:
        probe.close()


# ------------------------------------------------------------------ 1-4. the receive configurations
@full_size
@pytest.mark.parametrize("shape", RX_SHAPES[1:], ids=[s[0] for s in RX_SHAPES[1:]])
def test_rx_bench_shape(qrl, oracle, monkeypatch, shape):
    run_rx_shape(qrl, oracle, shape, monkeypatch)


def test_rx_harness_reduced(qrl, oracle, monkeypatch):
    """the harness at 33 channels x 2^17, K = 4, overlapped, host input: the windows, classes, twin passes and the oracle bookkeeping
    on a size the host-thread build of the library runs"""
    run_rx_shape(qrl, oracle, REDUCED, monkeypatch, host=True)


@full_size
def test_headline(qrl, oracle, monkeypatch):
    """run_ours: 64 ch x 2^22 overlapped calls back to back on the caller's stream (three passes against the serialised twin, the
    classes, the oracle), then the fused front end against a QRL_FSK_FRONTEND=0 twin, then the e2e calls: pinned-host gr_complex,
    sc16 and sc8 read after every call against device-input twins fed the same (host-converted) values"""
    import torch
    shape = RX_SHAPES[0]
    sh = run_rx_shape(qrl, oracle, shape, monkeypatch)
    tag, _, Cn, T, K, _ = shape
    peak = Peak(tag + " front end / e2e", False)
    L = qrl.load_library()
    cuts = [(0, T)] * K
    with caller_stream(False) as s:
        sh.X = sh.slab()
        a = b = None
        try:
            a = sh.make(s, True, profile=True)
            b = sh.make(s, True, profile=True, env={"QRL_FSK_FRONTEND": "0"}, monkeypatch=monkeypatch)
            lockstep(a, b, sh.feed, sh.feed, K, 1, False, where="QRL_FSK_FRONTEND=0")
            assert_fused(a, b, len(slice_outputs(cuts, 2)))
            b.close()
            b = None
            peak.sample()

            def host_call(fn, Xh, scale=None):
                def feed(blk, k):
                    args = (blk._h, C.c_void_p(Xh[:, k * DELTA:].data_ptr()), T, sh.S) + ((C.c_float(scale),) if scale else ()) + (0,)
                    assert fn(*args) == 0
                return feed

            # gr_complex from pinned host memory, the bench's e2e leg
            Xh = torch.empty(sh.X.shape, dtype=torch.complex64, pin_memory=True)
            Xh.copy_(sh.X)
            for fmt, mul, lo, hi, dt, scale, fn in (("gr_complex", None, 0, 0, None, None, L.qrl_rx_work),
                                                   ("sc16", 20000.0, -32768, 32767, torch.int16, 1.0 / 32767.0, L.qrl_rx_work_sc16),
                                                   ("sc8", 100.0, -128, 127, torch.int8, 1.0 / 128.0, L.qrl_rx_work_sc8)):
                if mul is None:
                    Xin, Xf = Xh, sh.X
                else:                           # the bench's conversion; the twin gets float32(v) * float32(scale), made here
                    Xq = torch.view_as_real(sh.X).mul(mul).round_().clamp_(lo, hi).to(dt)
                    Xin = torch.empty(Xq.shape, dtype=dt, pin_memory=True)
                    Xin.copy_(Xq)
                    Xf = torch.view_as_complex((Xq.to(torch.float32) * torch.tensor(scale, dtype=torch.float32, device="cuda")).contiguous())
                    del Xq
                e2e = sh.make(s, True)
                twin = sh.make(s, False)
                try:
                    peak.sample()
                    lockstep(e2e, twin, host_call(fn, Xin, scale), lambda blk, k: sh.feed(blk, k, Xf), K, 1, False, where=fmt)
                finally:
                    e2e.close(); twin.close()
                del Xin, Xf
        finally:
            for h in (a, b):
                if h is not None:
                    h.close()
            sh.X = None
            free_device()
    peak.report()


# ------------------------------------------------------------------ 5. mixed: three handles at once
@full_size
def test_mixed_concurrent_handles(qrl, oracle, monkeypatch):
    """mixed_config_block: the three handles of sharding.shard_channels for 128 channels, each on its own stream; every step issues
    all three calls before reading any of them"""
    import torch
    from qradiolink_b200 import sharding
    order, total, T, K = MIXED
    modes = [order[c % 3] for c in range(total)]
    mine = sharding.shard_channels(modes, 1, 0)
    peak = Peak("cfg4_mixed", False)
    shapes, blocks, streams, rows, oracles = {}, {}, {}, {}, {}
    try:
        for m, chans in mine.items():
            sh = shapes[m] = RxShape(qrl, oracle, "mixed_" + m, m, len(chans), T, K, False)
            peak.need(sh.Cn * sh.S * 8 + (2 << 30), "the %s slab and handle" % m)
            oracles[m] = Background(oracle_rx(m, oracle, sh.B, sh.spots, T, K), sh.chans)
            streams[m] = torch.cuda.Stream()
            blocks[m] = sh.make(streams[m], False)
            sh.X = sh.slab()
            rows[m] = {c: [[] for _ in range(RX[m][2])] for c in sh.chans}
            assert_partition(qrl, blocks[m], default_partition(m, sh.Cn))
        torch.cuda.synchronize()
        peak.sample()
        for k in range(K):
            for m, blk in blocks.items():
                shapes[m].feed(blk, k)
            for m, blk in blocks.items():
                ports = port_views(blk)
                assert_classes(ports, shapes[m].reps, shapes[m].spots, (m, k))
                for c, arrs in host_rows(ports, shapes[m].chans).items():
                    for p, a in enumerate(arrs):
                        rows[m][c][p].append(a)
        for m, sh in shapes.items():
            want = oracles[m].join()
            for c in sh.chans:
                assert_oracle(m, [np.concatenate(r) for r in rows[m][c]], want[c], K * T, ("mixed", m, c))
    finally:
        for blk in blocks.values():
            blk.close()
        for sh in shapes.values():
            sh.X = None
        for st in streams.values():
            st.synchronize()
        free_device()
    peak.report()


# ------------------------------------------------------------------ 6. 4FSK TX
@full_size
def test_4fsk_tx(qrl, oracle):
    """tx_config_block: 64 ch x 1024 bytes per call (4 096 000 IQ samples per channel), K calls on different bytes: IQ bit-identical to
    oracle.Tx fed each class's bytes call by call, every channel equal to its representative"""
    import torch
    Cn, n, K, db = TX_SHAPE
    Sb = n + (K - 1) * db
    nout = n * 4000
    B = np.random.default_rng(5000).integers(0, 256, (P, Sb), dtype=np.uint8)
    spots = {c: 1 + c for c in spot_shifts(Cn)}
    reps = representatives(Cn, spots)
    chans = sorted(set(reps.values()) | set(spots))
    L = qrl.load_library()
    peak = Peak("cfg5_4fsk_tx", False)
    peak.need(Cn * nout * 8 * 2 + (2 << 30), "the IQ buffer and the handle")
    D = torch.from_numpy(np.stack([tx_channel(B, "bytes", spots, c) for c in range(Cn)])).cuda()
    orc = {c: oracle.Tx(oracle.MOD_4FSK, 25, 1000000, 1700, 3500, 1) for c in chans}
    with caller_stream(False) as s:
        tx = qrl.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=Cn, max_items=n)
        try:
            tx.set_stream(s.cuda_stream)
            out = torch.empty((Cn, nout), dtype=torch.complex64, device="cuda")
            n2 = C.c_long()
            for k in range(K):
                tx.work_device(D[:, k * db:].data_ptr(), n, Sb)
                tx.sync()
                assert L.qrl_tx_read(tx._h, C.c_void_p(out.data_ptr()), nout, C.byref(n2), 1) == 0 and n2.value == nout
                peak.sample()
                V = out.view(torch.int64)
                assert_classes([(V, np.full(Cn, nout, np.int64), 8)], reps, spots, ("tx", k))
                got = {c: out[c].cpu().numpy() for c in chans}

                def one(c, k=k, got=got):
                    w = orc[c].work(tx_channel(B, "bytes", spots, c)[k * db: k * db + n])
                    assert len(w) == nout and np.array_equal(got[c].view(np.uint32), w.view(np.uint32)), ("tx", k, c)
                parallel(one, chans)
        finally:
            tx.close()
            free_device()
    peak.report()


# ------------------------------------------------------------------ 7. the channelizer
@full_size
def test_pfb_channelizer_m10(qrl, oracle):
    """pfb_config_block: M = 10, the 341-tap prototype, 2^27 wideband samples per call, K calls: all 10 rows bit-identical to
    oracle.PfbChannelizer fed the same stream"""
    import torch
    M, n_t, N, K = PFB_SHAPE
    L = qrl.load_library()
    taps = np.zeros(n_t, np.float32)
    assert L.qrl_firdes_low_pass_2(1.0, 250000.0, 5000.0, 2000.0, 60.0, 5, taps.ctypes.data_as(C.c_void_p), n_t) == n_t
    S = N + (K - 1) * DELTA
    peak = Peak("pfb_channelizer_m10", False)
    peak.need(3 * S * 8 + (2 << 30), "the stream and the handle")
    g = torch.Generator(device="cuda")
    g.manual_seed(27)
    x = torch.view_as_complex(torch.randn((S, 2), device="cuda", generator=g) * 0.3)
    xh = x.cpu().numpy()
    o = oracle.PfbChannelizer(M, taps)
    with caller_stream(False) as s:
        ch = qrl.PfbChannelizer(M, taps, max_in=N)
        try:
            ch.set_stream(s.cuda_stream)
            for k in range(K):
                ch.work_device(x[k * DELTA:].data_ptr(), N)
                ch.sync()
                ptr, stride, items = ch.out_device()
                peak.sample()
                got = torch.as_tensor(_DevArray(ptr, (M, stride), 8), device="cuda")[:, :items].cpu().numpy()
                want = o.work(xh[k * DELTA: k * DELTA + N])
                assert want.shape == (M, items), (k, want.shape, items)
                assert np.array_equal(got, want.view(np.int64)), k
        finally:
            ch.close()
            del x
            free_device()
    peak.report()


# ------------------------------------------------------------------ 8. the MMDVM demodulator
@full_size
def test_mmdvm_demod_7ch(qrl, oracle):
    """mmdvm_config_block: MmdvmDemod(7, 5000) driven as its call() drives it (qrl_pfb_work on the device stream, the channel chains
    on the channelizer's output slab), 2^26 wideband samples per call: the int16 rows equal the oracle channelizer + MmdvmRx"""
    import torch
    from qradiolink_b200.mmdvm import _low_pass_2
    nch, fw, N, K = MMDVM_SHAPE
    S = N + (K - 1) * DELTA
    L = qrl.load_library()
    peak = Peak("mmdvm_demod_7ch", False)
    peak.need(S * 8 * 3 + (2 << 30), "the stream and the handles")
    g = torch.Generator(device="cuda")
    g.manual_seed(26)
    x = torch.view_as_complex(torch.randn((S, 2), device="cuda", generator=g) * 0.05)
    tt = torch.arange(S, device="cuda", dtype=torch.float64)
    for p in qrl.mmdvm_port_map(nch):
        f = p * 25000.0 if p < 5 else (p - 10) * 25000.0
        x += (0.1 * torch.polar(torch.ones(S, device="cuda", dtype=torch.float64), 2 * np.pi * ((f + 900.0) * tt / 250000.0 % 1.0))).to(torch.complex64)
    del tt
    xh = x.cpu().numpy()
    taps = _low_pass_2(L, 1, 250000, fw, 2000, 60)
    ports = qrl.mmdvm_port_map(nch)
    och, orx = oracle.PfbChannelizer(10, taps), [oracle.MmdvmRx(fw) for _ in range(nch)]
    got, want = [[] for _ in range(nch)], [[] for _ in range(nch)]
    with caller_stream(False) as s:
        dem = qrl.MmdvmDemod(nch, fw, max_in=N)
        try:
            dem.channelizer.set_stream(s.cuda_stream); dem.channels.set_stream(s.cuda_stream)
            cnt = C.c_long()
            for k in range(K):
                pf = dem.channelizer
                assert L.qrl_pfb_work(pf._h, C.c_void_p(x[k * DELTA:].data_ptr()), N, 0, 1, C.byref(cnt)) == 0
                ptr, stride, items = pf.out_device()
                m = dem.channels.work_device(ptr, items, stride)
                out = dem.channels._read(m)[0]
                peak.sample()
                chan = och.work(xh[k * DELTA: k * DELTA + N])

                def one(c, chan=chan, out=out):
                    got[c].append(out[c].copy())
                    want[c].append(orx[c].work(chan[ports[c]])[0])
                parallel(one, range(nch))
        finally:
            dem.close()
            del x
            free_device()
    for c in range(nch):
        g_, w_ = np.concatenate(got[c]), np.concatenate(want[c])
        m = min(len(g_), len(w_))
        assert m > K * N * 24 // 250 - 1000 and abs(len(g_) - len(w_)) <= 1, (c, len(g_), len(w_))
        assert np.array_equal(g_[:m], w_[:m]), c
    peak.report()


# ------------------------------------------------------------------ 9. the display spectrum
@full_size
def test_spectrum_32k_64streams(qrl, oracle):
    """spectrum_config_block: 64 streams at 32 768 points, N + 1 samples per call and a get after each, K calls on different samples:
    every stream within check() of the oracle, with the oracle's ready / not-ready sequence"""
    import torch
    Sn, N, K, d = SPECTRUM_SHAPE
    width = N + 1 + (K - 1) * d
    stride = width + (width & 1)
    rng = np.random.default_rng(32768)
    X = ((rng.standard_normal((Sn, stride)) + 1j * rng.standard_normal((Sn, stride))) * 0.2).astype(np.complex64)
    t = np.arange(stride)
    for i in range(Sn):
        X[i] += (0.3 * np.exp(2j * np.pi * (0.1234 + 0.003 * i) * t)).astype(np.complex64)
    L = qrl.load_library()
    peak = Peak("spectrum_32k_64streams", False)
    Xd = torch.from_numpy(X).cuda()
    orc = []
    for _ in range(Sn):
        o = oracle.Spectrum(N, oracle.WIN_BLACKMAN_HARRIS)
        o.set_enabled(True)
        orc.append(o)
    nfft = C.c_uint()
    ready = []
    with caller_stream(False) as s:
        sp = qrl.Spectrum(N, 5, n_streams=Sn, max_samples=2 * N)
        try:
            sp.set_stream(s.cuda_stream)
            sp.set_enabled(True)
            out = torch.empty((Sn, N), dtype=torch.float32, device="cuda")
            for k in range(K):
                sp.work_device(Xd[:, k * d:].data_ptr(), N + 1, stride)
                assert L.qrl_spectrum_get(sp._h, C.c_void_p(out.data_ptr()), N, 1, C.byref(nfft)) == 0
                got = out.cpu().numpy()
                peak.sample()
                for i, o in enumerate(orc):
                    o.work(X[i, k * d: k * d + N + 1])
                    w = o.get()
                    assert (w is not None) == (nfft.value == N), (k, i, nfft.value)
                    if w is not None:
                        check(got[i], w, (k, i))
                ready.append(nfft.value == N)
        finally:
            sp.close()
            free_device()
    assert any(ready), ready
    peak.report()
