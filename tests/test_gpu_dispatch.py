"""GPU tier: the channel-count and knob-selected kernel paths of every chain against the oracle.

qrl_rx_create / qrl_rx_work pick kernels, windows, streams and SM partitions from the channel count and from the QRL_* knobs of
DESIGN.md section 10 (many mode, the NBFM de-emphasis split, the FEC stream's partition, the symbol-sync window, slice cuts, the
rotator pass).  Each case here reaches one of those paths at a channel count where a batched kernel goes wrong without a small-C
test noticing: a partial last 32-channel group, a channel reading its neighbour's ring column, a scratch region indexed per group.

Inputs: every slab is built from P = 7 base signals (7 is coprime to 32 and to the 4 channels of a Viterbi CTA).  Channel c carries
base c mod 7, except the spot channels (0, 31, 32, 33, both lanes that bound the last group, C - 1 and two seeded random ones), which
carry a unique np.roll of their base.  The slab is gathered on the device from the base rows, so the host rebuilds any channel bit
for bit.  Checks: every port of every channel equals the port of its class representative, bitwise; every port of the
representatives and of every spot channel equals the oracle, bitwise; the ports have a minimum length and frames are recovered where
the chain decodes.  Each case also asserts the path it names where the ABI shows it (qrl_rx_sm_partition, the NBFM split's stage-5
launches under qrl_rx_profile)."""
import ctypes as C
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest

from tests import freedv_oracle as FO
from tests import siggen
from tests.test_gpu_am import am_signal
from tests.test_gpu_bpsk_2fsk import make_signals as bpsk_2fsk_signals
from tests.test_gpu_dsss import dsss_channels
from tests.test_gpu_freedv import rx_signal as freedv_signal
from tests.test_gpu_m17 import m17_like_signal
from tests.test_gpu_wbfm import wbfm_signal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 7
KMAXSUB = 16            # qrl_rx::kMaxSub (qrl_b200.cu): the largest QRL_NSUB / QRL_FIR_GROUP the handle accepts
SLACK = 160             # tail latency an RX port may differ from the oracle fed the same cuts (as in the per-chain tests)
ANALOG = {"nbfm", "am", "usb", "lsb", "wbfm", "freedv_usb", "freedv_lsb"}


# ------------------------------------------------------------------ base signals (reuse the per-chain tests' generators)
def _ssb_signal(sb, T):
    n = np.arange(T)
    X = np.zeros((P, T), np.complex64)
    sign = -1.0 if sb else 1.0
    for c in range(P):
        rng = np.random.default_rng(40 + c)
        x = 0.05 * np.exp(2j * np.pi * sign * (700 + 150 * c) * n / 1e6) * (1 + 0.5 * np.sin(2 * np.pi * 3 * n / 1e6))
        x = x + 0.03 * np.exp(2j * np.pi * sign * 1900 * n / 1e6) + 0.002 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))
        x[:1234] = 0
        X[c] = x.astype(np.complex64)
    return X, None


def _tx_burst(O, seed, T, kind, txargs, nbytes=None, frames=None, fo=100.0, snr=20.0, amp=0.1, phase=False):
    rng = np.random.default_rng(seed)
    X = np.zeros((P, T), np.complex64)
    payloads = []
    for c in range(P):
        if frames:
            data, pl = siggen.frames_4fsk(rng, frames)
            payloads.append(pl)
        else:
            data = rng.integers(0, 256, nbytes, dtype=np.uint8)
        iq = O.Tx(getattr(O, kind), *txargs).work(data)
        X[c] = siggen.channel(iq, rng, fo_hz=rng.uniform(-fo, fo), phase=rng.uniform(0, 6.28) if phase else 0.0,
                              delay=int(rng.integers(0, 300)), snr_db=snr, amp=amp, total=T)
    return X, (payloads or None)


def _gen(name, O, T):
    if name == "nbfm":
        return siggen.gen_nbfm_channels(P, T, seed0=1, lead_zeros=777), None
    if name == "am":
        return am_signal(np.random.default_rng(65), P, T), None
    if name in ("usb", "lsb"):
        return _ssb_signal(name == "lsb", T)
    if name == "wbfm":
        return wbfm_signal(np.random.default_rng(80), P, T), None
    if name.startswith("freedv"):
        sb = name.endswith("lsb")
        return freedv_signal(sb, P, T, 300 + sb), None
    if name in ("4fsk", "4fsk_disc"):
        return siggen.gen_4fsk_channels(P, T, seed0=1000, fm=name == "4fsk")
    if name == "4fsk1k":
        return _tx_burst(O, 77, T, "MOD_4FSK", (50, 1000000, 1700, 2000, 1), nbytes=120, amp=0.8)
    if name == "4fsk10k":
        return _tx_burst(O, 78, T, "MOD_4FSK", (5, 1000000, 1700, 20000, 1), nbytes=1200)
    if name == "4fsk100k":
        return _tx_burst(O, 79, T, "MOD_4FSK", (2, 1000000, 1700, 125000, 1), nbytes=12000)
    if name == "qpsk":
        return siggen.gen_qpsk_channels(P, T, seed0=2000)
    if name == "qpsk20k":
        return _tx_burst(O, 61, T, "MOD_QPSK", (100, 1000000, 1700, 6500, 0), frames=int(T / 1e6 * 105), fo=40, snr=18.0,
                         amp=0.2, phase=True)
    if name in ("bpsk", "2fsk"):
        return bpsk_2fsk_signals(O, name, P, T, 31 if name == "2fsk" else 32)
    if name == "2fsk_band":
        return _tx_burst(O, 35, T, "MOD_2FSK", (25, 1000000, 1700, 4000, 0), frames=max(4, int(T / 1e6 * 2000 / 80) - 6), fo=60)
    if name == "gmsk":
        return _tx_burst(O, 75, T, "MOD_2FSK", (25, 1000000, 1700, 4000, 1), nbytes=int(T / 1e6 * 2000 / 8), amp=0.4, phase=True)
    if name in ("m17", "dmr"):
        rng = np.random.default_rng(90 if name == "m17" else 91)
        return np.stack([m17_like_signal(rng, T) for _ in range(P)]), None
    if name == "dsss":
        X, _ = dsss_channels(O, P, (T + 999999) // 1000000, 9100)
        return np.ascontiguousarray(X[:, :T]), None
    raise KeyError(name)


class _FreedvRxOracle:
    """tests/freedv_oracle.FreedvRx behind the oracle.Rx interface (ports accumulate until read)"""

    def __init__(self, sb):
        self.o, self.acc = FO.FreedvRx(125, 1000000, 2500, 200, sb), [[], []]

    def set_carrier_offset(self, hz):
        self.o.set_carrier_offset(hz)

    def work(self, x):
        for p, v in enumerate(self.o.work(x)):
            self.acc[p].append(v)

    def port(self, p):
        return np.concatenate(self.acc[p])


# name -> (factory(qrl, C, max_samples), oracle factory(O), ports, T, per-port minimum lengths, frame check (port, sync, bits, len))
F4 = (0xED89AA, 24, 7)
RX = {
    "nbfm": (lambda q, n, m: q.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_NBFM, 125, 1000000, 1700, 5000, 0), 2, 1 << 18, (4000, 1500), None),
    "am": (lambda q, n, m: q.make_gr_demod_am(125, 1000000, 1700, 5000, n_channels=n, max_samples=m),
           lambda O: O.Rx(O.DEMOD_AM, 125, 1000000, 1700, 5000, 0), 2, 1 << 18, (4000, 1500), None),
    "usb": (lambda q, n, m: q.make_gr_demod_ssb(125, 1000000, 1700, 2700, 0, n_channels=n, max_samples=m),
            lambda O: O.Rx(O.DEMOD_SSB, 125, 1000000, 1700, 2700, 0), 2, 1 << 18, (1500, 1500), None),
    "lsb": (lambda q, n, m: q.make_gr_demod_ssb(125, 1000000, 1700, 2700, 1, n_channels=n, max_samples=m),
            lambda O: O.Rx(O.DEMOD_SSB, 125, 1000000, 1700, 2700, 1), 2, 1 << 18, (1500, 1500), None),
    "wbfm": (lambda q, n, m: q.make_gr_demod_wbfm(125, 1000000, 1700, 75000, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_WBFM, 125, 1000000, 1700, 75000, 0), 2, 1 << 17, (20000, 800), None),
    "freedv_usb": (lambda q, n, m: q.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=n, max_samples=m),
                   lambda O: _FreedvRxOracle(0), 2, 1 << 18, (2000, 2000), None),
    "freedv_lsb": (lambda q, n, m: q.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 1, n_channels=n, max_samples=m),
                   lambda O: _FreedvRxOracle(1), 2, 1 << 18, (2000, 2000), None),
    "4fsk": (lambda q, n, m: q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_4FSK, 5, 1000000, 1700, 3000, 1), 3, 1 << 19, (10000, 1000, 900), (2,) + F4),
    "4fsk_disc": (lambda q, n, m: q.make_gr_demod_4fsk(5, 1000000, 1700, 4000, False, n_channels=n, max_samples=m),
                  lambda O: O.Rx(O.DEMOD_4FSK, 5, 1000000, 1700, 4000, 0), 3, 1 << 19, (10000, 1000, 900), (2,) + F4),
    "4fsk1k": (lambda q, n, m: q.make_gr_demod_4fsk(10, 1000000, 1700, 2000, True, n_channels=n, max_samples=m),
               lambda O: O.Rx(O.DEMOD_4FSK, 10, 1000000, 1700, 2000, 1), 3, 1 << 19, (5000, 500, 450), None),
    "4fsk10k": (lambda q, n, m: q.make_gr_demod_4fsk(1, 1000000, 1700, 20000, True, n_channels=n, max_samples=m),
                lambda O: O.Rx(O.DEMOD_4FSK, 1, 1000000, 1700, 20000, 1), 3, 1 << 18, (20000, 2500, 2400), None),
    "4fsk100k": (lambda q, n, m: q.make_gr_demod_4fsk(2, 1000000, 1700, 125000, True, n_channels=n, max_samples=m),
                 lambda O: O.Rx(O.DEMOD_4FSK, 2, 1000000, 1700, 125000, 1), 3, 1 << 18, (100000, 20000, 20000), None),
    "qpsk": (lambda q, n, m: q.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_QPSK, 2, 1000000, 1700, 160000, 0), 3, 1 << 18, (100000, 60000, 60000), (2, 0xDE98AA, 24, 1516)),
    "qpsk20k": (lambda q, n, m: q.make_gr_demod_qpsk(25, 1000000, 1700, 6500, n_channels=n, max_samples=m),
                lambda O: O.Rx(O.DEMOD_QPSK, 25, 1000000, 1700, 6500, 0), 3, 1 << 19, (20000, 5000, 5000), (2,) + F4),
    "bpsk": (lambda q, n, m: q.make_gr_demod_bpsk(5, 1000000, 1700, 2400, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_BPSK, 5, 1000000, 1700, 2400, 0), 4, 1 << 19, (10000, 2000, 900, 900), ((2, 3),) + F4),
    "2fsk": (lambda q, n, m: q.make_gr_demod_2fsk(5, 1000000, 1700, 4000, True, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_2FSK, 5, 1000000, 1700, 4000, 1), 4, 1 << 19, (20000, 2000, 900, 900), ((2, 3),) + F4),
    "2fsk_band": (lambda q, n, m: q.make_gr_demod_2fsk(5, 1000000, 1700, 4000, False, n_channels=n, max_samples=m),
                  lambda O: O.Rx(O.DEMOD_2FSK, 5, 1000000, 1700, 4000, 0), 4, 1 << 19, (20000, 2000, 900, 900), ((2, 3),) + F4),
    "gmsk": (lambda q, n, m: q.make_gr_demod_gmsk(5, 1000000, 1700, 4000, n_channels=n, max_samples=m),
             lambda O: O.Rx(O.DEMOD_GMSK, 5, 1000000, 1700, 4000, 0), 4, 1 << 18, (10000, 1000, 450, 450), None),
    "m17": (lambda q, n, m: q.make_gr_demod_m17(n_channels=n, max_samples=m),
            lambda O: O.Rx(O.DEMOD_M17, 125, 1000000, 1700, 9000, 0), 3, 1 << 18, (6000, 1200, 2400), None),
    "dmr": (lambda q, n, m: q.make_gr_demod_dmr(n_channels=n, max_samples=m),
            lambda O: O.Rx(O.DEMOD_DMR, 5, 1000000, 0, 0, 0), 4, 1 << 18, (6000, 1200, 2400, 6000), None),
    "dsss": (lambda q, n, m: q.make_gr_demod_dsss(n_channels=n, max_samples=m),
             # 16 symbols/s: the decoded-bit ports stay empty at this length (test_gpu_dsss decodes 26 s of signal)
             lambda O: O.Rx(O.DEMOD_DSSS, 25, 1000000, 1700, 150, 0), 4, 3 << 20, (16000, 20, 0, 0), None),
}

# Rows outside RX run through the harness below when passed as `row`: RX's six fields plus a seventh, gen(O, T) -> (the P base
# signals, payloads or None) (tests/reference_instances.py: the reference instances RX does not hold).  `name` then only keys the caches.
_BASES, _ORACLE = {}, {}


def bases(name, O, T, row=None):
    if (name, T) not in _BASES:
        _BASES[(name, T)] = row[6](O, T) if row is not None and len(row) > 6 else _gen(name, O, T)
    return _BASES[(name, T)]


# ------------------------------------------------------------------ slabs: classes, spot channels, device gather
def spot_shifts(Cn):
    """spot channel -> its unique roll of the base signal"""
    last = 32 * ((Cn - 1) // 32)
    s = {c for c in (0, 31, 32, 33, last, Cn - 1) if c < Cn}
    rng = np.random.default_rng(Cn)
    s |= {int(v) for v in rng.choice(Cn, size=min(2, Cn), replace=False)}
    return {c: 1009 + 97 * c for c in sorted(s)}


def representatives(Cn, spots):
    reps = {}
    for c in range(Cn):
        if c not in spots and c % P not in reps:
            reps[c % P] = c
    assert len(reps) == min(P, Cn - len(spots))       # every class has one (a handle of fewer than P plain channels: each its own)
    return reps


def host_channel(B, spots, c):
    return np.roll(B[c % P], spots[c]) if c in spots else B[c % P]


HOST_MAX = 97          # up to this many channels the slab is a host array fed through qrl_rx_work (so these cases also run on the
                       # host-thread build of the library, tools/emu); the larger ones are gathered on the device


def make_slab(B, Cn, spots):
    if Cn <= HOST_MAX:
        return np.stack([host_channel(B, spots, c) for c in range(Cn)])
    return device_slab(B, Cn, spots)


def free_device():
    if "torch" in sys.modules:
        import torch
        if torch.cuda.is_available():
            torch.cuda.empty_cache()


def device_slab(B, Cn, spots, stride=None):
    """[Cn][stride] complex64 on the device: an index gather of the base rows, the spot channels rolled (exact operations only)"""
    import torch
    T = B.shape[1]
    Bd = torch.from_numpy(np.ascontiguousarray(B)).cuda()
    X = torch.zeros((Cn, stride or T), dtype=torch.complex64, device="cuda")
    X[:, :T] = Bd.index_select(0, torch.arange(Cn, device="cuda") % P)
    for c, s in spots.items():
        X[c, :T] = torch.roll(Bd[c % P], s)
    del Bd
    return X


# ------------------------------------------------------------------ path introspection through the existing ABI
def sm_partition(blk):
    a, b = C.c_int(-1), C.c_int(-1)
    assert blk._L.qrl_rx_sm_partition(blk._h, C.byref(a), C.byref(b)) == 0
    return a.value, b.value


def stage_launches(blk, stage):
    ms, n = C.c_double(), C.c_long()
    assert blk._L.qrl_rx_profile_read(blk._h, stage, C.byref(ms), C.byref(n)) == 0
    return n.value


_GREEN = []


def green_contexts(qrl):
    """True when the driver grants the SM partition (a 3-channel 4FSK handle has one by default)"""
    if not _GREEN:
        blk = qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=3, max_samples=1000)
        _GREEN.append(sm_partition(blk) != (0, 0))
        blk.close()
    return _GREEN[0]


def assert_partition(qrl, blk, on, loop_sms=None):
    part = sm_partition(blk)
    if not on:
        assert part == (0, 0), part
    elif not green_contexts(qrl):
        warnings.warn("the driver refused green contexts: SM-partition assertion skipped, parity still checked")
    else:
        assert part[0] > 0 and part[1] > 0, part
        if loop_sms is not None:
            assert part[0] == loop_sms, part


def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------ the RX harness
def run_rx(blk, X, cuts, events=(), read_every=1):
    """feed the slab (host array or device tensor) in `cuts` (list of (lo, hi)); events: (cut index, channel or -1, carrier offset
    Hz) applied before the cut.  Returns per call the ports read after it, or None for a call not read: with overlapped calls a read
    joins the call's tail, so read_every > 1 issues the calls in between back to back"""
    calls = []
    for k, (lo, hi) in enumerate(cuts):
        for (ek, ch, hz) in events:
            if ek == k:
                blk.set_carrier_offset(hz, channel=ch)
        if isinstance(X, np.ndarray):
            blk.work(X[:, lo:hi])
        else:
            blk.work_device(X[:, lo:].data_ptr(), hi - lo, X.shape[1])
        read = (k + 1) % read_every == 0 or k == len(cuts) - 1
        calls.append([blk.read_port(p) for p in range(blk.nports)] if read else None)
    return calls


def concat_calls(calls, nports, Cn):
    return [[np.concatenate([calls[k][p][c] for k in range(len(calls))]) for c in range(Cn)] for p in range(nports)]


def oracle_ports(name, O, B, spots, c, cuts, events, setters=(), row=None):
    """setters: (PARAM key, value) applied before the first sample"""
    row = row or RX[name]
    key = (name, B.shape[1], c % P, spots.get(c), tuple(cuts), tuple((k, hz) for (k, ch, hz) in events if ch in (-1, c)), tuple(setters))
    if key not in _ORACLE:
        x = host_channel(B, spots, c)
        rx = row[1](O)
        for pkey, value in setters:
            rx.set_param(pkey, value)
        for k, (lo, hi) in enumerate(cuts):
            for (ek, ch, hz) in events:
                if ek == k and ch in (-1, c):
                    rx.set_carrier_offset(hz)
            rx.work(x[lo:hi])
        _ORACLE[key] = [rx.port(p) for p in range(row[2])]
    return _ORACLE[key]


def check_rx(name, O, B, payloads, got, spots, cuts, events=(), frames=True, setters=(), row=None):
    """got[p][c]: the whole stream of port p on channel c; setters: (PARAM key, value) the handle had before its first sample"""
    row = row or RX[name]
    nports, fr = row[2], row[5]
    mins = [m * cuts[-1][1] // row[3] for m in row[4]]         # the minimum lengths scale with the stream's length
    Cn = len(got[0])
    reps = representatives(Cn, spots)
    for p in range(nports):
        for c in range(Cn):
            if c not in spots:
                assert np.array_equal(got[p][c], got[p][reps[c % P]]), "%s: port %d of channel %d differs from channel %d" % (name, p, c, reps[c % P])
    for c in sorted(set(reps.values()) | set(spots)):
        want = oracle_ports(name, O, B, spots, c, cuts, events, setters, row)
        for p in range(nports):
            g, w = got[p][c], want[p]
            n = min(len(g), len(w))
            assert abs(len(g) - len(w)) <= SLACK and n >= mins[p], (name, c, p, len(g), len(w))
            assert np.array_equal(g[:n], w[:n]), "%s: port %d of channel %d differs from the oracle" % (name, p, c)
    if frames and fr and payloads:
        ports, sync, sbits, flen = fr
        for k, c in reps.items():        # the 4-port chains: the better of the two decoders (one runs behind delay(1))
            good = max(siggen.count_good_frames(got[p][c], sync, sbits, flen, payloads[k])[0] for p in np.atleast_1d(ports))
            assert good >= 1 and good >= len(payloads[k]) - 6, (name, c, good, len(payloads[k]))


def ragged(T):
    """one call under 256 outputs of any stage (untiled fir_ccf_ring / qdemod_fir_fff) between two large ones"""
    a = T // 2 + 13
    return [(0, a), (a, a + 101), (a + 101, T)]


def equal_cuts(T, K):
    return [(k * (T // K), (k + 1) * (T // K)) for k in range(K)]


def run_case(qrl, O, name, Cn, T=None, cuts=None, overlap=False, events=(), profile=False, frames=True, row=None):
    """build the slab, run one handle, check everything; returns the handle (caller closes).  Overlapped: the handle reads after every
    call; a serialised twin gives every call's reference ports; two more overlapped handles issue the calls back to back, one read
    every second call and one read only after the last, so the calls in between really run under each other's tails"""
    row = row or RX[name]
    T = T or row[3]
    B, payloads = bases(name, O, T, row)
    spots = spot_shifts(Cn)
    cuts = cuts or ragged(T)
    maxs = max(hi - lo for lo, hi in cuts)
    X = make_slab(B, Cn, spots)
    blk = row[0](qrl, Cn, maxs)
    try:
        if profile:
            assert blk._L.qrl_rx_profile(blk._h, 1) == 0
        if overlap:
            blk.set_overlap(True)
        calls = run_rx(blk, X, cuts, events)
        if overlap:         # every call equals the serialised handle's
            ser = row[0](qrl, Cn, maxs)
            try:
                want = run_rx(ser, X, cuts, events)
            finally:
                ser.close()
            for read_every in (1, 2, len(cuts)):
                if read_every == 1:
                    got_calls = calls
                else:
                    b2b = row[0](qrl, Cn, maxs)
                    try:
                        b2b.set_overlap(True)
                        got_calls = run_rx(b2b, X, cuts, events, read_every=read_every)
                    finally:
                        b2b.close()
                for k in range(len(cuts)):
                    if got_calls[k] is not None:
                        for p in range(blk.nports):
                            for c in range(Cn):
                                assert np.array_equal(got_calls[k][p][c], want[k][p][c]), (name, read_every, k, p, c)
        got = concat_calls(calls, blk.nports, Cn)
        check_rx(name, O, B, payloads, got, spots, cuts, events, frames=frames and T == row[3], row=row)
    except BaseException:
        blk.close()
        raise
    finally:
        del X
        free_device()
    return blk


def default_partition(name, Cn):
    """mirrors qrl_rx_create: many mode (no partition) when the loop CTAs exceed 44 or an analog chain has more than 64 channels;
    the NBFM split counts two CTAs per channel; QPSK never takes a partition"""
    groups = (Cn + 31) // 32
    if name.startswith("qpsk"):
        return False
    if name in ANALOG:
        big = 2 * Cn if (name == "nbfm" and Cn <= n_sm()) else min(Cn, 44)
        return big <= 44 and Cn <= 64
    return groups <= 44


# ------------------------------------------------------------------ 1. channel-count sweep of every receive chain
@pytest.mark.parametrize("Cn", [33, 97])
@pytest.mark.parametrize("name", list(RX))
def test_rx_channel_count_sweep(qrl, oracle, name, Cn):
    """C = 33: one-lane last group; C = 97: four groups, a one-lane last group, C mod 4 = 1 -- the analog chains in many mode
    (no partition), the digital chains' Viterbi on the loop partition."""
    blk = run_case(qrl, oracle, name, Cn, profile=name == "nbfm")
    try:
        assert_partition(qrl, blk, default_partition(name, Cn))
        if name == "nbfm":                  # C <= SM count: the de-emphasis runs split, as stage 5
            assert stage_launches(blk, 5) > 0
    finally:
        blk.close()


# ------------------------------------------------------------------ 2. thresholds at their natural sizes
@pytest.mark.parametrize("which", ["64", "65", "nsm", "nsm+1"])
def test_nbfm_many_and_split_thresholds(qrl, oracle, which):
    """h->many = C > 64 for the analog chains; nbfm_split = C <= SM count (read from the device, not assumed)"""
    Cn = {"64": 64, "65": 65, "nsm": n_sm(), "nsm+1": n_sm() + 1}[which]
    blk = run_case(qrl, oracle, "nbfm", Cn, T=1 << 17, profile=True)
    try:
        assert_partition(qrl, blk, default_partition("nbfm", Cn))
        split = stage_launches(blk, 5)
        assert (split > 0) == (Cn <= n_sm()), (Cn, split)
    finally:
        blk.close()


@pytest.mark.parametrize("Cn", [64, 65])
@pytest.mark.parametrize("name", ["am", "usb"])
def test_analog_many_threshold(qrl, oracle, name, Cn):
    """`analog_kind && h->C > 64` (qrl_b200.cu, qrl_rx_create) at the boundary itself: 64 channels keep the partition (44 loop CTAs),
    65 go to many mode.  NBFM cannot show it: its split already counts two loop CTAs per channel."""
    blk = run_case(qrl, oracle, name, Cn, T=1 << 17)
    try:
        assert_partition(qrl, blk, Cn <= 64)
    finally:
        blk.close()


def test_qpsk_many_mode_threshold(qrl, oracle):
    """C = 705: 2 * ceil(C / 32) = 46 loop CTAs > 44 puts QPSK in many mode -- agc_costas_kernel<32, ...> and the generic 64-row
    symbol sync (qrl_b200.cu: `h->many = big_ctas > 44 ...`, `small_win = h->many && ...`).  QPSK never takes a partition, so the
    ABI shows no difference; parity at this size is the check."""
    blk = run_case(qrl, oracle, "qpsk", 705, T=1 << 16, cuts=[(0, 40000), (40000, 40100), (40100, 1 << 16)])
    try:
        assert_partition(qrl, blk, False)
    finally:
        blk.close()


@pytest.mark.parametrize("Cn,K,T", [(65, 3, 3 << 17), (1409, 4, 1 << 17)])
def test_4fsk_overlapped_thresholds(qrl, oracle, Cn, K, T):
    """overlapped 4FSK-FM calls against the serialised handle and the oracle.  C = 65: three groups put the Viterbi stream on the
    loop partition (FEC not on the wide partition once groups > 2).  C = 1409: 45 groups > 44 -> many mode, no partition."""
    blk = run_case(qrl, oracle, "4fsk", Cn, T=T, cuts=equal_cuts(T, K), overlap=True)
    try:
        assert_partition(qrl, blk, default_partition("4fsk", Cn))
    finally:
        blk.close()


# ------------------------------------------------------------------ 3. every knob-selected variant at C = 33
KNOBS = [
    # id, chain, env, overlapped, expected partition (True / False / loop SM count), NBFM split expected
    ("many-qpsk", "qpsk", {"QRL_MANY_CHANNELS": "1"}, False, False, None),
    ("many-qpsk20k", "qpsk20k", {"QRL_MANY_CHANNELS": "1"}, False, False, None),
    ("many-am", "am", {"QRL_MANY_CHANNELS": "1"}, False, False, None),
    # without the split NBFM counts one loop CTA per channel: 33 <= 44, so the handle leaves many mode and takes a partition
    ("nbfm-no-split", "nbfm", {"QRL_NBFM_NO_SPLIT": "1"}, False, True, False),
    ("nbfm-no-split-0", "nbfm", {"QRL_NBFM_NO_SPLIT": "0"}, False, True, False),
    ("many-0-nbfm", "nbfm", {"QRL_MANY_CHANNELS": "0"}, False, True, True),
    ("fec-on-par-0", "4fsk", {"QRL_FEC_ON_PAR": "0"}, True, True, None),
    ("fec-on-par-1", "4fsk", {"QRL_FEC_ON_PAR": "1"}, True, True, None),
    ("ss-ch-256", "4fsk", {"QRL_SS_CH": "256"}, False, True, None),
    ("ss-ch-512", "4fsk", {"QRL_SS_CH": "512"}, False, True, None),
    # M17's low sps leaves no room for the replicated tap bank next to a 512-row window, so symsync_kernel variant 1 runs (selected in
    # qrl_rx_work's run_ext: `const bool rep = smem_rep <= 220 * 1024 && !h->dmr`; the ABI does not show it)
    ("ss-ch-512-m17", "m17", {"QRL_SS_CH": "512"}, False, True, None),
    ("nsub-1", "4fsk", {"QRL_NSUB": "1"}, True, True, None),
    ("nsub-max", "4fsk", {"QRL_NSUB": str(KMAXSUB)}, True, True, None),
    ("fir-group-1", "4fsk", {"QRL_FIR_GROUP": "1"}, True, True, None),
    ("no-sm-partition", "4fsk", {"QRL_NO_SM_PARTITION": "1"}, False, False, None),
    ("loop-sms-8", "am", {"QRL_LOOP_SMS": "8"}, False, 8, None),          # AM at C = 33 would take 40 loop SMs
]


@pytest.mark.parametrize("case", KNOBS, ids=[k[0] for k in KNOBS])
def test_knob_selected_variants(qrl, oracle, monkeypatch, case):
    _, name, env, overlap, part, split = case
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    T = RX[name][3]
    blk = run_case(qrl, oracle, name, 33, cuts=equal_cuts(T, 4) if overlap else None, overlap=overlap, profile=split is not None)
    try:
        assert_partition(qrl, blk, bool(part), loop_sms=part if part is not True and part else None)
        if split is not None:
            assert (stage_launches(blk, 5) > 0) == split
    finally:
        blk.close()


_LEAN_CHILD = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
import qradiolink_b200 as q
X = np.load(sys.argv[2])
blk = q.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=X.shape[0], max_samples=X.shape[1])
blk.work(X)
np.savez(sys.argv[3], *[np.concatenate(blk.read_port(p)) for p in range(3)], *[np.array([len(v) for v in blk.read_port(p)]) for p in range(3)])
blk.close()
"""


def test_qpsk_generic_symbol_sync_in_a_fresh_process(qrl, oracle, tmp_path):
    """QRL_QPSK_LEAN_SS=0 (read once per process into a static): the generic 128-row, 3-stage QPSK symbol sync.  A child process
    with the knob set runs 33 channels; its ports must equal this process's lean handle and the oracle."""
    name, Cn, T = "qpsk", 33, 1 << 18
    B, payloads = bases(name, oracle, T)
    spots = spot_shifts(Cn)
    Xh = np.stack([host_channel(B, spots, c) for c in range(Cn)])
    np.save(tmp_path / "x.npy", Xh)
    env = dict(os.environ, QRL_QPSK_LEAN_SS="0")
    r = subprocess.run([sys.executable, "-c", _LEAN_CHILD, ROOT, str(tmp_path / "x.npy"), str(tmp_path / "out.npz")],
                       env=env, cwd=ROOT, timeout=600, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    z = np.load(tmp_path / "out.npz")
    got = []
    for p in range(3):
        flat, counts = z["arr_%d" % p], z["arr_%d" % (p + 3)]
        got.append(np.split(flat, np.cumsum(counts)[:-1]))
    lean = RX[name][0](qrl, Cn, T)
    try:
        lean.work(Xh)
        for p in range(3):
            ref = lean.read_port(p)
            for c in range(Cn):
                assert np.array_equal(got[p][c], ref[c]), (p, c)
    finally:
        lean.close()
    check_rx(name, oracle, B, payloads, got, spots, [(0, T)])


# ------------------------------------------------------------------ 4. carrier offset on every stage-1 shape
OFFSET_EVENTS = [(0, -1, 1250.0), (2, -1, -2600.5)]


@pytest.mark.parametrize("name", ["wbfm", "m17", "dmr", "qpsk", "4fsk10k", "4fsk100k"])
def test_carrier_offset_rotator_pass(qrl, oracle, name):
    """shapes other than /50, /100, /25, /125 rotate in a rotator_kernel pre-pass (`h->rot_fused = h->rot_active && poly_shape && ...`
    in qrl_rx_work): an offset on every channel, a retune of all of them mid-stream and of one spot channel alone.  The pass shows
    as one more launch per call than the same handle without an offset."""
    events = OFFSET_EVENTS + [(2, 32, 777.0)]
    blk = run_case(qrl, oracle, name, 33, events=events)
    plain = run_case(qrl, oracle, name, 33)
    try:
        assert blk.launches - plain.launches == len(ragged(RX[name][3])), (blk.launches, plain.launches)
    finally:
        blk.close(); plain.close()


def test_carrier_offset_forced_pass_equals_fused(qrl, oracle, monkeypatch):
    """4FSK-2k fuses the rotator into stage 1; QRL_ROTATOR_PASS (read on every call) forces the pre-pass: same ports, same oracle,
    and one rotator_kernel launch more per call"""
    name, Cn = "4fsk", 33
    events = OFFSET_EVENTS + [(2, 32, 777.0)]
    T = RX[name][3]
    B, _ = bases(name, oracle, T)
    spots = spot_shifts(Cn)
    X = make_slab(B, Cn, spots)
    a, b = RX[name][0](qrl, Cn, T), RX[name][0](qrl, Cn, T)
    try:
        cuts = ragged(T)
        monkeypatch.setenv("QRL_ROTATOR_PASS", "1")
        got_pass = concat_calls(run_rx(a, X, cuts, events), 3, Cn)
        monkeypatch.delenv("QRL_ROTATOR_PASS")
        got_fused = concat_calls(run_rx(b, X, cuts, events), 3, Cn)
        for p in range(3):
            for c in range(Cn):
                assert np.array_equal(got_pass[p][c], got_fused[p][c]), (p, c)
        assert a.launches - b.launches == len(cuts), (a.launches, b.launches)
        check_rx(name, oracle, B, None, got_pass, spots, cuts, events)
    finally:
        a.close(); b.close()
        del X
        free_device()


# ------------------------------------------------------------------ 5. TX channel counts
TX = {
    # name: (factory(qrl, C, max_items), oracle factory(O), input kind, items per call)
    "4fsk2kfm": (lambda q, n, m: q.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=n, max_items=m),
                 lambda O: O.Tx(O.MOD_4FSK, 25, 1000000, 1700, 3500, 1), "bytes", 40),
    "4fsk2k": (lambda q, n, m: q.make_gr_mod_4fsk(25, 1000000, 1700, 4000, False, n_channels=n, max_items=m),
               lambda O: O.Tx(O.MOD_4FSK, 25, 1000000, 1700, 4000, 0), "bytes", 40),
    "4fsk100k": (lambda q, n, m: q.make_gr_mod_4fsk(2, 1000000, 1700, 125000, True, n_channels=n, max_items=m),
                 lambda O: O.Tx(O.MOD_4FSK, 2, 1000000, 1700, 125000, 1), "bytes", 600),
    "qpsk": (lambda q, n, m: q.make_gr_mod_qpsk(4, 1000000, 1700, 160000, n_channels=n, max_items=m),
             lambda O: O.Tx(O.MOD_QPSK, 4, 1000000, 1700, 160000, 0), "bytes", 600),
    "qpsk20k": (lambda q, n, m: q.make_gr_mod_qpsk(100, 1000000, 1700, 6500, n_channels=n, max_items=m),
                lambda O: O.Tx(O.MOD_QPSK, 100, 1000000, 1700, 6500, 0), "bytes", 60),
    "bpsk": (lambda q, n, m: q.make_gr_mod_bpsk(250, 1000000, 1700, 2800, n_channels=n, max_items=m),
             lambda O: O.Tx(O.MOD_BPSK, 250, 1000000, 1700, 2800, 0), "bytes", 20),
    "2fsk": (lambda q, n, m: q.make_gr_mod_2fsk(25, 1000000, 1700, 4000, True, n_channels=n, max_items=m),
             lambda O: O.Tx(O.MOD_2FSK, 25, 1000000, 1700, 4000, 1), "bytes", 30),
    "2fsk_band": (lambda q, n, m: q.make_gr_mod_2fsk(25, 1000000, 1700, 4000, False, n_channels=n, max_items=m),
                  lambda O: O.Tx(O.MOD_2FSK, 25, 1000000, 1700, 4000, 0), "bytes", 30),
    "gmsk": (lambda q, n, m: q.make_gr_mod_gmsk(50, 1000000, 1700, 4000, n_channels=n, max_items=m),
             lambda O: O.Tx(O.MOD_GMSK, 50, 1000000, 1700, 4000, 0), "bytes", 20),
    "m17": (lambda q, n, m: q.make_gr_mod_m17(n_channels=n, max_items=m),
            lambda O: O.Tx(O.MOD_M17, 125, 1000000, 1700, 9000, 0), "bytes", 60),
    "dmr": (lambda q, n, m: q.make_gr_mod_dmr(n_channels=n, max_items=m),
            lambda O: O.Tx(O.MOD_DMR, 125, 1000000, 1700, 5000, 0), "bytes", 60),
    "dsss": (lambda q, n, m: q.make_gr_mod_dsss(n_channels=n, max_items=m),
             lambda O: O.Tx(O.MOD_DSSS, 25, 1000000, 1700, 200, 0), "bytes", 1),
    "nbfm": (lambda q, n, m: q.make_gr_mod_nbfm(20, 1000000, 1700, 5000, n_channels=n, max_items=m),
             lambda O: O.Tx(O.MOD_NBFM, 20, 1000000, 1700, 5000, 0), "audio", 1500),
    "usb": (lambda q, n, m: q.make_gr_mod_ssb(125, 1000000, 1700, 2700, 0, n_channels=n, max_items=m),
            lambda O: O.Tx(O.MOD_SSB, 125, 1000000, 1700, 2700, 0), "audio", 1500),
    "lsb": (lambda q, n, m: q.make_gr_mod_ssb(125, 1000000, 1700, 2700, 1, n_channels=n, max_items=m),
            lambda O: O.Tx(O.MOD_SSB, 125, 1000000, 1700, 2700, 1), "audio", 1500),
    "am": (lambda q, n, m: q.make_gr_mod_am(125, 1000000, 1700, 5000, n_channels=n, max_items=m),
           lambda O: O.Tx(O.MOD_AM, 125, 1000000, 1700, 5000, 0), "audio", 1500),
    "freedv": (lambda q, n, m: q.make_gr_mod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=n, max_items=m),
               lambda O: FO.FreedvTx(125, 1000000, 2500, 200, 0), "modem", 1500),
}


def tx_bases(kind, n):
    rng = np.random.default_rng(4242 + n)
    if kind == "bytes":
        return rng.integers(0, 256, (P, n), dtype=np.uint8)
    t = np.arange(n) / 8000.0
    audio = np.stack([0.5 * np.sin(2 * np.pi * (500 + 170 * c) * t) + 0.3 * np.sin(2 * np.pi * 1900 * t + c) for c in range(P)])
    if kind == "audio":
        return audio.astype(np.float32)
    return (8000 * audio + 800 * rng.standard_normal(audio.shape)).astype(np.int16)


def tx_channel(B, kind, spots, c):
    """spot channels: frame bytes XOR a per-channel constant (DSSS has too few bytes for distinct rolls), audio rolled"""
    if c not in spots:
        return B[c % P]
    if kind == "bytes":
        return B[c % P] ^ np.uint8(1 + c % 255)
    return np.roll(B[c % P], spots[c])


@pytest.mark.parametrize("Cn", [33, 97])
@pytest.mark.parametrize("name", list(TX))
def test_tx_channel_count_sweep(qrl, oracle, name, Cn):
    """every modulator at C = 33 and 97 (tx_bits_kernel: one lane per channel, a partial last warp), two calls (state carried)"""
    factory, ofactory, kind, n = TX[name]
    B = tx_bases(kind, 2 * n)
    spots = {c: 1 + c for c in spot_shifts(Cn)}
    D = np.stack([tx_channel(B, kind, spots, c) for c in range(Cn)])
    tx = factory(qrl, Cn, n)
    try:
        work = {"bytes": tx.work, "audio": tx.work_audio, "modem": tx.work_modem}[kind]
        calls = [work(D[:, :n]), work(D[:, n:])]
    finally:
        tx.close()
    reps = representatives(Cn, spots)
    assert max(np.max(np.abs(got[reps[1]])) for got in calls) > 0       # (DMR: the first call is all latency)
    for got in calls:
        assert got.shape[1] >= n
        for c in range(Cn):
            if c not in spots:
                assert np.array_equal(got[c], got[reps[c % P]]), (name, c)
    for c in sorted(set(reps.values()) | set(spots)):
        o = ofactory(oracle)
        for k, got in enumerate(calls):
            want = o.work(D[c, k * n:(k + 1) * n])
            assert len(want) == got.shape[1] and np.array_equal(got[c], want), (name, c, k)


# ------------------------------------------------------------------ 6. the standalone decimating FIR beyond its grid cap
@pytest.mark.parametrize("D,ntaps,Cn", [(1, 33, 300), (31, 20, 97), (31, 100, 97), (33, 419, 64), (64, 5, 40), (64, 200, 40),
                                        (125, 64, 33), (125, 300, 33)])
def test_fir_decim_device_beyond_grid_cap(qrl, oracle, D, ntaps, Cn):
    """qrl_fir_decim_ccf_device caps its grid at 16 CTAs per SM (8 outputs each): nout ~ 40 000 runs the grid-stride loop.  Strides
    differ from T and nout; bitwise against oracle.fir_decim_ccf, and within 1e-5 relative RMS of a float64 statement of
    y[m] = sum_k h[k] x[m D - k] (x[i < 0] = 0)."""
    import torch
    rng = np.random.default_rng(D * 1000 + ntaps)
    nout = 40000 + D % 7
    T = (nout - 1) * D + 1 + int(rng.integers(0, D))
    assert (T + D - 1) // D == nout and nout > 16 * n_sm() * 8
    taps = (rng.standard_normal(ntaps) / np.sqrt(ntaps)).astype(np.float32)
    B = (rng.standard_normal((P, T)) + 1j * rng.standard_normal((P, T))).astype(np.complex64)
    spots = spot_shifts(Cn)
    xs, ys = T + 3, nout + 5
    X = device_slab(B, Cn, spots, stride=xs)
    Y = torch.full((Cn, ys), complex(7.0, 7.0), dtype=torch.complex64, device="cuda")
    L = qrl.load_library()
    rc = L.qrl_fir_decim_ccf_device(taps.ctypes.data_as(C.c_void_p), ntaps, D, C.c_void_p(X.data_ptr()), T, xs,
                                    C.c_void_p(Y.data_ptr()), ys, Cn, None)
    assert rc == 0
    got = Y.cpu().numpy()
    del X, Y
    torch.cuda.empty_cache()
    assert np.all(got[:, nout:] == np.complex64(7 + 7j))          # the padding columns stay untouched
    got = got[:, :nout]
    reps = representatives(Cn, spots)
    for c in range(Cn):
        if c not in spots:
            assert np.array_equal(got[c], got[reps[c % P]]), c
    h64 = taps.astype(np.float64)
    for c in sorted(set(reps.values()) | set(spots)):
        x = host_channel(B, spots, c)
        want = oracle.fir_decim_ccf(taps, D, x)
        assert len(want) == nout and np.array_equal(got[c], want), c
        xp = np.concatenate([np.zeros(ntaps - 1), x.astype(np.complex128)])
        y64 = np.zeros(nout, np.complex128)
        for k in range(ntaps):
            y64 += h64[k] * xp[ntaps - 1 - k: ntaps - 1 - k + (nout - 1) * D + 1: D]
        err = np.sqrt(np.mean(np.abs(got[c] - y64) ** 2) / np.mean(np.abs(y64) ** 2))
        assert err <= 1e-5, (c, err)
