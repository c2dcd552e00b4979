"""GPU tier: the reference instances no other table holds (tests/reference_instances.py), against the oracle.

Receivers: QPSK-2K (sps 125: /100 to 10 ksps, 2727 stage-1 taps, 5 samples per symbol, FLL, lean symbol sync), BPSK-1K
(clock_recovery_mm at omega 10), 2FSK-1K-FM and 2FSK-1K (sps 10: /50 to 20 ksps, RRC of 351 taps, the band-filter detector at 20 ksps)
and GMSK-10K (x2/25 to 80 ksps).  Each runs 3 channels of the oracle's own frames through a channel with ragged cuts, then 33 and 97
channels through test_gpu_dispatch's class and spot-channel harness; QPSK-2K also at 704 and 705 channels, either side of the many-mode
switch.  Every port is bit-identical to the oracle and at least N - 6 of the N payloads come back.  BPSK-1K and the 2FSK-1K receivers
run again with their clock or FLL limit reached (reference_instances.STRESS_RX).  Transmitters: USB-CW and FreeDV
2700/200 on both side bands, bit-identical over uneven calls; USB-CW also loops back through the USB receiver."""
import time

import numpy as np
import pytest

from tests import reference_instances as R
from tests import test_gpu_dispatch as D
from tests.test_gpu_freedv import tx_parity_case

pytestmark = pytest.mark.gpu

# stage 1 of the /100 and /50 chains is a register-tiled polyphase FIR with the carrier rotator fused in; GMSK-10K's x2/25
# resampler is not, so a carrier offset costs it one rotator_kernel launch per call
FUSED_ROTATOR = {"qpsk2k": True, "bpsk1k": True, "2fsk1kfm": True, "2fsk1k": True, "gmsk10k": False}


def free_mib():
    import torch
    return torch.cuda.mem_get_info()[0] / 2 ** 20


def report(tag, t0, free0, free1):
    """duration and device memory of a case, printed with -s (the rings and ports of these handles have never been sized before).
    The library's buffers come from cudaMalloc, which torch does not count, and NVML may not list this process, so the figure is the
    drop in the device's free memory from before the case to the moment after its last call with its handles open (every buffer of
    a handle is allocated at create, so that is their peak).  It is device-wide: another process allocating in between shows too."""
    print("\n[reference instance] %s: %.1f s; %.0f MiB of device memory taken with the handles open after their last call"
          % (tag, time.time() - t0, free0 - free1))


def cuts_for(T):
    """a 1-sample call, calls that are no multiple of /100, /50 or /12.5, and one under 256 outputs of any stage"""
    a = T // 3 + 7
    return [(0, 1), (1, a), (a, a + 101), (a + 101, 2 * T // 3 + 33), (2 * T // 3 + 33, T)]


@pytest.mark.parametrize("name", sorted(R.NEW_RX))
def test_rx_instance_parity(qrl, oracle, name):
    """3 plain channels (each its own class, no spot rolls), ragged cuts: every port against the oracle, payloads recovered.  A twin
    handle with a carrier offset on every channel and a retune mid-stream matches the oracle retuned the same way, and shows the
    stage-1 path by its launches: no extra launch where the rotator is fused into the tiled FIR, one per call where it is not."""
    t0, free0 = time.time(), free_mib()
    row = R.NEW_RX[name]
    T = row[3]
    B, payloads = D.bases(name, oracle, T, row)
    cuts = cuts_for(T)
    X = D.make_slab(B, 3, {})
    maxs = max(hi - lo for lo, hi in cuts)
    blk, twin = row[0](qrl, 3, maxs), row[0](qrl, 3, maxs)
    try:
        got = D.concat_calls(D.run_rx(blk, X, cuts), blk.nports, 3)
        D.check_rx(name, oracle, B, payloads, got, {}, cuts, row=row)
        events = [(0, -1, 310.0), (3, -1, -475.5)]
        got_off = D.concat_calls(D.run_rx(twin, X, cuts, events), twin.nports, 3)
        free1 = free_mib()
        D.check_rx(name, oracle, B, payloads, got_off, {}, cuts, events, frames=False, row=row)
        extra = twin.launches - blk.launches
        assert extra == (0 if FUSED_ROTATOR[name] else len(cuts)), (name, twin.launches, blk.launches)
    finally:
        blk.close(); twin.close()
    report("%s parity, 3 ch x %d" % (name, T), t0, free0, free1)


@pytest.mark.parametrize("name", sorted(R.STRESS_RX))
def test_rx_instance_loop_limits(qrl, oracle, name):
    """the loop clamps no frame-carrying channel reaches (reference_instances.STRESS_RX): BPSK-1K's omega limit under a symbol rate
    1 % fast, the 4 kHz FLL limit of BPSK-1K and both 2FSK-1K receivers under an offset sweeping to 9 kHz.  3 channels, ragged cuts,
    every port bit-identical to the oracle; no payload check (the loops sit at their limits)"""
    t0, free0 = time.time(), free_mib()
    row = R.STRESS_RX[name][1]
    T = row[3]
    B, _ = D.bases(name, oracle, T, row)
    cuts = cuts_for(T)
    X = D.make_slab(B, 3, {})
    blk = row[0](qrl, 3, max(hi - lo for lo, hi in cuts))
    try:
        got = D.concat_calls(D.run_rx(blk, X, cuts), blk.nports, 3)
        free1 = free_mib()
        D.check_rx(name, oracle, B, None, got, {}, cuts, frames=False, row=row)
    finally:
        blk.close()
    report("%s, 3 ch x %d" % (name, T), t0, free0, free1)


@pytest.mark.parametrize("Cn", [33, 97])
@pytest.mark.parametrize("name", sorted(R.NEW_RX))
def test_rx_instance_channel_counts(qrl, oracle, name, Cn):
    """C = 33 (a one-lane last group) and C = 97 (four groups): classes, spot channels and representatives against the oracle"""
    t0, free0 = time.time(), free_mib()
    blk = D.run_case(qrl, oracle, name, Cn, row=R.NEW_RX[name])
    try:
        free1 = free_mib()
        D.assert_partition(qrl, blk, D.default_partition(name, Cn))
    finally:
        blk.close()
    report("%s, %d channels" % (name, Cn), t0, free0, free1)


@pytest.mark.parametrize("Cn", [704, 705])
def test_qpsk_2k_either_side_of_many_mode(qrl, oracle, monkeypatch, Cn):
    """2 ceil(C / 32) loop CTAs: 44 at C = 704, 46 at 705, which puts QPSK in many mode (32-row AGC / Costas windows, the 64-row
    symbol sync).  A probe handle asking for an SM partition (QRL_QPSK_PARTITION=1) shows the mode: only many mode refuses it.
    Parity of the representatives and spot channels against the oracle over 2^18 samples with ragged cuts."""
    t0, free0 = time.time(), free_mib()
    T = 1 << 18
    need = Cn * T * 8 * 4                 # the device slab, the handle's input copy and rings, the ports: a generous bound
    import torch
    free = torch.cuda.mem_get_info()[0]
    if need > free:
        pytest.skip("QPSK-2K at %d channels x %d samples wants about %.1f GiB, %.1f GiB free" % (Cn, T, need / 2 ** 30, free / 2 ** 30))
    monkeypatch.setenv("QRL_QPSK_PARTITION", "1")
    try:
        probe = R.NEW_RX["qpsk2k"][0](qrl, Cn, 4096)
    finally:
        monkeypatch.delenv("QRL_QPSK_PARTITION")
    try:
        D.assert_partition(qrl, probe, Cn <= 704)
    finally:
        probe.close()
    blk = D.run_case(qrl, oracle, "qpsk2k", Cn, T=T, cuts=[(0, 100001), (100001, 100078), (100078, T)], row=R.NEW_RX["qpsk2k"])
    try:
        free1 = free_mib()
        D.assert_partition(qrl, blk, False)
    finally:
        blk.close()
    report("qpsk2k, %d channels x %d" % (Cn, T), t0, free0, free1)


# ------------------------------------------------------------------ transmit instances
def test_tx_usb_cw_matches_oracle_and_loops_back(qrl, oracle):
    """gr_mod_base's _usb_cw (side-band filter 1000 Hz wide): bit-identical to the oracle over three uneven calls; the IQ through
    the device USB receiver gives back each channel's tone within 10 Hz"""
    C, n = 2, 8000
    tones = (600.0, 850.0)
    t = np.arange(n) / 8000.0
    audio = np.stack([(0.6 * np.sin(2 * np.pi * f * t)).astype(np.float32) for f in tones])
    tx = qrl.make_gr_mod_ssb(125, 1000000, 1700, 1000, 0, n_channels=C, max_items=n)
    try:
        got = np.concatenate([tx.work_audio(audio[:, a:b]) for a, b in ((0, 1), (1, 2999), (2999, n))], axis=1)
    finally:
        tx.close()
    for c in range(C):
        want = oracle.Tx(oracle.MOD_SSB, 125, 1000000, 1700, 1000, 0).work(audio[c])
        assert got.shape[1] == len(want) > (n - 8) * 125, (got.shape, len(want))
        assert np.array_equal(got[c], want), c
    rx = qrl.make_gr_demod_ssb(125, 1000000, 1700, 2700, 0, n_channels=C, max_samples=got.shape[1])
    try:
        rx.work(np.ascontiguousarray(got))
        aud = rx.read_port(1)
    finally:
        rx.close()
    for c, f in enumerate(tones):
        a = aud[c][2000:]
        spec = np.abs(np.fft.rfft(a * np.hanning(len(a)), 8 * len(a)))
        fb = np.fft.rfftfreq(8 * len(a), 1 / 8000.0)
        assert abs(fb[np.argmax(spec)] - f) < 10.0, (c, f, fb[np.argmax(spec)])


@pytest.mark.parametrize("sb", [0, 1])
def test_tx_freedv_2700_200_matches_oracle(qrl, sb):
    """_freedv_tx800XA_usb / _lsb and _freedv_tx1600_lsb: the 2700 / 200 Hz side-band filter pair"""
    tx_parity_case(qrl, 200, sb)


def test_tx_2fsk_1k_matches_oracle(qrl, oracle):
    """_2fsk_1k (the band-filter 2FSK modulator at 50 samples per symbol, feeding the 2FSK-1K receiver): three uneven calls"""
    C, n = 2, 60
    data = np.random.default_rng(5210).integers(0, 256, (C, n), dtype=np.uint8)
    tx = qrl.make_gr_mod_2fsk(50, 1000000, 1700, 2000, False, n_channels=C, max_items=n)
    try:
        got = np.concatenate([tx.work(data[:, a:b]) for a, b in ((0, 1), (1, 23), (23, n))], axis=1)
    finally:
        tx.close()
    for c in range(C):
        want = oracle.Tx(oracle.MOD_2FSK, 50, 1000000, 1700, 2000, 0).work(data[c])
        assert got.shape[1] == len(want) and np.array_equal(got[c], want), c
