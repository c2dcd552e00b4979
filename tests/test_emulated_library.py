"""CPU tier: the library's OWN sources (qradiolink_b200/csrc/*.cu, *.cuh) compiled for host threads by tools/emu/build_emulated_lib.py
and driven through the real C ABI and the real Python wrappers -- handle creation, buffer sizing, launch geometry, slice pipelining,
the warp-specialised TMA producer / consumer kernels, the lean symbol-sync recurrence -- against the oracle and the committed golden
vectors.  The test bodies are the GPU tier's own (tests/test_golden.py, tests/test_gpu_*.py), called with the emulated build.

TEST INFRASTRUCTURE (DESIGN.md section 10a): the emulated library is built into a temporary directory, patched into the ctypes
loader for this module only and removed again; the package has no switch for it and no CPU fallback.  It says nothing about timing,
races on real hardware or the memory model -- that is the GPU tier's job; what it does catch is wrong indexing, wrong buffer sizes,
wrong launch geometry, state that does not carry across calls, and barrier mistakes (it found a missing __syncthreads in the SSB
audio kernel that the GPU's scheduling had been hiding)."""
import ctypes
import os
import sys

import numpy as np
import pytest

from tests.golden import cases
from tests import test_gpu_dispatch as D
from tests.test_gpu_dispatch import RX, TX, tx_bases

pytestmark = pytest.mark.timeout(900)      # pytest-timeout: a scheduling bug in the emulator must fail, not hang the tier

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_qrl(tmp_path_factory):
    sys.path.insert(0, os.path.join(ROOT, "tools", "emu"))
    from build_emulated_lib import build
    lib_path, n_sites = build(str(tmp_path_factory.mktemp("qrl_emu")))
    assert n_sites >= 60                                   # every kernel<<<...>>> launch site of the three translation units
    import qradiolink_b200 as q
    from qradiolink_b200 import lib as L
    saved = (L._LIB_PATH, L._LIB)
    L._LIB_PATH, L._LIB = lib_path, None
    q.load_library()
    assert L.device_count() == 1
    yield q
    L._LIB_PATH, L._LIB = saved


def rx_through_the_emulated_library(qrl, O, name, row, T):
    """2 channels, a 1-sample call and cuts that are no multiple of the decimation, every port bit-identical to the oracle under the
    length rules of test_gpu_dispatch.check_rx: port 0 as long as the oracle's, the others within SLACK, and empty only where the row's
    minimum length scaled to T is 0 and the oracle's port is empty too.  row: a row of test_gpu_dispatch.RX or of its form; the stream
    is the first T samples of the row's base signals"""
    B, _ = D.bases(name, O, row[3], row)
    X = np.ascontiguousarray(B[:2, :T])
    cuts = [(0, 1), (1, 30001), (30001, 30078), (30078, T)]
    blk = row[0](qrl, 2, max(hi - lo for lo, hi in cuts))
    try:
        got = D.concat_calls(D.run_rx(blk, X, cuts), blk.nports, 2)
    finally:
        blk.close()
    for c in range(2):
        rx = row[1](O)
        for lo, hi in cuts:
            rx.work(X[c, lo:hi])
        for p in range(blk.nports):
            g, w = got[p][c], rx.port(p)
            n = min(len(g), len(w))
            filled = n > 0 or (row[4][p] * T // row[3] == 0 and len(g) == len(w) == 0)
            assert abs(len(g) - len(w)) <= D.SLACK and filled and (p > 0 or len(g) == len(w)), (name, c, p, len(g), len(w))
            assert np.array_equal(g[:n], w[:n]), "%s: port %d of channel %d differs from the oracle" % (name, p, c)


# the cheaper golden cases (the 250 ksps QPSK chain takes minutes under emulation: GPU tier only)
@pytest.mark.parametrize("name", ["4fsk_2k_fm", "nbfm_2500", "am_5000", "bpsk_2k", "2fsk_2k_fm", "ssb_usb", "wbfm_75k", "m17"])
def test_golden_rx_through_the_emulated_library(emu_qrl, oracle, name):
    from tests import test_golden as TG
    assert name in cases.RX_CASES
    TG.test_golden_rx_cuda(emu_qrl, oracle, name)


@pytest.mark.parametrize("name", sorted(cases.TX_CASES))
def test_golden_tx_through_the_emulated_library(emu_qrl, name):
    from tests import test_golden as TG
    TG.test_golden_tx_cuda(emu_qrl, name)


# every row of the GPU tier's TX channel-count table, plus 4FSK-FM at 64 bytes per call (the three-stream pipelined path)
@pytest.mark.parametrize("name,n", [(k, TX[k][3]) for k in TX] + [("4fsk2kfm", 64)])
def test_tx_chain_through_the_emulated_library(emu_qrl, oracle, name, n):
    """2 channels, two calls (state carried across them), every output bit-identical to the oracle.  4FSK-FM runs its bit chain in
    8 slices per call (qrl_tx_profile stage 0) from 64 bytes per call on, in one launch per call below."""
    factory, ofactory, kind, _ = TX[name]
    D = tx_bases(kind, 2 * n)[:2]
    lib = emu_qrl.load_library()
    tx = factory(emu_qrl, 2, n)
    try:
        lib.qrl_tx_profile(tx._h, 1)
        work = {"bytes": tx.work, "audio": tx.work_audio, "modem": tx.work_modem}[kind]
        calls = [work(D[:, :n]), work(D[:, n:])]
        ms, cnt = ctypes.c_double(), ctypes.c_long()
        assert lib.qrl_tx_profile_read(tx._h, 0, ctypes.byref(ms), ctypes.byref(cnt)) == 0
    finally:
        tx.close()
    if name == "4fsk2kfm":
        assert cnt.value == (2 * 8 if n >= 64 else 0), (n, cnt.value)
    for c in range(2):
        o = ofactory(oracle)
        for k, got in enumerate(calls):
            want = o.work(D[c, k * n:(k + 1) * n])
            assert len(want) == got.shape[1] and np.array_equal(got[c], want), (name, c, k)


def test_tx_set_filter_width_and_ctcss_through_the_emulated_library(emu_qrl, oracle):
    """gr_mod_nbfm / gr_mod_ssb / gr_mod_am::set_filter_width and gr_mod_nbfm::set_ctcss between calls (tests/test_gpu_tx.py): new taps
    meet the rings' history, the tone source keeps its phase."""
    from tests import test_gpu_tx as TT
    TT.test_tx_nbfm_set_filter_width_mid_stream(emu_qrl, oracle)
    for kind in ("usb", "am"):
        TT.test_tx_ssb_am_set_filter_width_mid_stream(emu_qrl, oracle, kind)
    TT.nbfm_ctcss_case(emu_qrl, oracle)


def test_dmr_chain_through_the_emulated_library(emu_qrl, oracle):
    """QRL_DEMOD_DMR has not run on a GPU yet (tests/test_gpu_dmr.py is opt-in): here its real host path -- create, x3/125 generic
    stage 1, 1-tap stage 2, float port 3, symbol-sync variant 3, scaling epilogue, hard bits -- runs against the oracle."""
    from tests import test_gpu_dmr as TD
    TD.test_dmr_parity_chunked(emu_qrl, oracle)
    TD.test_dmr_refuses_overlapped_calls(emu_qrl)


def test_m17_modulator_through_the_emulated_library(emu_qrl, oracle):
    """QRL_MOD_M17 (tests/test_gpu_m17_tx.py is opt-in until a GPU run): real host path, state carried across three calls."""
    C, n = 2, 48
    data = np.random.default_rng(5400).integers(0, 256, (C, n), dtype=np.uint8)
    tx = emu_qrl.make_gr_mod_m17(n_channels=C, max_items=n)
    got = np.concatenate([tx.work(data[:, a:b]) for a, b in ((0, 1), (1, 20), (20, n))], axis=1)
    for c in range(C):
        want = oracle.Tx(oracle.MOD_M17, 125, 1000000, 1700, 9000, 0).work(data[c])
        assert got.shape[1] == len(want) == n * 4 * 5 * 125 // 3
        assert np.array_equal(got[c], want), c


def test_overlapped_calls_through_the_emulated_library(emu_qrl, oracle):
    """QRL_PARAM_OVERLAP_CALLS (double-buffered ports, ring fences, tail joins): same stream as serialised calls and as the oracle."""
    from tests import siggen
    from tests.test_gpu_4fsk import run_oracle, compare
    C, T = 3, 150000
    X, _ = siggen.gen_4fsk_channels(C, T, seed0=1000)
    want = run_oracle(oracle, X)
    blk = emu_qrl.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=C, max_samples=70001)
    blk.set_overlap(True)
    acc = [[[] for _ in range(C)] for _ in range(3)]
    lo, i, sizes = 0, 0, [1, 49, 50, 51, 70001, 12345, 33333, 7]
    while lo < T:
        n = min(sizes[i % len(sizes)], T - lo); i += 1
        blk.work(X[:, lo:lo + n]); lo += n
        for p in range(3):
            for c, v in enumerate(blk.read_port(p)):
                acc[p][c].append(v)
    compare([[np.concatenate(acc[p][c]) for c in range(C)] for p in range(3)], want, exact_float=True)


def test_channelizer_and_deframer_through_the_emulated_library(emu_qrl, oracle):
    from tests import test_gpu_pfb as TP
    from tests import test_gpu_framing as TF
    TP.test_channelizer_reference_config_bit_identical_and_chunked(emu_qrl, oracle)
    TP.test_synthesizer_matches_oracle_and_loops_back(emu_qrl, oracle)
    TF.test_deframer_record_overflow_drops_like_the_oracle(emu_qrl, oracle)


@pytest.mark.parametrize("single", [False, True])
def test_mmdvm_tx_zero_idle_through_the_emulated_library(emu_qrl, oracle, single):
    """gr_zero_idle_bursts(0) on the MMDVM modulators (qrl_mmdvm_tx_zero_samples): host bookkeeping of the tags + the clearing kernel
    between the stages, against the oracle, before GPU time is spent on it."""
    from tests import test_gpu_mmdvm as TM
    TM.zero_idle_case(emu_qrl, oracle, single, q=1)


def test_rx_reset_restarts_the_rotator_phase_through_the_emulated_library(emu_qrl):
    """qrl_rx_reset keeps each channel's carrier offset and restarts its phase at 0 (tests/test_gpu_rx_reset.py on every chain): a
    2500 Hz offset set after the first 20 000 samples, then a reset, must leave the next stream bit-identical to a fresh handle that
    had the offset before its first call"""
    from tests import siggen
    X = siggen.gen_nbfm_channels(1, 100000, seed0=5500)
    a = emu_qrl.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=1, max_samples=50000)
    b = emu_qrl.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=1, max_samples=50000)
    try:
        a.work(X[:, :20000])
        a.set_carrier_offset(2500.0)
        a.work(X[:, 20000:50000])
        a.reset()
        b.set_carrier_offset(2500.0)
        for blk in (a, b):
            blk.work(X[:, 50000:])
        for p in range(2):
            g, w = a.read_port(p)[0], b.read_port(p)[0]
            assert len(g) == len(w) > 0 and np.array_equal(g.view(np.uint8), w.view(np.uint8)), p
    finally:
        a.close(); b.close()


def test_rssi_switched_off_and_on_restarts_the_tap_through_the_emulated_library(emu_qrl, oracle):
    """QRL_PARAM_RSSI from 0 to 1 starts the tap afresh (tests/test_gpu_rx_reset.py): on for a loud call, off for a call 40 dB
    quieter, on again; the next call must read what rssi_block constructed at the re-enable reads"""
    from tests import siggen
    X = siggen.gen_nbfm_channels(1, 72000, seed0=5600)
    X[:, 50000:] *= np.float32(0.01)
    blk = emu_qrl.make_gr_demod_nbfm(125, 1000000, 1700, 5000, n_channels=1, max_samples=50000)
    try:
        blk.enable_rssi(True)
        blk.work(X[:, :50000])
        blk.enable_rssi(False)
        blk.work(X[:, 50000:70000])
        blk.enable_rssi(True)
        blk.work(X[:, 70000:])
        p0 = blk.read_port(0)[0]
        want = oracle.Rssi(0.0).work(p0)
        assert len(p0) > 0 and abs(float(blk.rssi()[0]) - want) < 1e-3, (float(blk.rssi()[0]), want)
    finally:
        blk.close()


def test_qpsk_chain_through_the_emulated_library(emu_qrl, oracle):
    """The QPSK-250k chain's loop kernels hand blocks between warps through 3-deep shared-memory rings (AGC -> Costas -> bulk store;
    symbol sync -> second Costas -> feed-forward epilogue): a short ragged stream through the real host code and kernels, ports
    bit-identical to the oracle.  (The golden QPSK case and the GPU tier's QPSK tests also pass under emulation; they take minutes.)"""
    from tests import siggen
    C, T = 2, 36000
    X, _ = siggen.gen_qpsk_channels(C, T, seed0=2300)
    blk = emu_qrl.make_gr_demod_qpsk(2, 1000000, 1700, 160000, n_channels=C, max_samples=20001)
    acc = [[[] for _ in range(C)] for _ in range(3)]
    lo = 0
    for n in (1, 20001, 3, T - 20005):
        blk.work(X[:, lo:lo + n]); lo += n
        for p in range(3):
            for c, v in enumerate(blk.read_port(p)):
                acc[p][c].append(v)
    assert lo == T
    for c in range(C):
        rx = oracle.Rx(oracle.DEMOD_QPSK, 2, 1000000, 1700, 160000, 0)
        rx.work(X[c])
        for p in range(3):
            g, w = np.concatenate(acc[p][c]), rx.port(p)
            n = min(len(g), len(w))
            assert n >= len(w) - (160 if p == 2 else 8), (c, p, len(g), len(w))
            assert np.array_equal(g[:n], w[:n]), (c, p)
        assert len(np.concatenate(acc[2][c])) > 3000           # several Viterbi frames came out


# stream lengths of the RX rows (default 60 000 samples, long enough for the first Viterbi frames): 4FSK-1K needs 120 000 for its
# first; the 250 ksps QPSK and 4FSK-100K chains, the slowest under emulation, decode within 40 000
RX_T = {"4fsk1k": 120000, "qpsk": 40000, "4fsk100k": 40000}


@pytest.mark.parametrize("name", sorted(RX))
def test_rx_chain_through_the_emulated_library(emu_qrl, oracle, name):
    """every receive chain of the GPU tier's channel-count table -- its create path, slice function and ports -- on the host-thread
    build, against the oracle"""
    rx_through_the_emulated_library(emu_qrl, oracle, name, RX[name], RX_T.get(name, 60000))
