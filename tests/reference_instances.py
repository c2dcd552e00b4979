"""Every receive and transmit instance the reference builds, and the test that holds it to the oracle.

gr_demod_base.cpp and gr_mod_base.cpp construct a fixed set of hier blocks, one per mode a user can pick; those instances are what the
library has to reproduce.  One row per instance: its line, the factory and its arguments as the reference passes them
(INTERNAL_DEFAULT_SAMPLE_RATE written as 1000000, freedv_api::MODE_x as the string "MODE_x", other identifiers as strings), what the
suite runs for it, and the test.  What the suite runs is a key of test_gpu_dispatch.RX / TX or a name of test_gpu_tx.TX_CASES where one
of those tables already holds the instance (the factory and oracle arguments are read from that row, not restated here), else the
oracle construction itself.  Receivers also name the transmit instance whose output the test demodulates and the frames it must
recover.  tests/test_reference_instances.py checks the table against the reference's sources where those exist, and every row
against the table it points into."""
from typing import NamedTuple

import numpy as np

from tests import siggen
from tests.test_gpu_dispatch import F4, P, RX, TX, _tx_burst
from tests.test_gpu_tx import TX_CASES

FILES = {True: "src/gr/gr_demod_base.cpp", False: "src/gr/gr_mod_base.cpp"}
RATE = 1000000                   # INTERNAL_DEFAULT_SAMPLE_RATE


class Instance(NamedTuple):
    var: str                     # the member gr_demod_base / gr_mod_base assigns
    line: int                    # its line in FILES[rx]
    factory: str
    args: tuple                  # as the reference passes them
    suite: object                # RX / TX key, TX_CASES name, or (oracle class, oracle kind, oracle args)
    test: str                    # "tests/<module>.py::<test>"
    feed: str = None             # receivers: the transmit instance feeding the test (None: a synthetic signal)

    @property
    def rx(self):
        return self.factory.startswith("make_gr_demod_")


DISPATCH, TXT, BPSK2FSK, FREEDV = "tests/test_gpu_dispatch.py", "tests/test_gpu_tx.py", "tests/test_gpu_bpsk_2fsk.py", "tests/test_gpu_freedv.py"
NEW = "tests/test_gpu_reference_instances.py"
SWEEP = DISPATCH + "::test_rx_channel_count_sweep"
TXSWEEP = DISPATCH + "::test_tx_channel_count_sweep"
ALL_TX = TXT + "::test_tx_all_digital_modes"
D2, M2 = "make_gr_demod_2fsk", "make_gr_mod_2fsk"

RX_INSTANCES = [
    Instance("_2fsk_2k_fm", 203, D2, (5, RATE, 1700, 4000, True), "2fsk", BPSK2FSK + "::test_2fsk_2k_fm_parity", "_2fsk_2k_fm"),
    Instance("_2fsk_1k_fm", 204, D2, (10, RATE, 1700, 2500, True), "2fsk1kfm", NEW + "::test_rx_instance_parity", "_2fsk_1k_fm"),
    Instance("_2fsk_2k", 205, D2, (5, RATE, 1700, 4000, False), "2fsk_band", BPSK2FSK + "::test_2fsk_2k_band_filter_variant", "_2fsk_2k"),
    Instance("_2fsk_1k", 206, D2, (10, RATE, 1700, 2000, False), "2fsk1k", NEW + "::test_rx_instance_parity", "_2fsk_1k"),
    Instance("_2fsk_10k", 207, D2, (1, RATE, 1700, 25000, True), ("Rx", "DEMOD_2FSK", (1, RATE, 1700, 25000, 1)),
             "tests/test_gpu_fast_modes.py::test_fast_mode_parity", "_2fsk_10k"),
    Instance("_gmsk_2k", 208, "make_gr_demod_gmsk", (5, RATE, 1700, 4000), "gmsk", SWEEP, "_2fsk_2k_fm"),
    Instance("_gmsk_1k", 209, "make_gr_demod_gmsk", (10, RATE, 1700, 2000), ("Rx", "DEMOD_GMSK", (10, RATE, 1700, 2000, 0)),
             BPSK2FSK + "::test_gmsk_demod_parity", "_2fsk_1k_fm"),
    Instance("_gmsk_10k", 210, "make_gr_demod_gmsk", (1, RATE, 1700, 20000), "gmsk10k", NEW + "::test_rx_instance_parity", "_gmsk_10k"),
    Instance("_4fsk_2k", 211, "make_gr_demod_4fsk", (5, RATE, 1700, 4000, False), "4fsk_disc", SWEEP, "_4fsk_2k"),
    Instance("_4fsk_2k_fm", 212, "make_gr_demod_4fsk", (5, RATE, 1700, 3000, True), "4fsk", SWEEP, "_4fsk_2k_fm"),
    Instance("_4fsk_1k_fm", 213, "make_gr_demod_4fsk", (10, RATE, 1700, 2000, True), "4fsk1k", SWEEP, "_4fsk_1k_fm"),
    Instance("_4fsk_10k_fm", 214, "make_gr_demod_4fsk", (1, RATE, 1700, 20000, True), "4fsk10k", SWEEP, "_4fsk_10k_fm"),
    Instance("_am", 215, "make_gr_demod_am", (125, RATE, 1700, 5000), "am", SWEEP),
    Instance("_bpsk_1k", 216, "make_gr_demod_bpsk", (10, RATE, 1700, 1300), "bpsk1k", NEW + "::test_rx_instance_parity", "_bpsk_1k"),
    Instance("_bpsk_2k", 217, "make_gr_demod_bpsk", (5, RATE, 1700, 2400), "bpsk", BPSK2FSK + "::test_bpsk_2k_parity", "_bpsk_2k"),
    Instance("_bpsk_dsss_8", 218, "make_gr_demod_dsss", (25, RATE, 1700, 150), "dsss", "tests/test_gpu_dsss.py::test_dsss_parity_and_decoded_bytes",
             "_bpsk_dsss_8"),
    Instance("_fm_2500", 219, "make_gr_demod_nbfm", (125, RATE, 1700, 2500), ("Rx", "DEMOD_NBFM", (125, RATE, 1700, 2500, 0)),
             "tests/test_gpu_nbfm.py::test_nbfm_parity"),
    Instance("_fm_5000", 220, "make_gr_demod_nbfm", (125, RATE, 1700, 5000), "nbfm", SWEEP),
    Instance("_qpsk_2k", 221, "make_gr_demod_qpsk", (125, RATE, 1700, 1300), "qpsk2k", NEW + "::test_rx_instance_parity", "_qpsk_2k"),
    Instance("_qpsk_10k", 222, "make_gr_demod_qpsk", (25, RATE, 1700, 6500), "qpsk20k", SWEEP, "_qpsk_10k"),
    Instance("_qpsk_250k", 223, "make_gr_demod_qpsk", (2, RATE, 1700, 160000), "qpsk", SWEEP, "_qpsk_250k"),
    Instance("_qpsk_video", 224, "make_gr_demod_qpsk", (2, RATE, 1700, 160000), "qpsk", SWEEP, "_qpsk_video"),
    Instance("_4fsk_96k", 225, "make_gr_demod_4fsk", (2, RATE, 1700, 125000, True), "4fsk100k", SWEEP, "_4fsk_96k"),
    Instance("_usb", 226, "make_gr_demod_ssb", (125, RATE, 1700, 2700, 0), "usb", SWEEP),
    Instance("_lsb", 227, "make_gr_demod_ssb", (125, RATE, 1700, 2700, 1), "lsb", SWEEP),
    Instance("_wfm", 228, "make_gr_demod_wbfm", (125, RATE, 1700, 75000), "wbfm", SWEEP),
] + [
    Instance("_freedv_rx%s_%s" % (mode, "lsb" if sb else "usb"), line, "make_gr_demod_freedv", (125, RATE, 1700, fw, lo, "MODE_" + mode, sb),
             ("FreedvRx", None, (125, RATE, fw, lo, sb)), FREEDV + "::test_freedv_rx_parity")
    for mode, fw, lo, sb, line in (("1600", 2500, 200, 0, 229), ("700C", 2400, 600, 0, 233), ("700D", 2400, 600, 0, 235),
                                   ("800XA", 2500, 0, 0, 238), ("1600", 2500, 200, 1, 241), ("700C", 2400, 600, 1, 244),
                                   ("700D", 2400, 600, 1, 246), ("800XA", 2500, 0, 1, 248))
] + [
    Instance("_mmdvm_demod", 250, "make_gr_demod_mmdvm", (), ("MmdvmRx", None, (5000, True)), "tests/test_gpu_mmdvm.py::test_single_channel_mmdvm_blocks"),
    Instance("_mmdvm_demod_multi", 251, "make_gr_demod_mmdvm_multi2",
             ("burst_timer", "_mmdvm_channels", "mmdvm_channel_separation", "_use_tdma"), ("MmdvmRx", None, (5000, False)),
             "tests/test_gpu_mmdvm.py::test_rx_channel_chains_match_the_oracle"),
    Instance("_m17_demod", 252, "make_gr_demod_m17", (), "m17", SWEEP),
    Instance("_dmr_demod", 253, "make_gr_demod_dmr", (5, RATE), "dmr", SWEEP),
]

TX_INSTANCES = [
    Instance("_2fsk_2k_fm", 155, M2, (25, 1000000, 1700, 4000, True), "2fsk2kfm", ALL_TX),
    Instance("_2fsk_1k_fm", 156, M2, (50, 1000000, 1700, 2500, True), "2fsk1kfm", ALL_TX),
    Instance("_2fsk_2k", 157, M2, (25, 1000000, 1700, 4000, False), "2fsk2k", ALL_TX),
    Instance("_2fsk_1k", 158, M2, (50, 1000000, 1700, 2000, False), ("Tx", "MOD_2FSK", (50, 1000000, 1700, 2000, 0)),
             NEW + "::test_tx_2fsk_1k_matches_oracle"),
    Instance("_2fsk_10k", 159, M2, (5, 1000000, 1700, 25000, True), "2fsk10kfm", ALL_TX),
] + [
    Instance("_gmsk_%s" % k, line, "make_gr_mod_gmsk", (sps, 1000000, 1700, fw), ("Tx", "MOD_GMSK", (sps, 1000000, 1700, fw, 0)),
             TXT + "::test_tx_gmsk_matches_oracle_and_loops_back")
    for k, line, sps, fw in (("2k", 160, 50, 4000), ("1k", 161, 100, 2000), ("10k", 162, 10, 20000))
] + [
    Instance("_4fsk_2k", 163, "make_gr_mod_4fsk", (25, 1000000, 1700, 4000, False), "4fsk2k", ALL_TX),
    Instance("_4fsk_2k_fm", 164, "make_gr_mod_4fsk", (25, 1000000, 1700, 3500, True), "4fsk2kfm", TXSWEEP),
    Instance("_4fsk_1k_fm", 165, "make_gr_mod_4fsk", (50, 1000000, 1700, 2000, True), "4fsk1kfm", ALL_TX),
    Instance("_4fsk_10k_fm", 166, "make_gr_mod_4fsk", (5, 1000000, 1700, 20000, True), "4fsk10kfm", ALL_TX),
    Instance("_am", 167, "make_gr_mod_am", (125, 1000000, 1700, 5000), "am", TXSWEEP),
    Instance("_bpsk_1k", 168, "make_gr_mod_bpsk", (500, 1000000, 1700, 1500), "bpsk1k", ALL_TX),
    Instance("_bpsk_2k", 169, "make_gr_mod_bpsk", (250, 1000000, 1700, 2800), "bpsk2k", ALL_TX),
    Instance("_bpsk_dsss_8", 170, "make_gr_mod_dsss", (25, 1000000, 1700, 200), "dsss", TXSWEEP),
    Instance("_fm_2500", 171, "make_gr_mod_nbfm", (20, 1000000, 1700, 2500), ("Tx", "MOD_NBFM", (20, 1000000, 1700, 2500, 0)),
             TXT + "::test_tx_analog_modulators"),
    Instance("_fm_5000", 172, "make_gr_mod_nbfm", (20, 1000000, 1700, 5000), "nbfm", TXSWEEP),
    Instance("_qpsk_2k", 173, "make_gr_mod_qpsk", (500, 1000000, 1700, 1300), "qpsk2k", ALL_TX),
    Instance("_qpsk_10k", 174, "make_gr_mod_qpsk", (100, 1000000, 1700, 6500), "qpsk20k", ALL_TX),
    Instance("_qpsk_250k", 175, "make_gr_mod_qpsk", (4, 1000000, 1700, 160000), "qpsk", TXSWEEP),
    Instance("_qpsk_video", 176, "make_gr_mod_qpsk", (4, 1000000, 1700, 160000), "qpsk", TXSWEEP),
    Instance("_4fsk_96k", 177, "make_gr_mod_4fsk", (2, 1000000, 1700, 125000, True), "4fsk100k", ALL_TX),
    Instance("_usb", 178, "make_gr_mod_ssb", (125, 1000000, 1700, 2700, 0), "usb", TXSWEEP),
    Instance("_lsb", 179, "make_gr_mod_ssb", (125, 1000000, 1700, 2700, 1), "lsb", TXSWEEP),
    Instance("_usb_cw", 180, "make_gr_mod_ssb", (125, 1000000, 1700, 1000, 0), ("Tx", "MOD_SSB", (125, 1000000, 1700, 1000, 0)),
             NEW + "::test_tx_usb_cw_matches_oracle_and_loops_back"),
] + [
    Instance("_freedv_tx%s_%s" % (mode, "lsb" if sb else "usb"), line, "make_gr_mod_freedv", (125, 1000000, 1700, fw, lo, "MODE_" + mode, sb),
             ("FreedvTx", None, (125, 1000000, fw, lo, sb)), test)
    for mode, fw, lo, sb, line, test in (
        ("1600", 2500, 200, 0, 181, TXSWEEP),
        ("700C", 2700, 300, 0, 186, FREEDV + "::test_freedv_tx_parity_and_bb_gain"),
        ("700D", 2700, 300, 0, 188, FREEDV + "::test_freedv_tx_parity_and_bb_gain"),
        ("800XA", 2700, 200, 0, 191, NEW + "::test_tx_freedv_2700_200_matches_oracle"),
        ("1600", 2700, 200, 1, 194, NEW + "::test_tx_freedv_2700_200_matches_oracle"),
        ("700C", 2700, 300, 1, 197, FREEDV + "::test_freedv_tx_parity_and_bb_gain"),
        ("700D", 2700, 300, 1, 199, FREEDV + "::test_freedv_tx_parity_and_bb_gain"),
        ("800XA", 2700, 200, 1, 202, NEW + "::test_tx_freedv_2700_200_matches_oracle"))
] + [
    Instance("_mmdvm_mod", 204, "make_gr_mod_mmdvm", (), ("MmdvmTx", None, (5000, True)), "tests/test_gpu_mmdvm.py::test_single_channel_mmdvm_blocks"),
    Instance("_mmdvm_mod_multi", 205, "make_gr_mod_mmdvm_multi2",
             ("burst_timer", "_mmdvm_channels", "mmdvm_channel_separation", "_use_tdma"), ("MmdvmTx", None, (5000, False)),
             "tests/test_gpu_mmdvm.py::test_tx_channel_chains_match_the_oracle"),
    Instance("_m17_mod", 206, "make_gr_mod_m17", (), "m17", TXSWEEP),
    Instance("_dmr_mod", 207, "make_gr_mod_dmr", (), "dmr", TXSWEEP),
]

INSTANCES = RX_INSTANCES + TX_INSTANCES
TX_BY_VAR = {i.var: i for i in TX_INSTANCES}


# ------------------------------------------------------------------ the receive instances test_gpu_dispatch.RX does not hold
N_FRAMES = 24          # frames per channel: the payload check asks for N - 6 back, the first ones fall into acquisition


def _burst(seed, tx_var, fo=150.0):
    """P channels of N_FRAMES voice frames from the oracle's modulator of the feeding instance, through the channel of
    test_gpu_bpsk_2fsk.py (offset, phase, delay up to 300 samples, 18 dB SNR, amplitude 0.1)"""
    def gen(O, T):
        okind, oargs = oracle_of(TX_BY_VAR[tx_var])[1:]
        return _tx_burst(O, seed, T, okind, oargs, frames=N_FRAMES, fo=fo, snr=18.0, amp=0.1, phase=True)
    return gen


# name -> test_gpu_dispatch.RX's six fields (factory, oracle factory, ports, T, minimum port lengths at T, frames) and the base
# signals gen(O, T) -> (P channels, payloads); the dispatch harness takes such a row as its `row` argument.
# T carries the preamble, N_FRAMES frames and the tail at the feeding modulator's 4000 (QPSK-2K), 8000 (1K) or 800 (GMSK-10K)
# samples per byte, plus the channel's delay; the minimum lengths are 90 % of what the oracle gives at T.
NEW_RX = {
    "qpsk2k": (lambda q, n, m: q.make_gr_demod_qpsk(125, RATE, 1700, 1300, n_channels=n, max_samples=m),
               lambda O: O.Rx(O.DEMOD_QPSK, 125, RATE, 1700, 1300, 0), 3, 1150000, (10000, 2000, 1900), (2,) + F4,
               _burst(221, "_qpsk_2k")),
    "bpsk1k": (lambda q, n, m: q.make_gr_demod_bpsk(10, RATE, 1700, 1300, n_channels=n, max_samples=m),
               lambda O: O.Rx(O.DEMOD_BPSK, 10, RATE, 1700, 1300, 0), 4, 2250000, (40000, 4000, 1900, 1900), ((2, 3),) + F4,
               _burst(216, "_bpsk_1k")),
    "2fsk1kfm": (lambda q, n, m: q.make_gr_demod_2fsk(10, RATE, 1700, 2500, True, n_channels=n, max_samples=m),
                 lambda O: O.Rx(O.DEMOD_2FSK, 10, RATE, 1700, 2500, 1), 4, 2250000, (40000, 4000, 1900, 1900), ((2, 3),) + F4,
                 _burst(204, "_2fsk_1k_fm")),
    "2fsk1k": (lambda q, n, m: q.make_gr_demod_2fsk(10, RATE, 1700, 2000, False, n_channels=n, max_samples=m),
               lambda O: O.Rx(O.DEMOD_2FSK, 10, RATE, 1700, 2000, 0), 4, 2250000, (40000, 4000, 1900, 1900), ((2, 3),) + F4,
               _burst(206, "_2fsk_1k", fo=60.0)),
    "gmsk10k": (lambda q, n, m: q.make_gr_demod_gmsk(1, RATE, 1700, 20000, n_channels=n, max_samples=m),
                lambda O: O.Rx(O.DEMOD_GMSK, 1, RATE, 1700, 20000, 0), 4, 230000, (16000, 4000, 1900, 1900), ((2, 3),) + F4,
                _burst(210, "_gmsk_10k")),
}


# ------------------------------------------------------------------ the same receivers with their loop limits reached
def _rate(x, up, down):
    """the modulator's output resampled by up / down (scipy's polyphase resampler): every symbol lasts up / down as long"""
    from scipy.signal import resample_poly
    return resample_poly(x, up, down).astype(np.complex64)


def _chirp(x, f_end, fs=1e6):
    """a carrier offset sweeping linearly from 0 to f_end Hz over the signal"""
    n = np.arange(len(x))
    return (x * np.exp(2j * np.pi * np.cumsum(f_end * n / len(x)) / fs)).astype(np.complex64)


def _stressed(seed, tx_var, bend):
    """P channels of random bytes from the feeding modulator, bent by `bend` (the whole stream at once), then the channel of _burst
    without its offset; no payloads: the loops sit at their limits, where the frames are not expected to survive"""
    def gen(O, T):
        okind, oargs = oracle_of(TX_BY_VAR[tx_var])[1:]
        X = np.zeros((P, T), np.complex64)
        for c in range(P):
            rng = np.random.default_rng(seed + c)
            iq = bend(O.Tx(getattr(O, okind), *oargs).work(rng.integers(0, 256, 320, dtype=np.uint8)))
            X[c] = siggen.channel(iq, rng, phase=rng.uniform(0, 6.28), delay=int(rng.integers(0, 300)), snr_db=18.0, amp=0.1, total=T)
        return X, None
    return gen


# The limits the channels of NEW_RX never reach.  BPSK-1K: clock_recovery_mm clamps omega to 10 +- 0.01 (omega_lim = 0.001 sps), and
# a symbol rate 1 % fast drives it there within 2.25 M samples (the loop's gain_omega of 2.5e-5 makes it slow); the band-edge FLL of
# BPSK-1K and of both 2FSK-1K receivers clamps at 2 pi 0.2 rad per 20 ksps sample = 4 kHz, which an offset sweeping to 9 kHz passes.
# (QPSK-2K's FLL limit, 2 pi 0.4 at 10 ksps = 4 kHz, lies at the edge of its 5 kHz stage-1 low-pass: a signal out there is filtered
# away before the FLL sees it; GMSK has no FLL and its period clamp is +-0.05 samples.)  Same handles, no frame check.
def _stress_row(name, T, mins, gen):
    return NEW_RX[name][:3] + (T, mins, None, gen)


STRESS_RX = {
    "bpsk1k-rate": ("bpsk1k", _stress_row("bpsk1k", 2250000, (40000, 4000, 1900, 1900),
                                          _stressed(4216, "_bpsk_1k", lambda x: _rate(x, 99, 100)))),
    "bpsk1k-sweep": ("bpsk1k", _stress_row("bpsk1k", 800000, (14000, 1400, 650, 650),
                                           _stressed(4217, "_bpsk_1k", lambda x: _chirp(x[:800000], 9000.0)))),
    "2fsk1kfm-sweep": ("2fsk1kfm", _stress_row("2fsk1kfm", 800000, (14000, 1400, 650, 650),
                                               _stressed(4204, "_2fsk_1k_fm", lambda x: _chirp(x[:800000], 9000.0)))),
    "2fsk1k-sweep": ("2fsk1k", _stress_row("2fsk1k", 800000, (14000, 1400, 650, 650),
                                           _stressed(4206, "_2fsk_1k", lambda x: _chirp(x[:800000], 9000.0)))),
}


# ------------------------------------------------------------------ reading what a row runs
class _Recorder:
    """stands in for the package or the oracle module: records the call a factory lambda makes"""

    def __getattr__(self, name):
        if name.startswith(("make_", "Rx", "Tx")):
            return lambda *a, **kw: (name,) + tuple(a)
        return name


def suite_row(inst):
    """the row of test_gpu_dispatch.RX / TX, NEW_RX or test_gpu_tx.TX_CASES the instance points at, or None"""
    if not isinstance(inst.suite, str):
        return None
    if inst.rx:
        return NEW_RX[inst.suite] if inst.suite in NEW_RX else RX[inst.suite]
    for case in TX_CASES:
        if case[0] == inst.suite:
            return case
    return TX[inst.suite]


def factory_of(inst):
    """(factory name, positional arguments) the suite's handle is made with, or None where the test builds it itself"""
    row = suite_row(inst)
    if row is None:
        return None
    if isinstance(row[0], str):                                   # TX_CASES
        return row[1], tuple(row[2])
    call = row[0](_Recorder(), 1, 1)
    return call[0], call[1:]


def oracle_of(inst):
    """(oracle class, kind, arguments) the suite compares the instance with"""
    row = suite_row(inst)
    if row is None:
        return tuple(inst.suite)
    if isinstance(row[0], str):                                   # TX_CASES
        return "Tx", row[3], tuple(row[4])
    if inst.var.startswith("_freedv"):
        return ("FreedvRx" if inst.rx else "FreedvTx", None, (125, RATE, inst.args[3], inst.args[4], inst.args[6]))
    call = row[1](_Recorder())
    return call[0], call[1], tuple(call[2:])


def frame_of(inst):
    """receivers: (ports, sync word, sync bits, frame bytes) the test finds its payloads with, None where it decodes no frames"""
    row = suite_row(inst)
    return row[5] if inst.rx and row is not None else None
