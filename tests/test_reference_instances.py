"""CPU tier: the reference's receive and transmit instances (tests/reference_instances.py).

The five receivers no other table holds -- QPSK-2K, BPSK-1K, 2FSK-1K-FM, 2FSK-1K and GMSK-10K -- each select create-time branches of
qrl_rx_create that nothing else reaches (QPSK sps >= 125: /100 to 10 ksps, 5 samples per symbol, 2727 stage-1 taps; 2FSK / GMSK
sps == 10 and sps == 1; BPSK at omega = 10).  Here the oracle itself recovers the frames its own modulator sends at each of them,
the host-thread build of the library is bit-identical to the oracle on a short ragged stream and with its loop limits reached, the table matches the rows it points
into, and, where the reference's sources are present, every instance they build has a row naming a test that exists."""
import os
import re

import numpy as np
import pytest

from tests import reference_instances as R
from tests import siggen
from tests import test_gpu_dispatch as D
from tests.test_emulated_library import emu_qrl, rx_through_the_emulated_library  # noqa: F401  (emu_qrl: module-scoped fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("QRL_REFERENCE", "/root/reference")      # where oracle/Makefile's REF points by default


# ------------------------------------------------------------------ the oracle against a known answer
@pytest.mark.parametrize("name", sorted(R.NEW_RX))
def test_oracle_loopback_recovers_frames(oracle, name):
    """oracle TX of the feeding instance -> channel -> oracle RX: at least N - 6 of the N payloads come back on a decoded port"""
    row = R.NEW_RX[name]
    ports, sync, sbits, flen = row[5]
    B, payloads = D.bases(name, oracle, row[3], row)
    for c in range(2):
        rx = row[1](oracle)
        rx.work(B[c])
        got = [rx.port(p) for p in range(row[2])]
        good = max(siggen.count_good_frames(got[p], sync, sbits, flen, payloads[c])[0] for p in np.atleast_1d(ports))
        assert len(payloads[c]) == R.N_FRAMES and good >= R.N_FRAMES - 6, (name, c, good)


# ------------------------------------------------------------------ the host-thread build of the library
# the frame-carrying rows on a short stream; the loop-limit rows (reference_instances.STRESS_RX) as long as the limit takes to reach
EMU_T = {"qpsk2k": 90000, "bpsk1k": 120000, "2fsk1kfm": 120000, "2fsk1k": 120000, "gmsk10k": 60000}
EMU_ROWS = {**{k: v for k, v in R.NEW_RX.items()}, **{k: v[1] for k, v in R.STRESS_RX.items()}}


@pytest.mark.parametrize("name", sorted(EMU_ROWS))
def test_rx_instance_through_the_emulated_library(emu_qrl, oracle, name):  # noqa: F811
    """2 channels, a 1-sample call and cuts that are no multiple of the decimation, every port bit-identical to the oracle (the
    length rules of test_gpu_dispatch.check_rx)"""
    row = EMU_ROWS[name]
    rx_through_the_emulated_library(emu_qrl, oracle, name, row, EMU_T.get(name, row[3]))


# ------------------------------------------------------------------ the lean QPSK symbol sync's proof at every QPSK instance
def _qpsk_symsync_constants(sps):
    """qrl_rx_create's QPSK symbol-sync constants in float32 (clock_loop_gains, qrl_design.hpp; the sps ladder of gr_demod_qpsk.cpp)"""
    f = np.float32
    if 4 < sps < 125:
        tsr, sym_sps = 40000, sps * 4 // 25
    elif sps >= 125:
        tsr, sym_sps = 10000, sps // 25
    else:
        tsr, sym_sps = 500000, sps
    symbol_rate = f(tsr) / f(sym_sps)
    sps_dev = f(200.0) / symbol_rate
    bw = f(2 * np.pi / (float(symbol_rate) / 10))
    alpha = f(2.0) / f(0.2869) * np.exp(-bw, dtype=f) * np.sinh(bw, dtype=f)
    maxp, minp = f(sym_sps) + sps_dev, f(sym_sps) - sps_dev
    n0 = int(np.floor(minp - abs(alpha)))
    return sym_sps, alpha, maxp, minp, f(n0), n0


@pytest.mark.parametrize("inst", [i for i in R.RX_INSTANCES if i.factory == "make_gr_demod_qpsk"], ids=lambda i: i.var)
def test_qpsk_lean_symbol_sync_window_proof(inst):
    """qpsk_symsync<128, 2, true> runs the lean recurrence only where lean_ok && window_sure hold (symsync_kernel, qrl_kernels.cuh);
    qrl_b200.cu selects it for every QPSK instance on the claim that they do.  QPSK-2K is the one with 5 samples per symbol.  This is a
    restatement of qrl_rx_create's constants and of the kernel's condition, not an observation of the kernel: it shows the proof holds
    for these constants as written here, and a change to the C++ constants does not reach this copy.  The device output itself is held
    to the oracle in tests/test_gpu_reference_instances.py, where the generic recurrence would give the same bits."""
    sym_sps, alpha, maxp, minp, fl0, n0 = _qpsk_symsync_constants(inst.args[0])
    assert sym_sps == {125: 5, 25: 4, 2: 2}[inst.args[0]]
    lean_ok = minp > abs(alpha) and fl0 >= 1.0
    window_sure = lean_ok and (maxp + abs(alpha) + 1 < fl0 + 3 - np.float32(1e-3)) and (minp - abs(alpha) > fl0 + np.float32(1e-3)) \
        and fl0 == n0
    assert lean_ok and window_sure, (inst.var, sym_sps, alpha, maxp, minp, n0)


def test_qpsk_2k_oracle_stage_one_and_shaping_taps(oracle):
    """the oracle's QPSK-2K filter designs: 2727 stage-1 taps (low_pass_2 at 1 Msps, 5 kHz, 1 kHz transition, 60 dB) and an
    11 x 5-tap RRC.  Only the oracle is read here; that the device runs the tiled /100 stage 1 with these taps shows in the GPU tier
    (ports bit-identical to this oracle, no rotator launch under a carrier offset)"""
    rx = oracle.Rx(oracle.DEMOD_QPSK, 125, 1000000, 1700, 1300, 0)
    assert len(rx.taps(0)) == 2727
    assert len(rx.taps(1)) == 55


# ------------------------------------------------------------------ the table
def _test_exists(test):
    path, name = test.split("::")
    src = open(os.path.join(ROOT, path)).read()
    return re.search(r"^def %s\(" % re.escape(name), src, re.M) is not None


def _norm(args):
    return tuple(int(a) if isinstance(a, bool) else a for a in args)


def test_rows_match_the_tables_they_point_into():
    """a row's factory and oracle are those of the suite row it names; its test and feeding instance exist"""
    seen = set()
    for inst in R.INSTANCES:
        assert (inst.rx, inst.var) not in seen, inst.var
        seen.add((inst.rx, inst.var))
        assert _test_exists(inst.test), inst
        assert inst.feed is None or inst.feed in R.TX_BY_VAR, inst
        fac = R.factory_of(inst)
        if fac is not None:
            assert fac[0] == inst.factory, (inst.var, fac)
            assert fac[1] == () or _norm(fac[1]) == _norm(inst.args), (inst.var, fac)
        cls, kind, oargs = R.oracle_of(inst)
        if cls in ("Rx", "Tx"):
            assert inst.factory.endswith("_" + kind.split("_", 1)[1].lower()), (inst.var, kind)
            if inst.args and inst.factory != "make_gr_demod_dmr":
                assert _norm(oargs[:len(inst.args)]) == _norm(inst.args[:len(oargs)]), (inst.var, oargs)
        if inst.feed is not None and R.frame_of(inst) is not None:
            assert R.oracle_of(R.TX_BY_VAR[inst.feed])[0] == "Tx"


_CALL = re.compile(r"^\s*(_\w+)\s*=\s*(make_gr_(?:de)?mod_\w+)\s*\((.*?)\)\s*;", re.S | re.M)


def _parse_arg(tok):
    tok = " ".join(tok.split())
    if tok == "INTERNAL_DEFAULT_SAMPLE_RATE":
        return R.RATE
    if tok in ("true", "false"):
        return tok == "true"
    m = re.fullmatch(r"(?:gr::vocoder::)?freedv_api::(MODE_\w+)", tok)
    if m:
        return m.group(1)
    return int(tok) if re.fullmatch(r"-?\d+", tok) else tok


def reference_instances(path):
    src = open(path).read()
    out = []
    for m in _CALL.finditer(src):
        args = tuple(_parse_arg(a) for a in m.group(3).split(",")) if m.group(3).strip() else ()
        out.append((m.group(1), src.count("\n", 0, m.start(1)) + 1, m.group(2), args))
    return out


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "src", "gr")), reason="the reference's sources are not on this machine")
@pytest.mark.parametrize("rx", [True, False], ids=["gr_demod_base", "gr_mod_base"])
def test_every_reference_instance_has_a_row(rx):
    found = reference_instances(os.path.join(REF, R.FILES[rx]))
    rows = {(i.var, i.line, i.factory, i.args) for i in R.INSTANCES if i.rx == rx}
    missing = [f for f in found if f not in rows]
    assert not missing, missing
    assert len(found) == len(rows), sorted(rows - set(found))
