"""GPU tier: FreeDV up to the codec2 modem boundary (QRL_DEMOD_FREEDV / QRL_MOD_FREEDV) against the CPU oracle, bit for bit: every
(filter_width, low_cutoff) pair of the reference's instances on both side bands with ragged chunks, the AGC setters and a carrier
retune mid-stream, the modulator with bb_gain changes, the known answers, and a TX -> RX loop-back of a multi-tone modem signal."""
import numpy as np
import pytest

from tests import freedv_oracle as FO
from tests import test_freedv as TF
from tests.golden import freedv_cases as F

pytestmark = pytest.mark.gpu

PAIRS = [(2500, 200), (2400, 600), (2500, 0)]          # gr_demod_base.cpp:229-249 (1600 / 700C-700D / 800XA)
SIZES = [1, 99999, 124, 1, 60000, 7, 125, 250]


def rx_signal(sb, C, T, seed):
    sign = -1.0 if sb else 1.0
    rng = np.random.default_rng(seed)
    n = np.arange(T)
    X = np.zeros((C, T), np.complex64)
    for c in range(C):
        x = 0.03 * np.exp(2j * np.pi * sign * (650 + 400 * c) * n / 1e6) * (1 + 0.7 * np.sin(2 * np.pi * 2 * n / 1e6))
        x = x + 0.01 * np.exp(2j * np.pi * sign * 2200 * n / 1e6) + 0.02 * np.exp(-2j * np.pi * sign * 1200 * n / 1e6)
        x = x + 0.003 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))
        x[:777] = 0
        X[c] = x.astype(np.complex64)
    return X


def run_chunked(blk, X, sizes, between=None):
    C, T = X.shape
    acc = [[[] for _ in range(C)] for _ in range(2)]
    a, i = 0, 0
    while a < T:
        m = min(sizes[i % len(sizes)], T - a); i += 1
        if between:
            between(a)
        blk.work(X[:, a:a + m]); a += m
        for p in range(2):
            for c, v in enumerate(blk.read_port(p)):
                acc[p][c].append(v)
    return [[np.concatenate(acc[p][c]) for c in range(C)] for p in range(2)]


@pytest.mark.parametrize("sb", [0, 1])
@pytest.mark.parametrize("fw,lo", PAIRS)
def test_freedv_rx_parity(qrl, sb, fw, lo):
    C, T = 3, 420000
    X = rx_signal(sb, C, T, 300 + fw + lo + sb)
    blk = qrl.make_gr_demod_freedv(125, 1000000, 1700, fw, lo, 0, sb, n_channels=C, max_samples=100000)
    assert blk.read_port(1)[0].dtype == np.int16
    got = run_chunked(blk, X, SIZES)
    for c in range(C):
        w0, w1 = FO.FreedvRx(125, 1000000, fw, lo, sb).work(X[c])
        assert len(got[0][c]) == len(w0) == len(got[1][c]) == len(w1) == T // 125
        assert np.array_equal(got[0][c], w0) and np.array_equal(got[1][c], w1), (c, sb, fw, lo)
        assert np.max(np.abs(w1[1000:].astype(np.int32))) > 1000        # the AGC lifted the modem samples


def test_freedv_rx_setters_mid_stream(qrl):
    """set_agc_attack / set_agc_decay (gr_demod_freedv.cpp:85-93) and a carrier retune between calls, the oracle cut the same way"""
    C, T = 3, 300000
    X = rx_signal(0, C, T, 900)
    sizes = [100124, 59876, 60000, 80000]
    events = {100124: ("attack", 0.5), 160000: ("decay", 0.02), 220000: ("retune", 350.0)}
    blk = qrl.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=C, max_samples=max(sizes))
    ors = [FO.FreedvRx(125, 1000000, 2500, 200, 0) for _ in range(C)]

    def apply(a):
        if a not in events:
            return
        kind, v = events[a]
        if kind == "retune":
            blk.set_carrier_offset(v)
            for o in ors:
                o.set_carrier_offset(v)
            return
        key = qrl.PARAM.AGC_ATTACK if kind == "attack" else qrl.PARAM.AGC_DECAY
        blk.set_param(key, v)
        for o in ors:
            o.set_param(key, v)

    got = [[[] for _ in range(C)] for _ in range(2)]
    want = [[[] for _ in range(C)] for _ in range(2)]
    a = 0
    for m in sizes:
        apply(a)
        blk.work(X[:, a:a + m])
        for p in range(2):
            for c, v in enumerate(blk.read_port(p)):
                got[p][c].append(v)
        for c in range(C):
            p0, p1 = ors[c].work(X[c, a:a + m])
            want[0][c].append(p0); want[1][c].append(p1)
        a += m
    base = [FO.FreedvRx(125, 1000000, 2500, 200, 0).work(X[c]) for c in range(C)]
    for c in range(C):
        for p in range(2):
            w = np.concatenate(want[p][c])
            assert np.array_equal(np.concatenate(got[p][c]), w), (c, p)
            assert not np.array_equal(w, base[c][p])                  # the setters changed the stream


@pytest.mark.parametrize("sb", [0, 1])
def test_freedv_tx_parity_and_bb_gain(qrl, sb):
    tx_parity_case(qrl, 300, sb)


def tx_parity_case(qrl, lo, sb):
    """make_gr_mod_freedv(125, 1e6, 1700, 2700, lo, ..., sb) against the oracle over ragged calls with two bb_gain changes"""
    C, n = 3, 9000
    rng = np.random.default_rng(950 + sb)
    t = np.arange(n) / 8000.0
    S = np.stack([(5000 * np.sin(2 * np.pi * (500 + 300 * c) * t) + 1500 * rng.standard_normal(n)).astype(np.int16) for c in range(C)])
    S[:, 3000:3600] = 0
    tx = qrl.make_gr_mod_freedv(125, 1000000, 1700, 2700, lo, 0, sb, n_channels=C, max_items=4000)
    ors = [FO.FreedvTx(125, 1000000, 2700, lo, sb) for _ in range(C)]
    a, i, sizes = 0, 0, [1, 4000, 511, 1, 2000, 2487]
    gains = {4001: 0.5, 6513: 1.7}
    while a < n:
        m = min(sizes[i % len(sizes)], n - a); i += 1
        if a in gains:
            tx.set_bb_gain(gains[a])
            for o in ors:
                o.set_bb_gain(gains[a])
        out = tx.work_modem(S[:, a:a + m])
        assert out.shape == (C, 125 * m)
        for c in range(C):
            assert np.array_equal(out[c].view(np.float32), ors[c].work(S[c, a:a + m]).view(np.float32)), (c, a, m)
        a += m


@pytest.mark.parametrize("name", sorted(F.RX_CASES))
def test_freedv_rx_golden(qrl, name):
    TF.golden_rx_through(qrl, name)


@pytest.mark.parametrize("name", sorted(F.TX_CASES))
def test_freedv_tx_golden(qrl, name):
    TF.golden_tx_through(qrl, name)


def test_freedv_einval(qrl):
    TF.einval_paths(qrl)


def test_freedv_loopback(qrl):
    """Device TX -> device RX: every tone of a multi-tone int16 modem signal comes back at its frequency within 2 Hz on port 0 of the
    USB handle, and the LSB handle on the same IQ sees at least 40 dB less power (port 0: port 1 sits behind an AGC that would lift the
    rejected side band)."""
    C, n = 3, 24000
    tones = [(500, 1100, 2100), (700, 1500, 2300), (400, 900, 1900)]
    t = np.arange(n) / 8000.0
    S = np.stack([sum(3000 * np.sin(2 * np.pi * f * t + k) for k, f in enumerate(tt)).astype(np.int16) for tt in tones])
    tx = qrl.make_gr_mod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=C, max_items=n)
    iq = tx.work_modem(S)
    assert iq.shape == (C, 125 * n)
    usb = qrl.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, n_channels=C, max_samples=iq.shape[1])
    lsb = qrl.make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 1, n_channels=C, max_samples=iq.shape[1])
    usb.work(iq); lsb.work(iq)
    u0, l0, u1 = usb.read_port(0), lsb.read_port(0), usb.read_port(1)
    for c in range(C):
        assert len(u0[c]) == len(u1[c]) == n
        y = u0[c][8000:].astype(np.complex128)                      # after the AGC has settled: 2 s
        spec = np.abs(np.fft.fft(y * np.hanning(len(y)), 8 * len(y)))
        f = np.fft.fftfreq(8 * len(y), 1 / 8000.0)
        for ft in tones[c]:
            sel = np.abs(f - ft) < 30
            fpk = f[sel][np.argmax(spec[sel])]
            assert abs(fpk - ft) <= 2.0, (c, ft, fpk)
        pu = np.mean(np.abs(u0[c][8000:]) ** 2)
        pl = np.mean(np.abs(l0[c][8000:]) ** 2)
        assert 10 * np.log10(pu / max(pl, 1e-30)) >= 40.0, (c, pu, pl)
        assert np.max(np.abs(u1[c][8000:].astype(np.int32))) > 1000


def test_freedv_cpp_mirror_loopback(tmp_path):
    """The C++ mirror (include/qrl_b200_gr.hpp make_gr_mod_freedv / make_gr_demod_freedv) runs the loop-back of tests/cpp."""
    import os
    import subprocess
    from tests.test_freedv import test_cpp_freedv_adapter_compiles
    test_cpp_freedv_adapter_compiles(tmp_path)
    out = subprocess.run([os.path.join(str(tmp_path), "test_freedv_adapter")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), out.stdout + out.stderr
