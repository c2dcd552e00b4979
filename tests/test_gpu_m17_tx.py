"""GPU tier: M17 modulator (gr_mod_m17.cpp: bytes -> dibits -> map -> RRC x5 -> x0.66666666 -> frequency modulator -> 24 ksps low-pass
-> x0.9 -> x125 / 3 rational interpolator) against the CPU oracle, state carried across calls, then CUDA TX -> CUDA M17 RX.
"""
import numpy as np
import pytest

from tests import siggen

pytestmark = [pytest.mark.gpu]


@pytest.mark.parametrize("cuts", [(), (100,), (1, 7, 150)])
def test_tx_m17_matches_oracle_and_streams(qrl, oracle, cuts):
    C, nbytes = 3, 300
    rng = np.random.default_rng(5400)
    data = rng.integers(0, 256, (C, nbytes), dtype=np.uint8)
    tx = qrl.make_gr_mod_m17(n_channels=C, max_items=nbytes)
    edges = [0, *cuts, nbytes]
    got = np.concatenate([tx.work(data[:, a:b]) for a, b in zip(edges[:-1], edges[1:])], axis=1)
    for c in range(C):
        want = oracle.Tx(oracle.MOD_M17, 125, 1000000, 1700, 9000, 0).work(data[c])
        assert got.shape[1] == len(want) == nbytes * 4 * 5 * 125 // 3, (got.shape, len(want))
        assert np.array_equal(got[c], want), c


def test_tx_m17_loops_back_through_the_cuda_receiver(qrl):
    rng = np.random.default_rng(5401)
    data = rng.integers(0, 256, 300, dtype=np.uint8)
    iq = qrl.make_gr_mod_m17(n_channels=1, max_items=len(data)).work(data[None, :])[0]
    x = siggen.channel(iq, rng, fo_hz=40, phase=0.3, delay=211, snr_db=30, amp=0.5, total=len(iq) + 30000)
    rx = qrl.make_gr_demod_m17(n_channels=1, max_samples=len(x))
    rx.work(x[None, :])
    bits, tx_bits = rx.read_port(2)[0], np.unpackbits(data)
    best = 0.0
    for off in range(60, 160):
        n = min(len(bits) - off, len(tx_bits)) - 100
        best = max(best, float(np.mean(bits[off:off + n] == tx_bits[:n])))
    assert best == 1.0
