"""GPU tier: DMR receive chain (gr_demod_dmr.cpp: x3/125 rational resampler to 24 ksps, quadrature demod, 0.2 roll-off symbol
filter tapped as float port 3, symbol sync with the PLAIN Mueller & Mueller detector, x0.9, phase modulator, hard bits) against the
CPU oracle: all four ports, ragged chunks.
"""
import numpy as np
import pytest

pytestmark = [pytest.mark.gpu]


def test_dmr_parity_chunked(qrl, oracle):
    from tests.test_gpu_m17 import m17_like_signal
    C, T = 3, 400000
    rng = np.random.default_rng(91)
    X = np.stack([m17_like_signal(rng, T) for _ in range(C)])
    blk = qrl.make_gr_demod_dmr(n_channels=C, max_samples=150000)
    assert blk.nports == 4
    acc = [[[] for _ in range(C)] for _ in range(4)]
    lo, i, sizes = 0, 0, [150000, 41, 125, 66667, 1, 99991]
    while lo < T:
        n = min(sizes[i % len(sizes)], T - lo); i += 1
        blk.work(X[:, lo:lo + n]); lo += n
        for p in range(4):
            for c, v in enumerate(blk.read_port(p)):
                acc[p][c].append(v)
    for c in range(C):
        rx = oracle.Rx(oracle.DEMOD_DMR, 5, 1000000, 0, 0, 0)
        rx.work(X[c])
        for p in range(4):
            got = np.concatenate(acc[p][c]); want = rx.port(p)
            assert got.dtype == want.dtype, (p, got.dtype, want.dtype)
            assert len(got) == len(want) and len(want) > 1000, (p, len(got), len(want))
            assert np.array_equal(got, want), (c, p)
    bits = np.concatenate(acc[2][0])
    assert bits.max() == 1 and 0.05 < bits.mean() < 0.95


def test_dmr_refuses_overlapped_calls(qrl):
    blk = qrl.make_gr_demod_dmr(n_channels=2, max_samples=1 << 16)
    with pytest.raises(Exception):
        blk.set_overlap(True)
