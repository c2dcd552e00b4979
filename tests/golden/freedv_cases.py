"""Seeded inputs of the FreeDV known-answer vectors (tests/golden/golden_freedv.json, made by tests/golden/make_golden_freedv.py)."""
import numpy as np

# name -> (sps, samp_rate, carrier_freq, filter_width, low_cutoff, sb): instances of gr_demod_base.cpp:229-249 / gr_mod_base.cpp:181-203
RX_CASES = {
    "freedv_rx_usb": (125, 1000000, 1700, 2500, 200, 0),
    "freedv_rx_lsb": (125, 1000000, 1700, 2400, 600, 1),
}
TX_CASES = {
    "freedv_tx_usb": (125, 1000000, 1700, 2500, 200, 0),
}


def rx_signal(name, C=2, T=150000):
    """[C][T] complex64 at 1 Msps: two tones inside the side band of the case, one outside it, and noise"""
    sb = RX_CASES[name][5]
    sign = -1.0 if sb else 1.0
    rng = np.random.default_rng(7100 + sb)
    n = np.arange(T)
    X = np.zeros((C, T), np.complex64)
    for c in range(C):
        x = 0.02 * np.exp(2j * np.pi * sign * (800 + 300 * c) * n / 1e6) + 0.01 * np.exp(2j * np.pi * sign * 1700 * n / 1e6)
        x = x + 0.01 * np.exp(-2j * np.pi * sign * 1000 * n / 1e6)
        x = x + 0.002 * (rng.standard_normal(T) + 1j * rng.standard_normal(T))
        X[c] = x.astype(np.complex64)
    return X


def tx_input(n=3000):
    """int16 modem samples at 8 ksps: two tones and noise (a stand-in for what freedv_tx_ss produces)"""
    rng = np.random.default_rng(7200)
    t = np.arange(n) / 8000.0
    return (6000 * np.sin(2 * np.pi * 900 * t) + 3000 * np.sin(2 * np.pi * 2100 * t) + 800 * rng.standard_normal(n)).astype(np.int16)
