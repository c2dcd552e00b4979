"""ctypes binding of the transmit-combiner oracle (tests/tx_combiner_oracle.c): N modulators interpolated to the device rate, each rotated
to its carrier offset there, summed, x 1 / C, x bb_gain -- gr_mod_mmdvm_multi's wiring with gr_mod_base's interpolator, restated on the
CPU.

TEST INFRASTRUCTURE ONLY.  The C file compiles tests/tx_frontend_oracle.c (and oracle/qrl_oracle.c) into its own translation unit, so it is
built here, with the oracle's compiler flags, into a per-user cache directory keyed by the sources' contents (the checkout may be
read-only); the product package never imports this module."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "tx_combiner_oracle.c")
_DEPS = [_SRC, os.path.join(_HERE, "tx_frontend_oracle.c"), os.path.join(_ROOT, "oracle", "qrl_oracle.c"),
         os.path.join(_ROOT, "oracle", "qrl_oracle.h")]
# oracle/Makefile's CFLAGS; -Bsymbolic keeps this copy's calls to the oracle's exported functions inside this library
_CFLAGS = ["-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=gnu11", "-w", "-shared", "-Wl,-Bsymbolic"]
_LIB = None


def build():
    h = hashlib.sha256()
    for p in _DEPS:
        h.update(open(p, "rb").read())
    h.update(" ".join(_CFLAGS).encode())
    d = os.path.join(tempfile.gettempdir(), "qrl_tx_combiner_oracle_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "libqrl_tx_combiner_oracle_%s.so" % h.hexdigest()[:16])
    if not os.path.exists(so):
        tmp = so + ".%d.tmp" % os.getpid()
        subprocess.check_call(["gcc"] + _CFLAGS + ["-o", tmp, _SRC, "-lm"])
        os.replace(tmp, so)
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        vp = C.c_void_p
        L.qo_tx_combiner_create.restype = vp
        L.qo_tx_combiner_create.argtypes = [C.c_int, C.c_int]
        L.qo_tx_combiner_destroy.argtypes = [vp]
        L.qo_tx_combiner_ntaps.argtypes = [vp]
        L.qo_tx_combiner_set_carrier_offset.argtypes = [vp, C.c_int, C.c_double]
        L.qo_tx_combiner_set_gain.argtypes = [vp, C.c_float]
        L.qo_tx_combiner_work.restype = C.c_long
        L.qo_tx_combiner_work.argtypes = [vp, vp, C.c_long, C.c_long, vp, C.c_long]
        _LIB = L
    return _LIB


class TxCombiner:
    """C channels at 1 Msps -> one stream at samp_rate: x N interpolator, device-rate rotator per channel, sum, x 1 / C, x gain."""

    def __init__(self, samp_rate, n_channels):
        self._h = lib().qo_tx_combiner_create(int(samp_rate), int(n_channels))
        if not self._h:
            raise ValueError("transmit combiner: samp_rate must be a multiple of 1e6 in [1e6, 32e6], n_channels >= 1")
        self.N, self.n_channels = int(samp_rate) // 1000000, int(n_channels)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().qo_tx_combiner_destroy(self._h); self._h = None

    @property
    def ntaps(self):
        return lib().qo_tx_combiner_ntaps(self._h)

    def set_carrier_offset(self, hz, channel=-1):
        lib().qo_tx_combiner_set_carrier_offset(self._h, int(channel), float(hz))

    def set_gain(self, g):
        lib().qo_tx_combiner_set_gain(self._h, float(g))

    def work(self, iq):
        """iq: complex64 [n_channels, n] -> complex64 [N n]"""
        iq = np.ascontiguousarray(iq, np.complex64).reshape(self.n_channels, -1)
        n = iq.shape[1]
        out = np.zeros(max(1, n * self.N), np.complex64)
        m = lib().qo_tx_combiner_work(self._h, iq.ctypes.data_as(C.c_void_p), n, n, out.ctypes.data_as(C.c_void_p), n * self.N)
        return out[:m].copy()
