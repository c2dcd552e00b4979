"""ctypes binding of the transmit front-end oracle (tests/tx_frontend_oracle.c): gr_mod_base's carrier-offset rotator at 1 Msps and x N
interpolator to the device rate, restated on the CPU.

TEST INFRASTRUCTURE ONLY.  The C file compiles oracle/qrl_oracle.c into its own translation unit, so it is built here, with the oracle's
compiler flags, into a per-user cache directory keyed by the sources' contents (the checkout may be read-only); the product package never
imports this module."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_SRC = os.path.join(_HERE, "tx_frontend_oracle.c")
_DEPS = [_SRC, os.path.join(_ROOT, "oracle", "qrl_oracle.c"), os.path.join(_ROOT, "oracle", "qrl_oracle.h")]
# oracle/Makefile's CFLAGS; -Bsymbolic keeps this copy's calls to the oracle's exported functions inside this library
_CFLAGS = ["-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=gnu11", "-w", "-shared", "-Wl,-Bsymbolic"]
_LIB = None


def build():
    h = hashlib.sha256()
    for p in _DEPS:
        h.update(open(p, "rb").read())
    h.update(" ".join(_CFLAGS).encode())
    d = os.path.join(tempfile.gettempdir(), "qrl_tx_frontend_oracle_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "libqrl_tx_frontend_oracle_%s.so" % h.hexdigest()[:16])
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
        L.qo_tx_frontend_create.restype = vp
        L.qo_tx_frontend_create.argtypes = [C.c_int]
        L.qo_tx_frontend_destroy.argtypes = [vp]
        L.qo_tx_frontend_ntaps.argtypes = [vp]
        L.qo_tx_frontend_set_carrier_offset.argtypes = [vp, C.c_double]
        L.qo_tx_frontend_work.restype = C.c_long
        L.qo_tx_frontend_work.argtypes = [vp, vp, C.c_long, vp, C.c_long]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class TxFrontend:
    """gr_mod_base transmit front end (gr_mod_base.cpp:38,211-293,799-805): rotator at 1 Msps + x N interpolator, one channel."""

    def __init__(self, samp_rate):
        self._h = lib().qo_tx_frontend_create(int(samp_rate))
        if not self._h:
            raise ValueError("transmit front end: samp_rate must be a multiple of 1e6 in [1e6, 32e6]")
        self.N = int(samp_rate) // 1000000

    def __del__(self):
        if getattr(self, "_h", None):
            lib().qo_tx_frontend_destroy(self._h); self._h = None

    @property
    def ntaps(self):
        return lib().qo_tx_frontend_ntaps(self._h)

    def set_carrier_offset(self, hz):
        lib().qo_tx_frontend_set_carrier_offset(self._h, float(hz))

    def work(self, iq):
        iq = np.ascontiguousarray(iq, np.complex64)
        cap = len(iq) * self.N
        out = np.zeros(max(1, cap), np.complex64)
        n = lib().qo_tx_frontend_work(self._h, _p(iq), len(iq), _p(out), cap)
        return out[:n].copy()
