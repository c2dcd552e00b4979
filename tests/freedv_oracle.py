"""ctypes binding of the FreeDV oracle (tests/freedv_oracle.c): gr_demod_freedv / gr_mod_freedv up to the codec2 modem boundary,
feedforward_agc_cc and the host-side speech helpers, restated on the CPU.

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
_SRC = os.path.join(_HERE, "freedv_oracle.c")
_DEPS = [_SRC, os.path.join(_ROOT, "oracle", "qrl_oracle.c"), os.path.join(_ROOT, "oracle", "qrl_oracle.h")]
# oracle/Makefile's CFLAGS; -Bsymbolic keeps this copy's calls to the oracle's exported functions inside this library
_CFLAGS = ["-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-std=gnu11", "-w", "-shared", "-Wl,-Bsymbolic"]
_LIB = None


def build():
    h = hashlib.sha256()
    for p in _DEPS:
        h.update(open(p, "rb").read())
    h.update(" ".join(_CFLAGS).encode())
    d = os.path.join(tempfile.gettempdir(), "qrl_freedv_oracle_%d" % os.getuid())
    os.makedirs(d, exist_ok=True)
    so = os.path.join(d, "libqrl_freedv_oracle_%s.so" % h.hexdigest()[:16])
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
        for side in ("rx", "tx"):
            getattr(L, "qo_freedv_%s_create" % side).restype = vp
            getattr(L, "qo_freedv_%s_create" % side).argtypes = [C.c_int] * 5
            getattr(L, "qo_freedv_%s_destroy" % side).argtypes = [vp]
            getattr(L, "qo_freedv_%s_taps" % side).argtypes = [vp, C.c_int, vp, C.c_int]
        L.qo_freedv_rx_set_param.argtypes = [vp, C.c_int, C.c_double]
        L.qo_freedv_rx_set_carrier_offset.argtypes = [vp, C.c_double]
        L.qo_freedv_rx_work.argtypes = [vp, vp, C.c_long]
        L.qo_freedv_rx_port_items.restype = C.c_long
        L.qo_freedv_rx_port_items.argtypes = [vp, C.c_int]
        L.qo_freedv_rx_port_data.restype = vp
        L.qo_freedv_rx_port_data.argtypes = [vp, C.c_int]
        L.qo_freedv_rx_clear.argtypes = [vp]
        L.qo_freedv_tx_set_bb_gain.argtypes = [vp, C.c_float]
        L.qo_freedv_tx_work.argtypes = [vp, vp, C.c_long]
        L.qo_freedv_tx_out_items.restype = C.c_long
        L.qo_freedv_tx_out_items.argtypes = [vp]
        L.qo_freedv_tx_out_data.restype = vp
        L.qo_freedv_tx_out_data.argtypes = [vp]
        L.qo_freedv_tx_out_clear.argtypes = [vp]
        L.qo_feedforward_agc_run.restype = C.c_long
        L.qo_feedforward_agc_run.argtypes = [vp, C.c_long, C.c_int, C.c_float, C.c_long, vp]
        L.qo_freedv_speech_out.argtypes = [vp, C.c_long, vp]
        L.qo_freedv_speech_in.restype = C.c_long
        L.qo_freedv_speech_in.argtypes = [vp, C.c_long, vp]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class FreedvRx:
    """One channel of gr_demod_freedv up to the input of freedv_rx_ss (gr_demod_freedv.cpp:31-81): port 0 = IQ at 8 ksps, port 1 = int16
    modem samples at 8 ksps."""

    def __init__(self, sps=125, samp_rate=1000000, filter_width=2500, low_cutoff=200, sb=0):
        self.h = lib().qo_freedv_rx_create(int(sps), int(samp_rate), int(filter_width), int(low_cutoff), int(sb))
        if not self.h:
            raise ValueError("oracle: gr_demod_freedv arguments out of range")

    def __del__(self):
        if getattr(self, "h", None):
            lib().qo_freedv_rx_destroy(self.h); self.h = None

    def set_param(self, key, value):
        if lib().qo_freedv_rx_set_param(self.h, int(key), float(value)) != 0:
            raise ValueError("oracle: no setter %r on gr_demod_freedv" % key)

    def set_carrier_offset(self, hz):
        lib().qo_freedv_rx_set_carrier_offset(self.h, float(hz))

    def work(self, iq):
        """-> (port 0 complex64, port 1 int16) produced by this call"""
        iq = np.ascontiguousarray(iq, np.complex64)
        L = lib()
        L.qo_freedv_rx_work(self.h, _p(iq), len(iq))
        n0, n1 = L.qo_freedv_rx_port_items(self.h, 0), L.qo_freedv_rx_port_items(self.h, 1)
        p0 = np.frombuffer(C.string_at(L.qo_freedv_rx_port_data(self.h, 0), 8 * n0), np.complex64).copy() if n0 else np.zeros(0, np.complex64)
        p1 = np.frombuffer(C.string_at(L.qo_freedv_rx_port_data(self.h, 1), 2 * n1), np.int16).copy() if n1 else np.zeros(0, np.int16)
        L.qo_freedv_rx_clear(self.h)
        return p0, p1

    def taps(self, which):
        """0 = stage-1 low-pass, 1 = side-band filter (complex64), 2 = audio band-pass"""
        out = np.zeros(2 * 4096, np.float32)
        n = lib().qo_freedv_rx_taps(self.h, which, _p(out), 4096)
        return out[: 2 * n].view(np.complex64).copy() if which == 1 else out[:n].copy()


class FreedvTx:
    """One channel of gr_mod_freedv behind freedv_tx_ss (gr_mod_freedv.cpp:27-85): int16 modem samples at 8 ksps -> complex64 at
    samp_rate, sps outputs per input sample."""

    def __init__(self, sps=125, samp_rate=1000000, filter_width=2500, low_cutoff=200, sb=0):
        self.h = lib().qo_freedv_tx_create(int(sps), int(samp_rate), int(filter_width), int(low_cutoff), int(sb))
        if not self.h:
            raise ValueError("oracle: gr_mod_freedv arguments out of range")

    def __del__(self):
        if getattr(self, "h", None):
            lib().qo_freedv_tx_destroy(self.h); self.h = None

    def set_bb_gain(self, g):
        lib().qo_freedv_tx_set_bb_gain(self.h, float(g))

    def work(self, s):
        s = np.ascontiguousarray(s, np.int16)
        L = lib()
        L.qo_freedv_tx_work(self.h, _p(s), len(s))
        n = L.qo_freedv_tx_out_items(self.h)
        out = np.frombuffer(C.string_at(L.qo_freedv_tx_out_data(self.h), 8 * n), np.complex64).copy() if n else np.zeros(0, np.complex64)
        L.qo_freedv_tx_out_clear(self.h)
        return out

    def taps(self, which):
        """0 = side-band filter (complex64), 1 = interpolator low-pass"""
        out = np.zeros(2 * 4096, np.float32)
        n = lib().qo_freedv_tx_taps(self.h, which, _p(out), 4096)
        return out[: 2 * n].view(np.complex64).copy() if which == 0 else out[:n].copy()


def feedforward_agc(x, N=512, ref=1.0, chunk=0):
    """analog::feedforward_agc_cc(N, ref) over one stream from zero history (qo_feedforward_agc_run), fed in chunks of `chunk` items"""
    x = np.ascontiguousarray(x, np.complex64)
    out = np.zeros(len(x), np.complex64)
    n = lib().qo_feedforward_agc_run(_p(x), len(x), int(N), float(ref), int(chunk), _p(out))
    return out[:n]


def freedv_speech_out(s):
    """RX speech side behind freedv_rx_ss: short_to_float(1, 32768) -> x2"""
    s = np.ascontiguousarray(s, np.int16)
    out = np.zeros(len(s), np.float32)
    lib().qo_freedv_speech_out(_p(s), len(s), _p(out))
    return out


def freedv_speech_in(audio):
    """TX speech side in front of freedv_tx_ss: band_pass(1, 8000, 200, 3500, 350, BH) -> float_to_short(1, 32765)"""
    audio = np.ascontiguousarray(audio, np.float32)
    out = np.zeros(len(audio), np.int16)
    n = lib().qo_freedv_speech_in(_p(audio), len(audio), _p(out))
    return out[:n]
