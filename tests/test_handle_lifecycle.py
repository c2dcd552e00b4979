"""Handle plumbing shared by the nine handle types (qradiolink_b200/csrc/qrl_handle.hpp): moving a handle onto a caller's stream and
back to one of its own leaves its outputs bit-identical to a twin that never moved; the NULL cases of *_destroy and qrl_pfb_set_stream;
the last error of a failed create; and handles created and run from two host threads at once, each on first use of its kernels'
shared-memory opt-in.

Runs under QRL_EMULATED_LIB=<libqrl_b200_emu.so> as well, except for the cases that need a real CUDA stream or real concurrency."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import siggen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMULATED = bool(os.environ.get("QRL_EMULATED_LIB"))
needs_real_gpu = pytest.mark.skipif(EMULATED, reason="needs a real CUDA device (torch streams, concurrent host threads)")


def _bits(rng, n, sync_words=()):
    """n random bits (one per byte) with the given (word, length) sync patterns planted at fixed places."""
    b = rng.integers(0, 2, n).astype(np.uint8)
    for k, (w, nb) in enumerate(sync_words):
        at = 40 + 150 * k
        b[at:at + nb] = [(w >> (nb - 1 - i)) & 1 for i in range(nb)]
    return b


# name -> (create(qrl), run(handle, call index) -> list of output arrays).  Small shapes: each runs in seconds under emulation.
def _rx(q):
    return q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=2, max_samples=40000)


def _rx_run(h, k):
    X, _ = siggen.gen_4fsk_channels(2, 40000, seed0=3000 + 10 * k)
    h.work(X)
    return [np.concatenate(h.read_port(p)) for p in range(3)]


def _tx(q):
    return q.make_gr_mod_4fsk(25, 1000000, 1700, 3500, True, n_channels=2, max_items=24)


def _tx_run(h, k):
    return [h.work(np.random.default_rng(3100 + k).integers(0, 256, (2, 24), dtype=np.uint8))]


def _frontend(q):
    return q.Frontend(2000000, n_channels=2, max_in=4096)


def _frontend_run(h, k):
    rng = np.random.default_rng(3200 + k)
    return [h.work((rng.standard_normal((2, 4000)) + 1j * rng.standard_normal((2, 4000))).astype(np.complex64))]


def _mmdvm_rx(q):
    return q.MmdvmChannelsRx(2, max_in=4096)


def _mmdvm_rx_run(h, k):
    rng = np.random.default_rng(3300 + k)
    out, db, items = h.work((0.3 * (rng.standard_normal((2, 4000)) + 1j * rng.standard_normal((2, 4000)))).astype(np.complex64))
    return [out, db, items]


def _mmdvm_tx(q):
    return q.MmdvmChannelsTx(2, max_in=4096)


def _mmdvm_tx_run(h, k):
    return [h.work(np.random.default_rng(3400 + k).integers(-8000, 8000, (2, 4000)).astype(np.int16))]


def _pfb(q):
    taps = np.random.default_rng(3500).standard_normal(341).astype(np.float32) * 0.05      # M = 10, 35 taps per branch: the tiled kernel
    return q.PfbChannelizer(10, taps, max_in=20000)


def _pfb_run(h, k):
    rng = np.random.default_rng(3600 + k)
    return [h.work((rng.standard_normal(20000 - 3 * k) + 1j * rng.standard_normal(20000 - 3 * k)).astype(np.complex64))]


def _spectrum(q):
    s = q.Spectrum(256, 5, n_streams=2, max_samples=1024)
    s.set_enabled(True)
    return s


def _spectrum_run(h, k):
    rng = np.random.default_rng(3700 + k)
    h.work((rng.standard_normal((2, 700)) + 1j * rng.standard_normal((2, 700))).astype(np.complex64))
    return [h.get_fft_data()]


def _deframer(q):
    return q.Deframer.for_mode("4FSK2K", n_channels=2, max_bits=2048)


def _deframer_run(h, k):
    rng = np.random.default_rng(3800 + k)
    frames = h.work([_bits(rng, 2000, [(0xED89, 16), (0x89EDAA, 24)]) for _ in range(2)])
    return [np.frombuffer(b"".join(t.to_bytes(4, "little") + p for ch in frames for t, p in ch), np.uint8), h.modem_sync.copy()]


def _dfbb(q):
    return q.DeframerBB(1, n_channels=2, max_bits=2048)


def _dfbb_run(h, k):
    rng = np.random.default_rng(3900 + k)
    return h.work([_bits(rng, 2000 - 7 * k, [(0x4C8A2B, 24), (0xED89, 16)]) for _ in range(2)])


HANDLES = {
    "rx": (_rx, _rx_run), "tx": (_tx, _tx_run), "frontend": (_frontend, _frontend_run), "mmdvm_rx": (_mmdvm_rx, _mmdvm_rx_run),
    "mmdvm_tx": (_mmdvm_tx, _mmdvm_tx_run), "pfb": (_pfb, _pfb_run), "spectrum": (_spectrum, _spectrum_run),
    "deframer": (_deframer, _deframer_run), "dfbb": (_dfbb, _dfbb_run),
}


def _same(got, want, where):
    assert len(got) == len(want), where
    for i, (g, w) in enumerate(zip(got, want)):
        if w is None:
            assert g is None, (where, i)
            continue
        g, w = np.asarray(g), np.asarray(w)
        assert g.shape == w.shape and g.dtype == w.dtype, (where, i, g.shape, w.shape)
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), (where, i)      # bit for bit


def _run_switching(qrl, name, streams):
    """One call on the handle's own stream, then one after each set_stream(s) of `streams`; a twin handle makes the same calls
    without ever switching.  Every call's outputs must be bit-identical."""
    create, run = HANDLES[name]
    L = qrl.load_library()
    h, twin = create(qrl), create(qrl)
    try:
        _same(run(h, 0), run(twin, 0), (name, "own stream"))
        for k, s in enumerate(streams, 1):
            if hasattr(h, "set_stream"):
                h.set_stream(s)
            else:                                       # DeframerBB's wrapper has no set_stream
                assert L.qrl_dfbb_set_stream(h._h, C.c_void_p(s)) == 0, k
            _same(run(h, k), run(twin, k), (name, "after set_stream", k))
    finally:
        h.close(); twin.close()


@pytest.mark.parametrize("name", sorted(HANDLES))
def test_set_stream_null_keeps_an_own_stream(qrl, name):
    """NULL: back to a stream of the handle's own (qrl_pfb_set_stream: keeps the current one)."""
    _run_switching(qrl, name, [None, None])


@needs_real_gpu
@pytest.mark.parametrize("name", sorted(HANDLES))
def test_set_stream_caller_stream_and_back(qrl, name):
    import torch
    s = torch.cuda.Stream()
    _run_switching(qrl, name, [s.cuda_stream, None])
    s.synchronize()


def test_null_handles_and_pfb_null_stream(qrl):
    L = qrl.load_library()
    for t in ("rx", "tx", "frontend", "mmdvm_rx", "mmdvm_tx", "spectrum"):
        assert getattr(L, "qrl_%s_destroy" % t)(None) == 0, t                    # QRL_OK
    for t in ("pfb", "deframer", "dfbb"):
        assert getattr(L, "qrl_%s_destroy" % t)(None) == -22, t                  # QRL_EINVAL
    for t in HANDLES:
        assert getattr(L, "qrl_%s_set_stream" % t)(None, None) == -22, t
    p = _pfb(qrl)
    assert L.qrl_pfb_set_stream(p._h, None) == 0             # keeps the current stream (outputs: test_set_stream_null_keeps_an_own_stream)
    p.close()


# a bad argument (QRL_EINVAL) and a device ordinal one past the last (QRL_ENODEV) for every create; the last error names the function
_CREATES = {
    "qrl_rx_create": lambda L, d, bad: L.qrl_rx_create(2, 5, 1000000, 1700, 3000, 1, 0 if bad else 1, 1024, d, C.byref(C.c_void_p())),
    "qrl_rx_create_freedv": lambda L, d, bad: L.qrl_rx_create_freedv(125, 1000000, 1700, 2000, 200, 0, 0 if bad else 1, 1024, d,
                                                                     C.byref(C.c_void_p())),
    "qrl_tx_create": lambda L, d, bad: L.qrl_tx_create(101, 25, 1000000, 1700, 3500, 1, 0 if bad else 1, 16, d, C.byref(C.c_void_p())),
    "qrl_tx_create_freedv": lambda L, d, bad: L.qrl_tx_create_freedv(125, 1000000, 1700, 2000, 200, 0, 0 if bad else 1, 16, d,
                                                                     C.byref(C.c_void_p())),
    "qrl_frontend_create": lambda L, d, bad: L.qrl_frontend_create(2000000, 0 if bad else 1, 4096, d, C.byref(C.c_void_p())),
    "qrl_mmdvm_rx_create": lambda L, d, bad: L.qrl_mmdvm_rx_create(0, 0 if bad else 1, None, 1, 5000, 4096, d, C.byref(C.c_void_p())),
    "qrl_mmdvm_tx_create": lambda L, d, bad: L.qrl_mmdvm_tx_create(0, 0 if bad else 1, None, 1, 5000, 4096, d, C.byref(C.c_void_p())),
    "qrl_pfb_create": lambda L, d, bad: L.qrl_pfb_create(201, 0 if bad else 10, np.ones(341, np.float32).ctypes.data_as(C.c_void_p), 341,
                                                         4096, d, C.byref(C.c_void_p())),
    "qrl_spectrum_create": lambda L, d, bad: L.qrl_spectrum_create(256, 5, 0 if bad else 1, 1024, d, C.byref(C.c_void_p())),
    "qrl_deframer_create": lambda L, d, bad: L.qrl_deframer_create(2, 64, 7, 0 if bad else 1, 2048, 8, d, C.byref(C.c_void_p())),
    "qrl_dfbb_create": lambda L, d, bad: L.qrl_dfbb_create(1, 0 if bad else 1, 2048, d, C.byref(C.c_void_p())),
}


@pytest.mark.parametrize("fn", sorted(_CREATES))
def test_failed_create_reports_the_create(qrl, fn):
    L = qrl.load_library()
    who = fn.replace("_freedv", "")                   # the FreeDV creates check their own arguments, then run the common create
    assert _CREATES[fn](L, 0, True) == -22                                       # QRL_EINVAL
    assert L.qrl_last_error(None).decode().startswith(who + ": "), L.qrl_last_error(None)
    assert _CREATES[fn](L, L.qrl_device_count(), False) == -19                   # QRL_ENODEV
    assert L.qrl_last_error(None).decode().startswith(who + ": "), L.qrl_last_error(None)


# two host threads, each creating and running a 4FSK-2k and an SSB receiver on device 0 at the same time, in a fresh process so that
# every kernel's shared-memory opt-in happens under the race; then the same handles' work serially, port for port
_THREADS_CHILD = r"""
import sys, threading
import numpy as np
sys.path.insert(0, sys.argv[1])
import qradiolink_b200 as q
from tests import siggen
C, T = 4, 1 << 17
X4, _ = siggen.gen_4fsk_channels(C, T, seed0=4000)
rng = np.random.default_rng(4100)
XS = (0.3 * (rng.standard_normal((C, T)) + 1j * rng.standard_normal((C, T)))).astype(np.complex64)

start = threading.Barrier(2)

def run():
    a = q.make_gr_demod_4fsk(5, 1000000, 1700, 3000, True, n_channels=C, max_samples=T)
    b = q.make_gr_demod_ssb(125, 1000000, 1700, 2700, 0, n_channels=C, max_samples=T)
    a.work(X4); b.work(XS)
    out = [np.concatenate(a.read_port(p)) for p in range(3)] + [np.concatenate(b.read_port(p)) for p in range(2)]
    a.close(); b.close()
    return out

res, errs = [None, None], []
def worker(i):
    try:
        start.wait()
        res[i] = run()
    except Exception as e:
        errs.append(repr(e))
ts = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
for t in ts:
    t.start()
for t in ts:
    t.join()
assert not errs, errs
serial = run()
for i in range(2):
    for p, (g, w) in enumerate(zip(res[i], serial)):
        assert g.shape == w.shape and np.array_equal(g.view(np.uint8), w.view(np.uint8)), (i, p)
print("ok")
"""


@needs_real_gpu
def test_two_host_threads_create_and_run_at_once(qrl):
    r = subprocess.run([sys.executable, "-c", _THREADS_CHILD, ROOT], cwd=ROOT, timeout=600, capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stderr[-2000:]
