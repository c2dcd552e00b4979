"""Front end at device rates >= 2 Msps: host-side mirror of gr_demod_base::set_samp_rate / set_carrier_offset for that case
(/root/reference/src/gr/gr_demod_base.cpp:1220-1225, 1303-1362): rotator at the device rate + rational_resampler_ccf(1, samp_rate / 1e6)
for a batch of channels.  The output stays in HBM in the layout RxBlock.work_device takes."""
import ctypes as C

import numpy as np

from .lib import Handle, check, load_library


class Frontend(Handle):
    ABI = "frontend"

    def __init__(self, samp_rate, n_channels=1, max_in=1 << 21, device=0):
        self._L = load_library()
        self.n_channels, self.max_in, self.decimation = int(n_channels), int(max_in), int(samp_rate) // 1000000
        self._create(self._L.qrl_frontend_create, int(samp_rate), self.n_channels, self.max_in, device)

    set_stream = Handle._set_stream

    def set_carrier_offset(self, hz, channel=-1):
        check(self._L.qrl_frontend_set_carrier_offset(self._h, channel, float(hz)), self._h, "qrl_frontend_set_carrier_offset")

    def work(self, iq):
        """iq at the device rate (host), complex64: [n_channels, T], one stream per channel, or [T], one wideband stream that every
        channel reads at its own carrier offset -> complex64 [n_channels, n_out] at 1 Msps."""
        iq = np.ascontiguousarray(iq, np.complex64)
        if iq.ndim == 1:
            T, stride = iq.shape[0], 0
        elif iq.ndim == 2 and iq.shape[0] == self.n_channels:
            T = stride = iq.shape[1]
        else:
            raise ValueError("Frontend.work: iq must be [T] (one shared stream) or [%d, T], got shape %s" % (self.n_channels, iq.shape))
        n = C.c_long()
        check(self._L.qrl_frontend_work(self._h, iq.ctypes.data_as(C.c_void_p), T, stride, 0, C.byref(n)), self._h, "qrl_frontend_work")
        out = np.zeros((self.n_channels, max(1, n.value)), np.complex64)
        check(self._L.qrl_frontend_read(self._h, out.ctypes.data_as(C.c_void_p), out.shape[1]), self._h, "qrl_frontend_read")
        return out[:, :n.value]

    def work_device(self, dev_ptr, T, stride):
        """device input: channel c reads dev_ptr[c * stride ..][:T]; stride 0 = one stream for every channel."""
        n = C.c_long()
        check(self._L.qrl_frontend_work(self._h, C.c_void_p(dev_ptr), T, stride, 1, C.byref(n)), self._h, "qrl_frontend_work")
        return n.value

    def out_device(self):
        """(device pointer, stride, items) of the last call's 1 Msps output: pass to RxBlock.work_device(ptr, items, stride)."""
        p, s, n = C.c_void_p(), C.c_long(), C.c_long()
        check(self._L.qrl_frontend_out_device(self._h, C.byref(p), C.byref(s), C.byref(n)), self._h, "qrl_frontend_out_device")
        return p.value, s.value, n.value


class TxFrontend(Handle):
    """Transmit side of the same pair, gr_mod_base::set_samp_rate / set_carrier_offset (gr_mod_base.cpp:38,211-293,799-805): rotator
    at 1 Msps + rational_resampler_ccf(samp_rate / 1e6, 1) behind the modulators, for a batch of channels.  Takes the layout
    TxBlock.out_device gives; the output at samp_rate stays in HBM until read."""
    ABI = "tx_frontend"

    def __init__(self, samp_rate, n_channels=1, max_in=1 << 16, device=0):
        self._L = load_library()
        self.n_channels, self.max_in, self.interpolation = int(n_channels), int(max_in), int(samp_rate) // 1000000
        self._create(self._L.qrl_tx_frontend_create, int(samp_rate), self.n_channels, self.max_in, device)

    set_stream = Handle._set_stream
    launches = property(Handle._launches)

    def set_carrier_offset(self, hz, channel=-1):
        check(self._L.qrl_tx_frontend_set_carrier_offset(self._h, channel, float(hz)), self._h, "qrl_tx_frontend_set_carrier_offset")

    def work(self, iq):
        """iq: complex64 [n_channels, n] at 1 Msps (host) -> complex64 [n_channels, N n] at the device rate."""
        iq = np.ascontiguousarray(iq, np.complex64)
        if iq.ndim == 1:
            iq = iq[None, :]
        n_in = iq.shape[1]
        n = C.c_long()
        check(self._L.qrl_tx_frontend_work(self._h, iq.ctypes.data_as(C.c_void_p), n_in, n_in, 0, C.byref(n)), self._h, "qrl_tx_frontend_work")
        out = np.zeros((self.n_channels, max(1, n.value)), np.complex64)
        check(self._L.qrl_tx_frontend_read(self._h, out.ctypes.data_as(C.c_void_p), out.shape[1]), self._h, "qrl_tx_frontend_read")
        return out[:, :n.value]

    def work_device(self, dev_ptr, n, stride):
        """device input, e.g. TxBlock.out_device()'s pointer and stride; returns the number of output items per channel (N n)."""
        out = C.c_long()
        check(self._L.qrl_tx_frontend_work(self._h, C.c_void_p(dev_ptr), n, stride, 1, C.byref(out)), self._h, "qrl_tx_frontend_work")
        return out.value

    def read(self):
        """complex64 [n_channels, items] of the last call (waits for the handle's stream)."""
        n = self.out_device()[2]
        out = np.zeros((self.n_channels, max(1, n)), np.complex64)
        check(self._L.qrl_tx_frontend_read(self._h, out.ctypes.data_as(C.c_void_p), out.shape[1]), self._h, "qrl_tx_frontend_read")
        return out[:, :n]

    def out_device(self):
        """(device pointer, stride, items) of the last call's output at the device rate, e.g. for Frontend.work_device(ptr, items, stride)."""
        p, s, n = C.c_void_p(), C.c_long(), C.c_long()
        check(self._L.qrl_tx_frontend_out_device(self._h, C.byref(p), C.byref(s), C.byref(n)), self._h, "qrl_tx_frontend_out_device")
        return p.value, s.value, n.value


class TxCombiner(Handle):
    """N modulators -> one SDR sink, gr_mod_mmdvm_multi's wiring (gr_mod_mmdvm_multi.cpp:53-125) with gr_mod_base's interpolator: per
    channel x samp_rate / 1e6, a rotator at the device rate (any offset within +-samp_rate / 2), add_cc, x 1 / C, x bb_gain.  The one
    summed stream stays in HBM until read."""
    ABI = "tx_combiner"

    def __init__(self, samp_rate, n_channels=1, max_in=1 << 16, device=0):
        self._L = load_library()
        self.n_channels, self.max_in, self.interpolation = int(n_channels), int(max_in), int(samp_rate) // 1000000
        self._create(self._L.qrl_tx_combiner_create, int(samp_rate), self.n_channels, self.max_in, device)

    set_stream = Handle._set_stream
    launches = property(Handle._launches)

    def set_carrier_offset(self, hz, channel=-1):
        check(self._L.qrl_tx_combiner_set_carrier_offset(self._h, channel, float(hz)), self._h, "qrl_tx_combiner_set_carrier_offset")

    def set_gain(self, g):
        check(self._L.qrl_tx_combiner_set_gain(self._h, float(g)), self._h, "qrl_tx_combiner_set_gain")

    def _work(self, rows, n, on_device):
        ptrs = (C.c_void_p * self.n_channels)(*rows)
        out = C.c_long()
        check(self._L.qrl_tx_combiner_work(self._h, ptrs, n, on_device, C.byref(out)), self._h, "qrl_tx_combiner_work")
        return out.value

    def work(self, iq):
        """iq: complex64 [n_channels, n] at 1 Msps (host) -> complex64 [N n] at the device rate."""
        iq = np.ascontiguousarray(iq, np.complex64)
        if iq.ndim != 2 or iq.shape[0] != self.n_channels:
            raise ValueError("TxCombiner.work: iq must be [n_channels, n]")
        self._work([iq.ctypes.data + c * iq.strides[0] for c in range(self.n_channels)], iq.shape[1], 0)
        return self.read()

    def work_device(self, rows, n):
        """rows: n_channels device addresses of n gr_complex each (e.g. TxBlock.out_device()'s pointer + c stride, or rows of several
        modulators on the combiner's stream); returns the number of output items (N n)."""
        if len(rows) != self.n_channels:
            raise ValueError("TxCombiner.work_device: need one row per channel")
        return self._work([int(r) for r in rows], n, 1)

    def read(self):
        """complex64 [items] of the last call (waits for the handle's stream)."""
        n = self.out_device()[1]
        out = np.zeros(max(1, n), np.complex64)
        check(self._L.qrl_tx_combiner_read(self._h, out.ctypes.data_as(C.c_void_p), n), self._h, "qrl_tx_combiner_read")
        return out[:n]

    def out_device(self):
        """(device pointer, items) of the last call's summed stream, e.g. for Frontend.work_device(ptr, items, 0)."""
        p, n = C.c_void_p(), C.c_long()
        check(self._L.qrl_tx_combiner_out_device(self._h, C.byref(p), C.byref(n)), self._h, "qrl_tx_combiner_out_device")
        return p.value, n.value
