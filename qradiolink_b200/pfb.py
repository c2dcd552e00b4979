"""Polyphase channelizer / synthesizer front end (SURVEY.md section 8f row 1): host-side mirror of
gr::filter::pfb_channelizer_ccf::make(M, taps, 1.0) behind blocks::stream_to_streams(M)
(/root/reference/src/gr/gr_demod_mmdvm_multi2.cpp:98-107) and gr::filter::pfb_synthesizer_ccf::make(M, taps, false)
(/root/reference/src/gr/gr_mod_mmdvm_multi2.cpp:90-92).  All arithmetic runs in libqrl_b200.so (CUDA)."""
import ctypes as C

import numpy as np

from .lib import Handle, check, load_library

PFB_CHANNELIZER, PFB_SYNTHESIZER = 201, 202


def mmdvm_port_map(num_channels):
    """Channelizer / synthesizer port of logical channel i as wired by the reference (channels 0..3 on ports 0..3,
    channel 4.. on ports 9, 8, ...: gr_demod_mmdvm_multi2.cpp:110-124, gr_mod_mmdvm_multi2.cpp:107-121)."""
    ports, m = [], 1
    for i in range(num_channels):
        if i <= 3:
            ports.append(i)
        else:
            ports.append(10 - m); m += 1
    return ports


class _Pfb(Handle):
    ABI = "pfb"

    def __init__(self, kind, M, taps, max_in, device=0):
        self._L = load_library()
        taps = np.ascontiguousarray(taps, np.float32)
        self.M, self.kind, self.max_in = int(M), kind, int(max_in)
        self._create(self._L.qrl_pfb_create, kind, self.M, taps.ctypes.data_as(C.c_void_p), len(taps), self.max_in, device)

    set_stream = Handle._set_stream
    sync = Handle._sync

    def out_device(self):
        """(device pointer, stride in items, valid items) of the last call's output."""
        d, s, n = C.c_void_p(), C.c_long(), C.c_long()
        check(self._L.qrl_pfb_out_device(self._h, C.byref(d), C.byref(s), C.byref(n)), self._h, "qrl_pfb_out_device")
        return d.value, s.value, n.value

    launches = property(Handle._launches)


class PfbChannelizer(_Pfb):
    """One wideband gr_complex stream -> M channels [M][n/M]; channel c is centred on +c*fs/M."""

    def __init__(self, M, taps, max_in=1 << 20, device=0):
        super().__init__(PFB_CHANNELIZER, M, taps, max_in, device)

    def work(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        n = C.c_long()
        check(self._L.qrl_pfb_work(self._h, x.ctypes.data_as(C.c_void_p), len(x), 0, 0, C.byref(n)), self._h, "qrl_pfb_work")
        out = np.zeros((self.M, max(1, n.value)), np.complex64)
        check(self._L.qrl_pfb_read(self._h, out.ctypes.data_as(C.c_void_p), out.shape[1]), self._h, "qrl_pfb_read")
        return out[:, :n.value]

    def work_device(self, dev_ptr, n):
        cnt = C.c_long()
        check(self._L.qrl_pfb_work(self._h, C.c_void_p(dev_ptr), n, 0, 1, C.byref(cnt)), self._h, "qrl_pfb_work")
        return cnt.value


class PfbSynthesizer(_Pfb):
    """M channels [M][n] -> one wideband gr_complex stream of n*M samples."""

    def __init__(self, M, taps, max_in=1 << 17, device=0):
        super().__init__(PFB_SYNTHESIZER, M, taps, max_in, device)

    def work(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        if x.shape[0] != self.M:
            raise ValueError("expected %d channels" % self.M)
        n = C.c_long()
        check(self._L.qrl_pfb_work(self._h, x.ctypes.data_as(C.c_void_p), x.shape[1], x.shape[1], 0, C.byref(n)), self._h, "qrl_pfb_work")
        out = np.zeros(max(1, n.value), np.complex64)
        check(self._L.qrl_pfb_read(self._h, out.ctypes.data_as(C.c_void_p), 0), self._h, "qrl_pfb_read")
        return out[:n.value]

    def work_device(self, dev_ptr, n, stride):
        cnt = C.c_long()
        check(self._L.qrl_pfb_work(self._h, C.c_void_p(dev_ptr), n, stride, 1, C.byref(cnt)), self._h, "qrl_pfb_work")
        return cnt.value
