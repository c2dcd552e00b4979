"""Display spectrum on the device: host-side mirror of rx_fft_c (/root/reference/src/gr/rx_fft.cpp:44-129; make_rx_fft_c(32768,
WIN_BLACKMAN_HARRIS) at gr_demod_base.cpp:166, read through gr_demod_base::get_FFT_data :978-986) for a batch of streams."""
import ctypes as C

import numpy as np

from .lib import Handle, check, load_library

WIN_HAMMING, WIN_HANN, WIN_BLACKMAN, WIN_RECTANGULAR, WIN_KAISER, WIN_BLACKMAN_HARRIS = 0, 1, 2, 3, 4, 5


class Spectrum(Handle):
    """make_rx_fft_c(fftsize, wintype) for n_streams streams; work() = one rx_fft_c::work call, get_fft_data() as in the reference
    (None while no spectrum is ready)."""
    ABI = "spectrum"

    def __init__(self, fft_size=32768, window=WIN_BLACKMAN_HARRIS, n_streams=1, max_samples=1 << 20, device=0):
        self._L = load_library()
        self.n_streams, self.fft_size, self.max_samples = int(n_streams), int(fft_size), int(max_samples)
        self._create(self._L.qrl_spectrum_create, self.fft_size, int(window), self.n_streams, self.max_samples, device)

    set_stream = Handle._set_stream

    def set_enabled(self, on):
        check(self._L.qrl_spectrum_set_enabled(self._h, int(bool(on))), self._h, "qrl_spectrum_set_enabled")

    def set_fft_size(self, n):
        check(self._L.qrl_spectrum_set_fft_size(self._h, int(n)), self._h, "qrl_spectrum_set_fft_size")
        self.fft_size = int(n)

    def work(self, iq):
        iq = np.ascontiguousarray(iq, np.complex64)
        if iq.ndim == 1:
            iq = iq[None, :]
        if iq.shape[0] != self.n_streams:
            raise ValueError("expected %d streams" % self.n_streams)
        T = iq.shape[1]
        check(self._L.qrl_spectrum_work(self._h, iq.ctypes.data_as(C.c_void_p), T, T, 0), self._h, "qrl_spectrum_work")

    def work_device(self, dev_ptr, T, stride):
        check(self._L.qrl_spectrum_work(self._h, C.c_void_p(dev_ptr), T, stride, 1), self._h, "qrl_spectrum_work")

    def get_fft_data(self):
        """float32 [n_streams, fft_size] dB, fft-shifted, or None when no spectrum is ready (fftSize = 0 in the reference)."""
        out = np.empty((self.n_streams, self.fft_size), np.float32)
        n = C.c_uint()
        check(self._L.qrl_spectrum_get(self._h, out.ctypes.data_as(C.c_void_p), self.fft_size, 0, C.byref(n)), self._h, "qrl_spectrum_get")
        return out if n.value else None

    launches = property(Handle._launches)
