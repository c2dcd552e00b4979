"""Host-side mirror of the reference's RX operator surface for the hot path.

`make_gr_demod_4fsk(sps, samp_rate, carrier_freq, filter_width, fm)` etc. take exactly the arguments of
the reference factories (/root/reference/src/gr/gr_demod_4fsk.h:51-53, gr_demod_qpsk.h:48-50,
gr_demod_nbfm.h:38-39) plus `n_channels`; the returned RxBlock has a GNU-Radio-shaped
`work(iq)` that consumes one chunk of the [channels, T] gr_complex stream and output ports
0..3 with the reference's io signature (gr_demod_4fsk.cpp:22-36).  `gr_bit_sink`, `gr_audio_sink`
and `gr_const_sink` restate the buffering / drop policy of the reference's sink blocks
(src/gr/gr_bit_sink.cpp:45-84, gr_audio_sink.cpp:49-90, gr_const_sink.cpp:48-87), which is what
gr_modem::demodulate() polls.  All DSP happens in libqrl_b200.so (CUDA); nothing here computes.
"""
import ctypes as C
import threading

import numpy as np

from .lib import KIND, PARAM, Handle, check, load_library


class RxBlock(Handle):
    """n_channels instances of one reference demod hier-block, batched on one GPU."""
    ABI = "rx"

    def __init__(self, kind, sps, samp_rate, carrier_freq, filter_width, flag=0, n_channels=1,
                 max_samples=1 << 20, device=0, low_cutoff=None):
        self._L = load_library()
        self.kind, self.n_channels, self.max_samples = kind, int(n_channels), int(max_samples)
        # constructor failures surface like the std::runtime_error RadioController::toggleRX catches
        if kind == KIND.DEMOD_FREEDV:
            self._create(self._L.qrl_rx_create_freedv, sps, samp_rate, carrier_freq, filter_width, int(low_cutoff), int(flag),
                         self.n_channels, self.max_samples, device)
        else:
            self._create(self._L.qrl_rx_create, kind, sps, samp_rate, carrier_freq, filter_width, int(flag),
                         self.n_channels, self.max_samples, device)
        self.nports = self._L.qrl_rx_num_ports(self._h)
        self._itemsize = [self._L.qrl_rx_port_itemsize(self._h, p) for p in range(self.nports)]

    # -- runtime setters (gr_demod_nbfm.h:47-49, gr_demod_base.cpp:1220-1225)
    def set_param(self, key, value, channel=-1):
        check(self._L.qrl_rx_set_param(self._h, channel, key, float(value)), self._h, "qrl_rx_set_param")

    def set_squelch(self, db):
        self.set_param(PARAM.SQUELCH_DB, db)

    def set_filter_width(self, width):
        self.set_param(PARAM.FILTER_WIDTH, width)

    def set_ctcss(self, value):
        """gr_demod_nbfm::set_ctcss (gr_demod_nbfm.cpp:97-121): 0 = no tone squelch; f = the CTCSS tone squelch at f Hz (audio gated)"""
        self.set_param(PARAM.CTCSS, value)

    def set_agc_attack(self, value):
        self.set_param(PARAM.AGC_ATTACK, value)

    def set_agc_decay(self, value):
        self.set_param(PARAM.AGC_DECAY, value)

    def set_gain(self, value):
        """gr_demod_ssb::set_gain (IF gain in front of the side-band filter)"""
        self.set_param(PARAM.GAIN, value)

    def set_carrier_offset(self, hz, channel=-1):
        self.set_param(PARAM.CARRIER_OFFSET_HZ, hz, channel)

    set_stream = Handle._set_stream

    def reset(self):
        check(self._L.qrl_rx_reset(self._h), self._h, "qrl_rx_reset")

    # -- streaming
    def work(self, iq):
        """iq: complex64 array [n_channels, T] in host memory (copied to the device inside the call)."""
        iq = np.ascontiguousarray(iq, np.complex64)
        if iq.ndim == 1:
            iq = iq[None, :]
        if iq.shape[0] != self.n_channels:
            raise ValueError("expected %d channels, got %d" % (self.n_channels, iq.shape[0]))
        T = iq.shape[1]
        check(self._L.qrl_rx_work(self._h, iq.ctypes.data_as(C.c_void_p), T, T, 0), self._h, "qrl_rx_work")

    def work_sc16(self, iq16, scale=1.0 / 32767.0):
        """iq16: int16 array [n_channels, T, 2] (interleaved I/Q as the SDR delivers it) in host memory; each component becomes
        float32(v) * float32(scale) on the device (qrl_rx_work_sc16: half the PCIe bytes of work())."""
        iq16 = np.ascontiguousarray(iq16, np.int16)
        if iq16.ndim == 2:
            iq16 = iq16[None, :, :]
        if iq16.shape[0] != self.n_channels or iq16.shape[2] != 2:
            raise ValueError("expected [%d][T][2] int16" % self.n_channels)
        T = iq16.shape[1]
        check(self._L.qrl_rx_work_sc16(self._h, iq16.ctypes.data_as(C.c_void_p), T, T, float(scale), 0), self._h, "qrl_rx_work_sc16")

    def work_sc8(self, iq8, scale=1.0 / 128.0):
        """iq8: int8 array [n_channels, T, 2] (HackRF-style interleaved I/Q) in host memory; float32(v) * float32(scale) on the device."""
        iq8 = np.ascontiguousarray(iq8, np.int8)
        if iq8.ndim == 2:
            iq8 = iq8[None, :, :]
        if iq8.shape[0] != self.n_channels or iq8.shape[2] != 2:
            raise ValueError("expected [%d][T][2] int8" % self.n_channels)
        T = iq8.shape[1]
        check(self._L.qrl_rx_work_sc8(self._h, iq8.ctypes.data_as(C.c_void_p), T, T, float(scale), 0), self._h, "qrl_rx_work_sc8")

    # -- one SDR stream for every channel (stride 0): each channel applies its own carrier offset to the same capture
    def work_shared(self, iq):
        """iq: complex64 array [T] in host memory, one stream feeding every channel (copied to the device once)."""
        iq = np.ascontiguousarray(iq, np.complex64)
        if iq.ndim != 1:
            raise ValueError("expected one stream [T], got shape %s" % (iq.shape,))
        check(self._L.qrl_rx_work(self._h, iq.ctypes.data_as(C.c_void_p), iq.shape[0], 0, 0), self._h, "qrl_rx_work")

    def work_shared_sc16(self, iq16, scale=1.0 / 32767.0):
        """iq16: int16 array [T, 2] in host memory, one stream feeding every channel (copied and converted once)."""
        iq16 = np.ascontiguousarray(iq16, np.int16)
        if iq16.ndim != 2 or iq16.shape[1] != 2:
            raise ValueError("expected one stream [T][2] int16, got shape %s" % (iq16.shape,))
        check(self._L.qrl_rx_work_sc16(self._h, iq16.ctypes.data_as(C.c_void_p), iq16.shape[0], 0, float(scale), 0), self._h,
              "qrl_rx_work_sc16")

    def work_shared_sc8(self, iq8, scale=1.0 / 128.0):
        """iq8: int8 array [T, 2] in host memory, one stream feeding every channel (copied and converted once)."""
        iq8 = np.ascontiguousarray(iq8, np.int8)
        if iq8.ndim != 2 or iq8.shape[1] != 2:
            raise ValueError("expected one stream [T][2] int8, got shape %s" % (iq8.shape,))
        check(self._L.qrl_rx_work_sc8(self._h, iq8.ctypes.data_as(C.c_void_p), iq8.shape[0], 0, float(scale), 0), self._h,
              "qrl_rx_work_sc8")

    def work_sc16_device(self, dev_ptr, T, stride, scale=1.0 / 32767.0):
        check(self._L.qrl_rx_work_sc16(self._h, C.c_void_p(dev_ptr), T, stride, float(scale), 1), self._h, "qrl_rx_work_sc16")

    def work_device(self, dev_ptr, T, stride):
        """iq already resident in HBM: dev_ptr = address of [n_channels][stride] complex64; stride 0 = one stream [T] for every
        channel, read in place."""
        check(self._L.qrl_rx_work(self._h, C.c_void_p(dev_ptr), T, stride, 1), self._h, "qrl_rx_work")

    sync = Handle._sync

    def set_overlap(self, on=True):
        """Streaming mode: the loop / FEC tail of work() call k runs under the parallel stages of call k+1; read_port(),
        sync() or join() wait for it."""
        self.set_param(PARAM.OVERLAP_CALLS, 1.0 if on else 0.0)

    def enable_rssi(self, on=True):
        self.set_param(PARAM.RSSI, 1.0 if on else 0.0)

    def rssi(self, level=0.0):
        """Per-channel RSSI in dB as rssi_block.cpp:25-45 would report it after the last work() (needs enable_rssi())."""
        out = np.zeros(self.n_channels, np.float32)
        check(self._L.qrl_rx_rssi(self._h, C.c_float(level), out.ctypes.data_as(C.c_void_p)), self._h, "qrl_rx_rssi")
        return out

    def join(self):
        check(self._L.qrl_rx_join(self._h), self._h, "qrl_rx_join")

    def read_port(self, port):
        """Returns a list (one entry per channel) of what the last work() produced on `port`."""
        isz = self._itemsize[port]
        dt = {8: np.complex64, 4: np.float32, 2: np.int16, 1: np.uint8}[isz]
        cap = C.c_long()
        data = C.c_void_p()
        cnts = C.c_void_p()
        check(self._L.qrl_rx_port_device(self._h, port, C.byref(data), C.byref(cap), C.byref(cnts)), self._h, "port_device")
        buf = np.zeros((self.n_channels, cap.value), dt)
        counts = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_rx_read_port(self._h, port, buf.ctypes.data_as(C.c_void_p), cap.value,
                                       counts.ctypes.data_as(C.c_void_p), 0), self._h, "qrl_rx_read_port")
        return [buf[c, :counts[c]].copy() for c in range(self.n_channels)]

    def read_port_counts(self, port):
        counts = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_rx_read_port(self._h, port, None, 0, counts.ctypes.data_as(C.c_void_p), 0), self._h, "read counts")
        return counts

    launches = property(Handle._launches)


def make_gr_demod_4fsk(sps, samp_rate, carrier_freq, filter_width, fm, n_channels=1, **kw):
    return RxBlock(KIND.DEMOD_4FSK, sps, samp_rate, carrier_freq, filter_width, int(bool(fm)), n_channels, **kw)


def make_gr_demod_qpsk(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    return RxBlock(KIND.DEMOD_QPSK, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_bpsk(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_demod_bpsk.h: 4 ports (IQ, constellation, bits, bits of the delayed decoder)."""
    return RxBlock(KIND.DEMOD_BPSK, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_2fsk(sps, samp_rate, carrier_freq, filter_width, fm, n_channels=1, **kw):
    """src/gr/gr_demod_2fsk.h: 4 ports (IQ, constellation, bits, bits of the delayed decoder)."""
    return RxBlock(KIND.DEMOD_2FSK, sps, samp_rate, carrier_freq, filter_width, int(bool(fm)), n_channels, **kw)


def make_gr_demod_ssb(sps, samp_rate, carrier_freq, filter_width, sb, n_channels=1, **kw):
    """src/gr/gr_demod_ssb.h: sb = 0 upper side band, 1 lower; ports (IQ, float audio)."""
    return RxBlock(KIND.DEMOD_SSB, sps, samp_rate, carrier_freq, filter_width, int(sb), n_channels, **kw)


def make_gr_demod_gmsk(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_demod_gmsk.h (instances gr_demod_base.cpp:208-210: sps 5 / 10 / 1 = GMSK2K / 1K / 10K); 4 ports like 2FSK."""
    return RxBlock(KIND.DEMOD_GMSK, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_m17(sps=125, samp_rate=1000000, carrier_freq=1700, filter_width=9000, n_channels=1, **kw):
    """src/gr/gr_demod_m17.h:41-42 (defaults as there); ports (IQ at 24 ksps, symbols, hard bits: 2 per symbol, no FEC)."""
    return RxBlock(KIND.DEMOD_M17, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_dmr(sps=5, samp_rate=1000000, n_channels=1, **kw):
    """src/gr/gr_demod_dmr.h:42 (instance gr_demod_base.cpp:253: make_gr_demod_dmr(5, 1e6)); ports (IQ at 24 ksps, symbols, hard bits:
    2 per symbol, float symbol-filter output)."""
    return RxBlock(KIND.DEMOD_DMR, sps, samp_rate, 0, 5000, 0, n_channels, **kw)


def make_gr_demod_dsss(sps=25, samp_rate=1000000, carrier_freq=1700, filter_width=150, n_channels=1, **kw):
    """src/gr/gr_demod_dsss.h (instance gr_demod_base.cpp:218: make_gr_demod_dsss(25, 1e6, 1700, 150)); Barker-13 BPSK, 16 symbols/s;
    ports (IQ at 5200 sps, symbols, decoded bits, decoded bits of the decoder behind delay(1))."""
    return RxBlock(KIND.DEMOD_DSSS, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_wbfm(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_demod_wbfm.h (instance gr_demod_base.cpp:228: make_gr_demod_wbfm(125, 1e6, 1700, 75000)); ports (IQ at 200 ksps,
    float audio at 8 ksps)."""
    return RxBlock(KIND.DEMOD_WBFM, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_am(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    """src/gr/gr_demod_am.h (instance gr_demod_base.cpp: make_gr_demod_am(125, 1e6, 1700, 5000)); ports (IQ, float audio)."""
    return RxBlock(KIND.DEMOD_AM, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_nbfm(sps, samp_rate, carrier_freq, filter_width, n_channels=1, **kw):
    return RxBlock(KIND.DEMOD_NBFM, sps, samp_rate, carrier_freq, filter_width, 0, n_channels, **kw)


def make_gr_demod_freedv(sps=125, samp_rate=8000, carrier_freq=1700, filter_width=2000, low_cutoff=200, mode=0, sb=0, n_channels=1, **kw):
    """src/gr/gr_demod_freedv.h:40-41 (defaults as there; instances gr_demod_base.cpp:229-249, e.g. (125, 1e6, 1700, 2500, 200, MODE_1600,
    0)) up to the input of codec2's freedv_rx_ss.  Ports: 0 = IQ at 8 ksps (sps x the input level: the reference's stage-1 taps), 1 = int16
    modem samples at 8 ksps, the samples freedv_rx_ss consumes (the reference's port 1 is float speech behind the vocoder).  `mode` is
    codec2's and only kept as an attribute for the adapter that runs the vocoder."""
    blk = RxBlock(KIND.DEMOD_FREEDV, sps, samp_rate, carrier_freq, filter_width, int(sb), n_channels, low_cutoff=low_cutoff, **kw)
    blk.mode = mode
    return blk


# ------------------------------------------------------------------ sink blocks (per channel)
class gr_bit_sink:
    """src/gr/gr_bit_sink.cpp: work() appends unless >1 Mi items are pending; get_data() -> None below 32 items."""

    def __init__(self):
        self._data = np.zeros(0, np.uint8)
        self._mutex = threading.Lock()      # work() and get_data() come from two threads (gr_bit_sink.cpp:47,70)

    def flush(self):
        with self._mutex:
            self._data = np.zeros(0, np.uint8)

    def work(self, items):
        if len(items) < 1:
            return 0
        with self._mutex:
            if len(self._data) > 1048576:
                return len(items)          # reader too slow: drop (gr_bit_sink.cpp:71-76)
            self._data = np.concatenate([self._data, np.asarray(items, np.uint8)])
        return len(items)

    def get_data(self):
        with self._mutex:
            if len(self._data) < 32:
                return None
            d, self._data = self._data, np.zeros(0, np.uint8)
        return d


class gr_audio_sink:
    """src/gr/gr_audio_sink.cpp: 640-sample packets; the buffer is cleared when more than 8000 samples wait."""

    def __init__(self):
        self._data = np.zeros(0, np.float32)
        self._mutex = threading.Lock()

    def flush(self):
        with self._mutex:
            self._data = np.zeros(0, np.float32)

    def work(self, items):
        if len(items) < 1:
            return 0
        with self._mutex:
            if len(self._data) > 8000:
                self._data = np.zeros(0, np.float32)
                return len(items)
            self._data = np.concatenate([self._data, np.asarray(items, np.float32)])
        return len(items)

    def get_data(self):
        with self._mutex:
            if len(self._data) < 640:
                return None
            d, self._data = self._data[:640], self._data[640:]
        return d


class gr_const_sink:
    """src/gr/gr_const_sink.cpp: constellation tap, drops when more than 256 items wait."""

    def __init__(self):
        self._data = np.zeros(0, np.complex64)
        self._mutex = threading.Lock()

    def flush(self):
        with self._mutex:
            self._data = np.zeros(0, np.complex64)

    def work(self, items):
        if len(items) < 1:
            return 0
        with self._mutex:
            if len(self._data) > 256:
                return len(items)
            self._data = np.concatenate([self._data, np.asarray(items, np.complex64)])
        return len(items)

    def get_data(self):
        with self._mutex:
            if len(self._data) < 32:
                return None
            d, self._data = self._data, np.zeros(0, np.complex64)
        return d


class gr_sample_sink:
    """src/gr/gr_sample_sink.cpp: time-domain display tap (gr_demod_base::get_sample_data, gr_demod_base.cpp:988-1006): disabled at
    start; keeps samples until more than 524288 wait; get_data hands out at most `window` of them (even count), None below 2."""

    def __init__(self):
        self._data = np.zeros(0, np.complex64)
        self._window = 8096
        self._enabled = False
        self._mutex = threading.Lock()

    def flush(self):
        with self._mutex:
            self._data = np.zeros(0, np.complex64)

    def set_sample_window(self, size):
        with self._mutex:
            self._window = int(size) + (int(size) % 2)

    def set_enabled(self, value):
        with self._mutex:
            self._enabled = bool(value)

    def work(self, items):
        if len(items) < 1 or not self._enabled:
            return len(items)
        with self._mutex:
            if len(self._data) > 524288:
                return len(items)
            self._data = np.concatenate([self._data, np.asarray(items, np.complex64)])
        return len(items)

    def get_data(self):
        with self._mutex:
            if len(self._data) < 2:
                return None
            size = min(len(self._data), self._window)
            size -= size % 2
            d, self._data = self._data[:size].copy(), self._data[size:]
        return d
