"""MMDVM multi-channel front end on the device: host-side mirrors of gr_demod_mmdvm_multi2 and gr_mod_mmdvm_multi2
(/root/reference/src/gr/gr_demod_mmdvm_multi2.cpp:30-127, gr_mod_mmdvm_multi2.cpp:28-131; instances gr_demod_base.cpp:251,
gr_mod_base.cpp:205) without their MMDVM-protocol sink / source: wideband gr_complex at 250 ksps <-> int16 discriminator /
modulator samples at 24 ksps for up to 7 channels.  The polyphase filter bank is qrl_pfb_*, the per-channel chains qrl_mmdvm_*;
everything between the wideband slab and the int16 rows stays in HBM."""
import ctypes as C

import numpy as np

from .lib import Handle, QrlError, check, load_library
from .pfb import PfbChannelizer, PfbSynthesizer, mmdvm_port_map

MAX_MMDVM_CHANNELS = 7            # src/bursttimer.h:28
MMDVM_SAMPLE_RATE = 250000        # src/config_mmdvm.h:4


def _low_pass_2(L, gain, fs, fc, tw, att):
    buf = np.zeros(16384, np.float32)
    n = L.qrl_firdes_low_pass_2(float(gain), float(fs), float(fc), float(tw), float(att), 5, buf.ctypes.data_as(C.c_void_p), len(buf))
    if n <= 0:
        raise QrlError("qrl_firdes_low_pass_2 failed")
    return buf[:n].copy()


class MmdvmChannelsRx(Handle):
    """The per-channel part alone (qrl_mmdvm_rx_*): rows of a [n_rows][stride] gr_complex slab at 25 ksps -> int16 at 24 ksps + RSSI."""
    ABI = "mmdvm_rx"

    def __init__(self, n_channels, rows=None, n_rows=None, filter_width=5000, max_in=1 << 16, device=0, single=False):
        """single=True: make_gr_demod_mmdvm (gr_demod_mmdvm.cpp:30-64) for n_channels independent 250 ksps streams."""
        self._L = load_library()
        self.n_channels = int(n_channels)
        self.n_rows = int(n_rows if n_rows is not None else n_channels)
        self.max_in = int(max_in)
        r = None if rows is None else np.ascontiguousarray(rows, np.int32)
        self._create(self._L.qrl_mmdvm_rx_create, int(bool(single)), self.n_channels, None if r is None else r.ctypes.data_as(C.c_void_p), self.n_rows,
                     int(filter_width), self.max_in, device)

    set_stream = Handle._set_stream

    def calibrate_rssi(self, level):
        check(self._L.qrl_mmdvm_rx_calibrate_rssi(self._h, float(level)), self._h, "qrl_mmdvm_rx_calibrate_rssi")

    def _read(self, n):
        out = np.zeros((self.n_channels, max(1, n)), np.int16)
        cap = n // 300 + 2
        db = np.zeros((self.n_channels, cap), np.float32)
        nr, first = C.c_int(), C.c_longlong()
        check(self._L.qrl_mmdvm_rx_read(self._h, out.ctypes.data_as(C.c_void_p), out.shape[1], db.ctypes.data_as(C.c_void_p), cap,
                                        C.byref(nr), C.byref(first)), self._h, "qrl_mmdvm_rx_read")
        return out[:, :n], db[:, :nr.value], first.value + 300 * np.arange(nr.value, dtype=np.int64)

    def work(self, slab):
        """slab: complex64 [n_rows, n] (host) -> (int16 [n_channels, n_out], rssi dB [n_channels, k], item offsets [k])."""
        slab = np.ascontiguousarray(slab, np.complex64)
        if slab.shape[0] != self.n_rows:
            raise ValueError("expected %d rows" % self.n_rows)
        n = C.c_long()
        check(self._L.qrl_mmdvm_rx_work(self._h, slab.ctypes.data_as(C.c_void_p), slab.shape[1], slab.shape[1], 0, C.byref(n)), self._h, "qrl_mmdvm_rx_work")
        return self._read(n.value)

    def work_device(self, dev_ptr, n, stride):
        cnt = C.c_long()
        check(self._L.qrl_mmdvm_rx_work(self._h, C.c_void_p(dev_ptr), n, stride, 1, C.byref(cnt)), self._h, "qrl_mmdvm_rx_work")
        return cnt.value

    launches = property(Handle._launches)


def mmdvm_tag_item(sample_index, single=False):
    """Item of the zero-idle block's own stream on which a "zero_samples" tag attached to int16 sample `sample_index` arrives: the sample
    itself for gr_mod_mmdvm (all blocks in front of gr_zero_idle_bursts are 1:1), floor(k * 25 / 24 + 1/2) behind the x25/24 resampler of
    gr_mod_mmdvm_multi2 (how GNU Radio's scheduler moves a tag across a block of relative rate 25/24)."""
    k = int(sample_index)
    return k if single else (2 * k * 25 + 24) // 48


class MmdvmChannelsTx(Handle):
    """The per-channel part alone (qrl_mmdvm_tx_*): int16 [n_channels][n] at 24 ksps -> rows of a [n_rows][stride] slab at 25 ksps."""
    ABI = "mmdvm_tx"

    def __init__(self, n_channels, rows=None, n_rows=None, filter_width=5000, max_in=1 << 16, device=0, single=False):
        """single=True: make_gr_mod_mmdvm (gr_mod_mmdvm.cpp:28-70) for n_channels independent streams, 250 ksps out."""
        self._L = load_library()
        self.n_channels = int(n_channels)
        self.n_rows = int(n_rows if n_rows is not None else n_channels)
        self.max_in = int(max_in)
        self.single = bool(single)
        r = None if rows is None else np.ascontiguousarray(rows, np.int32)
        self._create(self._L.qrl_mmdvm_tx_create, int(bool(single)), self.n_channels, None if r is None else r.ctypes.data_as(C.c_void_p), self.n_rows,
                     int(filter_width), self.max_in, device)

    set_stream = Handle._set_stream

    def set_bb_gain(self, g):
        check(self._L.qrl_mmdvm_tx_set_bb_gain(self._h, float(g)), self._h, "qrl_mmdvm_tx_set_bb_gain")

    def zero_samples(self, sample_index, n_samples, channel=-1):
        """The "zero_samples" tag of gr_mmdvm_source on int16 sample `sample_index` of `channel` (-1: all): gr_zero_idle_bursts(0) clears
        n_samples items of its stream from where the tag arrives (qrl_mmdvm_tx_zero_samples, mmdvm_tag_item)."""
        check(self._L.qrl_mmdvm_tx_zero_samples(self._h, int(channel), mmdvm_tag_item(sample_index, self.single), int(n_samples)), self._h,
              "qrl_mmdvm_tx_zero_samples")

    def work(self, samples):
        """samples: int16 [n_channels, n] (host) -> complex64 [n_rows, n_out] (unused rows zero)."""
        samples = np.ascontiguousarray(samples, np.int16)
        if samples.shape[0] != self.n_channels:
            raise ValueError("expected %d channels" % self.n_channels)
        n = C.c_long()
        check(self._L.qrl_mmdvm_tx_work(self._h, samples.ctypes.data_as(C.c_void_p), samples.shape[1], samples.shape[1], 0, C.byref(n)), self._h, "qrl_mmdvm_tx_work")
        out = np.zeros((self.n_rows, max(1, n.value)), np.complex64)
        check(self._L.qrl_mmdvm_tx_read(self._h, out.ctypes.data_as(C.c_void_p), out.shape[1]), self._h, "qrl_mmdvm_tx_read")
        return out[:, :n.value]

    def out_device(self):
        d, s, n = C.c_void_p(), C.c_long(), C.c_long()
        check(self._L.qrl_mmdvm_tx_out_device(self._h, C.byref(d), C.byref(s), C.byref(n)), self._h, "qrl_mmdvm_tx_out_device")
        return d.value, s.value, n.value

    launches = property(Handle._launches)


class MmdvmDemod:
    """make_gr_demod_mmdvm_multi2(burst_timer, num_channels, 25000, use_tdma, 125, 250000, 1700, filter_width) up to gr_mmdvm_sink:
    wideband gr_complex at 250 ksps -> int16 at 24 ksps for channels 0..num_channels-1 (port map of gr_demod_mmdvm_multi2.cpp:110-124)."""

    def __init__(self, num_channels=3, filter_width=5000, samp_rate=MMDVM_SAMPLE_RATE, max_in=1 << 18, device=0):
        L = load_library()
        self.num_channels = min(int(num_channels), MAX_MMDVM_CHANNELS)
        taps = _low_pass_2(L, 1, samp_rate, filter_width, 2000, 60)                        # gr_demod_mmdvm_multi2.cpp:56-57
        self.channelizer = PfbChannelizer(10, taps, max_in=max_in, device=device)
        self.channels = MmdvmChannelsRx(self.num_channels, rows=mmdvm_port_map(self.num_channels), n_rows=10, filter_width=filter_width,
                                        max_in=max_in // 10 + 16, device=device)

    def calibrate_rssi(self, level):
        self.channels.calibrate_rssi(level)

    def work(self, x):
        x = np.ascontiguousarray(x, np.complex64)
        n = C.c_long()
        pf = self.channelizer
        check(pf._L.qrl_pfb_work(pf._h, x.ctypes.data_as(C.c_void_p), len(x), 0, 0, C.byref(n)), pf._h, "qrl_pfb_work")
        ptr, stride, items = pf.out_device()
        pf.sync()
        m = self.channels.work_device(ptr, items, stride)
        return self.channels._read(m)

    def close(self):
        self.channelizer.close(); self.channels.close()


class MmdvmMod:
    """make_gr_mod_mmdvm_multi2(...) behind gr_mmdvm_source: int16 at 24 ksps per channel -> one wideband gr_complex stream at 250 ksps."""

    def __init__(self, num_channels=3, filter_width=5000, samp_rate=MMDVM_SAMPLE_RATE, max_in=1 << 15, device=0):
        L = load_library()
        self._L = L
        self.num_channels = min(int(num_channels), MAX_MMDVM_CHANNELS)
        taps = _low_pass_2(L, 10, samp_rate, filter_width, 2000, 60)                       # gr_mod_mmdvm_multi2.cpp:88-89
        self.channels = MmdvmChannelsTx(self.num_channels, rows=mmdvm_port_map(self.num_channels), n_rows=10, filter_width=filter_width,
                                        max_in=max_in, device=device)
        self.synthesizer = PfbSynthesizer(10, taps, max_in=max_in * 25 // 24 + 16, device=device)

    def set_bb_gain(self, g):
        self.channels.set_bb_gain(g)

    def zero_samples(self, sample_index, n_samples, channel=-1):
        self.channels.zero_samples(sample_index, n_samples, channel)

    def work(self, samples):
        samples = np.ascontiguousarray(samples, np.int16)
        n = C.c_long()
        ch = self.channels
        check(ch._L.qrl_mmdvm_tx_work(ch._h, samples.ctypes.data_as(C.c_void_p), samples.shape[1], samples.shape[1], 0, C.byref(n)), ch._h, "qrl_mmdvm_tx_work")
        ptr, stride, items = ch.out_device()
        check(ch._L.qrl_mmdvm_tx_sync(ch._h), ch._h, "qrl_mmdvm_tx_sync")
        sy = self.synthesizer
        wide = sy.work_device(ptr, items, stride)
        sy.sync()
        wptr, _, wn = sy.out_device()
        check(ch._L.qrl_mmdvm_tx_finish(ch._h, C.c_void_p(wptr), wn), ch._h, "qrl_mmdvm_tx_finish")
        check(ch._L.qrl_mmdvm_tx_sync(ch._h), ch._h, "qrl_mmdvm_tx_sync")
        out = np.zeros(max(1, wn), np.complex64)
        check(sy._L.qrl_pfb_read(sy._h, out.ctypes.data_as(C.c_void_p), 0), sy._h, "qrl_pfb_read")
        return out[:wn]

    def close(self):
        self.channels.close(); self.synthesizer.close()
