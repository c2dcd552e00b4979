"""DMR burst decoder on the device: gr_dmr_sink plus the per-burst FEC behind the DMR demodulator, for a batch of channels.

DmrBurstDecoder takes QRL_DEMOD_DMR's port 2 (one hard bit per byte) and returns, per burst in the order of gr_dmr_sink's
_frame_buffer, what DMRControl::addFrames reads of a DMRFrame: the sink's fields, the CACH, the slot type, validate()'s verdict and
IDs, the EMB of voice bursts B-F, the AMBE error count and the burst bytes as the reference leaves them.  The burst search, BPTC,
CRC, RS(12,9), trellis, Golay, QR and AMBE decoding run in libqrl_b200.so (qrl_dmr.cu); this module moves buffers."""
import ctypes as C

import numpy as np

from .lib import Handle, check, load_library

# one record of qrl_dmr_rx (include/qrl_b200.h)
DMR_RECORD = np.dtype([
    ("position", "<i8"), ("ts_index", "u1"), ("frame_type", "u1"), ("fn", "u1"), ("downlink", "u1"),
    ("cach_decoded", "u1"), ("at", "u1"), ("slot_no", "u1"), ("lcss", "u1"),
    ("color_code", "u1"), ("data_type", "u1"), ("valid", "u1"), ("flco", "u1"), ("fid", "u1"),
    ("emb_cc", "u1"), ("emb_pi", "u1"), ("emb_lcss", "u1"),
    ("src_id", "<u4"), ("dst_id", "<u4"), ("ambe_errors", "<i4"), ("cach", "u1", (3,)), ("frame", "u1", (33,))])
assert DMR_RECORD.itemsize == 72


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class DmrBurstDecoder(Handle):
    """gr_dmr_sink + DMRFrame decoding for n_channels channels of up to max_bits bits per call; up to max_bursts records per channel
    and call (more advance the state but are counted by dropped() instead of stored).  ambe_fec: Settings::dmr_vocoder, i.e. whether
    voice bursts go through CAMBEFEC::regenerateDMR.  Sink state carries across calls."""
    ABI = "dmr_rx"

    def __init__(self, n_channels, max_bits, max_bursts, ambe_fec=False, device=0):
        self._L = load_library()
        self.n_channels, self.max_bits, self.max_bursts = int(n_channels), int(max_bits), int(max_bursts)
        self._create(self._L.qrl_dmr_rx_create, self.n_channels, self.max_bits, self.max_bursts, int(bool(ambe_fec)), device)

    set_stream = Handle._set_stream
    sync = Handle._sync
    launches = property(Handle._launches)

    def reset(self, channel=-1):
        """gr_dmr_sink's constructor state for one channel (-1: every channel)"""
        check(self._L.qrl_dmr_rx_reset(self._h, int(channel)), self._h, "qrl_dmr_rx_reset")

    def dropped(self):
        d = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_dmr_rx_dropped(self._h, _p(d)), self._h, "qrl_dmr_rx_dropped")
        return d

    def out_device(self):
        """device pointers of the last call's [n_channels][max_bursts][72] records and [n_channels] counts"""
        r, c = C.c_void_p(), C.c_void_p()
        check(self._L.qrl_dmr_rx_out_device(self._h, C.byref(r), C.byref(c)), self._h, "qrl_dmr_rx_out_device")
        return r, c

    def read(self):
        """list per channel of a DMR_RECORD array, one entry per burst of the last call"""
        rec = np.zeros((self.n_channels, self.max_bursts), DMR_RECORD)
        cnt = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_dmr_rx_read(self._h, _p(rec), _p(cnt)), self._h, "qrl_dmr_rx_read")
        return [rec[c, :cnt[c]].copy() for c in range(self.n_channels)]

    def work(self, bits, counts=None, collect=True):
        """bits: [n_channels][stride] uint8 (one bit per byte, bit 0 used) or a list of per-channel arrays"""
        if isinstance(bits, (list, tuple)):
            stride = max([len(b) for b in bits] + [1])
            buf = np.zeros((self.n_channels, stride), np.uint8)
            cnt = np.zeros(self.n_channels, np.int32)
            for c, b in enumerate(bits):
                buf[c, :len(b)] = b
                cnt[c] = len(b)
        else:
            buf = np.ascontiguousarray(bits, np.uint8)
            cnt = np.full(self.n_channels, buf.shape[1], np.int32) if counts is None else np.ascontiguousarray(counts, np.int32)
        if buf.shape[0] != self.n_channels or cnt.shape != (self.n_channels,):
            raise ValueError("bits must be [n_channels][stride] with n_channels counts")
        check(self._L.qrl_dmr_rx_work(self._h, _p(buf), _p(cnt), buf.shape[1], 0), self._h, "qrl_dmr_rx_work")
        return self.read() if collect else None

    def work_from_demod(self, rx_block, collect=True):
        """decode the DMR demodulator's last port-2 output in place on the device (qrl_rx_port_device)"""
        data, cap, cnts = C.c_void_p(), C.c_long(), C.c_void_p()
        # the two handles run on different streams: the demodulator's call has to finish before the sink reads port 2.  The data
        # stays in HBM; only the host waits.  A caller that shares one stream between both handles (set_stream) needs no wait.
        check(self._L.qrl_rx_sync(rx_block._h), rx_block._h, "qrl_rx_sync")
        check(self._L.qrl_rx_port_device(rx_block._h, 2, C.byref(data), C.byref(cap), C.byref(cnts)), rx_block._h, "qrl_rx_port_device")
        check(self._L.qrl_dmr_rx_work(self._h, data, cnts, cap.value, 1), self._h, "qrl_dmr_rx_work")
        return self.read() if collect else None
