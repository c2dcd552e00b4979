"""DMR burst decoder on the device: gr_dmr_sink plus the per-burst FEC behind the DMR demodulator, for a batch of channels.

DmrBurstDecoder takes QRL_DEMOD_DMR's port 2 (one hard bit per byte) and returns, per burst in the order of gr_dmr_sink's
_frame_buffer, what DMRControl::addFrames reads of a DMRFrame: the sink's fields, the CACH, the slot type, validate()'s verdict and
IDs, the EMB of voice bursts B-F, the AMBE error count and the burst bytes as the reference leaves them.  The burst search, BPTC,
CRC, RS(12,9), trellis, Golay, QR and AMBE decoding run in libqrl_b200.so (qrl_dmr.cu); this module moves buffers.

DmrBurstEncoder is the other direction: per-channel ops (CSBK, voice header, vocoder frame, stop -- the calls gr_modem makes into
DMRControl) and 9-byte vocoder frames in, the bytes gr_dmr_source hands to the DMR modulator out, with one record per burst for its
tx_time and zero_samples tags.  The state machine and every encoder run in qrl_dmr.cu."""
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


# ---------------------------------------------------------------------------------------------------------------- transmit
OP_NONE, OP_CSBK, OP_HEADER, OP_AUDIO, OP_STOP = 0, 1, 2, 3, 4
KIND_CSBK, KIND_LC_HEADER, KIND_VOICE_SYNC, KIND_VOICE, KIND_TERMINATOR, KIND_EMPTY = 1, 2, 3, 4, 5, 6
TX_BURST_BYTES = 72            # 33 frame bytes + 39 zero bytes
TX_ZERO_OFFSET, TX_ZERO_SAMPLES = 33, 780     # gr_dmr_source's "zero_samples" tag: byte 33 of a burst, 39 * 4 * 5 samples
# one record of qrl_dmr_tx (include/qrl_b200.h)
DMR_TX_RECORD = np.dtype([("position", "<i8"), ("slot", "u1"), ("kind", "u1"), ("fn", "u1"), ("lcss", "u1"), ("op", "<i4")])
assert DMR_TX_RECORD.itemsize == 16


class _TxConfig(C.Structure):
    _fields_ = [("color_code", C.c_int), ("timeslot", C.c_int), ("src_id", C.c_uint), ("dst_id", C.c_uint), ("private_call", C.c_int),
                ("codec2", C.c_int), ("talker_alias_len", C.c_int), ("talker_alias", C.c_ubyte * 28)]


def dmr_tx_config(color_code=1, timeslot=1, src_id=1, dst_id=9, private_call=False, codec2=True, talker_alias=""):
    """qrl_dmr_tx_config from the Settings fields DMRControl reads (defaults: Settings' own).  codec2 is `not dmr_vocoder`;
    talker_alias is a str (or bytes) cut, as DMRControl copies it, to min(len(alias), 27) bytes of its UTF-8 form."""
    if isinstance(talker_alias, str):
        ta = talker_alias.encode("utf-8")[:min(len(talker_alias), 27)]
    else:
        ta = bytes(talker_alias)[:27]
    cfg = _TxConfig(int(color_code), int(timeslot), int(src_id), int(dst_id), int(bool(private_call)), int(bool(codec2)), len(ta))
    cfg.talker_alias[:len(ta)] = list(ta)
    return cfg


class DmrBurstEncoder(Handle):
    """DMRControl's transmit side plus gr_dmr_source's framing for n_channels channels, max_ops ops per channel and call (every op
    makes at most 4 bursts).  State carries across calls."""
    ABI = "dmr_tx"

    def __init__(self, n_channels=1, max_ops=64, device=0):
        self._L = load_library()
        self.n_channels, self.max_ops = int(n_channels), int(max_ops)
        self.max_bursts = 4 * self.max_ops
        self._create(self._L.qrl_dmr_tx_create, self.n_channels, self.max_ops, device)
        self._fed = 0          # bytes of this encoder handed to the modulator by feed()

    set_stream = Handle._set_stream
    sync = Handle._sync
    launches = property(Handle._launches)

    def set_config(self, cfg=None, channel=-1, **kw):
        """cfg: a dmr_tx_config(...) (or its keyword arguments); channel -1 = every channel"""
        cfg = dmr_tx_config(**kw) if cfg is None else cfg
        check(self._L.qrl_dmr_tx_set_config(self._h, int(channel), C.byref(cfg)), self._h, "qrl_dmr_tx_set_config")

    def reset(self, channel=-1):
        """DMRControl's constructor state under the config in force, byte position 0 (-1: every channel)"""
        check(self._L.qrl_dmr_tx_reset(self._h, int(channel)), self._h, "qrl_dmr_tx_reset")

    def out_device(self):
        """device pointers of the last call's [n_channels][stride] bytes, [n_channels] byte counts and records, and the stride"""
        b, s, c, r = C.c_void_p(), C.c_long(), C.c_void_p(), C.c_void_p()
        check(self._L.qrl_dmr_tx_out_device(self._h, C.byref(b), C.byref(s), C.byref(c), C.byref(r)), self._h, "qrl_dmr_tx_out_device")
        return b, s.value, c, r

    def work(self, ops, audio=None, collect=True):
        """ops [n_channels][K] of OP_*, audio [n_channels][K][9] -> (list per channel of its bytes, list per channel of DMR_TX_RECORD)"""
        ops = np.ascontiguousarray(ops, np.uint8)
        K = ops.shape[1]
        au = np.zeros((self.n_channels, K, 9), np.uint8) if audio is None else np.ascontiguousarray(audio, np.uint8)
        if ops.shape[0] != self.n_channels or au.shape != (self.n_channels, K, 9):
            raise ValueError("ops must be [n_channels][K], audio [n_channels][K][9]")
        check(self._L.qrl_dmr_tx_work(self._h, _p(ops), _p(au), K, 0), self._h, "qrl_dmr_tx_work")
        return self.read() if collect else None

    def work_device(self, ops_ptr, audio_ptr, K):
        """ops [n_channels][K] and audio [n_channels][K][9] already in this handle's GPU memory"""
        check(self._L.qrl_dmr_tx_work(self._h, C.c_void_p(ops_ptr), C.c_void_p(audio_ptr), int(K), 1), self._h, "qrl_dmr_tx_work")

    def read(self):
        stride = self.max_bursts * TX_BURST_BYTES
        out = np.zeros((self.n_channels, stride), np.uint8)
        rec = np.zeros((self.n_channels, self.max_bursts), DMR_TX_RECORD)
        cnt = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_dmr_tx_read(self._h, _p(out), stride, _p(rec), _p(cnt)), self._h, "qrl_dmr_tx_read")
        return ([out[c, :cnt[c]].copy() for c in range(self.n_channels)],
                [rec[c, :cnt[c] // TX_BURST_BYTES].copy() for c in range(self.n_channels)])

    def feed(self, tx_block):
        """hand the last call's bytes to a make_gr_mod_dmr block on the device, with gr_dmr_source's "zero_samples" tag registered
        (TxBlock.zero_samples) for every burst at the modulator's byte position, which counts the bytes this encoder has fed it (the
        block takes its input from this encoder alone).  Every channel must carry the same byte count: the modulator takes one count
        per call.  Returns the modulator's output (complex64 [n_channels, n_out])."""
        cnt = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_dmr_tx_read(self._h, None, 0, None, _p(cnt)), self._h, "qrl_dmr_tx_read")     # the counts alone
        n = int(cnt[0])
        if np.any(cnt != n):
            raise ValueError("DmrBurstEncoder.feed: the channels' byte counts differ; the modulator takes one count per call")
        for k in range(n // TX_BURST_BYTES):
            tx_block.zero_samples(self._fed + k * TX_BURST_BYTES + TX_ZERO_OFFSET, TX_ZERO_SAMPLES)
        b, stride, _, _ = self.out_device()
        # the two handles run on different streams: reading the counts synchronised the encoder's call before the modulator reads
        # its bytes, and reading the modulator's output below waits for the modulator before the encoder's next call overwrites them
        L = self._L
        check(L.qrl_tx_work(tx_block._h, b, n, stride, 1), tx_block._h, "qrl_tx_work")
        self._fed += n
        nout = C.c_long()
        check(L.qrl_tx_out_device(tx_block._h, None, None, C.byref(nout)), tx_block._h, "qrl_tx_out_device")
        out = np.zeros((self.n_channels, max(1, nout.value)), np.complex64)
        n2 = C.c_long()
        check(L.qrl_tx_read(tx_block._h, _p(out), max(1, nout.value), C.byref(n2), 0), tx_block._h, "qrl_tx_read")
        return out[:, :n2.value]
