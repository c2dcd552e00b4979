"""M17 frame codec on the device: the FEC half of gr_modem's M17 branches for a batch of channels.

M17Decoder takes the records of the layer-1 deframer (sync class 4) and returns, per record, what gr_modem reads after
M17FrameDecoder::decodeFrame: the frame type, the current LSF with its CRC verdict, and the current stream frame (frame number and
16-byte codec2 payload).  M17Encoder turns per-channel op sequences (start / stream frame / last frame) and codec2 payloads into
the bytes M17Transmitter and gr_modem::endTransmission push, the input of the M17 modulator.  The decorrelation, interleaving,
convolutional coding, puncturing, Viterbi decoding, Golay LICH coding and LSF reassembly run in libqrl_b200.so (qrl_m17.cu); this
module moves buffers and restates the LSF fill of M17Transmitter::start (m17_lsf) and the callsign decoding (m17_callsign)."""
import ctypes as C

import numpy as np

from .lib import Handle, check, load_library

OP_NONE, OP_START, OP_STREAM, OP_LAST = 0, 1, 2, 3
RX_RECORD_BYTES = 56          # {uint32 frame_type, lsf[30], lsf_valid, 0, stream_frame[18], 0, 0}
TX_STEP_BYTES = 96            # the longest op: 48-byte preamble + 48-byte LSF frame

_CHARS = "xABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789-/."
# the four special destinations of M17LinkSetupFrame::setDestination(int): ALL, ECHO, INFO, UNLINK
_SPECIAL_DST = {1: bytes([0xFF] * 6), 2: bytes([0, 0, 0, 0x0E, 0xD8, 0x7D]), 3: bytes([0, 0, 0, 0x0E, 0xCD, 0xB9]),
                4: bytes([0, 0, 0x45, 0x4F, 0x77, 0x45])}


def m17_crc16(data):
    """M17 CRC-16: polynomial 0x5935, initial value 0xFFFF, MSB first, no final XOR"""
    crc = 0xFFFF
    for b in bytes(data):
        crc ^= b << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x5935) if crc & 0x8000 else (crc << 1)
            crc &= 0xFFFF
    return crc


def m17_encode_callsign(callsign):
    """base-40 callsign, 6 bytes big endian; more than 9 characters encode as zeros, characters outside A-Z 0-9 - / . as 0"""
    if len(callsign) > 9:
        return bytes(6)
    v = 0
    for ch in reversed(callsign):
        v *= 40
        if "A" <= ch <= "Z":
            v += ord(ch) - ord("A") + 1
        elif "0" <= ch <= "9":
            v += ord(ch) - ord("0") + 27
        elif ch in "-/.":
            v += 37 + "-/.".index(ch)
    return (v & 0xFFFFFFFFFFFF).to_bytes(6, "big")


def m17_callsign(bytes6):
    """decode a 6-byte callsign field of a decoded LSF (all 0xFF: "BROADCAST")"""
    b = bytes(bytes6)
    if b == bytes([0xFF] * 6):
        return "BROADCAST"
    v, s = int.from_bytes(b, "big"), ""
    while v:
        s += _CHARS[v % 40]
        v //= 40
    return s


def m17_lsf(src, dst="", can=0, destination_type=0):
    """The 28 LSF bytes before the CRC (dst, src, type, meta) as M17Transmitter::start fills them: destination_type 0 encodes `dst`
    (an empty one leaves the broadcast address), 1 - 4 are ALL / ECHO / INFO / UNLINK; type = stream, voice, CAN; meta zero."""
    d = bytes([0xFF] * 6)
    if destination_type == 0:
        if dst:
            d = m17_encode_callsign(dst)
    elif destination_type in _SPECIAL_DST:
        d = _SPECIAL_DST[destination_type]
    t = 1 | (2 << 1) | ((int(can) & 0xF) << 7)
    return d + m17_encode_callsign(src) + bytes([t >> 8, t & 0xFF]) + bytes(14)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class M17Decoder(Handle):
    """M17FrameDecoder plus gr_modem's M17 record handling for n_channels channels; state (LSF, partial LSF from the LICH, segment
    map, stream frame) carries across calls."""
    ABI = "m17_rx"

    def __init__(self, n_channels=1, max_frames=64, device=0):
        self._L = load_library()
        self.n_channels, self.max_frames = int(n_channels), int(max_frames)
        self._create(self._L.qrl_m17_rx_create, self.n_channels, self.max_frames, device)

    set_stream = Handle._set_stream
    sync = Handle._sync
    launches = property(Handle._launches)

    def reset(self, channel):
        check(self._L.qrl_m17_rx_reset(self._h, int(channel)), self._h, "qrl_m17_rx_reset")

    def out_device(self):
        """device pointers of the last call's [n_channels][max_frames][56] records and [n_channels] counts"""
        r, c = C.c_void_p(), C.c_void_p()
        check(self._L.qrl_m17_rx_out_device(self._h, C.byref(r), C.byref(c)), self._h, "qrl_m17_rx_out_device")
        return r, c

    def read(self):
        """list per channel of (frame_type, lsf bytes[30], lsf_valid, stream_frame bytes[18])"""
        rec = np.zeros((self.n_channels, self.max_frames, RX_RECORD_BYTES), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_m17_rx_read(self._h, _p(rec), _p(cnt)), self._h, "qrl_m17_rx_read")
        self.raw, self.counts = rec, cnt
        return [[(int(r[:4].view(np.uint32)[0]), r[4:34].tobytes(), bool(r[34]), r[36:54].tobytes()) for r in rec[c, :cnt[c]]]
                for c in range(self.n_channels)]

    def work(self, records):
        """records: list per channel of (frame_type, payload bytes) -- what Deframer.work returns for the M17 mode"""
        rb = 8 + 48
        buf = np.zeros((self.n_channels, self.max_frames, rb), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        for c, recs in enumerate(records):
            if len(recs) > self.max_frames:
                raise ValueError("channel %d: %d records, max_frames is %d" % (c, len(recs), self.max_frames))
            cnt[c] = len(recs)
            for f, (ty, payload) in enumerate(recs):
                p = np.frombuffer(bytes(payload)[:46], np.uint8)
                buf[c, f, :4] = np.frombuffer(np.uint32(ty).tobytes(), np.uint8)
                buf[c, f, 4:8] = np.frombuffer(np.uint32(len(p)).tobytes(), np.uint8)
                buf[c, f, 8:8 + len(p)] = p
        check(self._L.qrl_m17_rx_work(self._h, _p(buf), _p(cnt), rb, self.max_frames, 0), self._h, "qrl_m17_rx_work")
        return self.read()

    def work_from_deframer(self, deframer, collect=True):
        """decode what the deframer's last call found, in place on the device (qrl_deframer_out_device)"""
        r, c = C.c_void_p(), C.c_void_p()
        check(self._L.qrl_deframer_out_device(deframer._h, C.byref(r), C.byref(c)), deframer._h, "qrl_deframer_out_device")
        check(self._L.qrl_deframer_sync(deframer._h), deframer._h, "qrl_deframer_sync")
        check(self._L.qrl_m17_rx_work(self._h, r, c, deframer.rec_bytes, deframer.max_frames, 1), self._h, "qrl_m17_rx_work")
        return self.read() if collect else None


class M17Encoder(Handle):
    """M17Transmitter::start / send and gr_modem::endTransmission's M17 tail for n_channels channels, max_steps ops per channel per
    call.  Frame number and LICH index carry across calls."""
    ABI = "m17_tx"

    def __init__(self, n_channels=1, max_steps=64, device=0):
        self._L = load_library()
        self.n_channels, self.max_steps = int(n_channels), int(max_steps)
        self._create(self._L.qrl_m17_tx_create, self.n_channels, self.max_steps, device)

    set_stream = Handle._set_stream
    sync = Handle._sync
    launches = property(Handle._launches)

    def set_lsf(self, channel, lsf28):
        b = np.frombuffer(bytes(lsf28), np.uint8)
        if len(b) != 28:
            raise ValueError("an LSF before its CRC has 28 bytes")
        check(self._L.qrl_m17_tx_set_lsf(self._h, int(channel), _p(b)), self._h, "qrl_m17_tx_set_lsf")

    def out_device(self):
        """device pointers of the last call's [n_channels][stride] bytes and [n_channels] counts, and the stride"""
        o, s, c = C.c_void_p(), C.c_long(), C.c_void_p()
        check(self._L.qrl_m17_tx_out_device(self._h, C.byref(o), C.byref(s), C.byref(c)), self._h, "qrl_m17_tx_out_device")
        return o, s.value, c

    def work(self, ops, payloads=None, collect=True):
        """ops [n_channels][K] of OP_*, payloads [n_channels][K][16] -> list per channel of the bytes produced"""
        ops = np.ascontiguousarray(ops, np.uint8)
        K = ops.shape[1]
        pl = np.zeros((self.n_channels, K, 16), np.uint8) if payloads is None else np.ascontiguousarray(payloads, np.uint8)
        if ops.shape[0] != self.n_channels or pl.shape != (self.n_channels, K, 16):
            raise ValueError("ops must be [n_channels][K], payloads [n_channels][K][16]")
        check(self._L.qrl_m17_tx_work(self._h, _p(ops), _p(pl), K, 0), self._h, "qrl_m17_tx_work")
        return self.read() if collect else None

    def read(self):
        stride = self.max_steps * TX_STEP_BYTES
        out = np.zeros((self.n_channels, stride), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_m17_tx_read(self._h, _p(out), stride, _p(cnt)), self._h, "qrl_m17_tx_read")
        return [out[c, :cnt[c]].copy() for c in range(self.n_channels)]
