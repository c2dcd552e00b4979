"""Layer-1 deframer on the device (SURVEY.md section 8f row 2): host-side mirror of gr_modem::synchronize / findSync /
packBytes (/root/reference/src/gr_modem.cpp:1119-1282, 980-994) for a batch of channels.  The search and the packing
run in libqrl_b200.so (CUDA); this class only moves buffers and splits the returned records."""
import ctypes as C

import numpy as np

from .lib import Handle, check, load_library

SYNC_1K, SYNC_NARROW, SYNC_WIDE = 1, 2, 3

# frame types = sync words (layer1framing.h:8-24)
FrameTypeVoice, FrameTypeVoice1, FrameTypeText, FrameTypeIP = 0xED89, 0xB5, 0x89EDAA, 0xDE98AA
FrameTypeVideo, FrameTypeCallsign, FrameTypeProto, FrameTypeEnd = 0x98DEAA, 0x8CC8DD, 0xED77AA, 0x4C8A2B

# (sync_class, bit_buf_len, rx_frame_length) per modem type as gr_modem::toggleRxMode sets them (gr_modem.cpp:203-322)
MODE_FRAMING = {
    "BPSK2K": (SYNC_NARROW, 64, 7), "BPSK1K": (SYNC_1K, 32, 4), "2FSK1KFM": (SYNC_1K, 32, 4), "2FSK1K": (SYNC_1K, 32, 4),
    "QPSK20K": (SYNC_NARROW, 384, 47), "QPSK2K": (SYNC_NARROW, 64, 7), "4FSK10KFM": (SYNC_NARROW, 384, 47),
    "2FSK10KFM": (SYNC_NARROW, 384, 47), "4FSK2K": (SYNC_NARROW, 64, 7), "4FSK2KFM": (SYNC_NARROW, 64, 7),
    "4FSK1KFM": (SYNC_1K, 32, 4), "QPSKVideo": (SYNC_WIDE, 3123 * 8, 3122), "2FSK2KFM": (SYNC_NARROW, 64, 7),
    "2FSK2K": (SYNC_NARROW, 64, 7), "QPSK250K": (SYNC_WIDE, 1517 * 8, 1516), "4FSK100K": (SYNC_WIDE, 623 * 8, 622),
}


SYNC_M17 = 4
FrameTypeM17Stream, FrameTypeM17LSF, FrameTypeM17EOT = 0xFF5D, 0x55F7, 0x555D555D
MODE_FRAMING["M17"] = (SYNC_M17, 46 * 8, 46)          # gr_modem.cpp:309-313


def frame(payloads, frame_types, one_k_mode=False, burst_ip=False, device=0):
    """gr_modem::frame (gr_modem.cpp:904-961) for a batch: list of payload bytes + list of frame types -> list of byte arrays for TxBlock.work."""
    L = load_library()
    Cn = len(payloads)
    n = max(1, max(len(p) for p in payloads))
    buf = np.zeros((Cn, n), np.uint8)
    lens = np.zeros(Cn, np.int32)
    for c, p in enumerate(payloads):
        buf[c, :len(p)] = np.frombuffer(bytes(p), np.uint8); lens[c] = len(p)
    types = np.asarray(frame_types, np.uint32)
    out = np.zeros((Cn, n + 16), np.uint8)
    olen = np.zeros(Cn, np.int32)
    check(L.qrl_frame_build(Cn, buf.ctypes.data_as(C.c_void_p), n, lens.ctypes.data_as(C.c_void_p), types.ctypes.data_as(C.c_void_p),
                            int(one_k_mode), int(burst_ip), out.ctypes.data_as(C.c_void_p), n + 16, olen.ctypes.data_as(C.c_void_p), 0, device, None),
          None, "qrl_frame_build")
    return [out[c, :olen[c]].copy() for c in range(Cn)]


class Deframer(Handle):
    ABI = "deframer"

    def __init__(self, sync_class, bit_buf_len, rx_frame_length, n_channels=1, max_bits=1 << 20, max_frames=None, device=0):
        self._L = load_library()
        self.n_channels, self.max_bits = int(n_channels), int(max_bits)
        self.max_frames = int(max_frames) if max_frames else max(4, self.max_bits // max(8, bit_buf_len - 8) + 2)
        self._create(self._L.qrl_deframer_create, sync_class, bit_buf_len, rx_frame_length, self.n_channels, self.max_bits, self.max_frames,
                     device)
        self.rec_bytes = self._L.qrl_deframer_record_bytes(self._h)

    @classmethod
    def for_mode(cls, mode, **kw):
        return cls(*MODE_FRAMING[mode], **kw)

    set_stream = Handle._set_stream

    def _collect(self):
        rec = np.zeros((self.n_channels, self.max_frames, self.rec_bytes), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        self.modem_sync = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_deframer_read(self._h, rec.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p),
                                        self.modem_sync.ctypes.data_as(C.c_void_p)), self._h, "qrl_deframer_read")
        out = []
        for c in range(self.n_channels):
            fr = []
            for r in rec[c, :cnt[c]]:
                ty, nb = int(r[:4].view(np.uint32)[0]), int(r[4:8].view(np.uint32)[0])
                fr.append((ty, r[8:8 + nb].tobytes()))
            out.append(fr)
        return out

    def work(self, bits_per_channel):
        """bits_per_channel: list of uint8 arrays (one decoded bit per byte) -> list (per channel) of (frame_type, payload)."""
        n = max(1, max(len(b) for b in bits_per_channel))
        buf = np.zeros((self.n_channels, n), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        for c, b in enumerate(bits_per_channel):
            buf[c, :len(b)] = b; cnt[c] = len(b)
        check(self._L.qrl_deframer_work(self._h, buf.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), n, 0),
              self._h, "qrl_deframer_work")
        return self._collect()

    def work_from_rx(self, rx, port=2):
        """Deframe what the last rx.work() left on `port` without leaving the GPU (qrl_rx_port_device)."""
        data, cap, cnts = C.c_void_p(), C.c_long(), C.c_void_p()
        check(self._L.qrl_rx_port_device(rx._h, port, C.byref(data), C.byref(cap), C.byref(cnts)), rx._h, "qrl_rx_port_device")
        rx.sync()
        check(self._L.qrl_deframer_work(self._h, data, cnts, cap.value, 1), self._h, "qrl_deframer_work")
        return self._collect()

    def work2(self, bits_a, bits_b):
        """Dual-decoder modes: per channel the LONGER of the two candidate streams of this call is deframed, the first on a tie
        (gr_modem::demodulate, gr_modem.cpp:1066-1085)."""
        n = max(1, max(len(b) for b in list(bits_a) + list(bits_b)))
        bufs, cnts = [], []
        for src in (bits_a, bits_b):
            buf = np.zeros((self.n_channels, n), np.uint8)
            cnt = np.zeros(self.n_channels, np.int32)
            for c, b in enumerate(src):
                buf[c, :len(b)] = b; cnt[c] = len(b)
            bufs.append(buf); cnts.append(cnt)
        check(self._L.qrl_deframer_work2(self._h, bufs[0].ctypes.data_as(C.c_void_p), cnts[0].ctypes.data_as(C.c_void_p),
                                         bufs[1].ctypes.data_as(C.c_void_p), cnts[1].ctypes.data_as(C.c_void_p), n, 0), self._h, "qrl_deframer_work2")
        return self._collect()

    def work2_from_dfbb(self, dfbb_a, dfbb_b):
        """Same, with both candidates still on the GPU (the outputs of two DeframerBB.work_from_rx calls)."""
        pa, sa, ca = dfbb_a.out_device()
        pb, sb, cb = dfbb_b.out_device()
        if sa != sb:
            raise ValueError("the two gr_deframer_bb handles must have the same max_bits")
        dfbb_a.sync(); dfbb_b.sync()
        check(self._L.qrl_deframer_work2(self._h, pa, ca, pb, cb, sa, 1), self._h, "qrl_deframer_work2")
        return self._collect()

    def dropped(self):
        """frames found beyond max_frames since creation, per channel"""
        d = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_deframer_dropped(self._h, d.ctypes.data_as(C.c_void_p)), self._h, "qrl_deframer_dropped")
        return d

    launches = property(Handle._launches)


class DeframerBB(Handle):
    """gr_deframer_bb (src/gr/gr_deframer_bb.cpp:83-185) for a batch of channels: modem_type 1 / 2 / 3 as gr_demod_base creates them
    (_deframer1/2, _deframer_700_1/2, _deframer_10k_1/2).  work() returns, per channel, the bit stream get_data() would hand to gr_modem."""
    ABI = "dfbb"

    def __init__(self, modem_type, n_channels=1, max_bits=1 << 20, device=0):
        self._L = load_library()
        self.n_channels, self.max_bits = int(n_channels), int(max_bits)
        self._create(self._L.qrl_dfbb_create, int(modem_type), self.n_channels, self.max_bits, device)

    sync = Handle._sync

    def out_device(self):
        p, s, c = C.c_void_p(), C.c_long(), C.c_void_p()
        check(self._L.qrl_dfbb_out_device(self._h, C.byref(p), C.byref(s), C.byref(c)), self._h, "qrl_dfbb_out_device")
        return p, s.value, c

    def _collect(self):
        cap = self.max_bits + 32
        out = np.zeros((self.n_channels, cap), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        check(self._L.qrl_dfbb_read(self._h, out.ctypes.data_as(C.c_void_p), cap, cnt.ctypes.data_as(C.c_void_p)), self._h, "qrl_dfbb_read")
        return [out[c, :cnt[c]].copy() for c in range(self.n_channels)]

    def work(self, bits_per_channel):
        n = max(1, max(len(b) for b in bits_per_channel))
        buf = np.zeros((self.n_channels, n), np.uint8)
        cnt = np.zeros(self.n_channels, np.int32)
        for c, b in enumerate(bits_per_channel):
            buf[c, :len(b)] = b; cnt[c] = len(b)
        check(self._L.qrl_dfbb_work(self._h, buf.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p), n, 0), self._h, "qrl_dfbb_work")
        return self._collect()

    def work_from_rx(self, rx, port, collect=True):
        """Deframe what the last rx.work() left on bit port 2 / 3 without leaving the GPU."""
        data, cap, cnts = C.c_void_p(), C.c_long(), C.c_void_p()
        check(self._L.qrl_rx_port_device(rx._h, port, C.byref(data), C.byref(cap), C.byref(cnts)), rx._h, "qrl_rx_port_device")
        rx.sync()
        check(self._L.qrl_dfbb_work(self._h, data, cnts, cap.value, 1), self._h, "qrl_dfbb_work")
        return self._collect() if collect else None
