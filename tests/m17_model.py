"""numpy restatement of the M17 frame codec (M17FrameDecoder / M17Transmitter and gr_modem's M17 branches), vectorised over frames.

TEST INFRASTRUCTURE: the expected values of the GPU tier (tests/test_gpu_m17_codec.py), where the compiled reference is absent.  It is
pinned to the reference's own code in the CPU tier (tests/test_m17_codec.py), and its constants are generated here from the M17
specification's definitions, independently of qrl_m17.cu."""
import numpy as np

from qradiolink_b200.m17 import m17_crc16

STREAM, LSF, EOT = 0xFF5D, 0x55F7, 0x555D555D

# puncture matrices: P1 = 1 followed by 15 x (1 0 1 1); P2 = 11 x 1 then 0
P1 = np.array([1] + [1, 0, 1, 1] * 15, np.uint8)
P2 = np.array([1] * 11 + [0], np.uint8)
# quadratic permutation polynomial interleaver over 368 bits: bit i goes to (45 i + 92 i^2) mod 368
QPP = np.array([(45 * i + 92 * i * i) % 368 for i in range(368)], np.int64)
# randomizer sequence of the M17 specification (46 bytes, XORed over the 368 payload bits of every frame)
RANDOMIZER = np.frombuffer(bytes.fromhex(
    "d6b5e23082ff8462ba4e9690d898dd5d0cc85243911df86e682f35da14eacd76198dd580d133871357182d2978c3"), np.uint8)


def _golay_rows():
    """row i = the 12 check bits of data bit i: (x^(11+i) mod g(x)) << 1 | overall parity, g = 0xC75 (the (23,12) Golay code)"""
    rows = []
    for i in range(12):
        r = 1 << (11 + i)
        for b in range(22, 10, -1):
            if r >> b & 1:
                r ^= 0xC75 << (b - 11)
        rows.append((r << 1) | ((1 + bin(r).count("1")) & 1))
    return rows


GOLAY_ENC = _golay_rows()
GOLAY_DEC = [sum(((GOLAY_ENC[k] >> j) & 1) << k for k in range(12)) for j in range(12)]     # the transpose = the inverse


def _mul(v, m):
    r = 0
    for i in range(12):
        if v >> i & 1:
            r ^= m[i]
    return r


def golay_encode(d):
    return (d << 12) | _mul(d, GOLAY_ENC)


def _error_of(s):
    """the error pattern M17's Golay decoder assumes for syndrome s (None: uncorrectable)"""
    pc = lambda v: bin(v).count("1")
    if pc(s) <= 3:
        return s
    for i in range(12):
        if pc(s ^ GOLAY_ENC[i]) <= 2:
            return ((1 << i) << 12) | (s ^ GOLAY_ENC[i])
    q = _mul(s, GOLAY_DEC)
    if pc(q) <= 3:
        return q << 12
    for i in range(12):
        if pc(q ^ GOLAY_DEC[i]) <= 2:
            return ((q ^ GOLAY_DEC[i]) << 12) | (1 << i)
    return None


GOLAY_ERR = [_error_of(s) for s in range(4096)]


def golay_decode(cw):
    e = GOLAY_ERR[(cw & 0xFFF) ^ _mul(cw >> 12, GOLAY_ENC)]
    return 0xFFFF if e is None else ((cw ^ e) >> 12) & 0xFFF


def bits_of(b):
    return np.unpackbits(np.asarray(b, np.uint8), axis=-1)


# ------------------------------------------------------------------------------------------------ transmit
def _conv(data_bits):
    """K = 5 encoder (G1 = 0x19, G2 = 0x17), zero state, 4 flush bits: [..., 2 n + 8] bits"""
    x = np.concatenate([np.zeros(data_bits.shape[:-1] + (4,), np.uint8), data_bits, np.zeros(data_bits.shape[:-1] + (4,), np.uint8)], -1)
    n = data_bits.shape[-1] + 4
    t = [x[..., 4 - k:4 - k + n] for k in range(5)]          # t[k] = input bit delayed by k
    g1 = t[0] ^ t[3] ^ t[4]                                   # 0x19: current, 3rd and 4th previous
    g2 = t[0] ^ t[1] ^ t[2] ^ t[4]                            # 0x17
    return np.stack([g1, g2], -1).reshape(data_bits.shape[:-1] + (2 * n,))


def _puncture(bits, p, n_out):
    keep = np.resize(p, bits.shape[-1]).astype(bool)
    return bits[..., keep][..., :n_out]


def _scramble(bits368):
    out = np.zeros_like(bits368)
    out[..., QPP] = bits368
    return out ^ bits_of(RANDOMIZER)


def lich_segments(lsf30):
    segs = []
    for n in range(6):
        ch = lsf30[5 * n:5 * n + 5]
        blocks = [ch[0] << 4 | ch[1] >> 4, (ch[1] & 15) << 8 | ch[2], ch[3] << 4 | ch[4] >> 4, (ch[4] & 15) << 8 | (n << 5)]
        segs.append(b"".join(golay_encode(int(b)).to_bytes(3, "big") for b in blocks))
    return segs


def lsf_frame(lsf30):
    bits = _puncture(_conv(bits_of(np.frombuffer(bytes(lsf30), np.uint8))), P1, 368)
    return bytes([0x55, 0xF7]) + np.packbits(_scramble(bits)).tobytes()


def stream_frame(lich12, fn, last, payload16):
    fnw = (fn & 0x7FFF) | (0x8000 if last else 0)
    data = bytes([fnw >> 8, fnw & 0xFF]) + bytes(payload16)
    bits = _puncture(_conv(bits_of(np.frombuffer(data, np.uint8))), P2, 272)
    return bytes([0xFF, 0x5D]) + np.packbits(_scramble(np.concatenate([bits_of(np.frombuffer(lich12, np.uint8)), bits]))).tobytes()


class Transmitter:
    """M17Transmitter (start / send) with gr_modem's endTransmission tail; the LSF comes in whole (28 bytes), as qrl_m17_tx_set_lsf takes it"""

    def __init__(self):
        self.fn, self.lich, self.lsf30 = 0, 0, None

    def set_lsf(self, lsf28):
        self.lsf30 = bytes(lsf28) + m17_crc16(bytes(lsf28)).to_bytes(2, "big")
        self.segs = lich_segments(np.frombuffer(self.lsf30, np.uint8).astype(int))

    def step(self, op, payload16):
        if op == 1:
            self.fn, self.lich = 0, 0
            return bytes([0x77] * 48) + lsf_frame(self.lsf30)
        if op in (2, 3):
            out = stream_frame(self.segs[self.lich], self.fn, op == 3, payload16)
            self.fn, self.lich = (self.fn + 1) & 0x7FF, (self.lich + 1) % 6
            return out + (bytes([0x55, 0x5D] * 8) if op == 3 else b"")
        return b""


# ------------------------------------------------------------------------------------------------ receive
def _descramble(payload46):
    """[N, 46] bytes -> [N, 368] deinterleaved bits"""
    b = bits_of(np.asarray(payload46, np.uint8)) ^ bits_of(RANDOMIZER)
    return b[:, QPP]


def viterbi(bits, p, n_out):
    """M17Viterbi::decodePunctured for [N, n_in] hard bits: uint16 metrics from 0, tie m0 >= m1 takes the upper predecessor,
    chainback over the last 8 n_out steps from state 0 with the reference's state update"""
    N, n_in = bits.shape
    syms, k, pi = [], 0, 0
    while k < n_in:
        s = []
        for _ in range(2):
            if p[pi]:
                s.append(bits[:, k].astype(np.int32) * 2); k += 1
            else:
                s.append(np.ones(N, np.int32))
            pi = (pi + 1) % len(p)
        syms.append(s)
    c0 = np.array([0, 0, 0, 0, 2, 2, 2, 2]); c1 = np.array([0, 2, 2, 0, 0, 2, 2, 0])
    prev = np.zeros((N, 16), np.int64)
    hist = np.zeros((len(syms), N, 16), bool)
    for t, (s0, s1) in enumerate(syms):
        met = np.abs(c0[None, :] - s0[:, None]) + np.abs(c1[None, :] - s1[:, None])     # [N, 8]
        lo, hi = prev[:, :8], prev[:, 8:]
        m0, m1, m2, m3 = lo + met, hi + 4 - met, lo + 4 - met, hi + met
        cur = np.empty_like(prev)
        cur[:, 0::2] = np.where(m0 >= m1, m1, m0); hist[t, :, 0::2] = m0 >= m1
        cur[:, 1::2] = np.where(m2 >= m3, m3, m2); hist[t, :, 1::2] = m2 >= m3
        prev = cur
    out = np.zeros((N, 8 * n_out), np.uint8)
    state = np.zeros(N, np.int64)
    pos = len(syms)
    for b in range(8 * n_out - 1, -1, -1):
        pos -= 1
        bit = hist[pos, np.arange(N), state >> 4]
        state = (state >> 1) | (bit.astype(np.int64) << 7)
        out[:, b] = bit
    return np.packbits(out, axis=1)


def decode_records(types, payloads):
    """per record: (kind, lsf30 or stream18, lich segment (6 bytes) or None) -- the per-frame half of M17FrameDecoder::decodeFrame"""
    types = np.asarray(types, np.uint32)
    payloads = np.asarray(payloads, np.uint8).reshape(-1, 46)
    bits = _descramble(payloads) if len(types) else np.zeros((0, 368), np.uint8)
    res = [None] * len(types)
    il, is_ = np.flatnonzero(types == LSF), np.flatnonzero(types == STREAM)
    for idx, first, p, n in ((il, 0, P1, 30), (is_, 96, P2, 18)):
        for k in range(0, len(idx), 8192):
            part = idx[k:k + 8192]
            for i, v in zip(part, viterbi(bits[part, first:], p, n)):
                res[i] = v.tobytes()
    lich = [None] * len(types)
    for i in is_:
        words = np.packbits(bits[i, :96]).tobytes()
        dec = [golay_decode(int.from_bytes(words[3 * k:3 * k + 3], "big")) for k in range(4)]
        if 0xFFFF not in dec:
            seg = [dec[0] >> 4, (dec[0] & 15) << 4 | dec[1] >> 8, dec[1] & 0xFF, dec[2] >> 4, (dec[2] & 15) << 4 | dec[3] >> 8, (dec[3] & 0xFF) >> 5]
            lich[i] = bytes(seg)
    return res, lich


def _valid(lsf):
    return m17_crc16(lsf[:28]) == int.from_bytes(lsf[28:30], "big")


CLEAR_LSF = bytes([0xFF] * 6 + [0] * 24)


class Decoder:
    """M17FrameDecoder + gr_modem's M17 record handling for one channel: records (type, 46 bytes) in, 56-byte snapshots out
    ({uint32 type, lsf 30, valid, 0, stream frame 18, 0, 0}, the layout of qrl_m17_rx_read)"""

    def __init__(self):
        self.reset()

    def reset(self):
        self.lsf, self.part, self.map, self.sf = CLEAR_LSF, bytearray(CLEAR_LSF), 0, bytes(18)

    def work(self, records, decoded=None):
        if not records:
            return []
        dec, lich = decoded or decode_records([t for t, _ in records], [np.frombuffer(bytes(p)[:46].ljust(46, b"\0"), np.uint8) for _, p in records])
        out = []
        for (t, _), d, seg in zip(records, dec, lich):
            if t == LSF:
                self.lsf = d
            elif t == STREAM:
                if seg is not None:
                    n = seg[5]
                    if n < 6:
                        self.part[5 * n:5 * n + 5] = seg[:5]
                    self.map |= 1 << n
                    if self.map == 0x3F:
                        if _valid(bytes(self.part)):
                            self.lsf = bytes(self.part)
                        self.map, self.part = 0, bytearray(CLEAR_LSF)
                self.sf = d
            v = _valid(self.lsf)
            out.append(int(t).to_bytes(4, "little") + self.lsf + bytes([v, 0]) + self.sf + b"\0\0")
            if t == EOT and v:
                self.reset()
        return out


def decode_channels(chans):
    """Decoder().work for every channel's record list, the per-frame half batched over all channels"""
    flat = [r for recs in chans for r in recs]
    if not flat:
        return [[] for _ in chans]
    dec, lich = decode_records([t for t, _ in flat], [np.frombuffer(bytes(p)[:46].ljust(46, b"\0"), np.uint8) for _, p in flat])
    out, k = [], 0
    for recs in chans:
        out.append(Decoder().work(recs, (dec[k:k + len(recs)], lich[k:k + len(recs)])))
        k += len(recs)
    return out
