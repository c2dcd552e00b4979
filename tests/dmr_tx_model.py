"""Plain-Python restatement of the DMR transmit side: DMRControl's transmit state machine (src/DMR/dmrcontrol.cpp:19-223) as
gr_modem drives it (gr_modem.cpp:676-678, 710-717, 747-802), the burst encoders behind DMRFrame (dmrframe.cpp:399-421, 460-501:
CDMRFullLC::encode, CDMRCSBK::get, CDMRSlotType::getData, CDMREmbeddedData::setLC / getData, CDMREMB::getData, CSync with
duplex = false) and gr_dmr_source's framing (gr/gr_dmr_source.cpp:58-126).  Written from the reference's lines, bit by bit.
Test infrastructure: tests/test_dmr_tx_codec.py and tests/test_gpu_dmr_tx_codec.py compare qrl_dmr.cu's transmit handle with it.
The FEC helpers (BPTC, CRC-CCITT, RS(12,9), the Golay check bits, the QR(15,7) remainder) come from tests/dmr_model.py."""
import numpy as np

from tests import dmr_model as M

OP_NONE, OP_CSBK, OP_HEADER, OP_AUDIO, OP_STOP = 0, 1, 2, 3, 4
KIND_CSBK, KIND_LC_HEADER, KIND_VOICE_SYNC, KIND_VOICE, KIND_TERMINATOR, KIND_EMPTY = 1, 2, 3, 4, 5, 6
IDLE, ACTIVE, ENDING = 0, 1, 2
FLCO_GROUP, FLCO_USER_USER = 0, 3
DT_VOICE_LC_HEADER, DT_TERMINATOR_WITH_LC, DT_CSBK = 1, 2, 3
CSBKO_BSDWNACT = 0x38
BURST_BYTES = 72                  # 33 frame bytes + 39 zero bytes (gr_dmr_source: FRAME_LENGTH_BYTES + 2 * CACH_LENGTH_BYTES)
ZERO_SAMPLES = 780                # DMR_ZERO_TX_LENGTH_SAMPLES = 39 * 4 * 5


class Config:
    """the Settings fields DMRControl reads; the defaults are Settings' (settings.cpp:85-94; dmr_vocoder = 0 means codec2)"""

    def __init__(self, color_code=1, timeslot=1, src_id=1, dst_id=9, private_call=False, codec2=True, talker_alias=b""):
        self.color_code, self.timeslot, self.src_id, self.dst_id = color_code, timeslot, src_id, dst_id
        self.private_call, self.codec2, self.talker_alias = bool(private_call), bool(codec2), bytes(talker_alias)[:27]

    def flco(self):
        return FLCO_USER_USER if self.private_call else FLCO_GROUP

    def ta27(self):
        return self.talker_alias + bytes(27 - len(self.talker_alias))


def lc_bytes(flco, fid, options, src, dst):
    """CDMRLC::getData (PF = R = 0)"""
    return bytes([flco & 0x3F, fid & 0xFF, options & 0xFF]) + (dst & 0xFFFFFF).to_bytes(3, "big") + (src & 0xFFFFFF).to_bytes(3, "big")


# ---------------------------------------------------------------- per-burst encoders (33 bytes)
def _slot_type_and_sync(fb, cc, dt):
    st = ((cc & 0xF) << 4) | (dt & 0xF)
    w = (st << 12) | M.golay_check(st)                 # Golay(20,8): the (23,12) code shortened to 8 data bits
    wb = [(w >> (19 - i)) & 1 for i in range(20)]
    fb[98:108], fb[156:166] = wb[:10], wb[10:]
    fb[108:156] = M.to_bits(M.SYNC_BYTES["ms_data"])


def csbk_payload(src, dst):
    """getStartCSBK's 12 CSBK bytes: CSBKO_BSDWNACT with LB set (setCSBKO's default), FID 0, data1 0, CBF 0, dst, src, then
    CRC-CCITT ^ 0xA5A5"""
    p = bytes([0x80 | CSBKO_BSDWNACT, 0, 0, 0]) + (dst & 0xFFFFFF).to_bytes(3, "big") + (src & 0xFFFFFF).to_bytes(3, "big")
    c = M.crc_ccitt(p)
    return p + bytes([(c >> 8) ^ 0xA5, (c & 0xFF) ^ 0xA5])


def csbk_burst(cc, src, dst):
    """getStartCSBK's frame: the CSBK bytes through BPTC, slot type, MS data sync"""
    fb = [0] * 264
    M.bptc_encode(csbk_payload(src, dst), fb)
    _slot_type_and_sync(fb, cc, DT_CSBK)
    return M.to_bytes(fb)


def lc_burst(lc9, dt, cc):
    """constructLCFrame: RS(12,9) parity ^ the header / terminator mask, BPTC, slot type, MS data sync"""
    m = 0x96 if dt == DT_VOICE_LC_HEADER else 0x99
    fb = [0] * 264
    M.bptc_encode(bytes(lc9) + bytes(x ^ m for x in M.rs129_parity(lc9)), fb)
    _slot_type_and_sync(fb, cc, dt)
    return M.to_bytes(fb)


def embedded_raw(lc9):
    """CDMREmbeddedData::setLC / encodeEmbeddedData: the 128 interleaved bits"""
    bits = M.to_bits(lc9)
    crc = sum(lc9) % 31
    data = [0] * 128
    for r, k in zip(range(2, 7), range(4, -1, -1)):
        data[16 * r + 10] = (crc >> k) & 1
    pos = list(range(0, 11)) + list(range(16, 27)) + [a for r in range(2, 7) for a in range(16 * r, 16 * r + 10)]
    for b, a in zip(bits, pos):
        data[a] = b
    for r in range(7):
        d = data[16 * r:16 * r + 16]
        for k, eq in enumerate(M.H15):
            d[11 + k] = sum(d[i] for i in eq) & 1
        d[15] = sum(d[:15]) & 1                        # Hamming(16,11,4): the (15,11) code plus overall parity
        data[16 * r:16 * r + 16] = d
    for a in range(16):
        data[112 + a] = sum(data[a + 16 * r] for r in range(7)) & 1
    raw, b = [0] * 128, 0
    for a in range(128):
        raw[a] = data[b]
        b += 16
        if b > 127:
            b -= 127
    return raw


def emb_word(cc, lcss, pi=0):
    """CDMREMB::getData: QR(16,7) = the (15,7) QR code (g = 0x139) plus overall parity"""
    v = ((cc & 0xF) << 3) | (pi << 2) | (lcss & 3)
    code = (v << 8) | M.poly_mod(v << 8, 14, 0x139, 8)
    return (code << 1) | (bin(code).count("1") & 1)


LCSS_OF_FN = {0: 0, 1: 1, 2: 3, 3: 3, 4: 2, 5: 0}


def voice_burst(audio27, fn, cc, emb_lc9):
    """getTxAudio's frame: setVoice (+ addVoiceSync at FN 0, setEmbeddedData otherwise); returns (bytes, lcss)"""
    ab = M.to_bits(audio27)
    fb = [0] * 264
    fb[0:108], fb[156:264] = ab[:108], ab[108:]
    if fn == 0:
        fb[108:156] = M.to_bits(M.SYNC_BYTES["ms_voice"])
        return M.to_bytes(fb), 0
    lcss = LCSS_OF_FN[fn]
    if 1 <= fn <= 4:
        fb[116:148] = embedded_raw(emb_lc9)[32 * (fn - 1):32 * fn]
    e = emb_word(cc, lcss)
    eb = [(e >> (15 - i)) & 1 for i in range(16)]
    fb[108:116], fb[148:156] = eb[:8], eb[8:]
    return M.to_bytes(fb), lcss


# ---------------------------------------------------------------- the state machine
class Channel:
    """DMRControl's transmit half for one channel, gr_modem's calls as ops, gr_dmr_source's byte stream"""

    def __init__(self, cfg=None):
        self.reset(cfg or Config())

    def reset(self, cfg):
        """DMRControl's constructor with `cfg` in force; byte position 0"""
        self.cfg = cfg
        self.state, self.fn, self.sf, self.pending, self.pos = IDLE, 0, 0, [], 0
        self._snapshot_lc()
        self.ta = cfg.ta27()

    def _snapshot_lc(self):
        c = self.cfg
        self.flco_tx = c.flco()
        self.lc_tx = lc_bytes(self.flco_tx, 0xC2 if c.codec2 else 0, 0, c.src_id, c.dst_id)
        self.emb_lc = self.lc_tx

    def _advance(self):
        """the frame / superframe counters after a voice burst, with the talker-alias LCs of superframes 1-4"""
        self.fn += 1
        if self.fn <= 5:
            return
        self.fn = 0
        self.sf = (self.sf + 1) % 5
        if self.sf == 0:
            self.emb_lc = self.lc_tx
            return
        i, flco, ta = (self.sf - 1) * 6, 3 + self.sf, self.ta
        if self.sf == 1:
            self.emb_lc = bytes([flco, 0, (1 << 6) | (0x1B << 1)]) + ta[i:i + 6]
        else:
            self.emb_lc = bytes([flco, 0, ta[i]]) + ta[i + 1:i + 7]

    def op(self, op, audio9=bytes(9)):
        """one gr_modem call; returns the frames gr_dmr_source gets: (kind, slot, fn, lcss, 33 bytes)"""
        c = self.cfg
        if op == OP_CSBK:
            b = csbk_burst(c.color_code, c.src_id, c.dst_id)
            return [(KIND_CSBK, c.timeslot, 0, 0, b)] * 3
        if op == OP_HEADER:
            self._snapshot_lc()
            b = lc_burst(self.lc_tx, DT_VOICE_LC_HEADER, c.color_code)
            self.fn, self.sf, self.state, self.ta = 0, 0, ACTIVE, c.ta27()       # initVoiceTX
            return [(KIND_LC_HEADER, c.timeslot, 0, 0, b)] * 2
        if op == OP_STOP:
            self.state = ENDING
            return []
        if op != OP_AUDIO or self.state == IDLE:
            return []
        self.pending.append(bytes(audio9))
        if len(self.pending) < 3:
            return []
        if self.state == ENDING and self.fn == 0:
            b = lc_burst(lc_bytes(self.flco_tx, 0, 0, c.src_id, c.dst_id), DT_TERMINATOR_WITH_LC, c.color_code)
            self.pending, self.state, self.sf = [], IDLE, 0
            t = (KIND_TERMINATOR, c.timeslot, 0, 0, b)
            e = (KIND_EMPTY, 0, 0, 0, bytes(33))
            return [t, t, e, e]
        audio, self.pending = b"".join(self.pending[:3]), self.pending[3:]
        fn = self.fn
        b, lcss = voice_burst(audio, fn, c.color_code, self.emb_lc)
        self._advance()
        return [(KIND_VOICE_SYNC if fn == 0 else KIND_VOICE, c.timeslot, fn, lcss, b)]

    def work(self, ops, audio):
        """ops [K], audio [K][9] -> (stream bytes, records); a record is (position, slot, kind, fn, lcss, op index)"""
        out, recs = bytearray(), []
        for k, op in enumerate(ops):
            for kind, slot, fn, lcss, b in self.op(int(op), bytes(audio[k])):
                recs.append((self.pos, slot, kind, fn, lcss, k))
                out += b + bytes(BURST_BYTES - 33)
                self.pos += BURST_BYTES
        return bytes(out), recs


def tags(records):
    """gr_dmr_source's tags of a channel's bursts: ("tx_time", byte, slot) on byte 0 and ("zero_samples", byte 33, 780)"""
    out = []
    for pos, slot, *_ in records:
        out += [("tx_time", pos, slot), ("zero_samples", pos + 33, ZERO_SAMPLES)]
    return out


def random_ops(rng, K, p=(0.04, 0.06, 0.8, 0.1)):
    """a stream of ops: CSBK, header, audio and stop with the given weights (none takes what is left)"""
    w = np.array([1.0 - sum(p)] + list(p))
    return rng.choice(5, K, p=w / w.sum()).astype(np.uint8)
