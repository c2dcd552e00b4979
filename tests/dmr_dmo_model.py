"""Plain-Python restatement of gr_dmr_dmo_sink (DMR direct mode, after MMDVM's DMRDMORX) sample by sample, in float32 with every
operation rounded where the reference's SSE code rounds it, plus stream builders for the tests.  The per-burst work (DMRFrame's
constructor, validate(), the EMB and the AMBE FEC) is tests/dmr_model.decode_burst.  Test infrastructure: tests/test_dmr_dmo_codec.py
and tests/test_gpu_dmr_dmo.py compare qrl_dmr.cu's DMO records with it."""
import numpy as np

from tests import dmr_model as M

RING = 1440
NOEND = 9999
MS_DATA_SYM, MS_VOICE_SYM = 0x76286E, 0x89D791          # the MS syncs' 24 symbols, +3 = 1
CTRL_NONE, CTRL_VOICE, CTRL_DATA = 0x00, 0x20, 0x40
R_NONE, R_DATA, R_VOICE = 0, 1, 2
F32 = np.float32
ZERO, TWO, FOUR = F32(0.0), F32(2.0), F32(4.0)


def slot_type2(w19):
    """CDMRSlotType2::decode2087 of its 19 code bits: colour code << 4 | data type.  Its DECODING_TABLE_1987 is the (19,8) syndrome
    table dmr_model builds (first least-weight pattern per syndrome), so this is DMRFrame's CDMRSlotType decode"""
    return ((w19 ^ M.GOLAY19[M.poly_mod(w19, 18, 0xC75, 11)]) >> 11) & 0xFF


def dibit(v, centre, threshold):
    s = F32(v - centre)
    if s < -threshold:
        return 3
    if s < ZERO:
        return 2
    if s < threshold:
        return 0
    return 1


class DmoSink:
    """gr_dmr_dmo_sink, with the members its constructor leaves uninitialised set to zero"""

    def __init__(self):
        self.buf = np.zeros(RING, np.float32)
        self.bits = [0] * 5
        self.data_ptr = self.bit_ptr = self.sync_ptr = 0
        self.end_ptr = NOEND
        self.max_corr = ZERO
        self.centre = [ZERO] * 4
        self.threshold = [ZERO] * 4
        self.avg_ptr = self.sync_count = 0
        self.state = R_NONE
        self.control = CTRL_NONE
        self.n = self.cc = 0
        self.pos = 0

    def _reset(self):
        self.sync_ptr, self.max_corr, self.sync_count, self.state, self.end_ptr, self.cc, self.n = 0, ZERO, 0, R_NONE, NOEND, 0, 0

    def _correlate(self, first):
        reg = self.bits[self.bit_ptr] & 0xFFFFFF
        data = bin(reg ^ MS_DATA_SYM).count("1") <= 2
        voice = bin(reg ^ MS_VOICE_SYM).count("1") <= 2
        if not (data or voice):
            return
        sym = MS_DATA_SYM if data else MS_VOICE_SYM
        p0 = (self.data_ptr + RING - 120 + 5) % RING
        vals = [self.buf[(p0 + 5 * i) % RING] for i in range(24)]
        corr, mn, mx = ZERO, F32(100.0), F32(-100.0)
        for i, val in enumerate(vals):
            if val > mx:
                mx = val
            if val < mn:
                mn = val
            corr = F32(corr + F32(F32(3.0 if sym >> (23 - i) & 1 else -3.0) * val))
        if not corr > self.max_corr:
            return
        centre = F32(F32(mx + mn) / TWO)
        threshold = F32(F32(mx - centre) / TWO)
        bits = 0
        for val in vals:
            bits = (bits << 2) | dibit(val, centre, threshold)
        if bin(bits ^ (M.MS_DATA if data else M.MS_VOICE)).count("1") > 3:
            return
        if first:
            self.threshold = [threshold] * 4
            self.centre = [centre] * 4
            self.avg_ptr = 0
        else:
            self.threshold[self.avg_ptr] = threshold
            self.centre[self.avg_ptr] = centre
            self.avg_ptr = (self.avg_ptr + 1) % 4
        self.max_corr = corr
        self.control = CTRL_DATA if data else CTRL_VOICE
        self.sync_ptr = self.data_ptr
        self.end_ptr = (self.data_ptr + 269) % RING

    def _frame(self):
        c, t = self.centre, self.threshold
        centre = F32(F32(F32(F32(c[0] + c[1]) + c[2]) + c[3]) / FOUR)
        threshold = F32(F32(F32(F32(t[0] + t[1]) + t[2]) + t[3]) / FOUR)
        p0 = (self.end_ptr + RING - 660 + 5 + 1) % RING
        bits = []
        for i in range(132):
            d = dibit(self.buf[(p0 + 5 * i) % RING], centre, threshold)
            bits += [d >> 1, d & 1]
        return bits

    def process(self, x):
        """processSample; returns the frames written as (frame_type, fn, colour code, 264 bits)"""
        out = []
        x = F32(x)
        self.buf[self.data_ptr] = x
        self.bits[self.bit_ptr] = ((self.bits[self.bit_ptr] << 1) | int(x > ZERO)) & 0xFFFFFFFF
        if self.state == R_NONE:
            self._correlate(True)
        elif (self.data_ptr + RING + 1 - self.sync_ptr) % RING <= 2:
            self._correlate(False)
        if self.data_ptr == self.end_ptr:
            fb = self._frame()
            write = lambda ft: out.append((ft, self.n, self.cc, fb))
            if self.control == CTRL_DATA:
                w19 = int("".join(map(str, fb[98:108] + fb[156:165])), 2)
                st = slot_type2(w19)
                dt = st & 0xF
                self.cc, self.sync_count, self.n = st >> 4, 0, 0
                if dt == 6:
                    self.state = R_DATA
                    write(0)
                elif dt in (7, 8, 10):
                    if self.state == R_DATA:
                        write(0)
                elif dt in (0, 1):
                    self.state = R_VOICE
                    write(0)
                elif dt == 2:
                    if self.state == R_VOICE:
                        write(0)
                        self._reset()
                else:
                    write(0)
                    self._reset()
            elif self.control == CTRL_VOICE:
                self.state, self.sync_count, self.n = R_VOICE, 0, 0
                write(2)
            else:
                if self.state != R_NONE:
                    self.sync_count += 1
                    if self.sync_count >= 13:
                        self._reset()
                if self.state == R_VOICE:
                    self.n = 0 if self.n >= 5 else self.n + 1
                    write(1)
                elif self.state == R_DATA:
                    write(0)
            self.max_corr = ZERO
            self.control = CTRL_NONE
        self.data_ptr = (self.data_ptr + 1) % RING
        self.bit_ptr = (self.bit_ptr + 1) % 5
        return out

    def work(self, x):
        """processSample over x; returns dicts in the form dmr_model.decode_burst takes, plus the colour code"""
        recs = []
        for v in np.asarray(x, np.float32):
            for ft, fn, cc, fb in self.process(v):
                recs.append(dict(position=self.pos, ts_index=0, frame_type=ft, fn=fn, downlink=0, bits=[0] * 24 + fb, cc=cc))
            self.pos += 1
        return recs


def decode(r, ambe_fec):
    """the record qrl_dmr_dmo_rx returns for a frame the sink wrote"""
    o = M.decode_burst(r, ambe_fec)
    o.update(slot_no=2, color_code=r["cc"])
    return o


class DmoDecoder:
    """DmoSink + decode per channel, across calls"""

    def __init__(self, n_channels, ambe_fec=False):
        self.sinks = [DmoSink() for _ in range(n_channels)]
        self.ambe_fec = ambe_fec

    def work(self, per_channel):
        return [[decode(r, self.ambe_fec) for r in s.work(x)] for s, x in zip(self.sinks, per_channel)]


# ---------------------------------------------------------------- stream builders (5 samples per symbol, dibit 01 = +3, 00 = +1,
# 10 = -1, 11 = -3, as the DMR modulator maps them)
LEVEL = {1: 3.0, 0: 1.0, 2: -1.0, 3: -3.0}


def burst_symbols(fb):
    """264 frame bits -> 132 symbol levels"""
    return [LEVEL[fb[2 * k] << 1 | fb[2 * k + 1]] for k in range(132)]


def to_samples(symbols, scale=0.3, dc=0.0, rng=None, noise=0.0, sps=5):
    x = np.repeat(np.asarray(symbols, np.float64) * scale + dc, sps)
    if rng is not None and noise:
        x = x + noise * rng.standard_normal(len(x))
    return x.astype(np.float32)


def random_symbols(rng, n):
    return [float(v) for v in rng.choice([-3.0, -1.0, 1.0, 3.0], n)]


def dmo_burst(fb, rng, gap=156):
    """one burst every 288 symbols (60 ms): the 132 burst symbols and `gap` symbols of the other (idle) slot"""
    return burst_symbols(fb) + random_symbols(rng, gap)


def voice_superframe(rng, cc=1, sync="ms_voice"):
    fbs = [M.voice_burst(rng, sync=sync)] + [M.voice_burst(rng, emb=(cc, 0, int(rng.integers(0, 4)))) for _ in range(5)]
    return sum((dmo_burst(fb, rng) for fb in fbs), [])
