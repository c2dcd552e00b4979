"""Plain-Python restatement of gr_dmr_sink and the per-burst DMRFrame work (constructor, setDownlink, validate), CDMREMB::putData and
CAMBEFEC::regenerateDMR, written bit by bit the way the reference walks them, plus the encoders the tests build streams with.
Test infrastructure: tests/test_dmr_codec.py and tests/test_gpu_dmr_codec.py compare qrl_dmr.cu's records with it."""
import itertools

import numpy as np

MS_DATA, MS_VOICE, BS_DATA, BS_VOICE = 0xD5D7F77FD757, 0x7F7D5DD57DFD, 0xDFF57D75DF5D, 0x755FD7DF75F7
DT_VOICE_SYNC, DT_VOICE = 0xF0, 0xF1
REC_FIELDS = ("position", "ts_index", "frame_type", "fn", "downlink", "cach_decoded", "at", "slot_no", "lcss", "color_code",
              "data_type", "valid", "flco", "fid", "emb_cc", "emb_pi", "emb_lcss", "src_id", "dst_id", "ambe_errors")


def poly_mod(r, top, g, deg):
    for b in range(top, deg - 1, -1):
        if r >> b & 1:
            r ^= g << (b - deg)
    return r


def syndrome_table(n, g, deg, max_w):
    """for each syndrome the first least-weight error pattern (itertools.combinations order), weights up to max_w; 0 elsewhere"""
    tab, seen = [0] * (1 << deg), {0}
    for w in range(1, max_w + 1):
        for pos in itertools.combinations(range(n), w):
            e = sum(1 << p for p in pos)
            s = poly_mod(e, n - 1, g, deg)
            if s not in seen:
                seen.add(s)
                tab[s] = e
    return tab


GOLAY23 = syndrome_table(23, 0xC75, 11, 3)
GOLAY19 = syndrome_table(19, 0xC75, 11, 5)
QR15 = syndrome_table(15, 0x139, 8, 4)


def golay_check(d):
    r = poly_mod(d << 11, 22, 0xC75, 11)
    par = (bin(d).count("1") + bin(r).count("1")) & 1
    return (r << 1) | par


def golay24_encode(d):
    return (d << 12) | golay_check(d)


def golay24_decode(a):
    """CGolay24128::decode24128: (valid, data)"""
    syn = poly_mod(a >> 1, 22, 0xC75, 11)
    out = a ^ (GOLAY23[syn] << 1)
    return bin(syn).count("1") < 3 or not (bin(out).count("1") & 1), out >> 12


def golay23_decode(b):
    return (b ^ GOLAY23[poly_mod(b, 22, 0xC75, 11)]) >> 11


def prng(u):
    p, v = 16 * u, 0
    for _ in range(24):
        p = (173 * p + 13849) & 0xFFFF
        v = (v << 1) | (p >> 15)
    return v


def crc_ccitt(data):
    crc = 0
    for b in data:
        crc ^= b << 8
        for _ in range(8):
            crc = ((crc << 1) ^ 0x1021) & 0xFFFF if crc & 0x8000 else (crc << 1) & 0xFFFF
    return ~crc & 0xFFFF


def gf_mul(a, b):
    r = 0
    for i in range(8):
        if b >> i & 1:
            r ^= a
        a = ((a << 1) ^ (0x11D if a & 0x80 else 0)) & 0x1FF
    return r & 0xFF


def rs129_parity(m9):
    g, par = (64, 56, 14), [0, 0, 0]
    for d in m9:
        d ^= par[2]
        par[2] = par[1] ^ gf_mul(g[2], d)
        par[1] = par[0] ^ gf_mul(g[1], d)
        par[0] = gf_mul(g[0], d)
    return bytes([par[2], par[1], par[0]])


# ---------------------------------------------------------------- bits <-> bytes; the BPTC and trellis skip frame bits 98..165
def to_bits(b):
    return [(x >> (7 - i)) & 1 for x in b for i in range(8)]


def to_bytes(bits):
    return bytes(int("".join(map(str, bits[i:i + 8])), 2) for i in range(0, len(bits), 8))


def info_bit(i):
    return i if i < 98 else i + 68


BPTC_DATA = [4 + k for k in range(8)] + [16 + m + 4 * (m // 11) for m in range(88)]
H15 = [(0, 1, 2, 3, 5, 7, 8), (1, 2, 3, 4, 6, 8, 9), (2, 3, 4, 5, 7, 9, 10), (0, 1, 2, 4, 6, 7, 10)]
H13 = [(0, 1, 3, 5, 6), (0, 1, 2, 4, 6, 7), (0, 1, 2, 3, 5, 7, 8), (0, 2, 4, 5, 8)]


def _ham_fix(v, eqs, nd):
    syn = sum((sum(v[i] for i in eq) & 1 ^ v[nd + k]) << k for k, eq in enumerate(eqs))
    if syn == 0:
        return False
    cols = {1 << k: nd + k for k in range(4)}
    for i in range(nd):
        cols.setdefault(sum(int(i in eq) << k for k, eq in enumerate(eqs)), i)
    if syn in cols:
        v[cols[syn]] ^= 1
        return True
    return False


def bptc_decode(fb):
    d = [fb[info_bit((a * 181) % 196)] for a in range(196)]
    for _ in range(5):
        fixing = False
        for c in range(15):
            idx = [c + 1 + 15 * a for a in range(13)]
            col = [d[i] for i in idx]
            if _ham_fix(col, H13, 9):
                fixing = True
                for i, v in zip(idx, col):
                    d[i] = v
        for r in range(9):
            row = d[r * 15 + 1: r * 15 + 16]
            if _ham_fix(row, H15, 11):
                fixing = True
                d[r * 15 + 1: r * 15 + 16] = row
        if not fixing:
            break
    return to_bytes([d[p] for p in BPTC_DATA])


def bptc_encode(payload, fb):
    d = [0] * 196
    for k, b in enumerate(to_bits(payload)):
        d[BPTC_DATA[k]] = b
    for r in range(9):
        row = d[r * 15 + 1: r * 15 + 16]
        for k, eq in enumerate(H15):
            row[11 + k] = sum(row[i] for i in eq) & 1
        d[r * 15 + 1: r * 15 + 16] = row
    for c in range(15):
        col = [d[c + 1 + 15 * a] for a in range(13)]
        for k, eq in enumerate(H13):
            col[9 + k] = sum(col[i] for i in eq) & 1
        for a in range(13):
            d[c + 1 + 15 * a] = col[a]
    for a in range(196):
        fb[info_bit((a * 181) % 196)] = d[a]


# ---------------------------------------------------------------- rate-3/4 trellis
TRELLIS_ORDER = [n for g in range(4) for n in range(98) if (n >> 1) & 3 == g]
_ROT = [0, 2, 0, 2, 4, 6, 4, 6]


def rev3(j):
    return ((j & 1) << 2) | (j & 2) | ((j >> 2) & 1)


def trellis_point(state, t):
    return (rev3((t + _ROT[state]) & 7) << 1) | (1 if 2 <= state <= 5 else 0)


# dibit pairs as (b1 b2)(b1 b2) with +3 = 01, +1 = 00, -1 = 10, -3 = 11; points 8-15 complement points 0-7
_BASE = [0x2, 0xA, 0x7, 0xF, 0xE, 0x6, 0xB, 0x3]
POINT_DIBITS = _BASE + [v ^ 0xF for v in _BASE]


def trellis_check(points):
    state, tribits = 0, []
    for i, pt in enumerate(points):
        t = next((j for j in range(8) if trellis_point(state, j) == pt), None)
        if t is None:
            return i, tribits
        tribits.append(t)
        state = t
    return (48 if tribits[48] else 999), tribits


def trellis_fix(points, fail):
    for _ in range(20):
        best_pos, best_val = 0, 0
        for i in range(16):
            points[fail] = i
            pos, _ = trellis_check(points)
            if pos == 999:
                return True
            if pos > best_pos:
                best_pos, best_val = pos, i
        points[fail] = best_val
        fail = best_pos
    return False


def trellis_points(fb):
    dib = [0] * 98
    for i in range(98):
        dib[TRELLIS_ORDER[i]] = fb[info_bit(2 * i)] << 1 | fb[info_bit(2 * i + 1)]
    return [POINT_DIBITS.index(dib[2 * i] << 2 | dib[2 * i + 1]) for i in range(49)]


def trellis_write(points, fb):
    for i in range(98):
        n = TRELLIS_ORDER[i]
        v = POINT_DIBITS[points[n >> 1]]
        db = v & 3 if n & 1 else v >> 2
        fb[info_bit(2 * i)], fb[info_bit(2 * i + 1)] = db >> 1, db & 1


def trellis_decode(fb):
    points = trellis_points(fb)
    fail, _ = trellis_check(points)
    if fail == 999:
        return points
    save = list(points)
    if trellis_fix(points, fail):
        return points
    if fail == 0:
        return None
    return save if trellis_fix(save, fail - 1) else None


def trellis_encode(payload18):
    """CDMRTrellis::encode's points for 18 payload bytes"""
    bits = to_bits(payload18)
    tribits = [bits[143 - 3 * i] << 2 | bits[142 - 3 * i] << 1 | bits[141 - 3 * i] for i in range(48)] + [0]
    points, state = [], 0
    for t in tribits:
        points.append(trellis_point(state, t))
        state = t
    return points


# ---------------------------------------------------------------- AMBE
def ambe_bit(f, t):
    base = 4 * (t % 18) + t // 18
    return base if f == 0 else (base + 120 if base + 72 >= 108 else base + 72) if f == 1 else base + 192


def ambe_regenerate(a, b, c):
    oa, ob = a, b
    ok, data = golay24_decode(a)
    if not ok:
        return 0xF00292, 0x0E0B20, 0, 10
    a = golay24_encode(data)
    p = prng(data) >> 1
    datb = golay23_decode(b ^ p)
    b = (((datb << 11) | (golay_check(datb) >> 1)) ^ p) & 0x7FFFFF
    ea, eb = bin(a ^ oa).count("1"), bin(b ^ ob).count("1")
    if ea >= 4 or (ea + eb >= 6 and ea >= 2):
        a, b, c = 0xF00292, 0x0E0B20, 0
    return a, b, c, ea + eb


def ambe_frame_encode(fb, f, a12, b12, c25):
    """put one AMBE frame (A data, B data, C bits) into frame bits fb"""
    a = golay24_encode(a12)
    b = (((b12 << 11) | (golay_check(b12) >> 1)) ^ (prng(a12) >> 1)) & 0x7FFFFF
    for t in range(24):
        fb[ambe_bit(f, t)] = (a >> (23 - t)) & 1
    for t in range(24, 47):
        fb[ambe_bit(f, t)] = (b >> (46 - t)) & 1
    for t in range(47, 72):
        fb[ambe_bit(f, t)] = (c25 >> (71 - t)) & 1


# ---------------------------------------------------------------- the sink
class Sink:
    """gr_dmr_sink::work, bit by bit"""

    def __init__(self):
        self.state, self.sr, self.btr, self.ftr = [0, 0], [0, 0], [0, 0], [0, 0]
        self.buf, self.downlink, self.next_slot, self.pos = [[], []], [1, 1], 0, 0

    def work(self, bits):
        out = []
        for i in range(2):
            if len(self.buf[i]) >= 864:
                del self.buf[i][:288]
        for b in bits:
            b = int(b) & 1
            ts = self.next_slot
            self.buf[ts].append(b)
            nxt = ts ^ 1
            st = self.state[ts]
            if st in (1, 2):
                if self.btr[ts] > 0:
                    self.btr[ts] -= 1
                    if self.btr[ts] == 0:
                        out.append(dict(position=self.pos, ts_index=ts, frame_type=0 if st == 1 else 2, fn=0,
                                        downlink=self.downlink[ts], bits=self.buf[ts][:288]))
                        self.state[ts] = 3 if st == 2 else 0
                        self.buf[ts] = []
                        self.next_slot = nxt
            elif st == 3 and self.ftr[ts] > 0:
                if len(self.buf[ts]) >= 288:
                    out.append(dict(position=self.pos, ts_index=ts, frame_type=1, fn=6 - self.ftr[ts], downlink=self.downlink[ts],
                                    bits=self.buf[ts][:288]))
                    self.buf[ts] = []
                    self.ftr[ts] -= 1
                    if self.ftr[ts] == 0:
                        self.state[ts] = 0
                    self.next_slot = nxt
            elif st == 0:
                self._find_sync(b, ts)
            self.pos += 1
        return out

    def _find_sync(self, b, ts):
        self.sr[ts] = ((self.sr[ts] << 1) | b) & ((1 << 64) - 1)
        t = self.sr[ts] & 0xFFFFFFFFFFFF
        if t in (BS_DATA, MS_DATA):
            self.state[ts] = 1
        elif t in (BS_VOICE, MS_VOICE):
            self.state[ts] = 2
        if t in (BS_DATA, BS_VOICE):
            self.downlink[ts] = 1
        elif t in (MS_DATA, MS_VOICE):
            self.downlink[ts] = 0
        if self.state[ts] != 0:
            if len(self.buf[ts]) < 180:
                self.state[ts], self.btr[ts], self.ftr[ts], self.buf[ts] = 0, 0, 0, []
                return
            del self.buf[ts][:len(self.buf[ts]) - 180]
            self.btr[ts] = 108
            if self.state[ts] == 2:
                self.ftr[ts] = 5


# ---------------------------------------------------------------- per-burst decode
def decode_burst(r, ambe_fec):
    """the record qrl_dmr.cu returns for a burst the sink cut (r: a dict from Sink.work)"""
    bits = r["bits"]
    cach, fb = to_bytes(bits[:24]), list(bits[24:])
    fr = to_bytes(fb)
    o = dict((k, r[k]) for k in ("position", "ts_index", "frame_type", "fn", "downlink"))
    o.update(cach_decoded=0, at=0, slot_no=0, lcss=0, color_code=255, valid=1, flco=0, fid=0, emb_cc=0, emb_pi=0, emb_lcss=0,
             src_id=0, dst_id=0, ambe_errors=-1)
    if r["downlink"]:
        at, tc, l1, l0 = cach[0] >> 7 & 1, cach[0] >> 3 & 1, cach[1] >> 7 & 1, cach[1] >> 3 & 1
        if (at ^ tc ^ l1) == (cach[1] >> 1 & 1) and (tc ^ l1 ^ l0) == (cach[2] >> 5 & 1) and (at ^ tc ^ l0) == (cach[2] >> 1 & 1):
            o.update(cach_decoded=1, at=at, slot_no=2 if tc else 1, lcss=l1 << 1 | l0)
    ft = r["frame_type"]
    if ft == 0:
        code = int("".join(map(str, fb[98:108] + fb[156:165])), 2)
        st = ((code ^ GOLAY19[poly_mod(code, 18, 0xC75, 11)]) >> 11) & 0xFF
        dt = st & 0xF
        o.update(color_code=st >> 4, data_type=dt, valid=0)
        if dt <= 7:
            pl = bytearray(bptc_decode(fb))
            ok = False
            id47, id79 = int.from_bytes(pl[4:7], "big"), int.from_bytes(pl[7:10], "big")
            if dt in (3, 4, 5):
                c = crc_ccitt(pl[:10])
                ok = (pl[10] ^ 0xA5) == c >> 8 and (pl[11] ^ 0xA5) == c & 0xFF
                if ok:
                    op = pl[0] & 0x3F
                    o.update(flco=op, fid=pl[1])
                    if op == 0x38:
                        o.update(src_id=id79)
                    elif op == 0x26 or (op == 0x24 and pl[3] != 0x80):
                        o.update(src_id=id47, dst_id=id79)
                    else:
                        o.update(dst_id=id47, src_id=id79)
            elif dt == 6:
                c = crc_ccitt(pl[:10])
                ok = (pl[10] ^ 0xCC) == c >> 8 and (pl[11] ^ 0xCC) == c & 0xFF
                dpf = pl[0] & 0xF
                if ok and dpf != 0xF:
                    o.update(dst_id=int.from_bytes(pl[2:5], "big"), src_id=int.from_bytes(pl[5:8], "big"))
                    if dpf == 0:
                        o.update(flco=pl[9] & 0x3F)
                        pl[9] &= 0xFE
                        c = crc_ccitt(pl[:10])
                        pl[10], pl[11] = (c >> 8) ^ 0xCC, (c & 0xFF) ^ 0xCC
            elif dt in (1, 2):
                m = 0x96 if dt == 1 else 0x99
                ok = rs129_parity(pl[:9]) == bytes(x ^ m for x in pl[9:12])
                if ok:
                    o.update(flco=pl[0] & 0x3F, fid=pl[1], dst_id=int.from_bytes(pl[3:6], "big"), src_id=int.from_bytes(pl[6:9], "big"))
            else:
                ok = True
            if ok:
                bptc_encode(pl, fb)
            o["valid"] = int(ok)
        elif dt == 8:
            pts = trellis_decode(fb)
            if pts is not None:
                trellis_write(pts, fb)
            o["valid"] = int(pts is not None)
    else:
        o["data_type"] = DT_VOICE if ft == 1 else DT_VOICE_SYNC
        if ambe_fec:
            errs = 0
            for f in range(3):
                a = int("".join(str(fb[ambe_bit(f, t)]) for t in range(24)), 2)
                b = int("".join(str(fb[ambe_bit(f, t)]) for t in range(24, 47)), 2)
                c = int("".join(str(fb[ambe_bit(f, t)]) for t in range(47, 72)), 2)
                a, b, c, e = ambe_regenerate(a, b, c)
                errs += e
                for t in range(24):
                    fb[ambe_bit(f, t)] = (a >> (23 - t)) & 1
                for t in range(24, 47):
                    fb[ambe_bit(f, t)] = (b >> (46 - t)) & 1
                for t in range(47, 72):
                    fb[ambe_bit(f, t)] = (c >> (71 - t)) & 1
            o["ambe_errors"] = errs
        if ft == 1:
            code = int("".join(map(str, fb[108:116] + fb[148:155])), 2)
            e8 = ((code ^ QR15[poly_mod(code, 14, 0x139, 8)]) >> 7) & 0xFF
            o.update(emb_cc=e8 >> 4, emb_pi=e8 >> 3 & 1, emb_lcss=e8 >> 1 & 3)
    o["cach"], o["frame"] = cach, to_bytes(fb)
    return o


class Decoder:
    """Sink + decode_burst per channel, across calls"""

    def __init__(self, n_channels, ambe_fec=False):
        self.sinks = [Sink() for _ in range(n_channels)]
        self.ambe_fec = ambe_fec

    def work(self, per_channel_bits):
        return [[decode_burst(r, self.ambe_fec) for r in s.work(b)] for s, b in zip(self.sinks, per_channel_bits)]


def records_equal(got, want):
    """got: a DMR_RECORD array of one channel, want: Decoder.work's list of that channel; returns a mismatch description or None"""
    if len(got) != len(want):
        return "count %d != %d" % (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        for k in REC_FIELDS:
            if int(g[k]) != int(w[k]):
                return "record %d field %s: %d != %d" % (i, k, int(g[k]), int(w[k]))
        if bytes(g["cach"]) != w["cach"] or bytes(g["frame"]) != w["frame"]:
            return "record %d bytes differ" % i
    return None


# ---------------------------------------------------------------- stream builders
SYNC_BYTES = {k: v.to_bytes(6, "big") for k, v in (("bs_data", BS_DATA), ("bs_voice", BS_VOICE), ("ms_data", MS_DATA),
                                                   ("ms_voice", MS_VOICE))}


def cach_bits(at, slot, lcss, good=True):
    tc, l1, l0 = int(slot == 2), lcss >> 1 & 1, lcss & 1
    h0, h1, h2 = at ^ tc ^ l1, tc ^ l1 ^ l0, at ^ tc ^ l0
    if not good:
        h0 ^= 1
    c = [0] * 24
    c[0], c[4], c[8], c[12], c[14], c[18], c[22] = at, tc, l1, l0, h0, h1, h2
    return c


def data_burst(cc, dt, payload12=None, points=None, sync="bs_data"):
    """264 frame bits: a BPTC payload (or trellis points for rate 3/4), the slot type for (cc, dt) and a sync word"""
    fb = [0] * 264
    if points is not None:
        trellis_write(points, fb)
    elif payload12 is not None:
        bptc_encode(bytes(payload12), fb)
    st = (cc << 4) | dt
    code = (st << 11) | poly_mod(st << 11, 18, 0xC75, 11)
    sb = [(code >> (18 - i)) & 1 for i in range(19)] + [0]
    fb[98:108], fb[156:166] = sb[:10], sb[10:]
    fb[108:156] = to_bits(SYNC_BYTES[sync])
    return fb


def voice_burst(rng, emb=None, sync=None, ambe=True):
    """264 frame bits of a voice burst: 3 AMBE frames (valid codewords when ambe) and either a sync word or an EMB (cc, pi, lcss)"""
    fb = [int(x) for x in rng.integers(0, 2, 264)]
    if ambe:
        for f in range(3):
            ambe_frame_encode(fb, f, int(rng.integers(0, 4096)), int(rng.integers(0, 4096)), int(rng.integers(0, 1 << 25)))
    if sync is not None:
        fb[108:156] = to_bits(SYNC_BYTES[sync])
    else:
        cc, pi, lcss = emb
        e8 = (cc << 4) | (pi << 3) | (lcss << 1)
        code = (e8 << 7) | poly_mod(e8 << 7, 14, 0x139, 8)
        eb = [(code >> (14 - i)) & 1 for i in range(15)] + [0]
        fb[108:116], fb[148:156] = eb[:8], eb[8:]
        fb[116:148] = [0] * 32
    return fb


def csbk_payload(op, fid, dst, src, mask=0xA5, b2=0, b3=0):
    p = bytearray([op & 0x3F, fid, b2, b3]) + dst.to_bytes(3, "big") + src.to_bytes(3, "big")
    c = crc_ccitt(p)
    return bytes(p) + bytes([(c >> 8) ^ mask, (c & 0xFF) ^ mask])


def lc_payload(flco, fid, dst, src, dt):
    p = bytes([flco, fid, 0]) + dst.to_bytes(3, "big") + src.to_bytes(3, "big")
    m = 0x96 if dt == 1 else 0x99
    return p + bytes(x ^ m for x in rs129_parity(p))


def data_header_payload(dpf, dst, src, b9=0):
    p = bytearray([dpf, 0]) + dst.to_bytes(3, "big") + src.to_bytes(3, "big") + bytes([1, b9])
    c = crc_ccitt(p)
    return bytes(p) + bytes([(c >> 8) ^ 0xCC, (c & 0xFF) ^ 0xCC])


def flip(fb, rng, n):
    fb = list(fb)
    for i in rng.choice(264, n, replace=False):
        fb[int(i)] ^= 1
    return fb


def mixed_stream(rng, n_slots_pairs=24, errors=(0, 1, 2, 3)):
    """a downlink stream alternating two slots: voice superframes and every data type, with bit errors; CACH with slot numbers"""
    out = []
    srcs = [int(rng.integers(1, 1 << 24)) for _ in range(2)]
    for k in range(n_slots_pairs):
        for slot in (1, 2):
            kind = int(rng.integers(0, 10))
            cc = int(rng.integers(0, 16))
            e = int(rng.choice(errors))
            if kind < 3:     # a voice superframe: A with sync, B-F with EMB
                fbs = [voice_burst(rng, sync="bs_voice", ambe=True)] + \
                      [voice_burst(rng, emb=(cc, int(rng.integers(0, 2)), int(rng.integers(0, 4))), ambe=bool(rng.integers(0, 4)))
                       for _ in range(5)]
            else:
                dt = [1, 2, 3, 4, 5, 6, 0, 7, 8, 9][int(rng.integers(0, 10))]
                dst = int(rng.integers(0, 1 << 24))
                if dt in (1, 2):
                    pl = lc_payload(int(rng.integers(0, 64)), 0, dst, srcs[slot - 1], dt)
                elif dt in (3, 4, 5):
                    pl = csbk_payload(int(rng.choice([0x04, 0x24, 0x26, 0x38, 0x3D, 0x1F])), 0x10, dst, srcs[slot - 1],
                                      b3=int(rng.choice([0, 0x80])))
                elif dt == 6:
                    pl = data_header_payload(int(rng.choice([0, 2, 3, 0xF])), dst, srcs[slot - 1], b9=int(rng.integers(0, 256)))
                else:
                    pl = bytes(int(x) for x in rng.integers(0, 256, 12))
                if dt == 8:
                    fbs = [data_burst(cc, dt, points=trellis_encode(bytes(int(x) for x in rng.integers(0, 256, 18))))]
                else:
                    fbs = [data_burst(cc, dt, payload12=pl)]
            for fb in fbs:
                out += cach_bits(int(rng.integers(0, 2)), slot, int(rng.integers(0, 4)), good=bool(rng.integers(0, 6))) + flip(fb, rng, e)
    return np.array(out, np.uint8)
