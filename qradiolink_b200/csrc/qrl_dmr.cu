// qrl_dmr.cu -- the DMR burst decoders (repeater and direct mode) and encoder on the device, part of libqrl_b200.so.
//
// qrl_dmr_rx_* takes QRL_DEMOD_DMR's port 2 (the hard bits gr_demod_base feeds to gr_dmr_sink, /root/reference/src/gr_demod_base.cpp:814)
// and returns, per burst, what DMRControl::addFrames reads of a DMRFrame.  Two kernels:
//   * dmr_sink_kernel, one warp per channel: gr_dmr_sink::work (/root/reference/src/gr/gr_dmr_sink.cpp).  While the active slot searches
//     (RECV_NONE) the warp tests 32 bit positions per step against the four sync words (zero errors), each lane building its 48-bit window
//     from the slot's shift register and the step's ballot; otherwise it jumps to the burst's end (108 bits after a sync, 288 bits per
//     voice burst).  A burst is cut from the slot's buffer, of which the last 288 bits are kept in a ring with a capped fill count.  The
//     reference's quirks stay: bits go only to the active slot's buffer, which flips only when a burst completes; a slot's buffer keeps the
//     bits of its last active period; a sync found with fewer than 180 bits buffered resets the slot; voice bursts B-F are cut by count.
//     The trim at the start of gr_dmr_sink::work (288 bits erased once a buffer holds >= 864) leaves >= 576, so it never changes a burst.
//   * dmr_decode_kernel, one warp per burst: DMRFrame's constructor (slot type, Golay(20,8)), setDownlink (CACH parity), validate()
//     (BPTC(196,96) with CRC-CCITT, RS(12,9) and the CSBK / data header / LC field parses, or the rate-3/4 trellis), CDMREMB::putData
//     (QR(16,7,6)) and CAMBEFEC::regenerateDMR (Golay(24,12) + PRNG + Golay(23,12), one AMBE frame per lane).
//
// Every constant comes from its definition: the syndrome tables of the (23,12) Golay code, the shortened (19,8) Golay code and the
// (15,7) QR code are built on the host once per device by enumerating error patterns by weight (the first pattern in lexicographic order
// of its bit positions wins a syndrome); the Golay check bits come from qrl_golay.cuh (g = 0xC75), the AMBE PRNG from its LCG, the CRC
// from x^16 + x^12 + x^5 + 1, RS(12,9) from GF(2^8) mod x^8 + x^4 + x^3 + x^2 + 1 with g(x) = (x + 2)(x + 4)(x + 8), the BPTC interleave
// from 181 i mod 196, the trellis interleave from the dibit order and its state table from the encoder's rotation rule.
#include "../../include/qrl_b200.h"
#include "qrl_golay.cuh"
#include "qrl_handle.hpp"

#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace {

constexpr int kRec = QRL_DMR_RECORD_BYTES;
constexpr int kBurstBits = 288;       // CACH (24) + burst (264)
constexpr int kSyncFill = 180;        // DATA_AND_SYNC_BITS: CACH + 108 payload bits + 48 sync bits
enum { RECV_NONE = 0, RECV_DATA = 1, RECV_VOICE_SYNC = 2, RECV_VOICE = 3 };
enum { FT_DATA = 0, FT_VOICE = 1, FT_VOICE_SYNC = 2 };
enum : unsigned char { DT_VOICE_PI_HEADER = 0, DT_VOICE_LC_HEADER = 1, DT_TERMINATOR_WITH_LC = 2, DT_CSBK = 3, DT_MBC_HEADER = 4,
                       DT_MBC_CONTINUATION = 5, DT_DATA_HEADER = 6, DT_RATE_12_DATA = 7, DT_RATE_34_DATA = 8, DT_VOICE_SYNC = 0xF0,
                       DT_VOICE = 0xF1 };
constexpr uint64_t kSyncMask = 0xFFFFFFFFFFFFull;
constexpr uint64_t kMsData = 0xD5D7F77FD757ull, kMsVoice = 0x7F7D5DD57DFDull, kBsData = 0xDFF57D75DF5Dull, kBsVoice = 0x755FD7DF75F7ull;

// ---- syndrome tables (host-built, once per device)
__device__ uint32_t d_golay23_err[2048];   // (23,12) Golay: syndrome -> the unique error pattern of weight <= 3
__device__ uint32_t d_golay19_err[2048];   // (19,8) shortened Golay of the slot type: weights <= 5; 0 where no such leader exists
__device__ uint16_t d_qr15_err[256];       // (15,7) QR of the EMB: weights <= 4

// remainder of pattern (degree < top + 1) divided by g (degree deg)
__host__ __device__ inline uint32_t poly_mod(uint32_t r, int top, uint32_t g, int deg)
{
    for (int b = top; b >= deg; b--)
        if (r >> b & 1u) r ^= g << (b - deg);
    return r;
}

// for each syndrome, the first error pattern of least weight (weights up to max_w; positions in lexicographic order)
template <class T>
std::vector<T> syndrome_table(int n, uint32_t g, int deg, int max_w)
{
    std::vector<T> tab(static_cast<size_t>(1) << deg, 0);
    std::vector<char> seen(tab.size(), 0);
    seen[0] = 1;
    for (int w = 1; w <= max_w; w++) {
        std::vector<int> pos(w);
        for (int i = 0; i < w; i++) pos[i] = i;
        while (true) {
            uint32_t e = 0;
            for (int p : pos) e |= 1u << p;
            const uint32_t s = poly_mod(e, n - 1, g, deg);
            if (!seen[s]) { seen[s] = 1; tab[s] = static_cast<T>(e); }
            int i = w - 1;
            while (i >= 0 && pos[i] == n - w + i) i--;
            if (i < 0) break;
            pos[i]++;
            for (int j = i + 1; j < w; j++) pos[j] = pos[j - 1] + 1;
        }
    }
    return tab;
}

int upload_dmr_tables(QrlHandleBase* h)
{
    return once_per_device(reinterpret_cast<const void*>(&upload_dmr_tables), h->device, [h]() -> int {
        const auto g23 = syndrome_table<uint32_t>(23, 0xC75, 11, 3);
        const auto g19 = syndrome_table<uint32_t>(19, 0xC75, 11, 5);
        const auto q15 = syndrome_table<uint16_t>(15, 0x139, 8, 4);
        QRL_CK(cudaMemcpyToSymbol(d_golay23_err, g23.data(), g23.size() * sizeof(uint32_t)));
        QRL_CK(cudaMemcpyToSymbol(d_golay19_err, g19.data(), g19.size() * sizeof(uint32_t)));
        QRL_CK(cudaMemcpyToSymbol(d_qr15_err, q15.data(), q15.size() * sizeof(uint16_t)));
        return QRL_OK;
    });
}

// ================================================================================================ burst search
struct DmrSlot {
    uint64_t sr;                 // _shift_register
    uint32_t state, btr, ftr;    // _state, _bits_to_receive, _frames_to_receive
    uint32_t fill, end;          // ring: bits buffered (capped at 288), next write index
    uint32_t downlink;
};
struct DmrChan {
    DmrSlot s[2];
    long long pos;               // bits consumed since create / reset
    uint32_t next_slot;
    int dropped;
};

__device__ __forceinline__ uint64_t sync_window(uint64_t sr, uint32_t word, int l)
{
    // the shift register after bits 0..l of this step went in (bit 0 of `word` is the step's first bit)
    const uint64_t v = static_cast<uint64_t>(__brev(word) >> (31 - l));
    return ((sr << (l + 1)) | v) & kSyncMask;
}

__global__ void __launch_bounds__(128)
dmr_sink_kernel(int C, const unsigned char* __restrict__ bits, long long stride, const int* __restrict__ counts, DmrChan* __restrict__ chans,
                unsigned char* __restrict__ rings, unsigned char* __restrict__ out, int max_bursts, int* __restrict__ out_counts)
{
    __shared__ unsigned char s_ring[4][2][kBurstBits];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * 4 + w;
    if (c >= C) return;
    unsigned char* ring_g = rings + static_cast<long long>(c) * 2 * kBurstBits;
    for (int i = lane; i < 2 * kBurstBits; i += 32) s_ring[w][i / kBurstBits][i % kBurstBits] = ring_g[i];
    __syncwarp();
    DmrChan ch = chans[c];
    DmrSlot s0 = ch.s[0], s1 = ch.s[1];     // the active slot is copied out and back, so no slot array is indexed at run time
    const unsigned char* in = bits + static_cast<long long>(c) * stride;
    const int n = max(counts[c], 0);
    int nrec = 0;
    // append in[p .. p + k) to slot ts's ring
    auto append = [&](DmrSlot& s, int ts, int p, int k) {
        for (int j = lane; j < k; j += 32) s_ring[w][ts][(s.end + j) % kBurstBits] = in[p + j] & 1u;
        s.end = (s.end + k) % kBurstBits;
        s.fill = min(s.fill + static_cast<uint32_t>(k), static_cast<uint32_t>(kBurstBits));
        __syncwarp();
    };
    // a completed burst: the ring holds exactly its 288 bits, oldest at `end`
    auto emit = [&](const DmrSlot& s, int ts, int last, int ftype, int fn) {
        if (nrec < max_bursts) {
            unsigned char* r = out + (static_cast<long long>(c) * max_bursts + nrec) * kRec;
            for (int j = lane; j < 36; j += 32) {
                uint32_t v = 0;
                for (int b = 0; b < 8; b++) v = (v << 1) | s_ring[w][ts][(s.end + 8 * j + b) % kBurstBits];
                r[36 + j] = static_cast<unsigned char>(v);
            }
            if (lane == 0) {
                const long long at = ch.pos + last;
                for (int b = 0; b < 8; b++) r[b] = static_cast<unsigned char>(at >> (8 * b));
                r[8] = static_cast<unsigned char>(ts); r[9] = static_cast<unsigned char>(ftype); r[10] = static_cast<unsigned char>(fn);
                r[11] = static_cast<unsigned char>(s.downlink);
            }
        } else {
            ch.dropped++;
        }
        nrec++;
    };
    int p = 0;
    while (p < n) {
        const int ts = static_cast<int>(ch.next_slot);
        DmrSlot s = ts ? s1 : s0;
        if (s.state == RECV_NONE) {
            const int k = min(32, n - p);
            const uint32_t word = __ballot_sync(0xffffffffu, lane < k && (in[p + lane] & 1u));
            const uint64_t win = sync_window(s.sr, word, lane);
            const bool hit = lane < k && (win == kMsData || win == kMsVoice || win == kBsData || win == kBsVoice);
            const uint32_t hits = __ballot_sync(0xffffffffu, hit);
            const int used = hits ? __ffs(hits) : k;
            const uint64_t hw = __shfl_sync(0xffffffffu, win, used - 1);
            append(s, ts, p, used);
            s.sr = (s.sr << used) | (used == 32 ? static_cast<uint64_t>(__brev(word)) : static_cast<uint64_t>(__brev(word) >> (32 - used)));
            p += used;
            if (hits) {
                s.state = (hw == kBsData || hw == kMsData) ? RECV_DATA : RECV_VOICE_SYNC;
                s.downlink = (hw == kBsData || hw == kBsVoice) ? 1u : 0u;
                if (s.fill < kSyncFill) {
                    s.state = RECV_NONE; s.btr = 0; s.ftr = 0; s.fill = 0;
                } else {
                    s.fill = kSyncFill;
                    s.btr = 108;
                    if (s.state == RECV_VOICE_SYNC) s.ftr = 5;
                }
            }
        } else if (s.state == RECV_DATA || s.state == RECV_VOICE_SYNC) {
            const int k = min(static_cast<int>(s.btr), n - p);
            append(s, ts, p, k);
            s.btr -= k;
            p += k;
            if (s.btr == 0) {
                emit(s, ts, p - 1, s.state == RECV_DATA ? FT_DATA : FT_VOICE_SYNC, 0);
                s.state = s.state == RECV_VOICE_SYNC ? RECV_VOICE : RECV_NONE;
                s.fill = 0;
                ch.next_slot ^= 1u;
            }
        } else {     // RECV_VOICE, ftr > 0
            const int k = min(kBurstBits - static_cast<int>(s.fill), n - p);
            append(s, ts, p, k);
            p += k;
            if (s.fill >= kBurstBits) {
                emit(s, ts, p - 1, FT_VOICE, 6 - static_cast<int>(s.ftr));
                s.fill = 0;
                if (--s.ftr == 0) s.state = RECV_NONE;
                ch.next_slot ^= 1u;
            }
        }
        if (ts) s1 = s;
        else s0 = s;
    }
    ch.s[0] = s0; ch.s[1] = s1;
    ch.pos += n;
    __syncwarp();
    for (int i = lane; i < 2 * kBurstBits; i += 32) ring_g[i] = s_ring[w][i / kBurstBits][i % kBurstBits];
    if (lane == 0) {
        chans[c] = ch;
        out_counts[c] = min(nrec, max_bursts);
    }
}

__global__ void dmr_reset_kernel(int C, int channel, DmrChan* __restrict__ chans)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C || (channel >= 0 && c != channel)) return;
    DmrChan ch = {};
    ch.s[0].downlink = ch.s[1].downlink = 1u;     // gr_dmr_sink's constructor: _downlink = true
    chans[c] = ch;
}

// ================================================================================================ per-burst decode
// frame bits are numbered 0..263 MSB first; the BPTC and the trellis both skip the 68 bits of slot type + sync + slot type (98..165)
__device__ __forceinline__ int info_bit(int i) { return i < 98 ? i : i + 68; }

__device__ __forceinline__ uint32_t crc_ccitt(const unsigned char* p, int n)
{
    uint32_t crc = 0;
    for (int i = 0; i < n; i++) {
        crc ^= static_cast<uint32_t>(p[i]) << 8;
        for (int b = 0; b < 8; b++) crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x1021u) & 0xFFFFu : (crc << 1) & 0xFFFFu;
    }
    return ~crc & 0xFFFFu;
}

// CCITT162 check of 12 bytes whose last two are masked with (m, m)
__device__ __forceinline__ bool crc_ok(const unsigned char* p, unsigned char m)
{
    const uint32_t crc = crc_ccitt(p, 10);
    return (p[10] ^ m) == (crc >> 8) && (p[11] ^ m) == (crc & 0xFF);
}

__device__ __forceinline__ uint32_t gf_mul(uint32_t a, uint32_t b)
{
    uint32_t r = 0;
    for (int i = 0; i < 8; i++) {
        if (b >> i & 1u) r ^= a;
        a = (a << 1) ^ ((a & 0x80u) ? 0x11Du : 0u);
    }
    return r & 0xFFu;
}

// CRS129::encode of 9 data bytes: par[2], par[1], par[0] are the parity bytes 9, 10, 11 of the codeword
__device__ void rs129_parity(const unsigned char* m, uint32_t* par)
{
    const uint32_t G[3] = { 64, 56, 14 };
    par[0] = par[1] = par[2] = 0;
    for (int i = 0; i < 9; i++) {
        const uint32_t d = m[i] ^ par[2];
        par[2] = par[1] ^ gf_mul(G[2], d);
        par[1] = par[0] ^ gf_mul(G[1], d);
        par[0] = gf_mul(G[0], d);
    }
}

// CRS129::check on 9 data bytes + 3 parity bytes
__device__ bool rs129_ok(const unsigned char* m)
{
    uint32_t par[3];
    rs129_parity(m, par);
    return m[9] == par[2] && m[10] == par[1] && m[11] == par[0];
}

// Hamming(15,11,3) rows and (13,9,3) columns of the BPTC: the syndrome bits of a row / column, data bits d[0..], parity after
__device__ __forceinline__ uint32_t ham15_parity(const unsigned char* d)
{
    return (d[0] ^ d[1] ^ d[2] ^ d[3] ^ d[5] ^ d[7] ^ d[8]) | (d[1] ^ d[2] ^ d[3] ^ d[4] ^ d[6] ^ d[8] ^ d[9]) << 1 |
           (d[2] ^ d[3] ^ d[4] ^ d[5] ^ d[7] ^ d[9] ^ d[10]) << 2 | (d[0] ^ d[1] ^ d[2] ^ d[4] ^ d[6] ^ d[7] ^ d[10]) << 3;
}
__device__ __forceinline__ uint32_t ham13_parity(const unsigned char* d, int s)     // d[k * s], k = 0..8
{
    const uint32_t a0 = d[0], a1 = d[s], a2 = d[2 * s], a3 = d[3 * s], a4 = d[4 * s], a5 = d[5 * s], a6 = d[6 * s], a7 = d[7 * s], a8 = d[8 * s];
    return (a0 ^ a1 ^ a3 ^ a5 ^ a6) | (a0 ^ a1 ^ a2 ^ a4 ^ a6 ^ a7) << 1 | (a0 ^ a1 ^ a2 ^ a3 ^ a5 ^ a7 ^ a8) << 2 | (a0 ^ a2 ^ a4 ^ a5 ^ a8) << 3;
}
// the position a syndrome points at: parity bit k for 1 << k, otherwise the data bit whose parity column equals it (-1: none)
__device__ __forceinline__ int ham_locate(uint32_t n, int nd, bool rows)
{
    if (n == 0) return -1;
    for (int k = 0; k < 4; k++) if (n == (1u << k)) return nd + k;
    unsigned char e[11];
    for (int i = 0; i < nd; i++) {
        for (int j = 0; j < 11; j++) e[j] = j == i;
        const uint32_t col = rows ? ham15_parity(e) : ham13_parity(e, 1);
        if (col == n) return i;
    }
    return -1;
}

// BPTC(196,96) data positions: rows 0-8 of the 13 x 15 matrix (after the unused R(3) bit at 0), minus the parity columns and R(2..0)
__device__ __forceinline__ int bptc_data_pos(int k)
{
    return k < 8 ? 4 + k : 16 + (k - 8) + 4 * ((k - 8) / 11);
}

// BPTC(196,96) decode (warp): fb = the 264 frame bits, d = 196 scratch bits, payload = the 12 data bytes; up to 5 passes of column
// then row corrections, as CBPTC19696::decodeErrorCheck
__device__ void bptc_decode(const unsigned char* fb, unsigned char* d, unsigned char* payload, int lane)
{
    for (int a = lane; a < 196; a += 32) d[a] = fb[info_bit((a * 181) % 196)];
    __syncwarp();
    for (int pass = 0; pass < 5; pass++) {
        bool fixed = false;
        if (lane < 15) {
            unsigned char* col = d + lane + 1;
            const uint32_t syn = ham13_parity(col, 15) ^ (col[9 * 15] | col[10 * 15] << 1 | col[11 * 15] << 2 | col[12 * 15] << 3);
            const int at = ham_locate(syn, 9, false);
            if (at >= 0) { col[at * 15] ^= 1u; fixed = true; }
        }
        __syncwarp();
        if (lane < 9) {
            unsigned char* row = d + lane * 15 + 1;
            const uint32_t syn = ham15_parity(row) ^ (row[11] | row[12] << 1 | row[13] << 2 | row[14] << 3);
            const int at = ham_locate(syn, 11, true);
            if (at >= 0) { row[at] ^= 1u; fixed = true; }
        }
        __syncwarp();
        if (!__any_sync(0xffffffffu, fixed)) break;
    }
    if (lane < 12) {
        uint32_t v = 0;
        for (int b = 0; b < 8; b++) v = (v << 1) | d[bptc_data_pos(8 * lane + b)];
        payload[lane] = static_cast<unsigned char>(v);
    }
    __syncwarp();
}

// BPTC(196,96) encode of 12 payload bytes into the frame bits (warp)
__device__ void bptc_encode(const unsigned char* payload, unsigned char* d, unsigned char* fb, int lane)
{
    for (int a = lane; a < 196; a += 32) d[a] = 0;
    __syncwarp();
    for (int k = lane; k < 96; k += 32) d[bptc_data_pos(k)] = (payload[k >> 3] >> (7 - (k & 7))) & 1u;
    __syncwarp();
    if (lane < 9) {
        unsigned char* row = d + lane * 15 + 1;
        const uint32_t p = ham15_parity(row);
        for (int k = 0; k < 4; k++) row[11 + k] = (p >> k) & 1u;
    }
    __syncwarp();
    if (lane < 15) {
        unsigned char* col = d + lane + 1;
        const uint32_t p = ham13_parity(col, 15);
        for (int k = 0; k < 4; k++) col[(9 + k) * 15] = (p >> k) & 1u;
    }
    __syncwarp();
    for (int a = lane; a < 196; a += 32) fb[info_bit((a * 181) % 196)] = d[a];
    __syncwarp();
}

// ---- rate-3/4 trellis.  Dibit i of the burst is dibit trellis_interleave(i) of the code: the 98 code dibits d ordered by (d >> 1) & 3,
// then by d.
__device__ __forceinline__ int trellis_interleave(int i)
{
    // group g = (d >> 1) & 3 holds 26, 24, 24, 24 dibits
    const int g = i < 26 ? 0 : (i - 2) / 24, r = i < 26 ? i : (i - 2) % 24;
    return 8 * (r >> 1) + 2 * g + (r & 1);
}
// constellation point -> dibit pair (values +3 +1 -1 -3 as 0..3 = b1 b2 bits: +3 = 01, +1 = 00, -1 = 10, -3 = 11): points 8-15 are
// points 0-7 with each dibit negated and its magnitude swapped (+1 <-> -3, -1 <-> +3)
__device__ __forceinline__ uint32_t point_dibits(uint32_t p)
{
    // points 0-7: (+1,-1) (-1,-1) (+3,-3) (-3,-3) (-3,-1) (+3,-1) (-1,-3) (+1,-3), 2 bits per dibit (b1 b2), first dibit high
    constexpr uint32_t base = (0x0u << 2 | 0x2u) | (0x2u << 2 | 0x2u) << 4 | (0x1u << 2 | 0x3u) << 8 | (0x3u << 2 | 0x3u) << 12 |
                              (0x3u << 2 | 0x2u) << 16 | (0x1u << 2 | 0x2u) << 20 | (0x2u << 2 | 0x3u) << 24 | (0x0u << 2 | 0x3u) << 28;
    const uint32_t v = (base >> (4 * (p & 7u))) & 0xFu;
    return p < 8 ? v : v ^ 0xFu;
}
__device__ __forceinline__ uint32_t rev3(uint32_t j) { return ((j & 1u) << 2) | (j & 2u) | ((j >> 2) & 1u); }

// CDMRTrellis::checkCode with point `at` replaced by `val` (at = -1: none): 999 when every point follows the state table and the last
// tribit is 0, otherwise the first failing position.  The state table (next point for state s, tribit t): row 0 is the bit-reversed
// tribit times 2; rows 2-5 add 1; row s is row 0 or row 2 rotated by 0, 2, 4 or 6 tribits -- so the tribit follows from the point.
__device__ int trellis_check(const unsigned char* pts, int at, uint32_t val, unsigned char* tribits)
{
    uint32_t state = 0;
    for (int i = 0; i < 49; i++) {
        const uint32_t pt = i == at ? val : pts[i];
        const uint32_t rot = (state == 1 || state == 3) ? 2 : (state == 4 || state == 6) ? 4 : (state == 5 || state == 7) ? 6 : 0;
        const uint32_t odd = (state >= 2 && state <= 5) ? 1u : 0u;
        if ((pt & 1u) != odd) return i;
        state = (rev3(pt >> 1) - rot) & 7u;
        if (tribits) tribits[i] = static_cast<unsigned char>(state);
    }
    return state != 0 ? 48 : 999;
}

// CDMRTrellis::fixCode, the 16 candidates of a round on lanes 0-15: the first that checks wins, otherwise the first with the furthest
// failing position moves the search on
__device__ bool trellis_fix(unsigned char* pts, int fail, int lane)
{
    for (int round = 0; round < 20; round++) {
        const int pos = lane < 16 ? trellis_check(pts, fail, static_cast<uint32_t>(lane), nullptr) : -1;
        const uint32_t ok = __ballot_sync(0xffffffffu, pos == 999);
        if (ok) {
            __syncwarp();
            if (lane == 0) pts[fail] = static_cast<unsigned char>(__ffs(ok) - 1);
            __syncwarp();
            return true;
        }
        int key = lane < 16 ? (pos << 4) | (15 - lane) : 0;
        for (int o = 16; o; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
        __syncwarp();
        if (lane == 0) pts[fail] = static_cast<unsigned char>(15 - (key & 15));
        __syncwarp();
        fail = key >> 4;
    }
    return false;
}

__device__ __forceinline__ uint32_t ambe_prng(uint32_t u)     // the 24-bit PRNG word of A's 12 data bits
{
    uint32_t p = 16u * u, v = 0;
    for (int i = 0; i < 24; i++) {
        p = (173u * p + 13849u) & 0xFFFFu;
        v = (v << 1) | (p >> 15);
    }
    return v;
}
__device__ __forceinline__ uint32_t golay23_decode(uint32_t code)      // CGolay24128::decode23127
{
    return (code ^ d_golay23_err[poly_mod(code, 22, 0xC75u, 11)]) >> 11;
}
// CAMBEFEC::regenerateDMR(a, b, c) for one AMBE frame: the error count; a, b, c regenerated (or set to the silence frame)
__device__ uint32_t ambe_regenerate(uint32_t& a, uint32_t& b, uint32_t& c)
{
    const uint32_t orig_a = a, orig_b = b;
    const uint32_t syn = poly_mod(a >> 1, 22, 0xC75u, 11);
    const uint32_t cw = a ^ (d_golay23_err[syn] << 1);
    if (!(__popc(syn) < 3 || !(__popc(cw) & 1))) { a = 0xF00292u; b = 0x0E0B20u; c = 0; return 10; }
    const uint32_t data = cw >> 12;
    a = (data << 12) | golay_check(data);
    const uint32_t p = ambe_prng(data) >> 1;
    const uint32_t datb = golay23_decode(b ^ p);
    b = (((datb << 11) | (golay_check(datb) >> 1)) ^ p) & 0x7FFFFFu;
    const uint32_t ea = __popc(a ^ orig_a), eb = __popc(b ^ orig_b);
    if (ea >= 4 || (ea + eb >= 6 && ea >= 2)) { a = 0xF00292u; b = 0x0E0B20u; c = 0; }
    return ea + eb;
}
// frame bit of bit t (0..71) of AMBE frame f: A = t 0..23, B = 24..46, C = 47..71 walk the 72 bits with stride 4; frames 2 and 3 sit
// 72 and 192 bits on, frame 2 skipping the 48 sync / EMB bits
__device__ __forceinline__ int ambe_bit(int f, int t)
{
    const int base = 4 * (t % 18) + t / 18;
    return f == 0 ? base : f == 1 ? (base + 72 >= 108 ? base + 120 : base + 72) : base + 192;
}

__device__ __forceinline__ uint32_t be24(const unsigned char* p) { return static_cast<uint32_t>(p[0]) << 16 | p[1] << 8 | p[2]; }

__global__ void __launch_bounds__(128)
dmr_decode_kernel(int C, int max_bursts, const int* __restrict__ counts, unsigned char* __restrict__ out, int ambe_fec, int dmo)
{
    __shared__ unsigned char s_fb[4][264];
    __shared__ unsigned char s_d[4][196];
    __shared__ unsigned char s_pl[4][12];
    __shared__ unsigned char s_pts[4][2][49];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long g = static_cast<long long>(blockIdx.x) * 4 + w;
    const int c = static_cast<int>(g / max_bursts), k = static_cast<int>(g % max_bursts);
    if (c >= C || k >= counts[c]) return;
    unsigned char* r = out + g * kRec;
    unsigned char* fb = s_fb[w];
    const unsigned char* fr = r + 39;
    for (int i = lane; i < 264; i += 32) fb[i] = (fr[i >> 3] >> (7 - (i & 7))) & 1u;
    __syncwarp();
    const int ftype = r[9];
    // DMRFrame::setDownlink: AT, TC, LS1, LS0 and their Hamming(7,4) parity h0-h2
    uint32_t cach_ok = 0, at = 0, slot = 0, lcss = 0;
    if (r[11]) {
        const uint32_t a = (r[36] >> 7) & 1u, tc = (r[36] >> 3) & 1u, l1 = (r[37] >> 7) & 1u, l0 = (r[37] >> 3) & 1u;
        if ((a ^ tc ^ l1) == ((r[37] >> 1) & 1u) && (tc ^ l1 ^ l0) == ((r[38] >> 5) & 1u) && (a ^ tc ^ l0) == ((r[38] >> 1) & 1u)) {
            cach_ok = 1; at = a; slot = tc ? 2 : 1; lcss = (l1 << 1) | l0;
        }
    }
    uint32_t cc = 255, dt = ftype == FT_VOICE ? DT_VOICE : DT_VOICE_SYNC, valid = 1, flco = 0, fid = 0, src = 0, dst = 0;
    uint32_t ecc = 0, epi = 0, elcss = 0;
    int ambe = -1;
    if (ftype == FT_DATA) {
        // CDMRSlotType::putData: 20 bits around the sync, the first 19 through the (19,8) Golay decoder
        const uint32_t code = (static_cast<uint32_t>(fr[12] & 0x3Fu) << 13) | (static_cast<uint32_t>(fr[13] >> 4) << 9) |
                              (static_cast<uint32_t>(fr[19] & 0x0Fu) << 5) | ((static_cast<uint32_t>(fr[20]) >> 3) & 0x1Fu);
        const uint32_t st = ((code ^ d_golay19_err[poly_mod(code, 18, 0xC75u, 11)]) >> 11) & 0xFFu;
        cc = st >> 4; dt = st & 0xFu;
        valid = 0;
        if (dt <= DT_RATE_12_DATA) {
            unsigned char* pl = s_pl[w];
            bptc_decode(fb, s_d[w], pl, lane);
            bool ok = false;
            if (lane == 0) {
                const uint32_t id47 = be24(pl + 4), id79 = be24(pl + 7);
                if (dt == DT_CSBK || dt == DT_MBC_HEADER || dt == DT_MBC_CONTINUATION) {
                    // CDMRCSBK::put checks every one of them with the CSBK mask (and makes the CSBK's type DT_CSBK, so get() re-encodes
                    // the same bytes); the IDs follow the opcode
                    ok = crc_ok(pl, 0xA5);
                    if (ok) {
                        flco = pl[0] & 0x3Fu; fid = pl[1];
                        if (flco == 0x38) src = id79;                                              // BSDWNACT
                        else if (flco == 0x26 || (flco == 0x24 && pl[3] != 0x80)) { src = id47; dst = id79; }   // NACKRSP, radio check ack
                        else { dst = id47; src = id79; }
                    }
                } else if (dt == DT_DATA_HEADER) {
                    ok = crc_ok(pl, 0xCC);
                    const uint32_t dpf = pl[0] & 0xFu;
                    if (ok && dpf != 0xF) {                    // proprietary: no IDs
                        dst = be24(pl + 2); src = be24(pl + 5);
                        if (dpf == 0) {                        // UDT: opcode, and get() clears bit 0 of byte 9 and recomputes the CRC
                            flco = pl[9] & 0x3Fu;
                            pl[9] &= 0xFEu;
                            const uint32_t crc = crc_ccitt(pl, 10);
                            pl[10] = static_cast<unsigned char>((crc >> 8) ^ 0xCC); pl[11] = static_cast<unsigned char>((crc & 0xFF) ^ 0xCC);
                        }
                    }
                } else if (dt == DT_VOICE_LC_HEADER || dt == DT_TERMINATOR_WITH_LC) {
                    const unsigned char m = dt == DT_VOICE_LC_HEADER ? 0x96 : 0x99;
                    unsigned char lc[12];
                    for (int i = 0; i < 12; i++) lc[i] = pl[i] ^ (i >= 9 ? m : 0);
                    ok = rs129_ok(lc);
                    if (ok) { flco = pl[0] & 0x3Fu; fid = pl[1]; dst = be24(pl + 3); src = be24(pl + 6); }
                } else {                                       // PI header, rate 1/2: decode and re-encode only
                    ok = true;
                }
            }
            ok = __shfl_sync(0xffffffffu, ok, 0);
            __syncwarp();
            if (ok) bptc_encode(pl, s_d[w], fb, lane);
            valid = ok;
        } else if (dt == DT_RATE_34_DATA) {
            unsigned char* dib = s_d[w];
            unsigned char* pts = s_pts[w][0];
            unsigned char* save = s_pts[w][1];
            for (int i = lane; i < 98; i += 32) dib[trellis_interleave(i)] = static_cast<unsigned char>(fb[info_bit(2 * i)] << 1 | fb[info_bit(2 * i + 1)]);
            __syncwarp();
            for (int i = lane; i < 49; i += 32) {
                const uint32_t v = static_cast<uint32_t>(dib[2 * i]) << 2 | dib[2 * i + 1];
                uint32_t p = 0;
                while (point_dibits(p) != v) p++;
                pts[i] = save[i] = static_cast<unsigned char>(p);
            }
            __syncwarp();
            const int fail = trellis_check(pts, -1, 0, nullptr);
            unsigned char* good = pts;
            bool ok = fail == 999;
            if (!ok) ok = trellis_fix(pts, fail, lane);
            if (!ok && fail != 0) { ok = trellis_fix(save, fail - 1, lane); good = save; }
            if (ok) {      // the re-encoded payload is the corrected code sequence
                for (int i = lane; i < 98; i += 32) {
                    const int d = trellis_interleave(i);
                    const uint32_t v = point_dibits(good[d >> 1]);
                    const uint32_t db = (d & 1) ? v & 3u : v >> 2;
                    fb[info_bit(2 * i)] = static_cast<unsigned char>(db >> 1);
                    fb[info_bit(2 * i + 1)] = static_cast<unsigned char>(db & 1u);
                }
            }
            valid = ok;
        }
    } else {
        if (ambe_fec) {
            uint32_t e = 0;
            if (lane < 3) {
                uint32_t a = 0, b = 0, cw = 0;
                for (int t = 0; t < 24; t++) a = (a << 1) | fb[ambe_bit(lane, t)];
                for (int t = 24; t < 47; t++) b = (b << 1) | fb[ambe_bit(lane, t)];
                for (int t = 47; t < 72; t++) cw = (cw << 1) | fb[ambe_bit(lane, t)];
                e = ambe_regenerate(a, b, cw);
                for (int t = 0; t < 24; t++) fb[ambe_bit(lane, t)] = (a >> (23 - t)) & 1u;
                for (int t = 24; t < 47; t++) fb[ambe_bit(lane, t)] = (b >> (46 - t)) & 1u;
                for (int t = 47; t < 72; t++) fb[ambe_bit(lane, t)] = (cw >> (71 - t)) & 1u;
            }
            ambe = static_cast<int>(__shfl_sync(0xffffffffu, e, 0) + __shfl_sync(0xffffffffu, e, 1) + __shfl_sync(0xffffffffu, e, 2));
        }
        if (ftype == FT_VOICE) {
            // CDMREMB::putData: the 16 EMB bits around the embedded signalling, the first 15 through the QR(15,7) decoder
            const uint32_t code = (static_cast<uint32_t>(fr[13] & 0x0Fu) << 11) | (static_cast<uint32_t>(fr[14] >> 4) << 7) |
                                  (static_cast<uint32_t>(fr[18] & 0x0Fu) << 3) | (static_cast<uint32_t>(fr[19]) >> 5);
            const uint32_t e8 = ((code ^ d_qr15_err[poly_mod(code, 14, 0x139u, 8)]) >> 7) & 0xFFu;
            ecc = e8 >> 4; epi = (e8 >> 3) & 1u; elcss = (e8 >> 1) & 3u;
        }
    }
    __syncwarp();
    for (int j = lane; j < 33; j += 32) {
        uint32_t v = 0;
        for (int b = 0; b < 8; b++) v = (v << 1) | fb[8 * j + b];
        r[39 + j] = static_cast<unsigned char>(v);
    }
    if (lane == 0) {
        // gr_dmr_dmo_sink::writeFrame sets the slot number and colour code after the constructor: the DMO sink wrote them already
        r[12] = static_cast<unsigned char>(cach_ok); r[13] = static_cast<unsigned char>(at);
        if (!dmo) { r[14] = static_cast<unsigned char>(slot); r[16] = static_cast<unsigned char>(cc); }
        r[15] = static_cast<unsigned char>(lcss); r[17] = static_cast<unsigned char>(dt);
        r[18] = static_cast<unsigned char>(valid); r[19] = static_cast<unsigned char>(flco); r[20] = static_cast<unsigned char>(fid);
        r[21] = static_cast<unsigned char>(ecc); r[22] = static_cast<unsigned char>(epi); r[23] = static_cast<unsigned char>(elcss);
        for (int b = 0; b < 4; b++) {
            r[24 + b] = static_cast<unsigned char>(src >> (8 * b));
            r[28 + b] = static_cast<unsigned char>(dst >> (8 * b));
            r[32 + b] = static_cast<unsigned char>(static_cast<uint32_t>(ambe) >> (8 * b));
        }
    }
}

// ================================================================================================ direct-mode (DMO) burst search
// gr_dmr_dmo_sink::processSample (MMDVM's DMRDMORX) on QRL_DEMOD_DMR's port 3: 24 ksps floats, 5 samples per symbol.  The sink keeps a
// 1440-sample ring (60 ms, one DMO burst period); every sign bit the reference shifts into its five per-phase registers is the sign of
// a ring sample, so the ring alone is saved between calls.  All float arithmetic is separate multiplies and adds in the reference's
// order (this file is compiled with -fmad=false), so every decision rounds as the reference's SSE code does.
constexpr int kDmoRing = 1440;                 // DMO_BUFFER_LENGTH_SAMPLES
constexpr uint32_t kDmoNoEnd = 9999;           // NOENDPTR
constexpr uint32_t kMsDataSym = 0x76286Eu, kMsVoiceSym = 0x89D791u;     // sign patterns of the MS syncs' 24 symbols (+3 = 1)
enum { DMO_NONE = 0, DMO_DATA = 1, DMO_VOICE = 2 };                      // RECV_NONE / RECV_DATA / RECV_VOICE
enum { CTRL_NONE = 0x00, CTRL_VOICE = 0x20, CTRL_DATA = 0x40 };

struct DmoChan {
    long long pos;               // samples consumed since create / reset; m_dataPtr = pos mod 1440, m_bitPtr = pos mod 5
    float max_corr, centre[4], threshold[4];
    uint32_t sync_ptr, end_ptr, avg_ptr, sync_count, state, control, n, cc;
    int dropped;
};

struct DmoCand {                 // correlateSync at one sample, before its acceptance test
    uint32_t kind;               // 0: the prefilter failed; CTRL_DATA / CTRL_VOICE
    float corr, centre, threshold;
    bool bytes_ok;               // the sliced sync is within MAX_SYNC_BYTES_ERRS of the sync bytes
};

__device__ __forceinline__ uint32_t dmo_dibit(float v, float centre, float threshold)
{
    const float s = v - centre;
    return s < -threshold ? 3u : s < 0.0f ? 2u : s < threshold ? 0u : 1u;
}

// correlateSync's sample-local part at ring index d (the ring holds the sample of d and the 115 before it)
__device__ DmoCand dmo_correlate(const float* ring, uint32_t d)
{
    DmoCand c = { 0u, 0.0f, 0.0f, 0.0f, false };
    const uint32_t p0 = (d + kDmoRing - 115) % kDmoRing;
    uint32_t reg = 0;
    for (int i = 0; i < 24; i++) reg = (reg << 1) | (ring[(p0 + 5 * i) % kDmoRing] > 0.0f ? 1u : 0u);
    const bool data = __popc(reg ^ kMsDataSym) <= 2, voice = __popc(reg ^ kMsVoiceSym) <= 2;
    if (!data && !voice) return c;
    const uint32_t sym = data ? kMsDataSym : kMsVoiceSym;
    float corr = 0.0f, mn = 100.0f, mx = -100.0f;
    for (int i = 0; i < 24; i++) {
        const float val = ring[(p0 + 5 * i) % kDmoRing];
        if (val > mx) mx = val;
        if (val < mn) mn = val;
        corr = corr + ((sym >> (23 - i) & 1u) ? 3.0f : -3.0f) * val;      // float(corrVal) * val, rounded, then the add
    }
    const float centre = (mx + mn) / 2.0f;
    const float threshold = (mx - centre) / 2.0f;
    uint64_t bits = 0;
    for (int i = 0; i < 24; i++) bits = (bits << 2) | dmo_dibit(ring[(p0 + 5 * i) % kDmoRing], centre, threshold);
    c.kind = data ? CTRL_DATA : CTRL_VOICE;
    c.corr = corr; c.centre = centre; c.threshold = threshold;
    const uint64_t e = bits ^ (data ? kMsData : kMsVoice);
    c.bytes_ok = __popc(static_cast<uint32_t>(e)) + __popc(static_cast<uint32_t>(e >> 32)) <= 3;
    return c;
}

// the acceptance branch of correlateSync (corr > m_maxCorr and the byte check passed)
__device__ __forceinline__ void dmo_accept(DmoChan& s, const DmoCand& c, uint32_t d, bool first)
{
    if (first) {
        for (int i = 0; i < 4; i++) { s.threshold[i] = c.threshold; s.centre[i] = c.centre; }
        s.avg_ptr = 0;
    } else {
        s.threshold[s.avg_ptr] = c.threshold; s.centre[s.avg_ptr] = c.centre;
        s.avg_ptr = (s.avg_ptr + 1) & 3u;
    }
    s.max_corr = c.corr;
    s.control = c.kind;
    s.sync_ptr = d;
    s.end_ptr = (d + 269) % kDmoRing;           // DMR_SLOT_TYPE_LENGTH_SAMPLES / 2 + DMR_INFO_LENGTH_SAMPLES / 2 - 1
}

__device__ __forceinline__ void dmo_sink_reset(DmoChan& s)     // gr_dmr_dmo_sink::reset(): the partial reset of the state machine
{
    s.sync_ptr = 0; s.max_corr = 0.0f; s.sync_count = 0; s.state = DMO_NONE; s.end_ptr = kDmoNoEnd; s.cc = 0; s.n = 0;
}

__global__ void __launch_bounds__(128)
dmr_dmo_sink_kernel(int C, const float* __restrict__ x, long long stride, int n_all, const int* __restrict__ counts,
                    DmoChan* __restrict__ chans, float* __restrict__ rings, unsigned char* __restrict__ out, int max_bursts,
                    int* __restrict__ out_counts)
{
    __shared__ float s_ring[4][kDmoRing];
    __shared__ unsigned char s_frame[4][36];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * 4 + w;
    if (c >= C) return;
    float* ring = s_ring[w];
    float* ring_g = rings + static_cast<long long>(c) * kDmoRing;
    for (int i = lane; i < kDmoRing; i += 32) ring[i] = ring_g[i];
    DmoChan s = chans[c];                   // every lane holds the same copy of the state
    const float* in = x + static_cast<long long>(c) * stride;
    const int n = counts ? min(max(counts[c], 0), n_all) : n_all;
    uint32_t d = static_cast<uint32_t>(s.pos % kDmoRing);
    int nrec = 0;
    __syncwarp();
    // the end of a slot at ring index d, sample p of this call (processSample's m_dataPtr == m_endPtr branch)
    auto end_event = [&](int p) {
        const float centre = (s.centre[0] + s.centre[1] + s.centre[2] + s.centre[3]) / 4.0f;
        const float threshold = (s.threshold[0] + s.threshold[1] + s.threshold[2] + s.threshold[3]) / 4.0f;
        const uint32_t p0 = (s.end_ptr + kDmoRing - 660 + 5 + 1) % kDmoRing;
        for (int j = lane; j < 33; j += 32) {
            uint32_t v = 0;
            for (int k = 0; k < 4; k++) v = (v << 2) | dmo_dibit(ring[(p0 + 5 * (4 * j + k)) % kDmoRing], centre, threshold);
            s_frame[w][j] = static_cast<unsigned char>(v);
        }
        __syncwarp();
        const unsigned char* fr = s_frame[w];
        int ftype = -1;                    // the frame writeFrame is called with, if any
        bool do_reset = false;
        if (s.control == CTRL_DATA) {
            // CDMRSlotType2::decode: the same 19 bits and the same (19,8) syndrome table as DMRFrame's CDMRSlotType
            const uint32_t code = (static_cast<uint32_t>(fr[12] & 0x3Fu) << 13) | (static_cast<uint32_t>(fr[13] >> 4) << 9) |
                                  (static_cast<uint32_t>(fr[19] & 0x0Fu) << 5) | ((static_cast<uint32_t>(fr[20]) >> 3) & 0x1Fu);
            const uint32_t st = ((code ^ d_golay19_err[poly_mod(code, 18, 0xC75u, 11)]) >> 11) & 0xFFu;
            const uint32_t dt = st & 0xFu;
            s.cc = st >> 4; s.sync_count = 0; s.n = 0;
            if (dt == DT_DATA_HEADER) { s.state = DMO_DATA; ftype = FT_DATA; }
            else if (dt == DT_RATE_12_DATA || dt == DT_RATE_34_DATA || dt == 0x0Au) { if (s.state == DMO_DATA) ftype = FT_DATA; }
            else if (dt == DT_VOICE_LC_HEADER || dt == DT_VOICE_PI_HEADER) { s.state = DMO_VOICE; ftype = FT_DATA; }
            else if (dt == DT_TERMINATOR_WITH_LC) { if (s.state == DMO_VOICE) { ftype = FT_DATA; do_reset = true; } }
            else { ftype = FT_DATA; do_reset = true; }
        } else if (s.control == CTRL_VOICE) {
            s.state = DMO_VOICE; s.sync_count = 0; s.n = 0;
            ftype = FT_VOICE_SYNC;
        } else {
            if (s.state != DMO_NONE && ++s.sync_count >= 13) dmo_sink_reset(s);
            if (s.state == DMO_VOICE) { s.n = s.n >= 5 ? 0 : s.n + 1; ftype = FT_VOICE; }
            else if (s.state == DMO_DATA) ftype = FT_DATA;
        }
        if (ftype >= 0) {
            if (nrec < max_bursts) {
                unsigned char* r = out + (static_cast<long long>(c) * max_bursts + nrec) * kRec;
                for (int j = lane; j < 33; j += 32) r[39 + j] = fr[j];
                if (lane == 0) {
                    const long long at = s.pos + p;
                    for (int b = 0; b < 8; b++) r[b] = static_cast<unsigned char>(at >> (8 * b));
                    r[8] = 0; r[9] = static_cast<unsigned char>(ftype); r[10] = static_cast<unsigned char>(s.n); r[11] = 0;
                    r[14] = 2; r[16] = static_cast<unsigned char>(s.cc);
                    r[36] = r[37] = r[38] = 0;
                }
            } else {
                s.dropped++;
            }
            nrec++;
        }
        if (do_reset) dmo_sink_reset(s);
        s.max_corr = 0.0f;
        s.control = CTRL_NONE;
        __syncwarp();
    };
    int p = 0;
    while (p < n) {
        if (s.state == DMO_NONE) {
            // searching: correlateSync(true) at every sample.  Lane l takes sample p + l; the step ends at the first sample whose
            // candidate beats m_maxCorr or that meets the (possibly stale) end pointer
            const int k = min(32, n - p);
            const uint32_t dl = (d + lane) % kDmoRing;
            float old = 0.0f;
            if (lane < k) { old = ring[dl]; ring[dl] = in[p + lane]; }
            __syncwarp();
            DmoCand cd = { 0u, 0.0f, 0.0f, 0.0f, false };
            if (lane < k) cd = dmo_correlate(ring, dl);
            const bool ev = lane < k && ((cd.kind && cd.corr > s.max_corr && cd.bytes_ok) || dl == s.end_ptr);
            const uint32_t evs = __ballot_sync(0xffffffffu, ev);
            const int used = evs ? __ffs(evs) : k;
            __syncwarp();
            if (lane >= used && lane < k) ring[dl] = old;     // samples after the event are not in the ring yet
            if (evs) {
                const int e = used - 1;
                const uint32_t de = (d + e) % kDmoRing;
                DmoCand ce;
                ce.kind = __shfl_sync(0xffffffffu, cd.kind, e);
                ce.corr = __shfl_sync(0xffffffffu, cd.corr, e);
                ce.centre = __shfl_sync(0xffffffffu, cd.centre, e);
                ce.threshold = __shfl_sync(0xffffffffu, cd.threshold, e);
                ce.bytes_ok = __shfl_sync(0xffffffffu, static_cast<int>(cd.bytes_ok), e) != 0;
                if (ce.kind && ce.corr > s.max_corr && ce.bytes_ok) dmo_accept(s, ce, de, true);
                __syncwarp();
                if (de == s.end_ptr) end_event(p + e);
            }
            __syncwarp();
            p += used;
            d = (d + used) % kDmoRing;
        } else {
            // locked: correlateSync(false) only at m_syncPtr - 1 .. m_syncPtr + 1, so jump to that window or the end pointer
            const uint32_t t_in = (d + kDmoRing + 1 - s.sync_ptr) % kDmoRing;            // 0..2: d lies in the window
            const uint32_t t_win = t_in <= 2 ? 0u : (s.sync_ptr + kDmoRing - 1 - d) % kDmoRing;
            const uint32_t t_end = s.end_ptr == kDmoNoEnd ? 0xFFFFFFFFu : (s.end_ptr + kDmoRing - d) % kDmoRing;
            const int m = static_cast<int>(min(static_cast<uint32_t>(n - p), min(t_win, t_end)));
            for (int j = lane; j < m; j += 32) ring[(d + j) % kDmoRing] = in[p + j];
            p += m;
            d = (d + m) % kDmoRing;
            __syncwarp();
            if (p >= n) break;
            // one sample, as processSample takes it
            if (lane == 0) ring[d] = in[p];
            __syncwarp();
            if ((d + kDmoRing + 1 - s.sync_ptr) % kDmoRing <= 2) {
                const DmoCand cd = dmo_correlate(ring, d);
                if (cd.kind && cd.corr > s.max_corr && cd.bytes_ok) dmo_accept(s, cd, d, false);
            }
            if (d == s.end_ptr) end_event(p);
            __syncwarp();
            p += 1;
            d = (d + 1) % kDmoRing;
        }
    }
    s.pos += n;
    __syncwarp();
    for (int i = lane; i < kDmoRing; i += 32) ring_g[i] = ring[i];
    if (lane == 0) {
        chans[c] = s;
        out_counts[c] = min(nrec, max_bursts);
    }
}

__global__ void dmr_dmo_reset_kernel(int C, int channel, DmoChan* __restrict__ chans, float* __restrict__ rings)
{
    // the constructor's state, with the members it leaves uninitialised (ring, bit registers, centre, threshold, control) zero
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const int c = static_cast<int>(i / kDmoRing), k = static_cast<int>(i % kDmoRing);
    if (c >= C || (channel >= 0 && c != channel)) return;
    rings[i] = 0.0f;
    if (k == 0) {
        DmoChan s = {};
        s.end_ptr = kDmoNoEnd;
        chans[c] = s;
    }
}

// ================================================================================================ transmit
// DMRControl's transmit state machine as gr_modem drives it, and the burst encoders behind DMRFrame (see qrl_b200.h, qrl_dmr_tx_*).
constexpr int kTxBurst = 72;                 // gr_dmr_source: 33 frame bytes + 39 zero bytes
constexpr int kTxRec = QRL_DMR_TX_RECORD_BYTES;
enum { TX_IDLE = 0, TX_ACTIVE = 1, TX_ENDING = 2 };
enum { OPX_NONE = 0, OPX_CSBK = 1, OPX_HEADER = 2, OPX_AUDIO = 3, OPX_STOP = 4 };
enum { BK_CSBK = 1, BK_LC_HEADER = 2, BK_VOICE_SYNC = 3, BK_VOICE = 4, BK_TERMINATOR = 5, BK_EMPTY = 6 };

struct DmrTxCfg {                            // the Settings fields DMRControl reads, per channel
    unsigned char cc, slot, flco, fid;       // fid: 0xC2 when the voice is codec2 (!dmr_vocoder)
    uint32_t src, dst;
    unsigned char ta[27];                    // talker alias, zero padded
};
struct DmrTxState {                          // DMRControl's transmit members, plus the byte position of gr_dmr_source's stream
    long long pos;
    unsigned char state, fn, sf, npend, flco_tx;
    unsigned char lc_tx[9], emb_lc[9], ta[27];
    unsigned char pend[18];                  // _tx_frames: up to two 9-byte vocoder frames wait for a third
};
struct DmrTxBurst {                          // what the encode warp needs beyond the channel's settings
    unsigned char kind, fn, lcss, cc;
    unsigned char lc[9];                     // LC header / terminator: the full LC; voice FN 1-4: the embedded LC
    unsigned char pad[3];
    int audio[3];                            // the three vocoder frames: op index of this call (>= 0) or carried frame -1 - j
};
struct DmrTxRecord { long long pos; unsigned char slot, kind, fn, lcss; int op; };
static_assert(sizeof(DmrTxRecord) == kTxRec, "record layout");

__host__ __device__ inline void lc_bytes(unsigned char* o, uint32_t flco, uint32_t fid, uint32_t options, uint32_t src, uint32_t dst)
{
    o[0] = static_cast<unsigned char>(flco & 0x3Fu); o[1] = static_cast<unsigned char>(fid); o[2] = static_cast<unsigned char>(options);
    o[3] = static_cast<unsigned char>(dst >> 16); o[4] = static_cast<unsigned char>(dst >> 8); o[5] = static_cast<unsigned char>(dst);
    o[6] = static_cast<unsigned char>(src >> 16); o[7] = static_cast<unsigned char>(src >> 8); o[8] = static_cast<unsigned char>(src);
}

// DMRControl's constructor with the channel's settings in force; channel < 0 = every channel
__global__ void dmr_tx_reset_kernel(int C, int channel, const DmrTxCfg* __restrict__ cfgs, DmrTxState* __restrict__ states)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C || (channel >= 0 && c != channel)) return;
    const DmrTxCfg g = cfgs[c];
    DmrTxState s = {};
    s.flco_tx = g.flco;
    lc_bytes(s.lc_tx, g.flco, g.fid, 0, g.src, g.dst);
    for (int i = 0; i < 9; i++) s.emb_lc[i] = s.lc_tx[i];
    for (int i = 0; i < 27; i++) s.ta[i] = g.ta[i];
    states[c] = s;
}

// one thread per channel, in op order: the state machine of DMRControl (dmrcontrol.cpp:44-223) under gr_modem's calls
// (gr_modem.cpp:676-678, 710-717, 747-802).  Writes a descriptor and a record per burst and the channel's byte count; the vocoder
// frames still waiting at the end of the call are copied into the state, the ones carried in are left in `prev` for the encoder.
__global__ void dmr_tx_scan_kernel(int C, int K, const unsigned char* __restrict__ ops, const unsigned char* __restrict__ audio,
                                   const DmrTxCfg* __restrict__ cfgs, DmrTxState* __restrict__ states, unsigned char* __restrict__ prev,
                                   DmrTxBurst* __restrict__ bursts, unsigned char* __restrict__ recs, int max_bursts, int* __restrict__ counts)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const DmrTxCfg g = cfgs[c];
    DmrTxState s = states[c];
    for (int i = 0; i < 18; i++) prev[static_cast<long long>(c) * 18 + i] = s.pend[i];
    int psrc[3] = { -1, -2, 0 };
    int nb = 0;
    DmrTxBurst* bo = bursts + static_cast<long long>(c) * max_bursts;
    DmrTxRecord* ro = reinterpret_cast<DmrTxRecord*>(recs) + static_cast<long long>(c) * max_bursts;
    auto emit = [&](int kind, int slot, int fn, int lcss, const unsigned char* lc, int k) {
        DmrTxBurst d = {};
        d.kind = static_cast<unsigned char>(kind); d.fn = static_cast<unsigned char>(fn); d.lcss = static_cast<unsigned char>(lcss);
        d.cc = g.cc;
        if (lc)
            for (int i = 0; i < 9; i++) d.lc[i] = lc[i];
        for (int j = 0; j < 3; j++) d.audio[j] = psrc[j];
        bo[nb] = d;
        DmrTxRecord r;
        r.pos = s.pos; r.slot = static_cast<unsigned char>(slot); r.kind = d.kind; r.fn = d.fn; r.lcss = d.lcss; r.op = k;
        ro[nb] = r;
        s.pos += kTxBurst;
        nb++;
    };
    for (int k = 0; k < K; k++) {
        const int op = ops[static_cast<long long>(c) * K + k];
        if (op == OPX_CSBK) {                                       // getStartCSBK: three CSBK frames
            for (int i = 0; i < 3; i++) emit(BK_CSBK, g.slot, 0, 0, nullptr, k);
        } else if (op == OPX_HEADER) {                              // getVoiceHeader (LC snapshot, two frames), initVoiceTX
            s.flco_tx = g.flco;
            lc_bytes(s.lc_tx, g.flco, g.fid, 0, g.src, g.dst);
            for (int i = 0; i < 9; i++) s.emb_lc[i] = s.lc_tx[i];
            for (int i = 0; i < 2; i++) emit(BK_LC_HEADER, g.slot, 0, 0, s.lc_tx, k);
            s.fn = 0; s.sf = 0; s.state = TX_ACTIVE;
            for (int i = 0; i < 27; i++) s.ta[i] = g.ta[i];
        } else if (op == OPX_STOP) {                                // stopVoiceTX, from any state
            s.state = TX_ENDING;
        } else if (op == OPX_AUDIO && s.state != TX_IDLE) {         // transmitDMR: addTxAudio, then getTxAudio at three frames
            psrc[s.npend++] = k;
            if (s.npend < 3) continue;
            if (s.state == TX_ENDING && s.fn == 0) {                // the terminator twice, two empty frames; clearTxAudio
                unsigned char lc[9];
                lc_bytes(lc, s.flco_tx, 0, 0, g.src, g.dst);
                emit(BK_TERMINATOR, g.slot, 0, 0, lc, k);
                emit(BK_TERMINATOR, g.slot, 0, 0, lc, k);
                emit(BK_EMPTY, 0, 0, 0, nullptr, k);
                emit(BK_EMPTY, 0, 0, 0, nullptr, k);
                s.npend = 0; s.state = TX_IDLE; s.sf = 0;
                continue;
            }
            const int fn = s.fn;
            emit(fn == 0 ? BK_VOICE_SYNC : BK_VOICE, g.slot, fn, fn == 1 ? 1 : fn == 4 ? 2 : (fn == 2 || fn == 3) ? 3 : 0, s.emb_lc, k);
            s.npend = 0;
            if (++s.fn > 5) {                                       // superframe: the voice LC, then the talker-alias LCs
                s.fn = 0;
                s.sf = s.sf >= 4 ? 0 : s.sf + 1;
                if (s.sf == 0) {
                    for (int i = 0; i < 9; i++) s.emb_lc[i] = s.lc_tx[i];
                } else {
                    const int i = (s.sf - 1) * 6;
                    const uint32_t flco = 3u + s.sf;
                    const unsigned char* t = s.ta;
                    if (s.sf == 1)
                        lc_bytes(s.emb_lc, flco, 0, (1u << 6) | (0x1Bu << 1), static_cast<uint32_t>(t[i + 3]) << 16 | t[i + 4] << 8 | t[i + 5],
                                 static_cast<uint32_t>(t[i]) << 16 | t[i + 1] << 8 | t[i + 2]);
                    else
                        lc_bytes(s.emb_lc, flco, 0, t[i], static_cast<uint32_t>(t[i + 4]) << 16 | t[i + 5] << 8 | t[i + 6],
                                 static_cast<uint32_t>(t[i + 1]) << 16 | t[i + 2] << 8 | t[i + 3]);
                }
            }
        }
    }
    // the frames still waiting: from this call's audio or carried in
    unsigned char pend[18];
    for (int j = 0; j < s.npend; j++)
        for (int i = 0; i < 9; i++)
            pend[9 * j + i] = psrc[j] >= 0 ? audio[(static_cast<long long>(c) * K + psrc[j]) * 9 + i] : s.pend[9 * (-1 - psrc[j]) + i];
    for (int i = 0; i < 9 * s.npend; i++) s.pend[i] = pend[i];
    states[c] = s;
    counts[c] = nb * kTxBurst;
}

// Hamming(16,11,4) of a row of the embedded LC: the (15,11) checks of the BPTC rows plus overall parity (CHamming::encode16114)
__device__ __forceinline__ void ham16_encode(unsigned char* d)
{
    const uint32_t p = ham15_parity(d);
    uint32_t all = 0;
    for (int k = 0; k < 4; k++) { d[11 + k] = (p >> k) & 1u; all ^= (p >> k) & 1u; }
    for (int i = 0; i < 11; i++) all ^= d[i];
    d[15] = static_cast<unsigned char>(all);
}

// one warp per burst (S warps share a channel's bursts): 33 frame bytes + 39 zero bytes at the burst's place in the stream
__global__ void __launch_bounds__(128)
dmr_tx_encode_kernel(int C, int K, int S, const unsigned char* __restrict__ audio, const unsigned char* __restrict__ prev,
                     const DmrTxCfg* __restrict__ cfgs, const DmrTxBurst* __restrict__ bursts, int max_bursts, const int* __restrict__ counts,
                     unsigned char* __restrict__ out, long long stride)
{
    __shared__ unsigned char s_fb[4][264];
    __shared__ unsigned char s_d[4][196];
    __shared__ unsigned char s_pl[4][28];
    __shared__ unsigned char s_emb[4][128];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long gw = static_cast<long long>(blockIdx.x) * 4 + w;
    const int c = static_cast<int>(gw / S), s0 = static_cast<int>(gw % S);
    if (c >= C) return;
    const int nb = counts[c] / kTxBurst;
    unsigned char* fb = s_fb[w];
    unsigned char* pl = s_pl[w];
    for (int b = s0; b < nb; b += S) {
        const DmrTxBurst d = bursts[static_cast<long long>(c) * max_bursts + b];
        uint32_t* o = reinterpret_cast<uint32_t*>(out + static_cast<long long>(c) * stride + static_cast<long long>(b) * kTxBurst);
        if (d.kind == BK_EMPTY) {                                   // DMRFrame(DMRFrameTypeData): 33 zero bytes
            if (lane < kTxBurst / 4) o[lane] = 0;
            continue;
        }
        if (d.kind == BK_CSBK || d.kind == BK_LC_HEADER || d.kind == BK_TERMINATOR) {
            const uint32_t dt = d.kind == BK_CSBK ? DT_CSBK : d.kind == BK_LC_HEADER ? DT_VOICE_LC_HEADER : DT_TERMINATOR_WITH_LC;
            if (lane == 0) {
                if (d.kind == BK_CSBK) {                            // CDMRCSBK::get: BSDWNACT with LB, FID / data1 / CBF 0, CRC ^ 0xA5A5
                    const DmrTxCfg& g = cfgs[c];
                    lc_bytes(pl + 1, 0, 0, 0, g.src, g.dst);            // dst at 4-6, src at 7-9
                    pl[0] = 0x80u | 0x38u;
                    const uint32_t crc = crc_ccitt(pl, 10);
                    pl[10] = static_cast<unsigned char>((crc >> 8) ^ 0xA5u); pl[11] = static_cast<unsigned char>((crc & 0xFFu) ^ 0xA5u);
                } else {                                            // CDMRFullLC::encode: RS(12,9) parity ^ the type's mask
                    const unsigned char m = d.kind == BK_LC_HEADER ? 0x96 : 0x99;
                    for (int i = 0; i < 9; i++) pl[i] = d.lc[i];
                    uint32_t par[3];
                    rs129_parity(pl, par);
                    pl[9] = static_cast<unsigned char>(par[2] ^ m); pl[10] = static_cast<unsigned char>(par[1] ^ m);
                    pl[11] = static_cast<unsigned char>(par[0] ^ m);
                }
            }
            __syncwarp();
            bptc_encode(pl, s_d[w], fb, lane);
            // CDMRSlotType::getData (Golay(20,8) of colour code and data type) and CSync::addDMRDataSync (MS sourced)
            const uint32_t st = (static_cast<uint32_t>(d.cc) << 4) | dt, w20 = (st << 12) | golay_check(st);
            for (int i = lane; i < 68; i += 32) {
                if (i < 20) fb[i < 10 ? 98 + i : 146 + i] = static_cast<unsigned char>((w20 >> (19 - i)) & 1u);
                else fb[88 + i] = static_cast<unsigned char>((kMsData >> (67 - i)) & 1u);
            }
        } else {                                                    // voice: setVoice, then the sync or the EMB + embedded fragment
            if (lane < 27) {
                const int src = d.audio[lane / 9];
                pl[lane] = src >= 0 ? audio[(static_cast<long long>(c) * K + src) * 9 + lane % 9]
                                    : prev[static_cast<long long>(c) * 18 + 9 * (-1 - src) + lane % 9];
            }
            __syncwarp();
            for (int i = lane; i < 216; i += 32) fb[i < 108 ? i : i + 48] = (pl[i >> 3] >> (7 - (i & 7))) & 1u;
            if (d.fn == 0) {
                for (int i = lane; i < 48; i += 32) fb[108 + i] = static_cast<unsigned char>((kMsVoice >> (47 - i)) & 1u);
            } else {
                unsigned char* e = s_emb[w];
                if (d.fn <= 4) {
                    // CDMREmbeddedData::encodeEmbeddedData: the 72 LC bits in rows of 11 / 10, the 5-bit checksum (sum of the bytes
                    // mod 31) in column 10 of rows 2-6, Hamming(16,11,4) rows, column parity in row 7
                    uint32_t sum = 0;
                    for (int i = 0; i < 9; i++) sum += d.lc[i];
                    const uint32_t crc = sum % 31u;
                    for (int a = lane; a < 128; a += 32) {
                        const int r = a >> 4, col = a & 15;
                        int j = -1;
                        uint32_t v = 0;
                        if (r < 2 && col < 11) j = 11 * r + col;
                        else if (r >= 2 && r < 7 && col < 10) j = 22 + 10 * (r - 2) + col;
                        else if (r >= 2 && r < 7 && col == 10) v = (crc >> (6 - r)) & 1u;
                        if (j >= 0) v = (d.lc[j >> 3] >> (7 - (j & 7))) & 1u;
                        e[a] = static_cast<unsigned char>(v);
                    }
                    __syncwarp();
                    if (lane < 7) ham16_encode(e + 16 * lane);
                    __syncwarp();
                    if (lane < 16) {
                        uint32_t p = 0;
                        for (int r = 0; r < 7; r++) p ^= e[16 * r + lane];
                        e[112 + lane] = static_cast<unsigned char>(p);
                    }
                    __syncwarp();
                    // packed downwards in columns: raw bit a is data bit 16 a mod 127 (bit 127 stays); fragment FN - 1 of 32 bits
                    const int a = 32 * (d.fn - 1) + lane;
                    fb[116 + lane] = e[a == 127 ? 127 : (16 * a) % 127];
                } else {
                    fb[116 + lane] = 0;                             // FN 5: CDMREmbeddedData::getData's null fragment
                }
                // CDMREMB::getData: QR(16,7) of colour code, PI 0, LCSS = the (15,7) QR code (g = 0x139) plus overall parity
                const uint32_t v = (static_cast<uint32_t>(d.cc) << 3) | d.lcss;
                const uint32_t code = (v << 8) | poly_mod(v << 8, 14, 0x139u, 8);
                const uint32_t w16 = (code << 1) | (__popc(code) & 1u);
                if (lane < 16) fb[lane < 8 ? 108 + lane : 140 + lane] = static_cast<unsigned char>((w16 >> (15 - lane)) & 1u);
            }
        }
        __syncwarp();
        if (lane < kTxBurst / 4) {
            uint32_t word = 0;
            for (int q = 0; q < 4; q++) {
                const int m = 4 * lane + q;
                uint32_t v = 0;
                if (m < 33)
                    for (int i = 0; i < 8; i++) v = (v << 1) | fb[8 * m + i];
                word |= v << (8 * q);
            }
            o[lane] = word;
        }
        __syncwarp();
    }
}

}  // namespace

struct qrl_dmr_rx : QrlHandleBase {
    int C = 0, max_bursts = 0, ambe_fec = 0;
    long max_bits = 0;
    DmrChan* d_chans = nullptr;
    unsigned char* d_rings = nullptr;
    unsigned char* d_out = nullptr;
    int* d_counts = nullptr;
    unsigned char* d_stage = nullptr;
    int* d_stage_counts = nullptr;
};

extern "C" {

int qrl_dmr_rx_destroy(qrl_dmr_rx* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_dmr_rx_create(int n_channels, long max_bits, int max_bursts, int ambe_fec, int device, qrl_dmr_rx** out)
{
    if (!out || n_channels < 1 || max_bits < 1 || max_bursts < 1) { set_err(nullptr, "qrl_dmr_rx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_dmr_rx_create", device)) return rc;
    qrl_dmr_rx* h = new qrl_dmr_rx();
    h->C = n_channels; h->max_bits = max_bits; h->max_bursts = max_bursts; h->ambe_fec = ambe_fec ? 1 : 0;
    auto fail = [&](int rc) { return create_failed(h, qrl_dmr_rx_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels);
    if ((rc = upload_dmr_tables(h)) || (rc = dev_alloc(h, &h->d_chans, C)) || (rc = dev_alloc(h, &h->d_rings, C * 2 * kBurstBits)) ||
        (rc = dev_alloc(h, &h->d_out, C * max_bursts * kRec)) || (rc = dev_alloc(h, &h->d_counts, C)) ||
        (rc = dev_alloc(h, &h->d_stage, C * static_cast<size_t>(max_bits), false)) || (rc = dev_alloc(h, &h->d_stage_counts, C)))
        return fail(rc);
    dmr_reset_kernel<<<(n_channels + 127) / 128, 128, 0, h->stream>>>(n_channels, -1, h->d_chans);
    h->launches++;
    if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create: state init failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_dmr_rx_set_stream(qrl_dmr_rx* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

int qrl_dmr_rx_work(qrl_dmr_rx* h, const unsigned char* bits, const int* counts, long stride, int on_device)
{
    if (!h || !bits || !counts || stride < 0) { set_err(h, "qrl_dmr_rx_work: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char* d_bits = bits;
    const int* d_cnt = counts;
    if (on_device) {
        int rc;
        if ((rc = check_device_ptr(h, bits, "qrl_dmr_rx_work")) || (rc = check_device_ptr(h, counts, "qrl_dmr_rx_work"))) return rc;
    } else {
        if (stride > h->max_bits) { set_err(h, "qrl_dmr_rx_work: stride exceeds max_bits"); return QRL_EINVAL; }
        for (int c = 0; c < h->C; c++)
            if (counts[c] < 0 || counts[c] > stride) { set_err(h, "qrl_dmr_rx_work: bad count"); return QRL_EINVAL; }
        if (stride > 0) QRL_CK(cudaMemcpyAsync(h->d_stage, bits, static_cast<size_t>(h->C) * stride, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage_counts, counts, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
        d_bits = h->d_stage; d_cnt = h->d_stage_counts;
    }
    dmr_sink_kernel<<<(h->C + 3) / 4, 128, 0, h->stream>>>(h->C, d_bits, stride, d_cnt, h->d_chans, h->d_rings, h->d_out, h->max_bursts, h->d_counts);
    h->launches++;
    QRL_CK(cudaGetLastError());
    const long long warps = static_cast<long long>(h->C) * h->max_bursts;
    dmr_decode_kernel<<<static_cast<unsigned>((warps + 3) / 4), 128, 0, h->stream>>>(h->C, h->max_bursts, h->d_counts, h->d_out, h->ambe_fec, 0);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_dmr_rx_record_bytes(qrl_dmr_rx* h) { return h ? kRec : 0; }

int qrl_dmr_rx_read(qrl_dmr_rx* h, unsigned char* records_host, int* counts_host)
{
    if (!h || !counts_host) { set_err(h, "qrl_dmr_rx_read: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (records_host)
        QRL_CK(cudaMemcpyAsync(records_host, h->d_out, static_cast<size_t>(h->C) * h->max_bursts * kRec, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_dmr_rx_out_device(qrl_dmr_rx* h, void** records, int** counts)
{
    if (!h) return QRL_EINVAL;
    if (records) *records = h->d_out;
    if (counts) *counts = h->d_counts;
    return QRL_OK;
}

int qrl_dmr_rx_dropped(qrl_dmr_rx* h, int* dropped_host)
{
    if (!h || !dropped_host) { set_err(h, "qrl_dmr_rx_dropped: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    std::vector<DmrChan> ch(h->C);
    QRL_CK(cudaMemcpyAsync(ch.data(), h->d_chans, sizeof(DmrChan) * h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    for (int c = 0; c < h->C; c++) dropped_host[c] = ch[c].dropped;
    return QRL_OK;
}

int qrl_dmr_rx_reset(qrl_dmr_rx* h, int channel)
{
    if (!h) return QRL_EINVAL;
    if (channel < -1 || channel >= h->C) { set_err(h, "qrl_dmr_rx_reset: channel out of range"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    dmr_reset_kernel<<<(h->C + 127) / 128, 128, 0, h->stream>>>(h->C, channel, h->d_chans);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_dmr_rx_sync(qrl_dmr_rx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_dmr_rx_launch_count(qrl_dmr_rx* h) { return h ? h->launches : 0; }

}  // extern "C"

// ================================================================================================ DMO receive handle
struct qrl_dmr_dmo_rx : QrlHandleBase {
    int C = 0, max_bursts = 0, ambe_fec = 0;
    long max_samples = 0;
    DmoChan* d_chans = nullptr;
    float* d_rings = nullptr;
    unsigned char* d_out = nullptr;
    int* d_counts = nullptr;
    float* d_stage = nullptr;
    int* d_stage_counts = nullptr;
};

extern "C" {

int qrl_dmr_dmo_rx_destroy(qrl_dmr_dmo_rx* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_dmr_dmo_rx_reset(qrl_dmr_dmo_rx* h, int channel)
{
    if (!h) return QRL_EINVAL;
    if (channel < -1 || channel >= h->C) { set_err(h, "qrl_dmr_dmo_rx_reset: channel out of range"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    const long long n = static_cast<long long>(h->C) * kDmoRing;
    dmr_dmo_reset_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, h->stream>>>(h->C, channel, h->d_chans, h->d_rings);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_dmr_dmo_rx_create(int n_channels, long max_samples, int max_bursts, int ambe_fec, int device, qrl_dmr_dmo_rx** out)
{
    if (!out || n_channels < 1 || max_samples < 1 || max_bursts < 1) { set_err(nullptr, "qrl_dmr_dmo_rx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_dmr_dmo_rx_create", device)) return rc;
    qrl_dmr_dmo_rx* h = new qrl_dmr_dmo_rx();
    h->C = n_channels; h->max_samples = max_samples; h->max_bursts = max_bursts; h->ambe_fec = ambe_fec ? 1 : 0;
    auto fail = [&](int rc) { return create_failed(h, qrl_dmr_dmo_rx_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels);
    if ((rc = upload_dmr_tables(h)) || (rc = dev_alloc(h, &h->d_chans, C)) || (rc = dev_alloc(h, &h->d_rings, C * kDmoRing)) ||
        (rc = dev_alloc(h, &h->d_out, C * max_bursts * kRec)) || (rc = dev_alloc(h, &h->d_counts, C)) ||
        (rc = dev_alloc(h, &h->d_stage, C * static_cast<size_t>(max_samples), false)) || (rc = dev_alloc(h, &h->d_stage_counts, C)))
        return fail(rc);
    if ((rc = qrl_dmr_dmo_rx_reset(h, -1))) return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create: state init failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_dmr_dmo_rx_set_stream(qrl_dmr_dmo_rx* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

int qrl_dmr_dmo_rx_work(qrl_dmr_dmo_rx* h, const float* samples, long n, const int* counts, long stride, int on_device)
{
    if (!h || !samples || n < 0 || n > h->max_samples || stride < n) {
        set_err(h, "qrl_dmr_dmo_rx_work: bad argument (0 <= n <= max_samples, stride >= n)");
        return QRL_EINVAL;
    }
    QRL_CK(cudaSetDevice(h->device));
    const float* d_x = samples;
    const int* d_cnt = counts;
    long d_stride = stride;
    if (on_device) {
        int rc;
        if ((rc = check_device_ptr(h, samples, "qrl_dmr_dmo_rx_work")) || (counts && (rc = check_device_ptr(h, counts, "qrl_dmr_dmo_rx_work"))))
            return rc;
    } else {
        if (counts)
            for (int c = 0; c < h->C; c++)
                if (counts[c] < 0 || counts[c] > n) { set_err(h, "qrl_dmr_dmo_rx_work: bad count"); return QRL_EINVAL; }
        if (n > 0)
            QRL_CK(cudaMemcpy2DAsync(h->d_stage, sizeof(float) * n, samples, sizeof(float) * stride, sizeof(float) * n, h->C,
                                     cudaMemcpyHostToDevice, h->stream));
        if (counts) {
            QRL_CK(cudaMemcpyAsync(h->d_stage_counts, counts, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
            d_cnt = h->d_stage_counts;
        }
        d_x = h->d_stage; d_stride = n;
    }
    dmr_dmo_sink_kernel<<<(h->C + 3) / 4, 128, 0, h->stream>>>(h->C, d_x, d_stride, static_cast<int>(n), d_cnt, h->d_chans, h->d_rings,
                                                              h->d_out, h->max_bursts, h->d_counts);
    h->launches++;
    QRL_CK(cudaGetLastError());
    const long long warps = static_cast<long long>(h->C) * h->max_bursts;
    dmr_decode_kernel<<<static_cast<unsigned>((warps + 3) / 4), 128, 0, h->stream>>>(h->C, h->max_bursts, h->d_counts, h->d_out, h->ambe_fec, 1);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_dmr_dmo_rx_record_bytes(qrl_dmr_dmo_rx* h) { return h ? kRec : 0; }

int qrl_dmr_dmo_rx_read(qrl_dmr_dmo_rx* h, unsigned char* records_host, int* counts_host)
{
    if (!h || !counts_host) { set_err(h, "qrl_dmr_dmo_rx_read: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (records_host)
        QRL_CK(cudaMemcpyAsync(records_host, h->d_out, static_cast<size_t>(h->C) * h->max_bursts * kRec, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_dmr_dmo_rx_out_device(qrl_dmr_dmo_rx* h, void** records, int** counts)
{
    if (!h) return QRL_EINVAL;
    if (records) *records = h->d_out;
    if (counts) *counts = h->d_counts;
    return QRL_OK;
}

int qrl_dmr_dmo_rx_dropped(qrl_dmr_dmo_rx* h, int* dropped_host)
{
    if (!h || !dropped_host) { set_err(h, "qrl_dmr_dmo_rx_dropped: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    std::vector<DmoChan> ch(h->C);
    QRL_CK(cudaMemcpyAsync(ch.data(), h->d_chans, sizeof(DmoChan) * h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    for (int c = 0; c < h->C; c++) dropped_host[c] = ch[c].dropped;
    return QRL_OK;
}

int qrl_dmr_dmo_rx_sync(qrl_dmr_dmo_rx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_dmr_dmo_rx_launch_count(qrl_dmr_dmo_rx* h) { return h ? h->launches : 0; }

}  // extern "C"

// ================================================================================================ transmit handle
struct qrl_dmr_tx : QrlHandleBase {
    int C = 0, max_ops = 0, max_bursts = 0;
    long out_stride = 0;
    DmrTxCfg* d_cfg = nullptr;
    DmrTxState* d_state = nullptr;
    DmrTxBurst* d_bursts = nullptr;
    unsigned char *d_recs = nullptr, *d_out = nullptr, *d_prev = nullptr, *d_ops = nullptr, *d_audio = nullptr;
    int* d_counts = nullptr;
};

namespace {
int tx_config(qrl_dmr_tx* h, const qrl_dmr_tx_config* in, DmrTxCfg* out)
{
    if (in->color_code < 0 || in->color_code > 15 || (in->timeslot != 1 && in->timeslot != 2) || in->src_id > 0xFFFFFFu ||
        in->dst_id > 0xFFFFFFu || (in->private_call != 0 && in->private_call != 1) || (in->codec2 != 0 && in->codec2 != 1) ||
        in->talker_alias_len < 0 || in->talker_alias_len > 27) {
        set_err(h, "qrl_dmr_tx_set_config: colour code 0-15, timeslot 1 or 2, 24-bit IDs, private_call and codec2 0 or 1, "
                   "talker_alias_len 0-27");
        return QRL_EINVAL;
    }
    *out = DmrTxCfg{};
    out->cc = static_cast<unsigned char>(in->color_code); out->slot = static_cast<unsigned char>(in->timeslot);
    out->flco = in->private_call ? 3 : 0; out->fid = in->codec2 ? 0xC2 : 0;
    out->src = in->src_id; out->dst = in->dst_id;
    for (int i = 0; i < in->talker_alias_len; i++) out->ta[i] = in->talker_alias[i];
    return QRL_OK;
}
}  // namespace

extern "C" {

int qrl_dmr_tx_destroy(qrl_dmr_tx* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_dmr_tx_set_config(qrl_dmr_tx* h, int channel, const qrl_dmr_tx_config* cfg)
{
    if (!h || !cfg) { set_err(h, "qrl_dmr_tx_set_config: bad argument"); return QRL_EINVAL; }
    if (channel < -1 || channel >= h->C) { set_err(h, "qrl_dmr_tx_set_config: channel out of range"); return QRL_ERANGE; }
    DmrTxCfg g;
    if (int rc = tx_config(h, cfg, &g)) return rc;
    QRL_CK(cudaSetDevice(h->device));
    const int n = channel < 0 ? h->C : 1;
    std::vector<DmrTxCfg> v(n, g);
    QRL_CK(cudaMemcpyAsync(h->d_cfg + (channel < 0 ? 0 : channel), v.data(), sizeof(DmrTxCfg) * n, cudaMemcpyHostToDevice, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_dmr_tx_reset(qrl_dmr_tx* h, int channel)
{
    if (!h) return QRL_EINVAL;
    if (channel < -1 || channel >= h->C) { set_err(h, "qrl_dmr_tx_reset: channel out of range"); return QRL_ERANGE; }
    QRL_CK(cudaSetDevice(h->device));
    dmr_tx_reset_kernel<<<(h->C + 127) / 128, 128, 0, h->stream>>>(h->C, channel, h->d_cfg, h->d_state);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_dmr_tx_create(int n_channels, int max_ops, int device, qrl_dmr_tx** out)
{
    if (!out || n_channels < 1 || max_ops < 1) { set_err(nullptr, "qrl_dmr_tx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_dmr_tx_create", device)) return rc;
    qrl_dmr_tx* h = new qrl_dmr_tx();
    h->C = n_channels; h->max_ops = max_ops; h->max_bursts = 4 * max_ops; h->out_stride = static_cast<long>(h->max_bursts) * kTxBurst;
    auto fail = [&](int rc) { return create_failed(h, qrl_dmr_tx_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels), B = C * h->max_bursts;
    if ((rc = dev_alloc(h, &h->d_cfg, C)) || (rc = dev_alloc(h, &h->d_state, C)) || (rc = dev_alloc(h, &h->d_bursts, B)) ||
        (rc = dev_alloc(h, &h->d_recs, B * kTxRec)) || (rc = dev_alloc(h, &h->d_out, C * h->out_stride, false)) ||
        (rc = dev_alloc(h, &h->d_prev, C * 18)) || (rc = dev_alloc(h, &h->d_ops, C * max_ops)) ||
        (rc = dev_alloc(h, &h->d_audio, C * max_ops * 9)) || (rc = dev_alloc(h, &h->d_counts, C)))
        return fail(rc);
    qrl_dmr_tx_config def = {};
    def.color_code = 1; def.timeslot = 1; def.src_id = 1; def.dst_id = 9; def.private_call = 0; def.codec2 = 1;
    if ((rc = qrl_dmr_tx_set_config(h, -1, &def)) || (rc = qrl_dmr_tx_reset(h, -1))) return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create: state init failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_dmr_tx_set_stream(qrl_dmr_tx* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

int qrl_dmr_tx_work(qrl_dmr_tx* h, const unsigned char* ops, const unsigned char* audio, int K, int on_device)
{
    if (!h || !ops || !audio) { set_err(h, "qrl_dmr_tx_work: bad argument"); return QRL_EINVAL; }
    if (K < 0 || K > h->max_ops) { set_err(h, "qrl_dmr_tx_work: K must be between 0 and max_ops"); return QRL_ERANGE; }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char *d_ops = ops, *d_audio = audio;
    if (on_device) {
        int rc;
        if ((rc = check_device_ptr(h, ops, "qrl_dmr_tx_work")) || (rc = check_device_ptr(h, audio, "qrl_dmr_tx_work"))) return rc;
    } else {
        if (K > 0) {
            QRL_CK(cudaMemcpyAsync(h->d_ops, ops, static_cast<size_t>(h->C) * K, cudaMemcpyHostToDevice, h->stream));
            QRL_CK(cudaMemcpyAsync(h->d_audio, audio, static_cast<size_t>(h->C) * K * 9, cudaMemcpyHostToDevice, h->stream));
        }
        d_ops = h->d_ops; d_audio = h->d_audio;
    }
    dmr_tx_scan_kernel<<<(h->C + 127) / 128, 128, 0, h->stream>>>(h->C, K, d_ops, d_audio, h->d_cfg, h->d_state, h->d_prev, h->d_bursts,
                                                                   h->d_recs, h->max_bursts, h->d_counts);
    h->launches++;
    QRL_CK(cudaGetLastError());
    if (K > 0) {
        // S warps per channel walk its bursts with stride S: steady voice makes one burst per three ops, a terminator four per op
        const int S = std::min(8, h->max_bursts);
        const long long warps = static_cast<long long>(h->C) * S;
        dmr_tx_encode_kernel<<<static_cast<unsigned>((warps + 3) / 4), 128, 0, h->stream>>>(h->C, K, S, d_audio, h->d_prev, h->d_cfg, h->d_bursts,
                                                                                         h->max_bursts, h->d_counts, h->d_out, h->out_stride);
        h->launches++;
        QRL_CK(cudaGetLastError());
    }
    return QRL_OK;
}

int qrl_dmr_tx_read(qrl_dmr_tx* h, unsigned char* bytes_host, long cap, unsigned char* records_host, int* counts_host)
{
    if (!h || !counts_host) { set_err(h, "qrl_dmr_tx_read: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (bytes_host && cap > 0)
        QRL_CK(cudaMemcpy2DAsync(bytes_host, static_cast<size_t>(cap), h->d_out, static_cast<size_t>(h->out_stride),
                                 static_cast<size_t>(cap < h->out_stride ? cap : h->out_stride), h->C, cudaMemcpyDeviceToHost, h->stream));
    if (records_host)
        QRL_CK(cudaMemcpyAsync(records_host, h->d_recs, static_cast<size_t>(h->C) * h->max_bursts * kTxRec, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_dmr_tx_out_device(qrl_dmr_tx* h, void** bytes, long* stride, int** counts, void** records)
{
    if (!h) return QRL_EINVAL;
    if (bytes) *bytes = h->d_out;
    if (stride) *stride = h->out_stride;
    if (counts) *counts = h->d_counts;
    if (records) *records = h->d_recs;
    return QRL_OK;
}

int qrl_dmr_tx_sync(qrl_dmr_tx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_dmr_tx_launch_count(qrl_dmr_tx* h) { return h ? h->launches : 0; }

}  // extern "C"
