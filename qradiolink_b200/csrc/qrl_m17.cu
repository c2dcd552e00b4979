// qrl_m17.cu -- the M17 frame codec on the device, part of libqrl_b200.so.
//
// Receive (qrl_m17_rx_*): M17FrameDecoder::decodeFrame plus the lines of gr_modem::processReceivedData that drive it
// (/root/reference/src/gr_modem.cpp:1370-1440; src/M17/M17/M17FrameDecoder.cpp) for a batch of channels, fed with the records of the
// layer-1 deframer (sync class 4).  Two kernels:
//   * m17_frame_kernel, one warp per (channel, record): every frame decodes independently of the others.  Derandomising and
//     deinterleaving are bit-parallel (a bit per lane); the punctured K = 5 Viterbi decoder keeps one trellis state per lane (16 states,
//     lanes 16-31 mirror 0-15), fetches the two predecessor metrics with __shfl_sync and stores the 16 decisions of a step with one
//     __ballot_sync; lane 0 walks the chainback.  The 4 Golay(24,12) words of a stream frame's LICH decode on lanes 0-3.
//   * m17_state_kernel, one thread per channel: walks that channel's records in order and applies what carries between frames --
//     LSF reassembly from the LICH segments, the CRC checks, the EOT reset -- and writes one snapshot per record.
// Transmit (qrl_m17_tx_*): M17Transmitter::start / send and gr_modem::endTransmission's M17 tail (gr_modem.cpp:680-735, 868-882;
// src/M17/M17/M17Transmitter.cpp).  m17_tx_scan_kernel (one thread per channel) turns the ops into output offsets, frame numbers and
// LICH indices, the only state that carries; m17_tx_encode_kernel (one warp per (channel, op)) encodes a frame bit-parallel.
//
// Every constant is generated from the M17 specification's definitions: the puncture matrices P1 / P2, the quadratic interleaver
// (45 i + 92 i^2) mod 368, the Golay(24,12) check matrix from the generator polynomial 0xC75, the CRC-16 (0x5935, init 0xFFFF) and the
// spec's randomizer sequence.  Where the reference decoder has a quirk (the Viterbi chainback, segment numbers 6 and 7) the kernels
// restate its observable result.
#include "../../include/qrl_b200.h"
#include "qrl_handle.hpp"

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

namespace {

enum : uint32_t { M17_STREAM = 0xFF5D, M17_LSF = 0x55F7, M17_EOT = 0x555D555D };     // layer1framing.h:21-23
enum { OP_NONE = 0, OP_START = 1, OP_STREAM = 2, OP_LAST = 3 };
constexpr int kRxRecord = 56;         // { uint32 type, lsf[30], lsf_valid, 0, stream_frame[18], 0, 0 }
constexpr int kStepMax = 96;          // bytes of the longest op (start: preamble + LSF frame)

// the randomizer ("decorrelator") sequence of the M17 specification, XORed over the 368 bits after the sync word of every frame
__device__ const unsigned char kRandomizer[46] = {
    0xd6, 0xb5, 0xe2, 0x30, 0x82, 0xff, 0x84, 0x62, 0xba, 0x4e, 0x96, 0x90, 0xd8, 0x98, 0xdd, 0x5d, 0x0c, 0xc8, 0x52, 0x43, 0x91, 0x1d, 0xf8,
    0x6e, 0x68, 0x2f, 0x35, 0xda, 0x14, 0xea, 0xcd, 0x76, 0x19, 0x8d, 0xd5, 0x80, 0xd1, 0x33, 0x87, 0x13, 0x57, 0x18, 0x2d, 0x29, 0x78, 0xc3 };

// ---- Golay(24,12): the 12 check bits of data d are ((d(x) x^11 mod g(x)) << 1) | overall parity, g(x) = 0xC75 (the (23,12) cyclic
// code, extended).  enc[i] = the check bits of data bit i; dec = its transpose, which is also its inverse (the code is self-dual).
struct GolayRows { uint16_t enc[12], dec[12]; };

__host__ __device__ constexpr uint16_t golay_check(uint32_t d)
{
    uint32_t r = d << 11;
    for (int b = 22; b >= 11; b--)
        if (r >> b & 1u) r ^= 0xC75u << (b - 11);
    int par = 0;
    for (int b = 0; b < 12; b++) par += static_cast<int>((d >> b) & 1u) + static_cast<int>((r >> b) & 1u);
    return static_cast<uint16_t>((r << 1) | (par & 1));
}

constexpr GolayRows make_golay_rows()
{
    GolayRows g{};
    for (int i = 0; i < 12; i++) g.enc[i] = golay_check(1u << i);
    for (int j = 0; j < 12; j++) {
        uint16_t v = 0;
        for (int k = 0; k < 12; k++) v |= static_cast<uint16_t>(((g.enc[k] >> j) & 1u) << k);
        g.dec[j] = v;
    }
    return g;
}

__device__ const GolayRows kGolay = make_golay_rows();

__device__ __forceinline__ uint32_t mat12(uint32_t v, const uint16_t* m)
{
    uint32_t r = 0;
    for (int i = 0; i < 12; i++) if (v >> i & 1u) r ^= m[i];
    return r;
}

// M17's Golay decoder (the error pattern it assumes for a syndrome: weight <= 3 in the check part, one data bit + <= 2 check bits, the
// same through the inverse syndrome); 0xFFFF = uncorrectable
__device__ uint32_t golay24_decode(uint32_t cw)
{
    const uint32_t s = (cw & 0xFFFu) ^ mat12(cw >> 12, kGolay.enc);
    uint32_t e = 0xFFFFFFFFu;
    if (__popc(s) <= 3) e = s;
    else {
        for (int i = 0; i < 12 && e == 0xFFFFFFFFu; i++)
            if (__popc(s ^ kGolay.enc[i]) <= 2) e = ((1u << i) << 12) | (s ^ kGolay.enc[i]);
        if (e == 0xFFFFFFFFu) {
            const uint32_t q = mat12(s, kGolay.dec);
            if (__popc(q) <= 3) e = q << 12;
            else
                for (int i = 0; i < 12 && e == 0xFFFFFFFFu; i++)
                    if (__popc(q ^ kGolay.dec[i]) <= 2) e = ((q ^ kGolay.dec[i]) << 12) | (1u << i);
        }
    }
    return e == 0xFFFFFFFFu ? 0xFFFFu : ((cw ^ e) >> 12) & 0xFFFu;
}

// ---- CRC-16 of the LSF: polynomial 0x5935, initial 0xFFFF, MSB first, over the first 28 bytes
__host__ __device__ inline uint16_t m17_crc(const unsigned char* p, int n)
{
    uint32_t crc = 0xFFFF;
    for (int i = 0; i < n; i++) {
        crc ^= static_cast<uint32_t>(p[i]) << 8;
        for (int j = 0; j < 8; j++) crc = (crc & 0x8000u) ? ((crc << 1) ^ 0x5935u) & 0xFFFFu : (crc << 1) & 0xFFFFu;
    }
    return static_cast<uint16_t>(crc);
}

__host__ __device__ inline bool lsf_valid(const unsigned char* lsf)
{
    const uint16_t c = m17_crc(lsf, 28);
    return lsf[28] == (c >> 8) && lsf[29] == (c & 0xFF);
}

// puncture matrices: P1 (LSF) = 1, then 15 x (1 0 1 1), 61 entries with 46 ones; P2 (stream) = 11 x 1, then 0
__device__ __forceinline__ bool p_keep(bool lsf, int i) { return lsf ? (i == 0 || ((i - 1) & 3) != 1) : i != 11; }
// index in the encoded stream of punctured bit q
__device__ __forceinline__ int p_source(bool lsf, int q)
{
    if (!lsf) return (q / 11) * 12 + q % 11;
    const int blk = q / 46, r = q % 46;
    if (r == 0) return blk * 61;
    const int b = (r - 1) / 3, m = (r - 1) % 3;
    return blk * 61 + 1 + 4 * b + (m == 0 ? 0 : m + 1);
}
__device__ __forceinline__ int qpp(int i) { return (45 * i + 92 * i * i) % 368; }

// ================================================================================================ receive
struct FrameOut {             // m17_frame_kernel -> m17_state_kernel, one per (channel, record)
    uint32_t type;
    unsigned char data[30];   // LSF: the decoded 30 bytes; stream: the 18-byte stream frame
    unsigned char seg[6];     // stream: the LICH segment (5 LSF bytes, segment number)
    unsigned char lich_ok, pad;
};

struct M17RxState {
    unsigned char lsf[30], part[30], sf[18];
    unsigned char map, valid;
};

__device__ __forceinline__ uint32_t ld_u32(const unsigned char* p)
{
    return static_cast<uint32_t>(p[0]) | static_cast<uint32_t>(p[1]) << 8 | static_cast<uint32_t>(p[2]) << 16 | static_cast<uint32_t>(p[3]) << 24;
}

__global__ void __launch_bounds__(128)
m17_frame_kernel(int C, int max_frames, const unsigned char* __restrict__ records, long long rec_bytes, const int* __restrict__ counts,
                 FrameOut* __restrict__ frames, int out_frames)
{
    __shared__ unsigned char s_bits[4][368];
    __shared__ uint16_t s_hist[4][244];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long g = static_cast<long long>(blockIdx.x) * 4 + w;
    const int c = static_cast<int>(g / max_frames), f = static_cast<int>(g % max_frames);
    if (c >= C) return;
    const int n = min(max(counts[c], 0), max_frames);
    if (f >= n) return;
    const unsigned char* rec = records + (static_cast<long long>(c) * max_frames + f) * rec_bytes;
    const uint32_t type = ld_u32(rec);
    FrameOut* o = frames + static_cast<long long>(c) * out_frames + f;
    if (lane == 0) o->type = type;
    if (type != M17_LSF && type != M17_STREAM) return;
    const bool lsf = type == M17_LSF;
    const unsigned char* p = rec + 8;
    unsigned char* bits = s_bits[w];
    // derandomise + deinterleave: deinterleaved bit i = received bit (45 i + 92 i^2) mod 368
    for (int i = lane; i < 368; i += 32) {
        const int s = qpp(i);
        bits[i] = static_cast<unsigned char>(((p[s >> 3] ^ kRandomizer[s >> 3]) >> (7 - (s & 7))) & 1u);
    }
    __syncwarp();
    if (!lsf) {
        // LICH: 4 x Golay(24,12), 24 bits MSB first each, on lanes 0-3
        uint32_t d = 0;
        if (lane < 4) {
            uint32_t cw = 0;
            for (int t = 0; t < 24; t++) cw = (cw << 1) | bits[24 * lane + t];
            d = golay24_decode(cw);
        }
        const uint32_t d0 = __shfl_sync(0xffffffffu, d, 0), d1 = __shfl_sync(0xffffffffu, d, 1);
        const uint32_t d2 = __shfl_sync(0xffffffffu, d, 2), d3 = __shfl_sync(0xffffffffu, d, 3);
        if (lane == 0) {
            const bool ok = d0 != 0xFFFFu && d1 != 0xFFFFu && d2 != 0xFFFFu && d3 != 0xFFFFu;
            o->lich_ok = ok;
            o->seg[0] = ok ? d0 >> 4 : 0;
            o->seg[1] = ok ? ((d0 & 0xF) << 4) | (d1 >> 8) : 0;
            o->seg[2] = ok ? d1 & 0xFF : 0;
            o->seg[3] = ok ? d2 >> 4 : 0;
            o->seg[4] = ok ? ((d2 & 0xF) << 4) | (d3 >> 8) : 0;
            o->seg[5] = ok ? (d3 & 0xFF) >> 5 : 0;
        }
    }
    // M17Viterbi::decodePunctured: hard symbols (0 / 2, a punctured one costs 1 against both branches), metrics from 0, no
    // normalisation (at most 244 steps x 4 stays far below 2^16), the upper predecessor wins a tie
    const int first = lsf ? 0 : 96, n_in = lsf ? 368 : 272, n_out = lsf ? 30 : 18, P = lsf ? 61 : 12;
    const int st = lane & 15, i = st >> 1;
    const int c0 = i >= 4 ? 2 : 0, c1 = ((i ^ (i >> 1)) & 1) * 2;
    uint32_t metric = 0;
    int pos = 0, pi = 0, bp = 0;
    while (bp < n_in) {
        int sym[2];
        for (int k = 0; k < 2; k++) {
            if (p_keep(lsf, pi)) sym[k] = bits[first + bp++] ? 2 : 0;
            else sym[k] = 1;
            if (++pi >= P) pi = 0;
        }
        const uint32_t m = abs(c0 - sym[0]) + abs(c1 - sym[1]);
        const uint32_t pa = __shfl_sync(0xffffffffu, metric, i), pb = __shfl_sync(0xffffffffu, metric, i + 8);
        const uint32_t ma = pa + ((st & 1) ? 4 - m : m), mb = pb + ((st & 1) ? m : 4 - m);
        const bool dec = ma >= mb;
        metric = dec ? mb : ma;
        const unsigned b = __ballot_sync(0xffffffffu, dec);
        if (lane == 0) s_hist[w][pos] = static_cast<uint16_t>(b & 0xFFFFu);
        pos++;
    }
    __syncwarp();
    // chainback from state 0 over the last 8 n_out steps, exactly as the reference walks it: decision bit (state >> 4) of the step,
    // state = (state >> 1) | bit << 7 on 8 bits.  The decoded bits go back into s_bits (free by now), then a byte per lane.
    if (lane == 0) {
        uint32_t state = 0;
        for (int b = 8 * n_out - 1; b >= 0; b--) {
            pos--;
            const uint32_t bit = (s_hist[w][pos] >> (state >> 4)) & 1u;
            state = ((state >> 1) | (bit << 7)) & 0xFFu;
            bits[b] = static_cast<unsigned char>(bit);
        }
    }
    __syncwarp();
    if (lane < n_out) {
        uint32_t v = 0;
        for (int k = 0; k < 8; k++) v = (v << 1) | bits[8 * lane + k];
        o->data[lane] = static_cast<unsigned char>(v);
    }
}

__device__ __forceinline__ void lsf_clear(unsigned char* l)
{
    for (int i = 0; i < 30; i++) l[i] = i < 6 ? 0xFF : 0;
}

__global__ void __launch_bounds__(128)
m17_state_kernel(int C, int max_frames, const int* __restrict__ counts, const FrameOut* __restrict__ frames, int out_frames,
                 M17RxState* __restrict__ states, unsigned char* __restrict__ out, int* __restrict__ out_counts)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    const int n = min(max(counts[c], 0), max_frames);
    M17RxState s = states[c];
    for (int f = 0; f < n; f++) {
        const FrameOut& fr = frames[static_cast<long long>(c) * out_frames + f];
        const uint32_t type = fr.type;
        if (type == M17_LSF) {
            // decodeLSF overwrites the LSF whether its CRC holds or not
            for (int k = 0; k < 30; k++) s.lsf[k] = fr.data[k];
            s.valid = lsf_valid(s.lsf);
        } else if (type == M17_STREAM) {
            if (fr.lich_ok) {
                const int num = fr.seg[5];
                // segment numbers 6 and 7 (only a miscorrected LICH has them) land past the partial LSF, in the stream frame the same
                // call then overwrites: their only lasting trace is the map bit, which keeps the map from reaching 0x3F until a reset
                if (num < 6)
                    for (int k = 0; k < 5; k++) s.part[5 * num + k] = fr.seg[k];
                s.map |= static_cast<unsigned char>(1u << num);
                if (s.map == 0x3F) {
                    if (lsf_valid(s.part)) { for (int k = 0; k < 30; k++) s.lsf[k] = s.part[k]; s.valid = 1; }
                    s.map = 0;
                    lsf_clear(s.part);
                }
            }
            for (int k = 0; k < 18; k++) s.sf[k] = fr.data[k];
        }
        uint32_t wds[kRxRecord / 4];
        unsigned char* b = reinterpret_cast<unsigned char*>(wds);
        wds[0] = type;
        for (int k = 0; k < 30; k++) b[4 + k] = s.lsf[k];
        b[34] = s.valid; b[35] = 0;
        for (int k = 0; k < 18; k++) b[36 + k] = s.sf[k];
        b[54] = 0; b[55] = 0;
        uint32_t* dst = reinterpret_cast<uint32_t*>(out + (static_cast<long long>(c) * out_frames + f) * kRxRecord);
        for (int k = 0; k < kRxRecord / 4; k++) dst[k] = wds[k];
        // gr_modem: an EOT record reports the current LSF, then resets the decoder if that LSF is valid
        if (type == M17_EOT && s.valid) {
            lsf_clear(s.lsf); lsf_clear(s.part);
            for (int k = 0; k < 18; k++) s.sf[k] = 0;
            s.map = 0; s.valid = 0;
        }
    }
    states[c] = s;
    out_counts[c] = n;
}

// M17FrameDecoder::reset (the decoder's initial state too): channel < 0 = every channel
__global__ void m17_rx_reset_kernel(int C, int channel, M17RxState* __restrict__ states)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C || (channel >= 0 && c != channel)) return;
    M17RxState s;
    lsf_clear(s.lsf); lsf_clear(s.part);
    for (int k = 0; k < 18; k++) s.sf[k] = 0;
    s.map = 0; s.valid = 0;
    states[c] = s;
}

// ================================================================================================ transmit
struct M17TxLsf { unsigned char lsf[30], lich[6][12]; };
struct M17TxState { uint32_t fn, lich; };
struct M17TxStep { int offset; uint16_t fn; unsigned char lich, op; };

__host__ __device__ inline int op_bytes(int op) { return op == OP_START ? 96 : op == OP_STREAM ? 48 : op == OP_LAST ? 64 : 0; }

// per channel, in op order: output offsets, frame numbers ((fn + 1) & 0x7FF, as M17Transmitter masks it) and LICH indices (mod 6);
// a start resets both counters.  An op value outside 0-3 is "none".
__global__ void m17_tx_scan_kernel(int C, int K, const unsigned char* __restrict__ ops, long long ops_stride, M17TxState* __restrict__ states,
                                   M17TxStep* __restrict__ steps, int max_steps, int* __restrict__ counts)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    M17TxState s = states[c];
    int off = 0;
    for (int k = 0; k < K; k++) {
        int op = ops[static_cast<long long>(c) * ops_stride + k];
        if (op > OP_LAST) op = OP_NONE;
        if (op == OP_START) { s.fn = 0; s.lich = 0; }
        M17TxStep st;
        st.offset = off; st.fn = static_cast<uint16_t>(s.fn); st.lich = static_cast<unsigned char>(s.lich); st.op = static_cast<unsigned char>(op);
        steps[static_cast<long long>(c) * max_steps + k] = st;
        if (op == OP_STREAM || op == OP_LAST) { s.fn = (s.fn + 1) & 0x07FFu; s.lich = (s.lich + 1) % 6u; }
        off += op_bytes(op);
    }
    states[c] = s;
    counts[c] = off;
}

// one warp per (channel, op): K = 5 convolutional code (G1 = 0x19, G2 = 0x17, zero start, 4 flush bits), puncture, LICH in front of a
// stream frame, interleave, randomise, sync word in front
__global__ void __launch_bounds__(128)
m17_tx_encode_kernel(int C, int K, const unsigned char* __restrict__ payloads, long long pl_stride, const M17TxLsf* __restrict__ lsfs,
                     const M17TxStep* __restrict__ steps, int max_steps, unsigned char* __restrict__ out, long long out_stride)
{
    __shared__ unsigned char s_bits[4][368];
    __shared__ unsigned char s_data[4][32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long g = static_cast<long long>(blockIdx.x) * 4 + w;
    const int c = static_cast<int>(g / K), k = static_cast<int>(g % K);
    if (c >= C) return;
    const M17TxStep st = steps[static_cast<long long>(c) * max_steps + k];
    if (st.op == OP_NONE) return;
    unsigned char* o = out + static_cast<long long>(c) * out_stride + st.offset;
    const M17TxLsf& L = lsfs[c];
    const bool lsf = st.op == OP_START;
    unsigned char* data = s_data[w];
    if (lsf) {
        for (int i = lane; i < 48; i += 32) o[i] = 0x77;
        o += 48;
        if (lane < 30) data[lane] = L.lsf[lane];
    } else {
        const uint32_t fnw = (st.fn & 0x7FFFu) | (st.op == OP_LAST ? 0x8000u : 0u);
        const unsigned char* pl = payloads + static_cast<long long>(c) * pl_stride + 16LL * k;
        if (lane < 18) data[lane] = lane == 0 ? static_cast<unsigned char>(fnw >> 8) : lane == 1 ? static_cast<unsigned char>(fnw & 0xFF) : pl[lane - 2];
    }
    __syncwarp();
    const int nbits = (lsf ? 30 : 18) * 8, first = lsf ? 0 : 96;
    unsigned char* bits = s_bits[w];
    for (int j = lane; j < 368; j += 32) {
        uint32_t v;
        if (j < first) v = (L.lich[st.lich][j >> 3] >> (7 - (j & 7))) & 1u;
        else {
            const int e = p_source(lsf, j - first), t = e >> 1;
            uint32_t x = 0;                  // bit d = input bit t - d (0 outside the frame: zero start, flush)
            for (int d = 0; d < 5; d++) {
                const int q = t - d;
                const uint32_t b = (q >= 0 && q < nbits) ? (data[q >> 3] >> (7 - (q & 7))) & 1u : 0u;
                x |= b << d;
            }
            v = (e & 1) ? __popc(x & 0x17u) & 1u : __popc(x & 0x19u) & 1u;
        }
        bits[qpp(j)] = static_cast<unsigned char>(v);
    }
    __syncwarp();
    if (lane < 2) o[lane] = lsf ? (lane ? 0xF7 : 0x55) : (lane ? 0x5D : 0xFF);
    for (int j = lane; j < 46; j += 32) {
        uint32_t v = 0;
        for (int b = 0; b < 8; b++) v = (v << 1) | bits[8 * j + b];
        o[2 + j] = static_cast<unsigned char>(v ^ kRandomizer[j]);
    }
    if (st.op == OP_LAST && lane < 16) o[48 + lane] = (lane & 1) ? 0x5D : 0x55;     // 8 x the EOT word's 0x555D
}

}  // namespace

struct qrl_m17_rx : QrlHandleBase {
    int C = 0, max_frames = 0;
    M17RxState* d_state = nullptr;
    FrameOut* d_frames = nullptr;
    unsigned char* d_out = nullptr;
    int* d_counts = nullptr;
    unsigned char* d_stage = nullptr;     // host input, staged (grown on demand; freed by destroy)
    size_t stage_bytes = 0;
    int* d_stage_counts = nullptr;
};

struct qrl_m17_tx : QrlHandleBase {
    int C = 0, max_steps = 0;
    long out_stride = 0;
    M17TxLsf* d_lsf = nullptr;
    M17TxState* d_state = nullptr;
    M17TxStep* d_steps = nullptr;
    unsigned char *d_out = nullptr, *d_ops = nullptr, *d_pl = nullptr;
    int* d_counts = nullptr;
};

extern "C" {

// ---------------------------------------------------------------------------------------------- receive
int qrl_m17_rx_destroy(qrl_m17_rx* h)
{
    if (!h) return QRL_EINVAL;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->d_stage) cudaFree(h->d_stage);
    return handle_close(h);
}

int qrl_m17_rx_create(int n_channels, int max_frames, int device, qrl_m17_rx** out)
{
    if (!out || n_channels < 1 || max_frames < 1) { set_err(nullptr, "qrl_m17_rx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_m17_rx_create", device)) return rc;
    qrl_m17_rx* h = new qrl_m17_rx();
    h->C = n_channels; h->max_frames = max_frames;
    auto fail = [&](int rc) { return create_failed(h, qrl_m17_rx_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels), F = C * max_frames;
    if ((rc = dev_alloc(h, &h->d_state, C)) || (rc = dev_alloc(h, &h->d_frames, F)) || (rc = dev_alloc(h, &h->d_out, F * kRxRecord)) ||
        (rc = dev_alloc(h, &h->d_counts, C)) || (rc = dev_alloc(h, &h->d_stage_counts, C)))
        return fail(rc);
    m17_rx_reset_kernel<<<(n_channels + 127) / 128, 128, 0, h->stream>>>(n_channels, -1, h->d_state);
    h->launches++;
    if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create: state init failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_m17_rx_set_stream(qrl_m17_rx* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

int qrl_m17_rx_work(qrl_m17_rx* h, const unsigned char* records, const int* frame_counts, int record_bytes, int max_frames, int on_device)
{
    if (!h || !records || !frame_counts) { set_err(nullptr, "qrl_m17_rx_work: bad argument"); return QRL_EINVAL; }
    if (record_bytes < 8 + 46 || max_frames < 1 || max_frames > h->max_frames) {
        set_err(h, "qrl_m17_rx_work: record_bytes must be >= 54 and max_frames between 1 and the handle's max_frames");
        return QRL_ERANGE;
    }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char* d_rec = records;
    const int* d_cnt = frame_counts;
    if (!on_device) {
        for (int c = 0; c < h->C; c++)
            if (frame_counts[c] < 0 || frame_counts[c] > max_frames) { set_err(h, "qrl_m17_rx_work: bad frame count"); return QRL_ERANGE; }
        const size_t bytes = static_cast<size_t>(h->C) * max_frames * record_bytes;
        if (bytes > h->stage_bytes) {
            QRL_CK(cudaStreamSynchronize(h->stream));
            if (h->d_stage) { cudaFree(h->d_stage); h->d_stage = nullptr; h->stage_bytes = 0; }
            QRL_CK(cudaMalloc(&h->d_stage, bytes));
            h->stage_bytes = bytes;
        }
        QRL_CK(cudaMemcpyAsync(h->d_stage, records, bytes, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage_counts, frame_counts, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
        d_rec = h->d_stage; d_cnt = h->d_stage_counts;
    }
    const long long warps = static_cast<long long>(h->C) * max_frames;
    m17_frame_kernel<<<static_cast<unsigned>((warps + 3) / 4), 128, 0, h->stream>>>(h->C, max_frames, d_rec, record_bytes, d_cnt, h->d_frames,
                                                                                 h->max_frames);
    h->launches++;
    QRL_CK(cudaGetLastError());
    m17_state_kernel<<<(h->C + 127) / 128, 128, 0, h->stream>>>(h->C, max_frames, d_cnt, h->d_frames, h->max_frames, h->d_state, h->d_out,
                                                                 h->d_counts);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_m17_rx_reset(qrl_m17_rx* h, int channel)
{
    if (!h) return QRL_EINVAL;
    if (channel < 0 || channel >= h->C) { set_err(h, "qrl_m17_rx_reset: channel out of range"); return QRL_ERANGE; }
    QRL_CK(cudaSetDevice(h->device));
    m17_rx_reset_kernel<<<(h->C + 127) / 128, 128, 0, h->stream>>>(h->C, channel, h->d_state);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_m17_rx_read(qrl_m17_rx* h, unsigned char* records_host, int* counts_host)
{
    if (!h || !counts_host) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (records_host)
        QRL_CK(cudaMemcpyAsync(records_host, h->d_out, static_cast<size_t>(h->C) * h->max_frames * kRxRecord, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_m17_rx_out_device(qrl_m17_rx* h, void** records, int** counts)
{
    if (!h) return QRL_EINVAL;
    if (records) *records = h->d_out;
    if (counts) *counts = h->d_counts;
    return QRL_OK;
}

int qrl_m17_rx_sync(qrl_m17_rx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_m17_rx_launch_count(qrl_m17_rx* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------- transmit
int qrl_m17_tx_destroy(qrl_m17_tx* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_m17_tx_create(int n_channels, int max_steps, int device, qrl_m17_tx** out)
{
    if (!out || n_channels < 1 || max_steps < 1) { set_err(nullptr, "qrl_m17_tx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_m17_tx_create", device)) return rc;
    qrl_m17_tx* h = new qrl_m17_tx();
    h->C = n_channels; h->max_steps = max_steps; h->out_stride = static_cast<long>(max_steps) * kStepMax;
    auto fail = [&](int rc) { return create_failed(h, qrl_m17_tx_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels), S = C * max_steps;
    if ((rc = dev_alloc(h, &h->d_lsf, C)) || (rc = dev_alloc(h, &h->d_state, C)) || (rc = dev_alloc(h, &h->d_steps, S)) ||
        (rc = dev_alloc(h, &h->d_out, C * h->out_stride)) || (rc = dev_alloc(h, &h->d_ops, S)) || (rc = dev_alloc(h, &h->d_pl, S * 16)) ||
        (rc = dev_alloc(h, &h->d_counts, C)))
        return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_m17_tx_set_stream(qrl_m17_tx* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

// M17LinkSetupFrame::updateCrc and generateLichSegment(0 .. 5) for one channel (host: once per transmission, not per frame)
int qrl_m17_tx_set_lsf(qrl_m17_tx* h, int channel, const unsigned char* lsf28)
{
    if (!h || !lsf28) { set_err(nullptr, "qrl_m17_tx_set_lsf: bad argument"); return QRL_EINVAL; }
    if (channel < 0 || channel >= h->C) { set_err(h, "qrl_m17_tx_set_lsf: channel out of range"); return QRL_ERANGE; }
    QRL_CK(cudaSetDevice(h->device));
    M17TxLsf L;
    for (int i = 0; i < 28; i++) L.lsf[i] = lsf28[i];
    const uint16_t crc = m17_crc(L.lsf, 28);
    L.lsf[28] = static_cast<unsigned char>(crc >> 8); L.lsf[29] = static_cast<unsigned char>(crc & 0xFF);
    for (int n = 0; n < 6; n++) {
        const unsigned char* ch = L.lsf + 5 * n;
        const uint32_t blk[4] = { static_cast<uint32_t>(ch[0] << 4 | ch[1] >> 4), static_cast<uint32_t>((ch[1] & 0xF) << 8 | ch[2]),
                                  static_cast<uint32_t>(ch[3] << 4 | ch[4] >> 4), static_cast<uint32_t>((ch[4] & 0xF) << 8 | (n << 5)) };
        for (int b = 0; b < 4; b++) {
            const uint32_t cw = (blk[b] << 12) | golay_check(blk[b]);
            L.lich[n][3 * b] = static_cast<unsigned char>(cw >> 16);
            L.lich[n][3 * b + 1] = static_cast<unsigned char>(cw >> 8);
            L.lich[n][3 * b + 2] = static_cast<unsigned char>(cw);
        }
    }
    QRL_CK(cudaMemcpyAsync(h->d_lsf + channel, &L, sizeof(L), cudaMemcpyHostToDevice, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_m17_tx_work(qrl_m17_tx* h, const unsigned char* ops, const unsigned char* payloads, int K, int on_device)
{
    if (!h || !ops || !payloads) { set_err(nullptr, "qrl_m17_tx_work: bad argument"); return QRL_EINVAL; }
    if (K < 0 || K > h->max_steps) { set_err(h, "qrl_m17_tx_work: K must be between 0 and max_steps"); return QRL_ERANGE; }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char *d_ops = ops, *d_pl = payloads;
    if (!on_device && K > 0) {
        QRL_CK(cudaMemcpyAsync(h->d_ops, ops, static_cast<size_t>(h->C) * K, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_pl, payloads, static_cast<size_t>(h->C) * K * 16, cudaMemcpyHostToDevice, h->stream));
        d_ops = h->d_ops; d_pl = h->d_pl;
    }
    m17_tx_scan_kernel<<<(h->C + 127) / 128, 128, 0, h->stream>>>(h->C, K, d_ops, K, h->d_state, h->d_steps, h->max_steps, h->d_counts);
    h->launches++;
    QRL_CK(cudaGetLastError());
    if (K > 0) {
        const long long warps = static_cast<long long>(h->C) * K;
        m17_tx_encode_kernel<<<static_cast<unsigned>((warps + 3) / 4), 128, 0, h->stream>>>(h->C, K, d_pl, 16LL * K, h->d_lsf, h->d_steps,
                                                                                         h->max_steps, h->d_out, h->out_stride);
        h->launches++;
        QRL_CK(cudaGetLastError());
    }
    return QRL_OK;
}

int qrl_m17_tx_read(qrl_m17_tx* h, unsigned char* out_host, long cap, int* counts_host)
{
    if (!h || !counts_host) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (out_host && cap > 0)
        QRL_CK(cudaMemcpy2DAsync(out_host, static_cast<size_t>(cap), h->d_out, static_cast<size_t>(h->out_stride),
                                 static_cast<size_t>(cap < h->out_stride ? cap : h->out_stride), h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_m17_tx_out_device(qrl_m17_tx* h, void** out, long* stride, int** counts)
{
    if (!h) return QRL_EINVAL;
    if (out) *out = h->d_out;
    if (stride) *stride = h->out_stride;
    if (counts) *counts = h->d_counts;
    return QRL_OK;
}

int qrl_m17_tx_sync(qrl_m17_tx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_m17_tx_launch_count(qrl_m17_tx* h) { return h ? h->launches : 0; }

}  // extern "C"
