// qrl_deframer.cu -- layer-1 deframer on the device (SURVEY.md section 8f row 2), part of libqrl_b200.so.
//
// Replaces the bit-serial CPU loop gr_modem::synchronize + findSync + packBytes
// (/root/reference/src/gr_modem.cpp:1119-1282, 980-994; sync words /root/reference/src/layer1framing.h:8-24) for a batch
// of channels: the decoded bits (one per byte, port 2 / 3 of the demodulators) never leave the GPU, only packed frames
// { type, length, payload } do.  Semantics are the reference's, bit for bit (oracle: qo_deframer_work):
//   * a shift register searches for a sync word; class 1 ("1K" modes) 8-bit 0xB5; class 2 (narrow modes) 16-bit 0xED89
//     first, then the 24-bit text / proto / video / callsign / end words; class 3 (QPSK250K, QPSKVideo, 4FSK100K) the
//     24-bit IP / video / end words; class 4 (M17) the 16-bit link-setup / stream words, then the 32-bit end-of-transmission word;
//   * after a sync the next bit_len bits are collected and packed MSB first; classes 2, 3: voice frames take
//     bit_buf_len bits into rx_frame_length + 1 bytes, all others bit_buf_len - 8 bits into rx_frame_length bytes;
//   * then the shift register is cleared (a sync word cannot straddle the end of a frame);
//   * _modem_sync: +8 (below 32) on a sync, -1 (above 0) per searched bit without one.
// One warp per channel: 32 bit positions are tested at once (the lane's shift register is rebuilt from a ballot of
// the 32 bits and the carried register), frames are packed a byte per lane.  State carries across calls.
#include "../../include/qrl_b200.h"
#include "qrl_handle.hpp"

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

namespace {

enum : uint32_t { FT_VOICE = 0xED89, FT_VOICE1 = 0xB5, FT_TEXT = 0x89EDAA, FT_IP = 0xDE98AA, FT_VIDEO = 0x98DEAA,
                  FT_CALLSIGN = 0x8CC8DD, FT_PROTO = 0xED77AA, FT_END = 0x4C8A2B,
                  FT_M17_STREAM = 0xFF5D, FT_M17_LSF = 0x55F7, FT_M17_EOT = 0x555D555D };     // layer1framing.h:21-23

struct DeframerState {
    uint32_t shift_reg;
    int sync_found;
    uint32_t cur_type;
    int bit_idx;
    int modem_sync;
};

__device__ __forceinline__ uint32_t match_sync(int sync_class, uint32_t sr)
{
    if (sync_class == 1) return (sr & 0xFFu) == FT_VOICE1 ? FT_VOICE1 : 0u;
    if (sync_class == 4) {          // ModemTypeM17 (gr_modem.cpp:1187-1207)
        const uint32_t t16 = sr & 0xFFFFu;
        if (t16 == FT_M17_LSF || t16 == FT_M17_STREAM) return t16;
        return sr == FT_M17_EOT ? FT_M17_EOT : 0u;
    }
    const uint32_t t24 = sr & 0xFFFFFFu;
    if (sync_class == 2) {
        if ((sr & 0xFFFFu) == FT_VOICE) return FT_VOICE;
        if (t24 == FT_TEXT || t24 == FT_PROTO || t24 == FT_VIDEO || t24 == FT_CALLSIGN || t24 == FT_END) return t24;
        return 0u;
    }
    if (t24 == FT_IP || t24 == FT_VIDEO || t24 == FT_END) return t24;
    return 0u;
}

__global__ void __launch_bounds__(128)
deframer_kernel(int C, int sync_class, int bit_buf_len, int rx_frame_length,
                const unsigned char* __restrict__ bits, long long bits_stride, const int* __restrict__ counts, int fixed_count,
                const unsigned char* __restrict__ bits2, const int* __restrict__ counts2,      // optional second stream: the longer one is taken
                DeframerState* __restrict__ states, unsigned char* __restrict__ bit_buf /*[C][bit_buf_len]*/,
                unsigned char* __restrict__ records, int rec_bytes, int max_frames, int* __restrict__ frame_counts,
                int* __restrict__ dropped /* [C], cumulative: frames found beyond max_frames */)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= C) return;
    const int c = warp;
    const unsigned char* b = bits + static_cast<long long>(c) * bits_stride;
    int n = counts ? counts[c] : fixed_count;
    if (bits2) {
        // gr_modem::demodulate (gr_modem.cpp:1066-1085): of the two deframed streams of a dual-decoder mode the longer one
        // goes to synchronize(), the first on a tie
        const int n2 = counts2[c];
        if (n2 > n) { n = n2; b = bits2 + static_cast<long long>(c) * bits_stride; }
    }
    n = n < 0 ? 0 : (static_cast<long long>(n) > bits_stride ? static_cast<int>(bits_stride) : n);     // a count can never exceed the row
    DeframerState st = states[c];
    __syncwarp();         // all lanes hold the state before lane 0 may store it back (n == 0: no collective in between)
    unsigned char* bb = bit_buf + static_cast<long long>(c) * bit_buf_len;
    unsigned char* rec = records + static_cast<long long>(c) * max_frames * rec_bytes;
    int found = 0, n_dropped = 0;
    int pos = 0;
    while (pos < n) {
        if (!st.sync_found) {
            const int v = min(32, n - pos);
            const unsigned bit = (lane < v) ? (b[pos + lane] & 1u) : 0u;
            const uint32_t wr = __brev(__ballot_sync(0xffffffffu, bit));      // bit 31 = the bit at pos
            // my shift register after consuming bits pos .. pos + lane
            const uint32_t sr = (lane == 31 ? 0u : (st.shift_reg << (lane + 1))) | (wr >> (31 - lane));
            const uint32_t ty = (lane < v) ? match_sync(sync_class, sr) : 0u;
            const unsigned hit = __ballot_sync(0xffffffffu, ty != 0u);
            if (hit == 0u) {
                st.shift_reg = __shfl_sync(0xffffffffu, sr, v - 1);
                st.modem_sync = max(0, st.modem_sync - v);
                pos += v;
            } else {
                const int f = __ffs(hit) - 1;
                st.cur_type = __shfl_sync(0xffffffffu, ty, f);
                st.shift_reg = __shfl_sync(0xffffffffu, sr, f);
                st.modem_sync = max(0, st.modem_sync - f);
                if (st.modem_sync < 32) st.modem_sync += 8;
                st.sync_found = 1; st.bit_idx = 0;
                pos += f + 1;
            }
        } else {
            int frame_length = rx_frame_length, bit_len = bit_buf_len;
            if (sync_class != 1 && sync_class != 4) {
                if (st.cur_type == FT_VOICE) frame_length++;
                else bit_len = bit_buf_len - 8;
            }
            const int take = min(bit_len - st.bit_idx, n - pos);
            const bool complete = st.bit_idx + take >= bit_len;
            if (complete && found < max_frames) {
                unsigned char* r = rec + static_cast<long long>(found) * rec_bytes;
                for (int i = lane; i < rec_bytes; i += 32) r[i] = 0;
                __syncwarp();
                if (lane == 0) {
                    reinterpret_cast<uint32_t*>(r)[0] = st.cur_type;
                    reinterpret_cast<uint32_t*>(r)[1] = static_cast<uint32_t>(frame_length);
                }
                // byte j of the frame = bits 8j .. 8j+7: the first bit_idx bits are staged in bb, the rest come from b
                for (int j = lane; j * 8 < bit_len && 8 + j < rec_bytes; j += 32) {
                    int t = 0;
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        const int q = j * 8 + k;
                        const unsigned bit = q < st.bit_idx ? bb[q] : b[pos + q - st.bit_idx];
                        t = (t << 1) | (bit & 1u);
                    }
                    r[8 + j] = static_cast<unsigned char>(t);
                }
            } else if (!complete) {
                for (int i = lane; i < take; i += 32) bb[st.bit_idx + i] = b[pos + i] & 1u;
            }
            __syncwarp();
            pos += take;
            if (complete) {
                if (found < max_frames) found++;
                else n_dropped++;
                st.sync_found = 0; st.shift_reg = 0; st.bit_idx = 0;
            } else st.bit_idx += take;
        }
    }
    if (lane == 0) { states[c] = st; frame_counts[c] = found; if (n_dropped) dropped[c] += n_dropped; }
}

// ----------------------------------------------------------------------------------------------------------------
// gr_deframer_bb (/root/reference/src/gr/gr_deframer_bb.cpp:83-185; behind ports 2 / 3 of the dual-decoder modes, gr_demod_base.cpp:
// _deframer1/2 type 1, _deframer_700_1/2 type 2, _deframer_10k_1/2 type 3) for a batch of channels, quirks included (oracle:
// qo_dfbb_work, pinned to the reference source in oracle/_ref): bit stream in, {matched sync word MSB first, the next bit_buf_len
// bits verbatim} stream out.  One warp per channel, same 32-positions-at-once search as above.
// ----------------------------------------------------------------------------------------------------------------
struct DfbbState { uint32_t shift_reg; int sync_found, idx; };

__device__ __forceinline__ uint32_t dfbb_match(int type, uint32_t sr)
{
    const uint32_t t = type != 2 ? (sr & 0xFFFFu) : (sr & 0xFFu);
    if (type == 2 && t == 0xB5u) return t;
    if (t == 0x89EDu || t == 0xED89u || t == 0x98DEu || t == 0xED77u || t == 0x8CC8u) return t;
    return (sr & 0xFFFFFFu) == 0x4C8A2Bu ? 0x4C8A2Bu : 0u;
}

__global__ void __launch_bounds__(128)
dfbb_kernel(int C, int type, int len, const unsigned char* __restrict__ bits, long long bits_stride, const int* __restrict__ counts,
            DfbbState* __restrict__ states, unsigned char* __restrict__ out, long long out_stride, int* __restrict__ out_counts)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= C) return;
    const int c = warp;
    const unsigned char* b = bits + static_cast<long long>(c) * bits_stride;
    int n = counts[c];
    n = n < 0 ? 0 : (static_cast<long long>(n) > bits_stride ? static_cast<int>(bits_stride) : n);
    DfbbState st = states[c];
    __syncwarp();
    unsigned char* o = out + static_cast<long long>(c) * out_stride;
    long long no = 0;
    int pos = 0;
    while (pos < n) {
        if (!st.sync_found) {
            const int v = min(32, n - pos);
            const unsigned bit = (lane < v) ? (b[pos + lane] & 1u) : 0u;
            const uint32_t wr = __brev(__ballot_sync(0xffffffffu, bit));
            const uint32_t sr = (lane == 31 ? 0u : (st.shift_reg << (lane + 1))) | (wr >> (31 - lane));
            const uint32_t ty = (lane < v) ? dfbb_match(type, sr) : 0u;
            const unsigned hit = __ballot_sync(0xffffffffu, ty != 0u);
            if (hit == 0u) {
                st.shift_reg = __shfl_sync(0xffffffffu, sr, v - 1);
                pos += v;
            } else {
                const int f = __ffs(hit) - 1;
                const uint32_t ft = __shfl_sync(0xffffffffu, ty, f);
                st.shift_reg = __shfl_sync(0xffffffffu, sr, f);
                const int nb = (type == 1 || type == 3) ? (ft != 0x4C8A2Bu ? 16 : 24) : 8;
                if (lane < nb && no + lane < out_stride) o[no + lane] = static_cast<unsigned char>((ft >> (nb - 1 - lane)) & 1u);
                no += nb;
                st.sync_found = 1; st.idx = 0;
                pos += f + 1;
            }
        } else {
            const int take = min(len - st.idx, n - pos);
            for (int i = lane; i < take; i += 32) if (no + i < out_stride) o[no + i] = b[pos + i] & 1u;
            no += take; pos += take; st.idx += take;
            if (st.idx >= len) { st.sync_found = 0; st.shift_reg = 0; st.idx = 0; }
        }
    }
    if (lane == 0) { states[c] = st; out_counts[c] = static_cast<int>(no < out_stride ? no : out_stride); }
}

}  // namespace

// gr_modem::frame (/root/reference/src/gr_modem.cpp:904-961) for a batch of channels: sync word (+ 10 x 0xAA in front of an IP frame in
// burst mode) + payload -> the byte vector gr_byte_source hands to the modulator.  One CTA per channel.
__global__ void __launch_bounds__(128)
frame_build_kernel(int C, const unsigned char* __restrict__ payload, long long payload_stride, const int* __restrict__ payload_len,
                   const unsigned* __restrict__ frame_type, int one_k_mode, int burst_ip,
                   unsigned char* __restrict__ out, long long out_stride, int* __restrict__ out_len)
{
    const int c = blockIdx.x;
    if (c >= C) return;
    const unsigned ft = frame_type[c];
    const int n = payload_len[c];
    unsigned char hdr[13]; int nh = 0;
    if (ft == FT_IP && burst_ip) for (int i = 0; i < 10; i++) hdr[nh++] = 0xAA;
    if (ft == FT_VOICE) {
        if (one_k_mode) hdr[nh++] = static_cast<unsigned char>(FT_VOICE1 & 0xFF);
        else { hdr[nh++] = static_cast<unsigned char>((FT_VOICE >> 8) & 0xFF); hdr[nh++] = static_cast<unsigned char>(FT_VOICE & 0xFF); hdr[nh++] = 0xAA; }
    } else if (ft == FT_TEXT || ft == FT_VIDEO || ft == FT_IP || ft == FT_PROTO) {
        hdr[nh++] = static_cast<unsigned char>((ft >> 16) & 0xFF); hdr[nh++] = static_cast<unsigned char>((ft >> 8) & 0xFF); hdr[nh++] = static_cast<unsigned char>(ft & 0xFF);
    }
    unsigned char* o = out + static_cast<long long>(c) * out_stride;
    const unsigned char* p = payload + static_cast<long long>(c) * payload_stride;
    for (int i = threadIdx.x; i < nh + n; i += blockDim.x) if (i < out_stride) o[i] = i < nh ? hdr[i] : p[i - nh];
    if (threadIdx.x == 0) out_len[c] = static_cast<int>(nh + n < out_stride ? nh + n : out_stride);
}

struct qrl_deframer : QrlHandleBase {
    int sync_class = 0, bit_buf_len = 0, rx_frame_length = 0, C = 0, max_frames = 0, rec_bytes = 0;
    long max_bits = 0;
    DeframerState* d_state = nullptr;
    unsigned char *d_bit_buf = nullptr, *d_records = nullptr, *d_stage = nullptr;
    unsigned char* d_stage2 = nullptr;
    int *d_counts = nullptr, *d_stage_counts = nullptr, *d_stage_counts2 = nullptr, *d_dropped = nullptr;
};

struct qrl_dfbb : QrlHandleBase {
    int type = 0, len = 0, C = 0;
    long max_bits = 0, out_stride = 0;
    DfbbState* d_state = nullptr;
    unsigned char *d_out = nullptr, *d_stage = nullptr;
    int *d_counts = nullptr, *d_stage_counts = nullptr;
};

extern "C" {

int qrl_deframer_destroy(qrl_deframer* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_deframer_create(int sync_class, int bit_buf_len, int rx_frame_length, int n_channels, long max_bits, int max_frames,
                        int device, qrl_deframer** out)
{
    if (!out || sync_class < 1 || sync_class > 4 || bit_buf_len < 16 || (bit_buf_len & 7) || rx_frame_length < 1 || n_channels < 1 ||
        max_bits < 1 || max_frames < 1) {
        set_err(nullptr, "qrl_deframer_create: bad argument");
        return QRL_EINVAL;
    }
    *out = nullptr;
    if (int rc = check_device("qrl_deframer_create", device)) return rc;
    qrl_deframer* h = new qrl_deframer();
    h->sync_class = sync_class; h->bit_buf_len = bit_buf_len; h->rx_frame_length = rx_frame_length; h->C = n_channels;
    h->max_bits = max_bits; h->max_frames = max_frames;
    h->rec_bytes = (8 + bit_buf_len / 8 + 7) & ~7;
    auto fail = [&](int rc) { return create_failed(h, qrl_deframer_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels);
    if ((rc = dev_alloc(h, &h->d_state, C)) || (rc = dev_alloc(h, &h->d_bit_buf, C * bit_buf_len)) ||
        (rc = dev_alloc(h, &h->d_records, C * max_frames * h->rec_bytes)) || (rc = dev_alloc(h, &h->d_counts, C)) ||
        (rc = dev_alloc(h, &h->d_stage, C * static_cast<size_t>(max_bits))) || (rc = dev_alloc(h, &h->d_stage_counts, C)) ||
        (rc = dev_alloc(h, &h->d_dropped, C)))
        return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_deframer_set_stream(qrl_deframer* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

int qrl_deframer_work(qrl_deframer* h, const unsigned char* bits, const int* counts, long stride, int on_device)
{
    if (!h || !bits || !counts || stride < 0) { set_err(nullptr, "qrl_deframer_work: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char* d_bits = bits; const int* d_cnt = counts; long long d_stride = stride;
    if (!on_device) {
        if (stride > h->max_bits) { set_err(nullptr, "qrl_deframer_work: stride exceeds max_bits"); return QRL_ERANGE; }
        for (int c = 0; c < h->C; c++) if (counts[c] < 0 || counts[c] > stride) { set_err(nullptr, "qrl_deframer_work: bad count"); return QRL_ERANGE; }
        QRL_CK(cudaMemcpyAsync(h->d_stage, bits, static_cast<size_t>(h->C) * stride, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage_counts, counts, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
        d_bits = h->d_stage; d_cnt = h->d_stage_counts;
    }
    const int warps_per_block = 4;
    deframer_kernel<<<(h->C + warps_per_block - 1) / warps_per_block, 32 * warps_per_block, 0, h->stream>>>(
        h->C, h->sync_class, h->bit_buf_len, h->rx_frame_length, d_bits, d_stride, d_cnt, 0, nullptr, nullptr,
        h->d_state, h->d_bit_buf, h->d_records, h->rec_bytes, h->max_frames, h->d_counts, h->d_dropped);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_deframer_work2(qrl_deframer* h, const unsigned char* bits_a, const int* counts_a, const unsigned char* bits_b, const int* counts_b,
                       long stride, int on_device)
{
    if (!h || !bits_a || !counts_a || !bits_b || !counts_b || stride < 0) { set_err(nullptr, "qrl_deframer_work2: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char *da = bits_a, *db = bits_b; const int *ca = counts_a, *cb = counts_b;
    if (!on_device) {
        if (stride > h->max_bits) { set_err(nullptr, "qrl_deframer_work2: stride exceeds max_bits"); return QRL_ERANGE; }
        if (!h->d_stage2) {
            int rc;
            if ((rc = dev_alloc(h, &h->d_stage2, static_cast<size_t>(h->C) * h->max_bits, false)) ||
                (rc = dev_alloc(h, &h->d_stage_counts2, h->C, false))) return rc;
        }
        QRL_CK(cudaMemcpyAsync(h->d_stage, bits_a, static_cast<size_t>(h->C) * stride, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage_counts, counts_a, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage2, bits_b, static_cast<size_t>(h->C) * stride, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage_counts2, counts_b, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
        da = h->d_stage; ca = h->d_stage_counts; db = h->d_stage2; cb = h->d_stage_counts2;
    }
    const int warps_per_block = 4;
    deframer_kernel<<<(h->C + warps_per_block - 1) / warps_per_block, 32 * warps_per_block, 0, h->stream>>>(
        h->C, h->sync_class, h->bit_buf_len, h->rx_frame_length, da, stride, ca, 0, db, cb,
        h->d_state, h->d_bit_buf, h->d_records, h->rec_bytes, h->max_frames, h->d_counts, h->d_dropped);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_deframer_dropped(qrl_deframer* h, int* dropped_host)
{
    if (!h || !dropped_host) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(dropped_host, h->d_dropped, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_deframer_record_bytes(qrl_deframer* h) { return h ? h->rec_bytes : 0; }

int qrl_deframer_read(qrl_deframer* h, unsigned char* records_host, int* frame_counts_host, int* modem_sync_host)
{
    if (!h || !frame_counts_host) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(frame_counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (records_host)
        QRL_CK(cudaMemcpyAsync(records_host, h->d_records, static_cast<size_t>(h->C) * h->max_frames * h->rec_bytes, cudaMemcpyDeviceToHost, h->stream));
    std::vector<DeframerState> st;
    if (modem_sync_host) {
        st.resize(h->C);
        QRL_CK(cudaMemcpyAsync(st.data(), h->d_state, sizeof(DeframerState) * h->C, cudaMemcpyDeviceToHost, h->stream));
    }
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (modem_sync_host) for (int c = 0; c < h->C; c++) modem_sync_host[c] = st[c].modem_sync;
    return QRL_OK;
}

int qrl_deframer_out_device(qrl_deframer* h, void** records, int** frame_counts)
{
    if (!h) return QRL_EINVAL;
    if (records) *records = h->d_records;
    if (frame_counts) *frame_counts = h->d_counts;
    return QRL_OK;
}

int qrl_deframer_sync(qrl_deframer* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_deframer_launch_count(qrl_deframer* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------- gr_modem::frame
int qrl_frame_build(int n_channels, const unsigned char* payload, long payload_stride, const int* payload_len, const unsigned* frame_type,
                    int one_k_mode, int burst_ip, unsigned char* out, long out_stride, int* out_len, int on_device, int device, void* cuda_stream)
{
    if (n_channels < 1 || !payload || !payload_len || !frame_type || !out || !out_len || payload_stride < 0 || out_stride < 1) {
        set_err(nullptr, "qrl_frame_build: bad argument"); return QRL_EINVAL;
    }
    if (qrl_device_count() <= device) { set_err(nullptr, "qrl_frame_build: no CUDA device (this library has no CPU fallback)"); return QRL_ENODEV; }
    auto ck = [](cudaError_t e, const char* what) { if (e != cudaSuccess) { set_err(nullptr, std::string(what) + ": " + cudaGetErrorString(e)); return false; } return true; };
    if (!ck(cudaSetDevice(device), "cudaSetDevice")) return QRL_ECUDA;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    if (on_device) {
        frame_build_kernel<<<n_channels, 128, 0, st>>>(n_channels, payload, payload_stride, payload_len, frame_type, one_k_mode, burst_ip, out, out_stride, out_len);
        return ck(cudaGetLastError(), "frame_build_kernel") ? QRL_OK : QRL_ECUDA;
    }
    const size_t C = static_cast<size_t>(n_channels);
    unsigned char *d_p = nullptr, *d_o = nullptr; int *d_l = nullptr, *d_ol = nullptr; unsigned* d_t = nullptr;
    bool ok = ck(cudaMalloc(&d_p, std::max<size_t>(16, C * payload_stride)), "cudaMalloc") && ck(cudaMalloc(&d_o, C * out_stride), "cudaMalloc") &&
              ck(cudaMalloc(&d_l, C * 4), "cudaMalloc") && ck(cudaMalloc(&d_ol, C * 4), "cudaMalloc") && ck(cudaMalloc(&d_t, C * 4), "cudaMalloc");
    if (ok) ok = ck(cudaMemcpyAsync(d_p, payload, C * payload_stride, cudaMemcpyHostToDevice, st), "copy") &&
                 ck(cudaMemcpyAsync(d_l, payload_len, C * 4, cudaMemcpyHostToDevice, st), "copy") && ck(cudaMemcpyAsync(d_t, frame_type, C * 4, cudaMemcpyHostToDevice, st), "copy");
    if (ok) {
        frame_build_kernel<<<n_channels, 128, 0, st>>>(n_channels, d_p, payload_stride, d_l, d_t, one_k_mode, burst_ip, d_o, out_stride, d_ol);
        ok = ck(cudaGetLastError(), "frame_build_kernel") && ck(cudaMemcpyAsync(out, d_o, C * out_stride, cudaMemcpyDeviceToHost, st), "copy") &&
             ck(cudaMemcpyAsync(out_len, d_ol, C * 4, cudaMemcpyDeviceToHost, st), "copy") && ck(cudaStreamSynchronize(st), "sync");
    }
    cudaFree(d_p); cudaFree(d_o); cudaFree(d_l); cudaFree(d_ol); cudaFree(d_t);
    return ok ? QRL_OK : QRL_ECUDA;
}

// ---------------------------------------------------------------------------------------------- gr_deframer_bb
int qrl_dfbb_destroy(qrl_dfbb* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_dfbb_create(int modem_type, int n_channels, long max_bits, int device, qrl_dfbb** out)
{
    if (!out || modem_type < 1 || modem_type > 3 || n_channels < 1 || max_bits < 1) { set_err(nullptr, "qrl_dfbb_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_dfbb_create", device)) return rc;
    qrl_dfbb* h = new qrl_dfbb();
    h->type = modem_type; h->len = modem_type == 1 ? 64 : (modem_type == 2 ? 32 : 384);      // gr_deframer_bb.cpp:36-47
    h->C = n_channels; h->max_bits = max_bits;
    h->out_stride = max_bits + 32;          // a call emits at most its input plus one sync word whose last bit just arrived
    auto fail = [&](int rc) { return create_failed(h, qrl_dfbb_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    const size_t C = static_cast<size_t>(n_channels);
    if ((rc = dev_alloc(h, &h->d_state, C)) || (rc = dev_alloc(h, &h->d_out, C * static_cast<size_t>(h->out_stride))) ||
        (rc = dev_alloc(h, &h->d_counts, C)) || (rc = dev_alloc(h, &h->d_stage, C * static_cast<size_t>(max_bits))) ||
        (rc = dev_alloc(h, &h->d_stage_counts, C)))
        return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_dfbb_set_stream(qrl_dfbb* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, cuda_stream);
}

int qrl_dfbb_work(qrl_dfbb* h, const unsigned char* bits, const int* counts, long stride, int on_device)
{
    if (!h || !bits || !counts || stride < 0) { set_err(nullptr, "qrl_dfbb_work: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    const unsigned char* d_bits = bits; const int* d_cnt = counts;
    if (stride > h->max_bits) { set_err(nullptr, "qrl_dfbb_work: stride exceeds max_bits"); return QRL_ERANGE; }
    if (!on_device) {
        for (int c = 0; c < h->C; c++) if (counts[c] < 0 || counts[c] > stride) { set_err(nullptr, "qrl_dfbb_work: bad count"); return QRL_ERANGE; }
        QRL_CK(cudaMemcpyAsync(h->d_stage, bits, static_cast<size_t>(h->C) * stride, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaMemcpyAsync(h->d_stage_counts, counts, sizeof(int) * h->C, cudaMemcpyHostToDevice, h->stream));
        d_bits = h->d_stage; d_cnt = h->d_stage_counts;
    }
    const int warps_per_block = 4;
    dfbb_kernel<<<(h->C + warps_per_block - 1) / warps_per_block, 32 * warps_per_block, 0, h->stream>>>(
        h->C, h->type, h->len, d_bits, stride, d_cnt, h->d_state, h->d_out, h->out_stride, h->d_counts);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_dfbb_out_device(qrl_dfbb* h, void** bits, long* stride, int** counts)
{
    if (!h) return QRL_EINVAL;
    if (bits) *bits = h->d_out;
    if (stride) *stride = h->out_stride;
    if (counts) *counts = h->d_counts;
    return QRL_OK;
}

int qrl_dfbb_read(qrl_dfbb* h, unsigned char* out_host, long cap, int* counts_host)
{
    if (!h || !counts_host) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpyAsync(counts_host, h->d_counts, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
    if (out_host && cap > 0)
        QRL_CK(cudaMemcpy2DAsync(out_host, static_cast<size_t>(cap), h->d_out, static_cast<size_t>(h->out_stride), static_cast<size_t>(std::min(cap, h->out_stride)), h->C,
                              cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_dfbb_sync(qrl_dfbb* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_dfbb_launch_count(qrl_dfbb* h) { return h ? h->launches : 0; }

}  // extern "C"
