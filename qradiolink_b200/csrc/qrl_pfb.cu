// qrl_pfb.cu -- polyphase channelizer / synthesizer (SURVEY.md section 8f row 1), part of libqrl_b200.so.
//
// Replaces gr::filter::pfb_channelizer_ccf(M, taps, 1.0) behind blocks::stream_to_streams(M)
// (/root/reference/src/gr/gr_demod_mmdvm_multi2.cpp:98-107) and gr::filter::pfb_synthesizer_ccf(M, taps, false)
// (/root/reference/src/gr/gr_mod_mmdvm_multi2.cpp:90-92).  The channelizer turns ONE wideband stream into the
// channel-major [M][T/M] layout that qrl_rx_work takes as a device-resident input; the synthesizer is its inverse.
//
//   channelizer: u_k[m] = sum_t taps[k + tM] * x[(m - t)M + (M-1-k)];  out_c[m] = sum_k u_k[m] * exp(+j 2 pi k c / M)
//   synthesizer: v_i[n] = sum_c in_c[n] * exp(+j 2 pi i c / M);        y[nM + i] = sum_t taps[i + tM] * v_i[n - t]
//
// Arithmetic order = the oracle's (oracle/qrl_oracle.c, "polyphase channelizer / synthesizer"): branch FIRs
// accumulate oldest sample first with fmaf; the M-point DFT is the direct sum over k ascending,
// re = fmaf(ur, wr, re); re = fmaf(-ui, wi, re); im = fmaf(ur, wi, im); im = fmaf(ui, wr, im), with twiddles
// (float)cos / (float)sin of the double angle.  Results are bit-identical to the oracle.
//
// Bound: 16 bytes of HBM traffic per wideband sample (8 read + 8 written) against 2*tpf + 4*M FFMA per sample
// (110 for the reference's M = 10, 341-tap prototype): FP32-issue bound, HBM roofline reported beside it.
// There is NO CPU fallback.
#include "../../include/qrl_b200.h"
#include "qrl_tma.cuh"
#include "qrl_handle.hpp"

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

using namespace qrl;

namespace {

// --------------------------------------------------------------------------------------------------------------
// Channelizer, register-tiled instance.  One CTA = TM = G*R consecutive output times of all M channels.
//   stage A: thread (k = tid % M, q = tid / M) holds the TPF taps of branch k in registers and slides over
//            R + TPF - 1 samples of stream M-1-k (stride M in the TMA-fetched window) -> R values of u_k
//   stage B: warp task (c, 32 consecutive m): 10-term DFT out of the transposed u buffer, coalesced 256-byte stores
// R*M mod 16 == 10 keeps the stage-A LDS.64 of a half warp on distinct banks for M = 10.
// The logical input stream is hist ++ x (hist = the previous call's tail, even length so that every window is
// 16-byte aligned for cp.async.bulk).
// --------------------------------------------------------------------------------------------------------------
template <int M, int TPF, int R, int G>
__global__ void __launch_bounds__(M * G)
pfb_chan_kernel(const float* __restrict__ bt /*[M][TPF]*/, const float* __restrict__ w /*[M][2]*/,
                const float2* __restrict__ hist, long long hist_len /* even */, const float2* __restrict__ x, long long n_x,
                long long frame0_e /* x-coordinate of stream sample (m = 0, j = 0): -pending */, long long frames,
                float2* __restrict__ out, long long out_stride, int use_tma)
{
    // x-coordinates: e >= 0 is x[e], e < 0 is hist[hist_len + e] (the previous calls' tail); hist_len is even, so an
    // even e is 16-byte aligned in either buffer and a window that starts on an even e can be fetched by cp.async.bulk
    constexpr int TM = G * R, SPAN = (TM + TPF - 1) * M, SPANP = (SPAN + 3) & ~1, TMP = TM + 1;
    extern __shared__ __align__(128) unsigned char smraw[];
    float2* win = reinterpret_cast<float2*>(smraw);                 // [SPANP]
    float2* ub = win + SPANP;                                       // [M][TMP]
    __shared__ __align__(8) uint64_t bar;
    const int tid = threadIdx.x;
    const long long m0 = static_cast<long long>(blockIdx.x) * TM;
    const long long e0 = frame0_e + (m0 - (TPF - 1)) * M;           // x-coordinate of the first sample stage A reads
    const int woff = static_cast<int>(e0 & 1);
    const long long e0p = e0 - woff;                                // even
    auto fetch = [&](long long e) {
        return e < 0 ? (e >= -hist_len ? hist[hist_len + e] : make_float2(0.0f, 0.0f)) : (e < n_x ? x[e] : make_float2(0.0f, 0.0f));
    };
    if (use_tma) {
        if (tid == 0) { mbar_init(&bar, 1); mbar_fence_init(); }
        __syncthreads();
        long long hi = e0p + SPANP;
        if (hi > n_x) hi = n_x & ~1LL;                              // the (short) rest is filled by the loop below
        if (hi < e0p) hi = e0p;
        if (tid == 0) {
            const long long n_h = e0p < 0 ? (hi < 0 ? hi - e0p : -e0p) : 0;
            const long long n_n = hi - e0p - n_h;
            mbar_expect_tx(&bar, static_cast<uint32_t>((hi - e0p) * 8));
            if (n_h > 0) bulk_g2s(win, hist + (hist_len + e0p), static_cast<uint32_t>(n_h * 8), &bar);
            if (n_n > 0) bulk_g2s(win + n_h, x + (e0p + n_h), static_cast<uint32_t>(n_n * 8), &bar);
        }
        for (long long i = hi - e0p + tid; i < SPANP; i += M * G) win[i] = fetch(e0p + i);
        mbar_wait(&bar, 0);
    } else {
        for (int i = tid; i < SPANP; i += M * G) win[i] = fetch(e0p + i);
    }
    __syncthreads();
    // ---- stage A
    {
        // thread -> (branch k, output group q).  The LDS.64 below touch float2 index R M q + (M - 1 - k) + const: a half-warp (16 consecutive
        // tids) is conflict-free when those are distinct mod 16.  With q = tid / M the group stride R M = 90 = 10 (mod 16) collides with
        // the k run of the neighbouring group (2-way conflicts on every load: 4 wavefronts instead of 2); visiting the groups
        // in the order 7 q' makes the stride 630 = 6 = -10 (mod 16), i.e. the index is 9 - tid (mod 16): distinct for any 16 consecutive tids.
        const int k = tid % M, qlin = tid / M;
        const int q = (M == 10 && R == 9 && G == 32) ? ((7 * qlin) & 31) : qlin;
        float h[TPF];
#pragma unroll
        for (int t = 0; t < TPF; t++) h[t] = bt[k * TPF + t];
        float2 acc[R];                                              // (re, im) pairs: one ffma2() (two FFMA) per tap and output
#pragma unroll
        for (int r = 0; r < R; r++) acc[r] = make_float2(0.0f, 0.0f);
        const float2* s = win + woff + (q * R) * M + (M - 1 - k);  // s[j*M] = stream sample at time (q*R - (TPF-1) + j)
#pragma unroll
        for (int j = 0; j < R + TPF - 1; j++) {
            const float2 v = s[j * M];
#pragma unroll
            for (int r = 0; r < R; r++) {
                const int t = r + TPF - 1 - j;                      // tap index for output r: sample time = m - t
                if (t >= 0 && t < TPF) ffma2(acc[r], h[t], v);
            }
        }
#pragma unroll
        for (int r = 0; r < R; r++) ub[k * TMP + q * R + r] = acc[r];
    }
    __syncthreads();
    // ---- stage B: warp w owns channel c = w, w + nwarps, ...: its M twiddles stay in registers
    {
        const int warp = tid >> 5, lane = tid & 31, nwarps = (M * G) >> 5;
        for (int c = warp; c < M; c += nwarps) {
            float wr[M], wi[M];
#pragma unroll
            for (int k = 0; k < M; k++) { const int qd = (k * c) % M; wr[k] = w[2 * qd]; wi[k] = w[2 * qd + 1]; }
            float2* orow = out + c * out_stride + m0;
            for (int m = lane; m < TM; m += 32) {
                if (m0 + m >= frames) break;
                float2 o = make_float2(0.0f, 0.0f);
#pragma unroll
                for (int k = 0; k < M; k++) {
                    const float2 u = ub[k * TMP + m];
                    // re += u.x wr; re += -u.y wi; im += u.x wi; im += u.y wr  ==  o += u.x (wr, wi); o += u.y (-wi, wr)   (two ffma2();
                    // fma(-a, b, c) and fma(a, -b, c) are the same operation)
                    ffma2_sp(o, u.x, wr[k], wi[k]);
                    ffma2_sp(o, u.y, -wi[k], wr[k]);
                }
                orow[m] = o;
            }
        }
    }
}

// --------------------------------------------------------------------------------------------------------------
// Every other shape (1 <= M <= 4096, up to 128 taps per branch): two kernels with the intermediate in HBM.
//   channelizer: pfb_fir_kernel<false> -> u [frames][M] (branch FIRs), pfb_dft_kernel<.., false> -> out [M][out_stride]
//   synthesizer: pfb_dft_kernel<.., true> -> v [hl + n][M] (hl = tpf-1 history columns recomputed from the input
//                history rows), pfb_fir_kernel<true> -> y [n][M]
// The round trip of u / v costs 16 B per wideband sample against 4 M FFMA of the DFT.
// --------------------------------------------------------------------------------------------------------------
constexpr int kFirThreads = 256, kFirR = 9;

// Branch FIR.  CTA = kb consecutive branches (kb = min(32, pow2 >= M)) x TB = (256 / kb) * R output times.  For a block of
// consecutive branches each time step reads one contiguous run of kb samples (channelizer: stream positions M-1-k; synthesizer:
// one row of v), so the shared window is [TB + tpf - 1][kb] at any M.  Thread (kk = tid % kb, g = tid / kb) computes the R
// consecutive times g R .. g R + R - 1 of branch k0 + kk: taps outer, newest-first index t = tpf-1 .. 0 (the oracle's oldest
// sample first), R window values held in registers and slid by one row per tap, so one tap load and one window load feed
// 2 R FFMA.  R = 9 keeps the window loads of a half warp on distinct banks for every kb < 16 (9 kb g mod 16 distinct).
template <bool SYN>
__global__ void __launch_bounds__(kFirThreads)
pfb_fir_kernel(int M, int tpf, int kb, const float* __restrict__ bt /*[M][tpf]*/, const float2* __restrict__ hist,
               long long hist_len, const float2* __restrict__ x, long long n_x, long long frame0_e, long long n_t,
               float2* __restrict__ out /*[n_t][M]*/)
{
    const int G = kFirThreads / kb, TB = G * kFirR, rows = TB + tpf - 1;
    extern __shared__ __align__(128) unsigned char smraw[];
    float2* win = reinterpret_cast<float2*>(smraw);                 // [rows][kb]
    float* hs = reinterpret_cast<float*>(win + rows * kb);          // [tpf][kb]
    const int tid = threadIdx.x;
    const long long m0 = static_cast<long long>(blockIdx.x) * TB;
    const int k0 = blockIdx.y * kb;
    for (int i = tid; i < tpf * kb; i += kFirThreads) {
        const int t = i / kb, k = k0 + i % kb;
        hs[i] = k < M ? bt[k * tpf + t] : 0.0f;
    }
    for (int i = tid; i < rows * kb; i += kFirThreads) {
        const int j = i / kb, k = k0 + i % kb;
        float2 v = make_float2(0.0f, 0.0f);
        if (k < M) {
            if (SYN) {                                              // x = v [n_t + tpf - 1][M]; window row j = v row m0 + j
                const long long r = m0 + j;
                if (r < n_t + tpf - 1) v = x[r * M + k];
            } else {                                                // stream sample (time m0 - (tpf-1) + j, position M-1-k)
                const long long e = frame0_e + (m0 - (tpf - 1) + j) * M + (M - 1 - k);
                if (e < 0) { if (e >= -hist_len) v = hist[hist_len + e]; }
                else if (e < n_x) v = x[e];
            }
        }
        win[i] = v;
    }
    __syncthreads();
    const int kk = tid % kb, g = tid / kb;
    if (k0 + kk >= M) return;
    const float2* s = win + (g * kFirR) * kb + kk;                  // s[j kb] = sample of output time g R at tap tpf-1-j
    float2 acc[kFirR], v[kFirR];
#pragma unroll
    for (int r = 0; r < kFirR; r++) { acc[r] = make_float2(0.0f, 0.0f); v[r] = s[r * kb]; }
    for (int t = tpf - 1;; t--) {
        const float h = hs[t * kb + kk];
#pragma unroll
        for (int r = 0; r < kFirR; r++) ffma2(acc[r], h, v[r]);    // v[r] = sample of output time g R + r at tap t
        if (t == 0) break;
#pragma unroll
        for (int r = 0; r < kFirR - 1; r++) v[r] = v[r + 1];
        v[kFirR - 1] = s[(kFirR + tpf - 1 - t) * kb];
    }
#pragma unroll
    for (int r = 0; r < kFirR; r++) {
        const long long m = m0 + g * kFirR + r;
        if (m < n_t) out[m * M + k0 + kk] = acc[r];
    }
}

// Exact-order DFT as a register-tiled complex "GEMM": out_p[t] = sum_k W[(k p) mod M] A[t][k], k ascending in one thread.
//   channelizer: A[t][k] = u[t M + k], out [p][out_stride] (p = channel c), stores coalesced along t
//   synthesizer: A[t][k] = input column t - hl of channel k (hist rows for t < hl), out [t][out_stride] (p = branch i),
//                stores coalesced along p
// CTA tile P = 4 PT outputs x T = 4 TT times (PT x TT = 256 threads); thread (pi, ti) owns p = pi + PT jp, t = ti + TT jt
// (jp, jt < 4): 16 complex accumulators.  k runs in chunks of KC: A staged as [KC][T + 1], the twiddle tile [KC][P] gathered
// once per chunk from the [M] table in shared memory, then 64 FFMA per 4 + 4 LDS.64 per k.
// A chunk past M is padded with zeros: fmaf(0, w, acc) returns acc bit for bit, because acc is never -0 (it starts at +0,
// and an fma only rounds to -0 from a -0 addend), so the padded terms leave every sum exactly the oracle's.
constexpr int kDftThreads = 256, kDftKc = 16;
template <int PT> constexpr int dft_smem(int M)
{
    return static_cast<int>(sizeof(float2)) * (M + kDftKc * (4 * (kDftThreads / PT) + 1) + kDftKc * 4 * PT);
}

template <int PT, bool SYN>
__global__ void __launch_bounds__(kDftThreads)
pfb_dft_kernel(int M, const float* __restrict__ wtab /*[M][2]*/, const float2* __restrict__ a, long long a_stride,
               const float2* __restrict__ hist /*SYN: [M][hl]*/, int hl, long long n_t, float2* __restrict__ out,
               long long out_stride)
{
    constexpr int TT = kDftThreads / PT, P = 4 * PT, T = 4 * TT, KC = kDftKc, TP = T + 1;
    extern __shared__ __align__(128) unsigned char smraw[];
    float2* wsm = reinterpret_cast<float2*>(smraw);                 // [M]
    float2* as = wsm + M;                                           // [KC][TP]
    float2* ws = as + KC * TP;                                      // [KC][P]
    const int tid = threadIdx.x;
    const long long t0 = static_cast<long long>(blockIdx.x) * T;
    const int p0 = blockIdx.y * P;
    const int pi = SYN ? tid % PT : tid / TT, ti = SYN ? tid / PT : tid % TT;
    for (int i = tid; i < M; i += kDftThreads) wsm[i] = make_float2(wtab[2 * i], wtab[2 * i + 1]);
    float2 acc[4][4];
#pragma unroll
    for (int jp = 0; jp < 4; jp++)
#pragma unroll
        for (int jt = 0; jt < 4; jt++) acc[jp][jt] = make_float2(0.0f, 0.0f);
    for (int k0 = 0; k0 < M; k0 += KC) {
        __syncthreads();                                            // the previous chunk is consumed (first: wsm is written)
        for (int i = tid; i < KC * T; i += kDftThreads) {
            const int kc = SYN ? i / T : i % KC, t = SYN ? i % T : i / KC;     // global reads contiguous along k / along t
            const int k = k0 + kc;
            const long long tt = t0 + t;
            float2 v = make_float2(0.0f, 0.0f);
            if (k < M && tt < n_t) {
                if (SYN) {
                    const long long n = tt - hl;
                    v = n < 0 ? hist[static_cast<long long>(k) * hl + hl + n] : a[k * a_stride + n];
                } else {
                    v = a[tt * a_stride + k];
                }
            }
            as[kc * TP + t] = v;
        }
        for (int i = tid; i < KC * P; i += kDftThreads) {
            const int k = k0 + i / P, p = p0 + i % P;
            ws[i] = (k < M && p < M) ? wsm[(k * p) % M] : make_float2(0.0f, 0.0f);
        }
        __syncthreads();
#pragma unroll
        for (int kc = 0; kc < KC; kc++) {
            float2 av[4], wv[4];
#pragma unroll
            for (int j = 0; j < 4; j++) { av[j] = as[kc * TP + ti + TT * j]; wv[j] = ws[kc * P + pi + PT * j]; }
#pragma unroll
            for (int jp = 0; jp < 4; jp++)
#pragma unroll
                for (int jt = 0; jt < 4; jt++) {
                    // re = fmaf(ur, wr, re); re = fmaf(-ui, wi, re); im = fmaf(ur, wi, im); im = fmaf(ui, wr, im)
                    ffma2_sp(acc[jp][jt], av[jt].x, wv[jp].x, wv[jp].y);
                    ffma2_sp(acc[jp][jt], av[jt].y, -wv[jp].y, wv[jp].x);
                }
        }
    }
#pragma unroll
    for (int jp = 0; jp < 4; jp++) {
        const int p = p0 + pi + PT * jp;
        if (p >= M) continue;
#pragma unroll
        for (int jt = 0; jt < 4; jt++) {
            const long long t = t0 + ti + TT * jt;
            if (t >= n_t) continue;
            if (SYN) out[t * out_stride + p] = acc[jp][jt];
            else out[p * out_stride + t] = acc[jp][jt];
        }
    }
}

// the last new_len samples of the stream (x-coordinates n_x - new_len .. n_x - 1) -> the other history buffer
__global__ void pfb_tail_kernel(const float2* __restrict__ hist, long long hist_len, const float2* __restrict__ x,
                                long long n_x, float2* __restrict__ dst, long long new_len)
{
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= new_len) return;
    const long long e = n_x - new_len + i;
    dst[i] = e < 0 ? (e >= -hist_len ? hist[hist_len + e] : make_float2(0.0f, 0.0f)) : x[e];
}

// --------------------------------------------------------------------------------------------------------------
// Synthesizer.  One CTA = TN = G*R consecutive input times n of all M channels.
//   stage A: thread (n lane-fastest, i): v_i[n] for n0 - (TPF-1) .. n0 + TN - 1 out of the [M][cols] input window
//            (the columns before the call come from the per-channel history rows)
//   stage B: thread (i = tid % M, q = tid / M): R outputs y[(n0 + qR + r) M + i], taps of branch i in registers,
//            sliding over v_i (contiguous in n); consecutive lanes write consecutive wideband samples
// --------------------------------------------------------------------------------------------------------------
template <int M, int TPF, int R, int G>
__global__ void __launch_bounds__(M * G)
pfb_synth_kernel(const float* __restrict__ bt, const float* __restrict__ w,
                 const float2* __restrict__ hist /*[M][TPF-1]*/, const float2* __restrict__ in, long long in_stride,
                 long long n_cols, float2* __restrict__ out)
{
    constexpr int TN = G * R, COLS = TN + TPF - 1, VP = COLS | 1;
    extern __shared__ __align__(16) unsigned char smraw[];
    float2* xin = reinterpret_cast<float2*>(smraw);                 // [M][COLS]
    float2* vb = xin + M * COLS;                                    // [M][VP]
    const int tid = threadIdx.x;
    const long long n0 = static_cast<long long>(blockIdx.x) * TN;
    for (int i = tid; i < M * COLS; i += M * G) {
        const int c = i / COLS, col = i % COLS;
        const long long n = n0 - (TPF - 1) + col;
        xin[i] = n < 0 ? hist[c * (TPF - 1) + (TPF - 1) + n] : (n < n_cols ? in[c * in_stride + n] : make_float2(0.0f, 0.0f));
    }
    __syncthreads();
    {
        const int warp = tid >> 5, lane = tid & 31, nwarps = (M * G) >> 5;
        for (int br = warp; br < M; br += nwarps) {              // warp owns branch br: twiddles in registers
            float wr[M], wi[M];
#pragma unroll
            for (int c = 0; c < M; c++) { const int qd = (br * c) % M; wr[c] = w[2 * qd]; wi[c] = w[2 * qd + 1]; }
            for (int col = lane; col < COLS; col += 32) {
                float2 o = make_float2(0.0f, 0.0f);
#pragma unroll
                for (int c = 0; c < M; c++) {
                    const float2 u = xin[c * COLS + col];
                    ffma2_sp(o, u.x, wr[c], wi[c]);             // re += u.x wr, im += u.x wi
                    ffma2_sp(o, u.y, -wi[c], wr[c]);            // re += -u.y wi, im += u.y wr
                }
                vb[br * VP + col] = o;
            }
        }
    }
    __syncthreads();
    {
        const int br = tid % M, q = tid / M;
        float h[TPF];
#pragma unroll
        for (int t = 0; t < TPF; t++) h[t] = bt[br * TPF + t];
        float2 acc[R];                                              // (re, im) pairs: one ffma2() (two FFMA) per tap and output
#pragma unroll
        for (int r = 0; r < R; r++) acc[r] = make_float2(0.0f, 0.0f);
        const float2* s = vb + br * VP + q * R;                     // s[j] = v_br[n0 + qR - (TPF-1) + j]
#pragma unroll
        for (int j = 0; j < R + TPF - 1; j++) {
            const float2 v = s[j];
#pragma unroll
            for (int r = 0; r < R; r++) {
                const int t = r + TPF - 1 - j;
                if (t >= 0 && t < TPF) ffma2(acc[r], h[t], v);
            }
        }
#pragma unroll
        for (int r = 0; r < R; r++) {
            const long long n = n0 + q * R + r;
            if (n < n_cols) out[n * M + br] = acc[r];
        }
    }
}

// new per-channel history rows: the last tpf-1 input columns of (hist ++ in)
__global__ void pfb_synth_tail_kernel(int M, int hl, const float2* __restrict__ hist, const float2* __restrict__ in,
                                      long long in_stride, long long n_cols, float2* __restrict__ dst)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * hl) return;
    const int c = i / hl, j = i % hl;
    const long long n = n_cols - hl + j;
    dst[i] = n < 0 ? hist[c * hl + hl + n] : in[c * in_stride + n];
}

}  // namespace

struct qrl_pfb : QrlHandleBase {        // err / device / stream / launches / allocs: qrl_handle.hpp
    int kind = 0, M = 0, tpf = 0;
    long max_in = 0;
    float *d_bt = nullptr, *d_w = nullptr;
    // channelizer: tail of the stream = [pad][(tpf-1)*M history][pend < M pending samples], hist_len even
    // synthesizer: [M][tpf-1] last input columns
    float2* d_hist[2] = { nullptr, nullptr }; int hist_cur = 0; long long hist_len = 0; int pend = 0;
    float2* d_stage = nullptr;          // staging for host input
    float2* d_out = nullptr; long long out_stride = 0; long long out_items = 0;
    float2* d_mid = nullptr;            // two-kernel shapes: channelizer u [frames][M], synthesizer v [tpf-1 + n][M]
    bool fast = false;
};

namespace {
constexpr int kFastM = 10, kFastTpf = 35, kChanR = 9, kChanG = 32, kSynR = 10, kSynG = 32;
// 4096 channels of 25 kHz = 102.4 Msps, the top of the receive front end's range
constexpr int kMaxM = 4096, kMaxTpf = 128;
// pfb_fir_kernel's window and taps: (256 / kb * R + tpf - 1) kb float2 + tpf kb float, at most 67 328 B (kb = 32, tpf = 128)
constexpr int kFirSmemMax = static_cast<int>(sizeof(float2)) * (kFirThreads * kFirR + (kMaxTpf - 1) * 32) + 4 * kMaxTpf * 32;
// pfb_dft_kernel: PT = 4 (16 outputs x 256 times per CTA) up to M = 16, PT = 16 (64 x 64) above
constexpr int kDftSmallM = 16;
int fir_kb(int M) { int kb = 1; while (kb < M && kb < 32) kb *= 2; return kb; }
int fir_smem(int tpf, int kb) { return static_cast<int>(sizeof(float2)) * ((kFirThreads / kb * kFirR + tpf - 1) * kb) + 4 * tpf * kb; }
template <bool SYN>
int launch_fir(qrl_pfb* h, const float2* hist, long long hist_len, const float2* x, long long n_x, long long frame0_e, long long n_t,
               float2* out)
{
    const int kb = fir_kb(h->M), tb = kFirThreads / kb * kFirR;
    if (int rc = smem_opt_in(h, pfb_fir_kernel<SYN>, kFirSmemMax)) return rc;
    pfb_fir_kernel<SYN><<<dim3(static_cast<unsigned>((n_t + tb - 1) / tb), static_cast<unsigned>((h->M + kb - 1) / kb)), kFirThreads,
                          fir_smem(h->tpf, kb), h->stream>>>(h->M, h->tpf, kb, h->d_bt, hist, hist_len, x, n_x, frame0_e, n_t, out);
    h->launches++;
    return QRL_OK;
}
template <int PT, bool SYN>
int launch_dft_pt(qrl_pfb* h, const float2* a, long long a_stride, const float2* hist, int hl, long long n_t, float2* out,
                  long long out_stride)
{
    constexpr int P = 4 * PT, T = 4 * (kDftThreads / PT);
    if (int rc = smem_opt_in(h, pfb_dft_kernel<PT, SYN>, dft_smem<PT>(PT == 4 ? kDftSmallM : kMaxM))) return rc;
    pfb_dft_kernel<PT, SYN><<<dim3(static_cast<unsigned>((n_t + T - 1) / T), static_cast<unsigned>((h->M + P - 1) / P)), kDftThreads,
                              dft_smem<PT>(h->M), h->stream>>>(h->M, h->d_w, a, a_stride, hist, hl, n_t, out, out_stride);
    h->launches++;
    return QRL_OK;
}
template <bool SYN>
int launch_dft(qrl_pfb* h, const float2* a, long long a_stride, const float2* hist, int hl, long long n_t, float2* out, long long out_stride)
{
    return h->M <= kDftSmallM ? launch_dft_pt<4, SYN>(h, a, a_stride, hist, hl, n_t, out, out_stride)
                              : launch_dft_pt<16, SYN>(h, a, a_stride, hist, hl, n_t, out, out_stride);
}
long long chan_hist_len(int tpf, int M, int pend) { return (static_cast<long long>(tpf - 1) * M + pend + 2) & ~1LL; }
}  // namespace

extern "C" {

int qrl_pfb_destroy(qrl_pfb* h)
{
    if (!h) return QRL_EINVAL;
    return handle_close(h);
}

int qrl_pfb_create(int kind, int M, const float* taps, int ntaps, long max_in, int device, qrl_pfb** out)
{
    if (M > kMaxM) {
        set_err(nullptr, "qrl_pfb_create: M above 4096 channels");
        return QRL_EINVAL;
    }
    if (!out || !taps || (kind != QRL_PFB_CHANNELIZER && kind != QRL_PFB_SYNTHESIZER) || M < 1 || ntaps < 1 ||
        max_in < 1 || (ntaps + M - 1) / M > kMaxTpf) {
        set_err(nullptr, "qrl_pfb_create: bad argument");
        return QRL_EINVAL;
    }
    *out = nullptr;
    if (int rc = check_device("qrl_pfb_create", device)) return rc;
    qrl_pfb* h = new qrl_pfb();
    h->kind = kind; h->M = M; h->tpf = (ntaps + M - 1) / M; h->max_in = max_in;
    auto fail = [&](int rc) { return create_failed(h, qrl_pfb_destroy, rc); };
    int rc = handle_open(h, device);
    if (rc) return fail(rc);
    // branch taps [M][tpf] (polyphase_filterbank::set_taps: filter k holds taps[k + t*M], zero padded) and twiddles
    std::vector<float> bt(static_cast<size_t>(M) * h->tpf, 0.0f), w(static_cast<size_t>(M) * 2);
    for (int j = 0; j < ntaps; j++) bt[static_cast<size_t>(j % M) * h->tpf + j / M] = taps[j];
    for (int q = 0; q < M; q++) {
        const double a = 2.0 * 3.14159265358979323846 * static_cast<double>(q) / static_cast<double>(M);
        w[2 * q] = static_cast<float>(std::cos(a)); w[2 * q + 1] = static_cast<float>(std::sin(a));
    }
    if ((rc = dev_alloc(h, &h->d_bt, bt.size(), false)) || (rc = dev_alloc(h, &h->d_w, w.size(), false)) ||
        (rc = upload_state(h, h->d_bt, bt.data(), bt.size() * 4)) || (rc = upload_state(h, h->d_w, w.data(), w.size() * 4))) return fail(rc);
    h->fast = (M == kFastM && h->tpf == kFastTpf);
    if (kind == QRL_PFB_CHANNELIZER) {
        const size_t hcap = static_cast<size_t>(h->tpf) * M + 4;
        if ((rc = dev_alloc(h, &h->d_hist[0], hcap)) || (rc = dev_alloc(h, &h->d_hist[1], hcap))) return fail(rc);
        h->pend = 0; h->hist_len = chan_hist_len(h->tpf, M, 0);
        h->out_stride = (max_in + M - 1) / M + 2;
        if ((rc = dev_alloc(h, &h->d_out, static_cast<size_t>(h->out_stride) * M))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_stage, static_cast<size_t>(max_in)))) return fail(rc);
        if (!h->fast && (rc = dev_alloc(h, &h->d_mid, static_cast<size_t>(h->out_stride) * M))) return fail(rc);
    } else {
        const size_t hl = static_cast<size_t>(std::max(1, h->tpf - 1)) * M;
        if ((rc = dev_alloc(h, &h->d_hist[0], hl)) || (rc = dev_alloc(h, &h->d_hist[1], hl))) return fail(rc);
        h->out_stride = max_in * M;
        if ((rc = dev_alloc(h, &h->d_out, static_cast<size_t>(max_in) * M))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_stage, static_cast<size_t>(max_in) * M))) return fail(rc);
        if (!h->fast && (rc = dev_alloc(h, &h->d_mid, static_cast<size_t>(max_in + h->tpf - 1) * M))) return fail(rc);
    }
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

int qrl_pfb_set_stream(qrl_pfb* h, void* cuda_stream)
{
    if (!h) return QRL_EINVAL;
    if (!cuda_stream) return QRL_OK;       // unlike the other handle types: NULL keeps the current stream
    return handle_set_stream(h, cuda_stream);
}

int qrl_pfb_work(qrl_pfb* h, const void* in, long n_in, long in_stride, int in_on_device, long* n_out)
{
    if (!h || (!in && n_in > 0) || n_in < 0 || n_in > h->max_in) { set_err(nullptr, "qrl_pfb_work: bad argument"); return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    const int M = h->M, tpf = h->tpf;
    const float2* hist = h->d_hist[h->hist_cur];
    float2* hist_next = h->d_hist[h->hist_cur ^ 1];
    if (h->kind == QRL_PFB_CHANNELIZER) {
        const float2* x = static_cast<const float2*>(in);
        if (!in_on_device && n_in > 0) {
            QRL_CK(cudaMemcpyAsync(h->d_stage, in, sizeof(float2) * n_in, cudaMemcpyHostToDevice, h->stream));
            x = h->d_stage;
        }
        const long long frames = (static_cast<long long>(h->pend) + n_in) / M;
        if (frames > 0) {
            if (h->fast) {
                constexpr int TM = kChanR * kChanG, SPAN = (TM + kFastTpf - 1) * kFastM, SPANP = (SPAN + 3) & ~1;
                const size_t smem = sizeof(float2) * (SPANP + kFastM * (TM + 1));
                auto kern = pfb_chan_kernel<kFastM, kFastTpf, kChanR, kChanG>;
                if (int rc = smem_opt_in(h, kern, static_cast<int>(smem))) return rc;
                const int use_tma = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
                kern<<<static_cast<unsigned>((frames + TM - 1) / TM), kFastM * kChanG, smem, h->stream>>>(
                    h->d_bt, h->d_w, hist, h->hist_len, x, n_in, -static_cast<long long>(h->pend), frames,
                    h->d_out, h->out_stride, use_tma);
                h->launches++;
            } else {
                if (int rc = launch_fir<false>(h, hist, h->hist_len, x, n_in, -static_cast<long long>(h->pend), frames, h->d_mid)) return rc;
                if (int rc = launch_dft<false>(h, h->d_mid, M, nullptr, 0, frames, h->d_out, h->out_stride)) return rc;
            }
        }
        const int new_pend = static_cast<int>((static_cast<long long>(h->pend) + n_in) % M);
        const long long new_len = chan_hist_len(tpf, M, new_pend);
        if (n_in > 0) {
            pfb_tail_kernel<<<static_cast<unsigned>((new_len + 255) / 256), 256, 0, h->stream>>>(hist, h->hist_len, x, n_in, hist_next, new_len);
            h->launches++;
            h->hist_cur ^= 1; h->hist_len = new_len; h->pend = new_pend;
        }
        h->out_items = frames;
        if (n_out) *n_out = static_cast<long>(frames);
    } else {
        const float2* x = static_cast<const float2*>(in);
        long long stride = in_stride;
        if (!in_on_device && n_in > 0) {
            QRL_CK(cudaMemcpy2DAsync(h->d_stage, sizeof(float2) * n_in, in, sizeof(float2) * in_stride, sizeof(float2) * n_in, M,
                                  cudaMemcpyHostToDevice, h->stream));
            x = h->d_stage; stride = n_in;
        }
        if (n_in > 0) {
            const int hl = tpf - 1;
            if (h->fast) {
                constexpr int TN = kSynR * kSynG, COLS = TN + kFastTpf - 1, VP = COLS | 1;
                const size_t smem = sizeof(float2) * (kFastM * COLS + kFastM * VP);
                auto kern = pfb_synth_kernel<kFastM, kFastTpf, kSynR, kSynG>;
                if (int rc = smem_opt_in(h, kern, static_cast<int>(smem))) return rc;
                kern<<<static_cast<unsigned>((n_in + TN - 1) / TN), kFastM * kSynG, smem, h->stream>>>(
                    h->d_bt, h->d_w, hist, x, stride, n_in, h->d_out);
                h->launches++;
            } else {
                if (int rc = launch_dft<true>(h, x, stride, hist, hl, hl + n_in, h->d_mid, M)) return rc;
                if (int rc = launch_fir<true>(h, nullptr, 0, h->d_mid, 0, 0, n_in, h->d_out)) return rc;
            }
            if (hl > 0) {
                pfb_synth_tail_kernel<<<(M * hl + 255) / 256, 256, 0, h->stream>>>(M, hl, hist, x, stride, n_in, hist_next);
                h->launches++;
                h->hist_cur ^= 1;
            }
        }
        h->out_items = static_cast<long long>(n_in) * M;
        if (n_out) *n_out = static_cast<long>(h->out_items);
    }
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_pfb_sync(qrl_pfb* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

int qrl_pfb_out_device(qrl_pfb* h, void** data, long* stride, long* items)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = h->d_out;
    if (stride) *stride = static_cast<long>(h->out_stride);
    if (items) *items = static_cast<long>(h->out_items);
    return QRL_OK;
}

int qrl_pfb_read(qrl_pfb* h, void* host_dst, long dst_stride)
{
    if (!h || !host_dst) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    if (h->out_items > 0) {
        if (h->kind == QRL_PFB_CHANNELIZER)
            QRL_CK(cudaMemcpy2DAsync(host_dst, sizeof(float2) * dst_stride, h->d_out, sizeof(float2) * h->out_stride,
                                  sizeof(float2) * h->out_items, h->M, cudaMemcpyDeviceToHost, h->stream));
        else
            QRL_CK(cudaMemcpyAsync(host_dst, h->d_out, sizeof(float2) * h->out_items, cudaMemcpyDeviceToHost, h->stream));
    }
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_pfb_launch_count(qrl_pfb* h) { return h ? h->launches : 0; }

}  // extern "C"
