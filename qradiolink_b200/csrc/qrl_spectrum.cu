// qrl_spectrum.cu -- the display spectrum on the device (SURVEY.md section 8f row 4), part of libqrl_b200.so.
//
// Replaces rx_fft_c (/root/reference/src/gr/rx_fft.cpp:44-129; instance gr_demod_base.cpp:166: 32768 points, Blackman-Harris) for a
// batch of streams (one wideband source per GPU, or every channel of a batch): samples x window fill an N-item buffer per stream;
// when the buffer is full at the NEXT incoming sample the forward FFT runs, volk_32fc_s32f_power_spectrum_32f(points, fft, N, N) turns
// it into dB and the block takes no more input (whole work() calls are skipped) until get has been called, which returns the points
// fft-shifted.  One qrl_spectrum_work call = one rx_fft_c::work call for every stream (all streams get the same number of samples,
// so the fill counter is host state).  Only the LAST trigger of a call has an observable result (each trigger overwrites the points),
// so one call costs at most one FFT per stream however long it is.
//
// The FFT is hand-written (no cuFFT): N = N1 x N2 (both powers of two, 16..256), four-step.
//   pass A: per column n2, a length-N1 FFT over x[n1 N2 + n2] * window, times the twiddle W_N^(n2 k1), stored in place as Y[k1][n2]
//           (a CTA takes 16 adjacent columns: 128-byte global segments, radix-2 stages in shared memory);
//   pass B: per row k1, a length-N2 FFT over Y[k1][.]; bin k = k1 + N1 k2 -> 3.0103 log2(|Y / N|^2) -> out[(k + N/2) mod N]
//           (a CTA takes 16 adjacent rows so that the shifted stores are 64-byte segments).
// Twiddles come from sincospif on exact arguments (j / L is exact in binary), so the float FFT stays within ~1e-6 relative of the
// oracle's double-precision definition (oracle/qrl_oracle.c qo_spectrum_*); tests hold it to 2e-4 dB on bins within 40 dB of the peak
// and every bin's amplitude to 2e-6 of the peak amplitude.
#include "../../include/qrl_b200.h"
#include "qrl_design.hpp"
#include "qrl_handle.hpp"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

namespace {

constexpr int kCols = 16;       // columns (pass A) / rows (pass B) per CTA

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// in-place radix-2 decimation-in-time FFTs of length L (log2 = LB) on kCols independent sequences held as s[seq * (L + 1) + i]
// (bit-reversed on load by the caller); tw[j] = e^{-2 pi i j / L}, j < L / 2
__device__ __forceinline__ void smem_fft(float2* s, const float2* tw, int L, int LB)
{
    const int half_total = kCols * (L >> 1);
    for (int st = 1; st <= LB; st++) {
        const int len = 1 << st, half = len >> 1, tstep = L >> st;
        for (int b = threadIdx.x; b < half_total; b += blockDim.x) {
            const int seq = b / (L >> 1), r = b - seq * (L >> 1);
            const int grp = r / half, j = r - grp * half;
            float2* base = s + seq * (L + 1) + grp * len;
            const float2 w = tw[j * tstep];
            const float2 u = base[j], v = cmul(base[j + half], w);
            base[j] = make_float2(u.x + v.x, u.y + v.y);
            base[j + half] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
}

// pass A: grid (N2 / kCols, streams)
__global__ void __launch_bounds__(256)
spectrum_pass_a_kernel(const float2* __restrict__ buf, const float* __restrict__ window, float2* __restrict__ work, int N1, int N2, int LB1)
{
    extern __shared__ float2 sm[];
    float2* tw = sm;                         // N1 / 2
    float2* s = sm + (N1 >> 1);              // kCols * (N1 + 1)
    const int N = N1 * N2;
    const long long so = static_cast<long long>(blockIdx.y) * N;
    const int col0 = blockIdx.x * kCols;
    for (int j = threadIdx.x; j < (N1 >> 1); j += blockDim.x) {
        float sn, cs; sincospif(-2.0f * static_cast<float>(j) / static_cast<float>(N1), &sn, &cs);
        tw[j] = make_float2(cs, sn);
    }
    for (int e = threadIdx.x; e < kCols * N1; e += blockDim.x) {
        const int n1 = e / kCols, cc = e - n1 * kCols;
        const int n = n1 * N2 + col0 + cc;
        const float2 v = buf[so + n];
        const float w = window[n];
        const int r = static_cast<int>(__brev(static_cast<unsigned>(n1)) >> (32 - LB1));
        s[cc * (N1 + 1) + r] = make_float2(v.x * w, v.y * w);           // d_sample_buffer[i] = in[i] * d_window[i] (rx_fft.cpp:95)
    }
    __syncthreads();
    smem_fft(s, tw, N1, LB1);
    for (int e = threadIdx.x; e < kCols * N1; e += blockDim.x) {
        const int k1 = e / kCols, cc = e - k1 * kCols;
        const int n2 = col0 + cc;
        float sn, cs; sincospif(-2.0f * static_cast<float>(n2 * k1) / static_cast<float>(N), &sn, &cs);    // n2 k1 < 2^16: exact
        work[so + static_cast<long long>(k1) * N2 + n2] = cmul(s[cc * (N1 + 1) + k1], make_float2(cs, sn));
    }
}

// pass B: grid (N1 / kCols, streams)
__global__ void __launch_bounds__(256)
spectrum_pass_b_kernel(const float2* __restrict__ work, float* __restrict__ points, int N1, int N2, int LB2)
{
    extern __shared__ float2 sm[];
    float2* tw = sm;                         // N2 / 2
    float2* s = sm + (N2 >> 1);              // kCols * (N2 + 1)
    const int N = N1 * N2;
    const long long so = static_cast<long long>(blockIdx.y) * N;
    const int row0 = blockIdx.x * kCols;
    for (int j = threadIdx.x; j < (N2 >> 1); j += blockDim.x) {
        float sn, cs; sincospif(-2.0f * static_cast<float>(j) / static_cast<float>(N2), &sn, &cs);
        tw[j] = make_float2(cs, sn);
    }
    for (int e = threadIdx.x; e < kCols * N2; e += blockDim.x) {
        const int rr = e / N2, n2 = e - rr * N2;
        const int r = static_cast<int>(__brev(static_cast<unsigned>(n2)) >> (32 - LB2));
        s[rr * (N2 + 1) + r] = work[so + static_cast<long long>(row0 + rr) * N2 + n2];
    }
    __syncthreads();
    smem_fft(s, tw, N2, LB2);
    const float inorm = 1.0f / static_cast<float>(N);
    for (int e = threadIdx.x; e < kCols * N2; e += blockDim.x) {
        const int k2 = e / kCols, rr = e - k2 * kCols;
        const float2 v = s[rr * (N2 + 1) + k2];
        const float re = v.x * inorm, im = v.y * inorm;
        float l = log2f(re * re + im * im);                              // volk_32fc_s32f_power_spectrum_32f (VOLK 2.x generic)
        if (fabsf(l) > 3.0e38f) l = copysignf(127.0f, l);      // log2f_non_ieee: an infinite log becomes -/+127
        const int k = row0 + rr + N1 * k2;
        points[so + ((k + (N >> 1)) & (N - 1))] = 3.01029995663981209120f * l;      // fft-shift of get_fft_data (rx_fft.cpp:122-124)
    }
}

// samples [i0, i1) of this call into the fill buffer at slot (slot0 + i - i0); slots stay below N by construction
__global__ void spectrum_fill_kernel(const float2* __restrict__ in, long long in_stride, long long i0, long long i1,
                                     float2* __restrict__ buf, int N, int slot0)
{
    const long long so = static_cast<long long>(blockIdx.y) * N;
    const float2* src = in + static_cast<long long>(blockIdx.y) * in_stride;
    for (long long i = i0 + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < i1; i += static_cast<long long>(gridDim.x) * blockDim.x)
        buf[so + slot0 + (i - i0)] = src[i];
}

}  // namespace

struct qrl_spectrum : QrlHandleBase {
    int N = 0, N1 = 0, N2 = 0, LB1 = 0, LB2 = 0, win = 0, S = 0;
    long max_samples = 0;
    bool enabled = false, data_ready = false;
    int push = 0;
    unsigned counter = 0;
    float2 *d_buf = nullptr, *d_work = nullptr, *d_stage = nullptr;
    float *d_window = nullptr, *d_points = nullptr;
};

namespace {
void spectrum_free_buffers(qrl_spectrum* h)
{
    for (void* p : { static_cast<void*>(h->d_buf), static_cast<void*>(h->d_work), static_cast<void*>(h->d_window), static_cast<void*>(h->d_points) })
        if (p) cudaFree(p);
    h->d_buf = h->d_work = nullptr; h->d_window = h->d_points = nullptr;
}
int spectrum_alloc_buffers(qrl_spectrum* h, int n)
{
    int lb = 0; while ((1 << lb) < n) lb++;
    h->N = n; h->LB1 = lb / 2; h->LB2 = lb - h->LB1; h->N1 = 1 << h->LB1; h->N2 = 1 << h->LB2;
    const size_t items = static_cast<size_t>(n) * h->S;
    QRL_CK(cudaMalloc(&h->d_buf, sizeof(float2) * items));
    QRL_CK(cudaMalloc(&h->d_work, sizeof(float2) * items));
    QRL_CK(cudaMalloc(&h->d_points, sizeof(float) * items));
    QRL_CK(cudaMalloc(&h->d_window, sizeof(float) * n));
    QRL_CK(cudaMemsetAsync(h->d_buf, 0, sizeof(float2) * items, h->stream));
    QRL_CK(cudaMemsetAsync(h->d_points, 0, sizeof(float) * items, h->stream));
    const std::vector<float> w = qrl::window_build(h->win, n);          // gr::filter::firdes::window(type, N, 6.76) (rx_fft.cpp:181)
    QRL_CK(cudaMemcpyAsync(h->d_window, w.data(), sizeof(float) * n, cudaMemcpyHostToDevice, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    h->counter = 0; h->data_ready = false;
    return QRL_OK;
}
}  // namespace

extern "C" {

int qrl_spectrum_create(int fft_size, int window_type, int n_streams, long max_samples, int device, qrl_spectrum** out)
{
    if (!out || n_streams <= 0 || max_samples <= 0) { set_err(nullptr, "qrl_spectrum_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (fft_size < 256 || fft_size > 65536 || (fft_size & (fft_size - 1))) {
        set_err(nullptr, "qrl_spectrum_create: fft_size must be a power of two in [256, 65536]"); return QRL_EINVAL;
    }
    if (window_type < 0 || window_type > 7) window_type = qrl::WIN_HAMMING;           // rx_fft.cpp:176-179
    if (window_type == qrl::WIN_KAISER || window_type > qrl::WIN_BLACKMAN_HARRIS) {
        set_err(nullptr, "qrl_spectrum_create: window type not built (Hamming, Hann, Blackman, rectangular, Blackman-Harris are)"); return QRL_EINVAL;
    }
    if (int rc = check_device("qrl_spectrum_create", device)) return rc;
    qrl_spectrum* h = new qrl_spectrum;
    h->S = n_streams; h->win = window_type; h->max_samples = max_samples;
    int rc = handle_open(h, device);
    if (!rc) rc = spectrum_alloc_buffers(h, fft_size);
    if (rc) return create_failed(h, qrl_spectrum_destroy, rc);
    *out = h;
    return QRL_OK;
}

int qrl_spectrum_destroy(qrl_spectrum* h)
{
    if (!h) return QRL_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    spectrum_free_buffers(h);
    return handle_close(h);
}

int qrl_spectrum_set_stream(qrl_spectrum* h, void* s)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, s);
}

int qrl_spectrum_set_enabled(qrl_spectrum* h, int enabled)      // rx_fft_c::set_enabled (rx_fft.cpp:103-108)
{
    if (!h) return QRL_EINVAL;
    h->enabled = enabled != 0;
    return QRL_OK;
}

int qrl_spectrum_set_fft_size(qrl_spectrum* h, int fft_size)    // rx_fft_c::set_fft_size (rx_fft.cpp:130-158): buffer and ready flag reset
{
    if (!h) return QRL_EINVAL;
    if (fft_size == h->N) return QRL_OK;
    if (fft_size < 256 || fft_size > 65536 || (fft_size & (fft_size - 1))) { h->err = "qrl_spectrum_set_fft_size: power of two in [256, 65536]"; return QRL_EINVAL; }
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaStreamSynchronize(h->stream));
    spectrum_free_buffers(h);
    return spectrum_alloc_buffers(h, fft_size);
}

int qrl_spectrum_work(qrl_spectrum* h, const float* iq, long T, long stride, int on_device)
{
    if (!h || !iq || T < 0) return QRL_EINVAL;
    if (T > h->max_samples) { h->err = "qrl_spectrum_work: T exceeds max_samples given at create"; return QRL_ERANGE; }
    if (T == 0 || h->push > 0 || !h->enabled) return QRL_OK;         // rx_fft.cpp:80-84: nobody is reading, the whole call is dropped
    QRL_CK(cudaSetDevice(h->device));
    const float2* x = reinterpret_cast<const float2*>(iq);
    long long xstride = stride;
    if (!on_device) {
        if (!h->d_stage) { int rc = dev_alloc(h, &h->d_stage, static_cast<size_t>(h->max_samples) * h->S, false); if (rc) return rc; }
        QRL_CK(cudaMemcpy2DAsync(h->d_stage, sizeof(float2) * h->max_samples, iq, sizeof(float2) * stride, sizeof(float2) * T, h->S,
                              cudaMemcpyHostToDevice, h->stream));
        x = h->d_stage; xstride = h->max_samples;
    }
    // sample i triggers the FFT when the fill counter has reached N on its arrival: c + i = k N (k >= 1)
    const long long N = h->N, c = h->counter;
    long long i_last = -1;
    if (c + T - 1 >= N) i_last = ((c + T - 1) / N) * N - c;            // largest i < T with (c + i) a positive multiple of N
    auto fill = [&](long long i0, long long i1, int slot0) {
        if (i1 <= i0) return;
        dim3 g(static_cast<unsigned>(std::min<long long>((i1 - i0 + 255) / 256, 1024)), h->S);
        spectrum_fill_kernel<<<g, 256, 0, h->stream>>>(x, xstride, i0, i1, h->d_buf, h->N, slot0);
        h->launches++;
    };
    if (i_last < 0) {
        fill(0, T, static_cast<int>(c));
        h->counter = static_cast<unsigned>(c + T);
    } else {
        // the N samples in front of the last trigger: the tail of what the buffer already holds + this call's [i_last - N, i_last)
        const long long from = std::max<long long>(0, i_last - N);
        fill(from, i_last, static_cast<int>(N - (i_last - from)));
        const size_t smem_a = sizeof(float2) * ((h->N1 >> 1) + kCols * (h->N1 + 1));
        const size_t smem_b = sizeof(float2) * ((h->N2 >> 1) + kCols * (h->N2 + 1));
        spectrum_pass_a_kernel<<<dim3(h->N2 / kCols, h->S), 256, smem_a, h->stream>>>(h->d_buf, h->d_window, h->d_work, h->N1, h->N2, h->LB1);
        spectrum_pass_b_kernel<<<dim3(h->N1 / kCols, h->S), 256, smem_b, h->stream>>>(h->d_work, h->d_points, h->N1, h->N2, h->LB2);
        h->launches += 2;
        h->data_ready = true;
        h->push += static_cast<int>((c + T - 1) / N);
        fill(i_last, T, 0);
        h->counter = static_cast<unsigned>(T - i_last);
    }
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_spectrum_get(qrl_spectrum* h, float* dst, long dst_stride, int dst_on_device, unsigned* fft_size)
{
    if (!h || !dst || !fft_size) return QRL_EINVAL;
    h->push = 0;                                                        // rx_fft.cpp:115: want more samples
    if (!h->data_ready) { *fft_size = 0; return QRL_OK; }
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaMemcpy2DAsync(dst, sizeof(float) * dst_stride, h->d_points, sizeof(float) * h->N, sizeof(float) * h->N, h->S,
                          dst_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    *fft_size = static_cast<unsigned>(h->N);
    h->data_ready = false;
    return QRL_OK;
}

long qrl_spectrum_launch_count(qrl_spectrum* h) { return h ? h->launches : 0; }

}  // extern "C"
