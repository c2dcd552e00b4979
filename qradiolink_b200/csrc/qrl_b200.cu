// qrl_b200.cu -- handles, stage orchestration and the C ABI (include/qrl_b200.h) of libqrl_b200.so.
//
// One qrl_rx handle = n_channels independent instances of ONE reference demod hier-block
// (/root/reference/src/gr/gr_demod_{nbfm,4fsk,qpsk}.cpp) running as batched CUDA kernels.  All
// per-channel DSP state (FIR history, resampler phase, loop filters, Viterbi start state, LFSR)
// lives in HBM between qrl_rx_work calls, so results do not depend on how the stream is chunked.
// There is NO CPU fallback: without a CUDA device every create call fails with QRL_ENODEV.
#include "../../include/qrl_b200.h"
#include "qrl_design.hpp"
#include "qrl_kernels.cuh"
#include "qrl_handle.hpp"

#include <cuda.h>

#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <type_traits>
#include <vector>

using namespace qrl;

namespace {

struct Ring {
    void* d = nullptr;
    unsigned mask = 0;
    long long stride = 0;   // items per channel (= capacity)
};

unsigned pow2_at_least(long long n)
{
    unsigned long long c = 64;
    while (c < static_cast<unsigned long long>(n)) c <<= 1;
    return static_cast<unsigned>(c);
}

// a polyphase interpolator's taps as L arms of nt taps each (arm p holds taps p, p + L, ...; zero past the end)
std::vector<float> make_arms(const std::vector<float>& taps, int L, int nt)
{
    std::vector<float> a(static_cast<size_t>(L) * nt, 0.0f);
    for (int p = 0; p < L; p++)
        for (int k = 0; k < nt; k++) { const size_t j = p + static_cast<size_t>(k) * L; if (j < taps.size()) a[p * nt + k] = taps[j]; }
    return a;
}

using HandleBase = QrlHandleBase;       // qrl_handle.hpp: shared by every handle type of the library

// the atan, tanh, MMSE and sine lookup tables, once per device (keyed by this function)
int upload_tables(HandleBase* h)
{
    return once_per_device(reinterpret_cast<const void*>(&upload_tables), h->device, [h]() -> int {
        auto at = atan_table(); auto th = tanh_table(); auto mm = mmse_table(); auto sn = fxpt_sine_table();
        cudaError_t e = cudaMemcpyToSymbol(d_atan_tab, at.data(), at.size() * 4);
        if (e == cudaSuccess) e = cudaMemcpyToSymbol(d_tanh_tab, th.data(), th.size() * 4);
        if (e == cudaSuccess) e = cudaMemcpyToSymbol(d_mmse_tab, mm.data(), mm.size() * 4);
        if (e == cudaSuccess) e = cudaMemcpyToSymbol(d_sine_tab, sn.data(), sn.size() * 4);
        if (e != cudaSuccess) { set_err(h, std::string("table upload: ") + cudaGetErrorString(e)); return QRL_ECUDA; }   // retried by the next create
        return QRL_OK;
    });
}

}  // namespace

// =====================================================================================================
struct qrl_rx : HandleBase {
    int kind = 0, sps = 0, samp_rate = 0, carrier_freq = 0, filter_width = 0, flag = 0, C = 0;
    long Tmax = 0;
    int nports = 3;
    // stage 1 (rational_resampler_ccf(1, D))
    int D1 = 1, L1 = 1, Q1 = 1, ntaps1 = 0, H = 0, hist_cur = 0;
    float* d_taps1 = nullptr;
    float2* d_hist[2] = { nullptr, nullptr };
    float2* d_in_staging = nullptr;
    short2* d_in_sc16 = nullptr;        // qrl_rx_work_sc16 with a host buffer: the int16 slab as it arrived over PCIe
    float2* d_in1 = nullptr;            // stride 0 (one stream for every channel): [Tmax] staging of host or converted input
    short2* d_in1_sc16 = nullptr;       // stride 0, sc16 / sc8 from a host buffer: [Tmax] pairs as they arrived over PCIe
    long long n_in = 0, n1 = 0;       // stage-1 progress (absolute input samples consumed / outputs produced)
    long long n_in_s = 0, n1_s = 0;   // progress of the per-slice stages behind it (equal to the above between calls)
    bool fir_group_forced = false;     // QRL_FIR_GROUP given: keep it in overlap mode too
    int fir_group = 4;                 // stage-1 launches cover this many slices (bigger launches, same pipeline depth)
    Ring r1;
    // stage 2: channel / shaping filter on the complex stream (port 0)
    float* d_taps2 = nullptr; int ntaps2 = 0; size_t taps2_cap = 0;     // floats allocated for d_taps2 (set_filter_width redesigns)
    float if_gain = 0.9f;              // gr_demod_ssb: multiply_const_cc(0.9) in front of the side-band filter (set_gain)
    Ring r2;
    float2* d_port0 = nullptr; long port0_cap = 0; long port0_n = 0;
    // stage 3: quadrature demod + RRC (4FSK-FM)
    float* d_taps3 = nullptr; int ntaps3 = 0; float qd_gain = 0;
    Ring r4;
    // PSK chains: agc2 + costas "PLL" loop stage (per sample), output ring r3 (interleaved)
    AgcCostasParams acp{};
    AgcCostasState* d_ac = nullptr;
    // NBFM: de-emphasis recurrence in its own kernel on s_loop2 (overlaps the next slice's squelch recurrence)
    NbfmDeemphState* d_nb2 = nullptr; Ring raud; bool nbfm_split = false;
    // NBFM: stream between the 2/5 resampler and the audio filter (copy, or ctcss_squelch_ff after set_ctcss(f))
    Ring rq; NbfmCtcss ctc{}; double* d_cenv = nullptr;
    // gr_demod_dsss: one chain kernel behind stage 1 (dsss_chain_kernel)
    DsssParams dsp{}; DsssState* d_ds = nullptr; float* d_ds_arms = nullptr; float2* d_ds_taps = nullptr;
    Ring ds_a, ds_c, ds_d; long long ds_o_call0 = 0;
    Ring r3;
    int sym_sps = 0;
    // BPSK / 2FSK: fll_band_edge_cc + second (delayed) decoder
    FllParams fllp{};
    FllState* d_fll = nullptr; float2* d_fll_hist = nullptr; float* d_fll_taps = nullptr;
    Ring rf;                       // FLL output (channel-major complex)
    ViterbiState* d_vs2 = nullptr;
    unsigned char* d_port3 = nullptr; int* d_port3_cnt = nullptr;
    // front-end rotator (carrier offset)
    std::vector<RotState> rot; RotState* d_rot = nullptr; bool rot_active = false; float2* d_rot_buf = nullptr;
    bool rot_fused = false;            // this call: the rotator runs inside the stage-1 kernel (register-tiled shapes)
    // non-FM FSK detectors: band-pass bank + symbol filter
    float* d_bank_taps = nullptr; int nt_bank = 0;
    float* d_symf_taps = nullptr; int nt_symf = 0;
    Ring rbank;                    // bank output (complex for 4FSK, float for 2FSK), channel-major
    // FreeDV: agc2_ff + audio band-pass + int16 conversion behind the side-band filter (AGC output ring: rstr)
    FreedvRxParams fdp{};
    FreedvRxState* d_fdv = nullptr;
    // SSB audio chain
    SsbParams ssbp{};
    SsbState* d_ssb = nullptr;
    Ring rclip, rstr;
    float* d_taps2c = nullptr;     // complex side-band filter taps
    // NBFM audio chain
    NbfmParams nbp{};
    NbfmState* d_nb = nullptr;
    Ring rg, rd, rr;
    float* d_env = nullptr; float* d_arm_taps = nullptr; float* d_audio_taps = nullptr;
    float* d_port1f = nullptr;
    int tsr = 0;
    std::vector<std::pair<void*, size_t>> zero_list;   // buffers qrl_rx_reset clears
    // symbol sync
    SymSyncParams ssp{};
    SymSyncState* d_ss = nullptr;
    float* d_ss_scratch = nullptr; int* d_ss_hdr = nullptr; long long ss_chunk_cap = 0, ss_chunk_off = 0;   // external symbol-sync epilogue
    cudaStream_t s_epi = nullptr;                        // wide-partition stream of the external epilogue
    bool gmsk = false;                                   // 2FSK code path running as gr_demod_gmsk (no FLL)
    bool m17 = false;                                    // 4FSK (fm) code path running as gr_demod_m17 (x3/125 front end, hard bits)
    int nt_arm1 = 0;                                     // taps per arm of a generic rational stage 1 (L1 > 1)
    bool dmr = false;                                    // M17 code path running as gr_demod_dmr (plain M&M detector, x0.9, float port 3)
    float* d_port3f = nullptr;                           // gr_demod_dmr port 3: symbol filter output, [C][port0_cap] floats
    // RSSI tap on port 0 (QRL_PARAM_RSSI): ring of |x|^2, carried IIR value, latest dB value per channel
    bool rssi_on = false; float* d_rssi_ring = nullptr; float* d_rssi_y = nullptr; float* d_rssi_db = nullptr; long long rssi_n = 0;
    // QRL_PARAM_OVERLAP_CALLS: the loop / FEC tail of call k runs under the parallel stages of call k+1.  Output ports
    // are double-buffered (alt_* = the buffers of the previous call), ring reuse is fenced slice by slice.
    bool many = false;                                   // many-channel geometry of the loop kernels (small windows, no SM partition)
    bool overlap = false;
    float2* alt_port0 = nullptr; float2* alt_port1 = nullptr; unsigned char* alt_port2 = nullptr; unsigned char* alt_port3 = nullptr;
    int *alt_port1_cnt = nullptr, *alt_port2_cnt = nullptr, *alt_port3_cnt = nullptr;
    long alt_port0_n = 0;
    cudaEvent_t ev_v[16] = { nullptr };                  // Viterbi of slice i done (kMaxSub entries)
    cudaEvent_t ev_tail[2][3] = { { nullptr } };         // s_loop / s_fec / s_epi at the end of a call, by call parity
    int call_parity = 0;
    long prev_T = -1;                  // length of the previous overlapped call (a change of length joins the tail, see qrl_rx_work)
    long long prev_k1[16] = { 0 }, cur_k1[16] = { 0 }; int prev_nsub = 0;      // stage-1 sample index at the end of each slice
    int ss_ch = 256;                                     // rows per symbol-sync window (256 x 3 stages or 512 x 2)
    float2* d_port1 = nullptr; long port1_cap = 0; int* d_port1_cnt = nullptr;
    Ring r5;   // soft bits (u8)
    ViterbiState* d_vs = nullptr;
    unsigned char* d_port2 = nullptr; long port2_cap = 0; int* d_port2_cnt = nullptr;
    long n1max = 0;
    // software pipeline inside one work() call: parallel stages on `stream`, loop stages on s_loop, FEC on s_fec
    static constexpr int kMaxSub = 16;
    int nsub = 12;
    bool nsub_forced = false;          // QRL_NSUB given
    cudaStream_t s_loop = nullptr, s_loop2 = nullptr, s_fec = nullptr;
    cudaEvent_t ev_start = nullptr, ev_a[kMaxSub] = { nullptr }, ev_b[kMaxSub] = { nullptr }, ev_c[kMaxSub] = { nullptr },
                ev_loop_done = nullptr, ev_loop2_done = nullptr, ev_fec_done = nullptr;
    long long* d_nsoft = nullptr;   // [kMaxSub][C] soft-bit write index snapshots
    // static SM partition (CUDA green contexts): the sequential loop / FEC kernels get a small private set of SMs so
    // their single dependent instruction streams never arbitrate with the FMA-bound FIR warps; the parallel stages
    // run on the remaining SMs through s_par.  Falls back to plain streams when the driver refuses.
    CUgreenCtx g_loop = nullptr, g_par = nullptr;
    cudaStream_t s_par = nullptr;
    cudaEvent_t ev_par_done = nullptr;
    int sm_loop = 0, sm_par = 0;
    cudaStream_t par() const { return s_par ? s_par : stream; }
    StageProfiler prof{ 8 };           // optional per-stage device timing (qrl_rx_profile)
};

namespace {

template <int D, int Q, int K, int NOUT, int NWARPS>
int launch_fir_poly(qrl_rx* h, const float2* iq, long long stride, long long T, long long k0, long long k1)
{
    constexpr int W = (NOUT + Q - 1) * D;
    const size_t smem = sizeof(float2) * ((W + 3) & ~1);
    if (int rc = smem_opt_in(h, fir_decim_poly_kernel<D, Q, K, NOUT, NWARPS>, (int)smem)) return rc;
    const long long nout = k1 - k0;
    dim3 grid(static_cast<unsigned>((nout + NOUT - 1) / NOUT), h->C);
    fir_decim_poly_kernel<D, Q, K, NOUT, NWARPS><<<grid, NWARPS * 32, smem, h->par()>>>(
        iq, stride, T, h->d_hist[h->hist_cur], h->H, h->d_taps1,
        static_cast<float2*>(h->r1.d), h->r1.mask, h->r1.stride, h->n_in, k0, k1, h->rot_fused ? h->d_rot : nullptr);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

template <int NTP, int K, int NTHREADS>
int launch_fir_d2(qrl_rx* h, const float2* iq, long long stride, long long T, long long k0, long long k1)
{
    constexpr int NOUT = NTHREADS * K;
    constexpr int W = 2 * (NOUT - 1) + NTP;
    const size_t smem = sizeof(float2) * (W + W / (2 * K) + 2);
    const long long nout = k1 - k0;
    dim3 grid(static_cast<unsigned>((nout + NOUT - 1) / NOUT), h->C);
    fir_decim2_kernel<NTP, K, NTHREADS><<<grid, NTHREADS, smem, h->par()>>>(
        iq, stride, T, h->d_hist[h->hist_cur], h->H, h->d_taps1,
        static_cast<float2*>(h->r1.d), h->r1.mask, h->r1.stride, h->n_in, k0, k1);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int launch_fir_resamp_2_25(qrl_rx* h, const float2* iq, long long stride, long long T, long long k0, long long k1)
{
    constexpr int L = 2, M = 25, NT = 105, NOUT = 512;
    constexpr int SPAN = (NOUT * M + L - 1) / L + NT + 1;
    const size_t smem = sizeof(float2) * SPAN;
    if (int rc = smem_opt_in(h, fir_resamp_ccf_kernel<L, M, NT, NOUT>, (int)smem)) return rc;
    dim3 grid(static_cast<unsigned>((k1 - k0 + NOUT - 1) / NOUT), h->C);
    fir_resamp_ccf_kernel<L, M, NT, NOUT><<<grid, 256, smem, h->par()>>>(iq, stride, T, h->d_hist[h->hist_cur], h->H, h->d_taps1,
        static_cast<float2*>(h->r1.d), h->r1.mask, h->r1.stride, h->n_in, k0, k1);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

using Stage1Launch = int (*)(qrl_rx*, const float2*, long long, long long, long long, long long);

// The register-tiled instance of the decimating stage 1 for the handle's (D, Q) shape, nullptr where none is built.  Only these
// instances rotate their window in shared memory (the carrier offset without an extra pass over HBM), so this one list decides both
// which kernel stage 1 runs and whether rx_work_impl needs the rotator pass.
Stage1Launch stage1_tiled(const qrl_rx* h)
{
    if (h->L1 != 1) return nullptr;
    if (h->D1 == 50 && h->Q1 == 9) return launch_fir_poly<50, 9, 8, 128, 8>;
    if (h->D1 == 100 && h->Q1 == 9) return launch_fir_poly<100, 9, 8, 64, 8>;      // 837 taps (4FSK-1k, QPSK-2k shape)
    if (h->D1 == 25 && h->Q1 == 9) return launch_fir_poly<25, 9, 8, 256, 8>;       // 209 taps (2FSK-2k)
    if (h->D1 == 125 && h->Q1 == 9) return launch_fir_poly<125, 9, 8, 48, 6>;      // 1045 taps (SSB)
    if (h->D1 == 25 && h->Q1 == 28) return launch_fir_poly<25, 28, 8, 192, 8>;     // 681 taps (QPSK-20k)
    if (h->D1 == 100 && h->Q1 == 28) return launch_fir_poly<100, 28, 8, 32, 4>;    // 2727 taps (QPSK-2k)
    return nullptr;
}

bool stage1_fuses_rotator(const qrl_rx* h) { return stage1_tiled(h) != nullptr; }

int stage1(qrl_rx* h, const float2* iq, long long stride, long long T, long long k0, long long k1)
{
    if (k1 <= k0) return QRL_OK;
    if (h->L1 == 2 && h->D1 == 25 && h->ntaps1 <= 210) return launch_fir_resamp_2_25(h, iq, stride, T, k0, k1);
    if (h->L1 > 2) {       // shape-generic rational resampler (M17: x3 / 125)
        const long long nout = k1 - k0;
        dim3 grid(static_cast<unsigned>((nout + 127) / 128), h->C);
        fir_resamp_hist_generic_kernel<<<grid, 128, 0, h->par()>>>(iq, stride, T, h->d_hist[h->hist_cur], h->H, h->d_taps1, h->nt_arm1,
            h->L1, h->D1, static_cast<float2*>(h->r1.d), h->r1.mask, h->r1.stride, h->n_in, k0, k1);
        h->launches++;
        QRL_CK(cudaGetLastError());
        return QRL_OK;
    }
    if (h->L1 != 1) { set_err(h, "stage-1 resampler shape not built"); return QRL_EINVAL; }
    if (Stage1Launch tiled = stage1_tiled(h)) return tiled(h, iq, stride, T, k0, k1);
    if (h->D1 == 2 && h->ntaps1 <= 56) return launch_fir_d2<56, 8, 128>(h, iq, stride, T, k0, k1);
    if (h->L1 == 1) {      // no register-tiled instance for this shape: one thread per output, same order, same history
        const long long nout = k1 - k0;
        dim3 grid(static_cast<unsigned>((nout + 127) / 128), h->C);
        fir_decim_hist_generic_kernel<<<grid, 128, 0, h->par()>>>(iq, stride, T, h->d_hist[h->hist_cur], h->H, h->d_taps1, h->ntaps1, h->D1,
            static_cast<float2*>(h->r1.d), h->r1.mask, h->r1.stride, h->n_in, k0, k1);
        h->launches++;
        QRL_CK(cudaGetLastError());
        return QRL_OK;
    }
    set_err(h, "stage-1 resampler shape not built (L=" + std::to_string(h->L1) + ", D=" + std::to_string(h->D1) + ", taps=" + std::to_string(h->ntaps1) + ")");
    return QRL_EINVAL;
}

template <class F>
F drv(const char* name)
{
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult st;
    if (cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &st) != cudaSuccess || st != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<F>(fn);
}

// split the device into {loop_sms} + {rest} and create the three internal streams; false -> caller falls back
bool make_sm_partition(qrl_rx* h, unsigned loop_sms, int prio, bool fec_on_par_default)
{
    if (const char* e = getenv("QRL_NO_SM_PARTITION")) { if (e[0] == '1') return false; }
    auto pDeviceGet = drv<CUresult (*)(CUdevice*, int)>("cuDeviceGet");
    auto pGetRes = drv<CUresult (*)(CUdevice, CUdevResource*, CUdevResourceType)>("cuDeviceGetDevResource");
    auto pSplit = drv<CUresult (*)(CUdevResource*, unsigned int*, const CUdevResource*, CUdevResource*, unsigned int, unsigned int)>("cuDevSmResourceSplitByCount");
    auto pDesc = drv<CUresult (*)(CUdevResourceDesc*, CUdevResource*, unsigned int)>("cuDevResourceGenerateDesc");
    auto pCreate = drv<CUresult (*)(CUgreenCtx*, CUdevResourceDesc, CUdevice, unsigned int)>("cuGreenCtxCreate");
    auto pStream = drv<CUresult (*)(CUstream*, CUgreenCtx, unsigned int, int)>("cuGreenCtxStreamCreate");
    if (!pDeviceGet || !pGetRes || !pSplit || !pDesc || !pCreate || !pStream) return false;
    CUdevice dev;
    if (pDeviceGet(&dev, h->device) != CUDA_SUCCESS) return false;
    CUdevResource all{}, grp{}, rest{};
    if (pGetRes(dev, &all, CU_DEV_RESOURCE_TYPE_SM) != CUDA_SUCCESS) return false;
    unsigned nb = 1;
    if (pSplit(&grp, &nb, &all, &rest, 0, loop_sms) != CUDA_SUCCESS || nb < 1) return false;
    CUdevResourceDesc d_loop, d_par;
    if (pDesc(&d_loop, &grp, 1) != CUDA_SUCCESS || pDesc(&d_par, &rest, 1) != CUDA_SUCCESS) return false;
    if (pCreate(&h->g_loop, d_loop, dev, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS) return false;
    if (pCreate(&h->g_par, d_par, dev, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS) return false;
    CUstream a = nullptr, b = nullptr, c = nullptr, d = nullptr;
    if (pStream(&a, h->g_loop, CU_STREAM_NON_BLOCKING, prio) != CUDA_SUCCESS) return false;
    // FEC (Viterbi) stream.  Up to 64 channels the step is the latency of the lone recurrence warps and the decoder runs on the wide
    // partition, off their SMs; with more channels the step is the sum of the parallel stages and the decoder stays in the loop
    // partition, out of their way.  QRL_FEC_ON_PAR=0/1 forces either.
    bool fec_on_par = fec_on_par_default;
    if (const char* e = getenv("QRL_FEC_ON_PAR")) fec_on_par = e[0] == '1';
    if (pStream(&b, fec_on_par ? h->g_par : h->g_loop, CU_STREAM_NON_BLOCKING, prio) != CUDA_SUCCESS) return false;
    if (pStream(&d, h->g_loop, CU_STREAM_NON_BLOCKING, prio) != CUDA_SUCCESS) return false;
    if (pStream(&c, h->g_par, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS) return false;
    CUstream e2 = nullptr;
    if (pStream(&e2, h->g_par, CU_STREAM_NON_BLOCKING, prio) != CUDA_SUCCESS) return false;
    h->s_loop = a; h->s_fec = b; h->s_par = c; h->s_loop2 = d; h->s_epi = e2;
    h->sm_loop = static_cast<int>(grp.sm.smCount); h->sm_par = static_cast<int>(rest.sm.smCount);
    return true;
}

// a carrier-offset change: from input sample n_in on, channel `channel` (every channel for channel < 0) turns by `inc` per sample,
// the phase kept continuous; returns whether any channel still rotates
bool retune(std::vector<RotState>& rot, int channel, unsigned inc, long long n_in)
{
    bool active = false;
    for (int c = 0; c < static_cast<int>(rot.size()); c++) {
        RotState& r = rot[c];
        if (channel < 0 || c == channel) {
            r.base = r.base + r.inc * static_cast<unsigned>(n_in - r.n_base);
            r.n_base = n_in;
            r.inc = inc;
        }
        if (r.inc != 0 || r.base != 0) active = true;
    }
    return active;
}

// interleaved = channel-interleaved layout [ceil(C/32)][slots][32] (allocated for the padded channel count)
// digital::fll_band_edge_cc::design_filter restated: returns lower[2N] | upper[2N] (complex, stored reversed)
std::vector<float> fll_design(float sps, float rolloff, int N)
{
    auto sinc = [](double x) { return x == 0 ? 1.0 : std::sin(kPi * x) / (kPi * x); };
    std::vector<float> bb(N), t(4 * N);
    const int M = static_cast<int>(std::rint(N / sps));
    float power = 0;
    for (int i = 0; i < N; i++) {
        const float k = static_cast<float>(-M + i * 2.0 / sps);
        const float tap = static_cast<float>(sinc(rolloff * k - 0.5) + sinc(rolloff * k + 0.5));
        power += tap; bb[i] = tap;
    }
    const int Nh = static_cast<int>((N - 1.0) / 2.0);
    for (int i = 0; i < N; i++) {
        const float tap = bb[i] / power;
        const float k = static_cast<float>((-Nh + i) / (2.0 * sps));
        const float ang = static_cast<float>(2.0 * kPi * (1 + rolloff) * k);
        t[2 * (N - i - 1)] = tap * cosf(-ang); t[2 * (N - i - 1) + 1] = tap * sinf(-ang);
        t[2 * N + 2 * (N - i - 1)] = tap * cosf(ang); t[2 * N + 2 * (N - i - 1) + 1] = tap * sinf(ang);
    }
    return t;
}

int make_ring(qrl_rx* h, Ring* r, size_t isz, long long min_items, bool interleaved = false)
{
    unsigned cap = pow2_at_least(min_items);
    r->mask = cap - 1;
    r->stride = cap;
    unsigned char* p = nullptr;
    const size_t nch = interleaved ? static_cast<size_t>((h->C + 31) / 32) * 32 : static_cast<size_t>(h->C);
    const size_t bytes = static_cast<size_t>(cap) * isz * nch;
    int rc = dev_alloc(h, &p, bytes, true);
    r->d = p;
    if (!rc) h->zero_list.emplace_back(p, bytes);
    return rc;
}

// low-rate stream filters: register-tiled instances for real calls, the one-thread-per-output kernels for slivers
int launch_fir_ccf_c(HandleBase* h, int C, cudaStream_t st, const float2* in, unsigned in_mask, long long in_stride, float2* out, unsigned out_mask, long long out_stride,
                     const float* taps, int ntaps, long long a0, long long a1, float2* lin, long long lin_stride, long long lin_base, int interleaved)
{
    const long long n = a1 - a0;
    if (n <= 0) return QRL_OK;
    constexpr int K = 8, NT = 128, TILE = K * NT;
    const int span = TILE + ntaps - 1;
    const size_t smem = sizeof(float) * ((ntaps + 1) & ~1) + sizeof(float2) * (span + (span >> 4) + 2);
    if (smem > 48 * 1024 && smem <= 100 * 1024) {            // long filters (gr_mod_am's 4545-tap output filter): opt in to the larger window once per device
        if (int rc = smem_opt_in(h, fir_ccf_ring_tiled_kernel<K, NT>, 100 * 1024)) return rc;
    }
    if (n >= 256 && smem <= 100 * 1024 && ntaps >= K) {      // (the tiled kernel's head / tail phases assume at least K taps)
        dim3 g(static_cast<unsigned>((n + TILE - 1) / TILE), C);
        fir_ccf_ring_tiled_kernel<K, NT><<<g, NT, smem, st>>>(in, in_mask, in_stride, out, out_mask, out_stride, taps, ntaps, a0, a1, lin, lin_stride, lin_base, interleaved);
    } else {
        dim3 g(static_cast<unsigned>((n + 255) / 256), C);
        fir_ccf_ring_kernel<<<g, 256, sizeof(float) * ntaps, st>>>(in, in_mask, in_stride, out, out_mask, out_stride, taps, ntaps, a0, a1, lin, lin_stride, lin_base, interleaved);
    }
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int launch_fir_ccf(qrl_rx* h, cudaStream_t st, const float2* in, unsigned in_mask, long long in_stride, float2* out, unsigned out_mask, long long out_stride,
                   const float* taps, int ntaps, long long a0, long long a1, float2* lin, long long lin_stride, long long lin_base, int interleaved)
{
    return launch_fir_ccf_c(h, h->C, st, in, in_mask, in_stride, out, out_mask, out_stride, taps, ntaps, a0, a1, lin, lin_stride, lin_base, interleaved);
}
int launch_qdemod_fir(qrl_rx* h, cudaStream_t st, const float2* in, unsigned in_mask, long long in_stride, float* out, unsigned out_mask, long long out_stride,
                      const float* taps, int ntaps, float gain, long long a0, long long a1)
{
    const long long n = a1 - a0;
    if (n <= 0) return QRL_OK;
    constexpr int K = 8, NT = 128, TILE = K * NT;
    const int span = TILE + ntaps - 1;
    const size_t smem = sizeof(float) * (ntaps + span + (span >> 5) + 2);
    if (n >= 256 && smem <= 48 * 1024 && ntaps >= K) {
        dim3 g(static_cast<unsigned>((n + TILE - 1) / TILE), h->C);
        qdemod_fir_fff_tiled_kernel<K, NT><<<g, NT, smem, st>>>(in, in_mask, in_stride, out, out_mask, out_stride, taps, ntaps, gain, a0, a1);
    } else {
        dim3 g(static_cast<unsigned>((n + 255) / 256), h->C);
        qdemod_fir_fff_kernel<<<g, 256, sizeof(float) * (2 * ntaps + 256), st>>>(in, in_mask, in_stride, out, out_mask, out_stride, taps, ntaps, gain, a0, a1, nullptr, 0);
    }
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

// symbols one CH-row symbol-sync window can hold (the shortest symbol period is min_period - |alpha|)
int symsync_maxs(const SymSyncParams& p, int CH)
{
    return static_cast<int>((CH + 1) / (p.min_period - fabsf(p.alpha)) + 3);
}

// dynamic shared memory of the 4FSK-FM symbol sync with the external epilogue: NST input stages of CH rows x 32 channels, the tap
// table, two symbol windows and the header; rep adds the replicated (conflict-free) interpolator bank.  rx_create chooses ss_ch and
// sizes the epilogue scratch with it, and the launch uses it, so the two always agree.
size_t symsync_ext_smem(const SymSyncParams& p, int CH, int NST, bool rep)
{
    return sizeof(float) * (NST * CH * 32 + SYMSYNC_TAB_FLOATS + 2 * (symsync_maxs(p, CH) + 2) * 32) + sizeof(int) * 64 + (rep ? 129 * 512 : 0);
}

// ---- the receive chains behind stage 1.  rx_work_impl cuts each call into slices, runs stage 1 and hands every slice to the
// slice function of the handle's chain, which queues the rest of that slice on the parallel, loop and FEC streams.

constexpr int kTileThreads = 256;       // CTA size of the per-output stream filters (Slice::gtile)

// slice i of a call: the stage-1 outputs [k0, k1) are new
struct Slice {
    int i;
    long long k0, k1, n_new;
    long long k_call0;          // stage-1 index of the call's first output (port 0 of the call starts there)
    long long* nsoft_i;         // [C] soft-bit write index snapshots of this slice
    cudaStream_t sp;            // stream of the parallel stages
    dim3 gtile;                 // kTileThreads-thread CTAs over the new outputs, one row per channel
    int groups;                 // CTAs of 32 channels (the loop kernels)
};

// `to` runs on behind everything queued on `from` so far
int hand_off(qrl_rx* h, cudaEvent_t ev, cudaStream_t from, cudaStream_t to)
{
    QRL_CK(cudaEventRecord(ev, from));
    QRL_CK(cudaStreamWaitEvent(to, ev, 0));
    return QRL_OK;
}

// fll_band_edge_cc (sequential, per sample) on the loop stream: r1 -> rf
void launch_fll(qrl_rx* h, const Slice& s)
{
    fll_kernel<32><<<s.groups, 32, 0, h->s_loop>>>(h->fllp, h->d_fll, h->d_fll_hist, h->C, h->d_fll_taps,
        static_cast<const float2*>(h->r1.d), h->r1.mask, h->r1.stride, s.k1,
        static_cast<float2*>(h->rf.d), h->rf.mask, h->rf.stride);
    h->launches++;
}

// the channel / shaping filter of a slice on `st`: `in` -> r2 (channel-interleaved when `interleaved`) and port 0
int launch_channel_filter(qrl_rx* h, const Slice& s, cudaStream_t st, const Ring& in, int interleaved)
{
    return launch_fir_ccf(h, st, static_cast<const float2*>(in.d), in.mask, in.stride, static_cast<float2*>(h->r2.d), h->r2.mask, h->r2.stride,
                          h->d_taps2, h->ntaps2, s.k0, s.k1, h->d_port0, h->port0_cap, s.k_call0, interleaved);
}

// one symbol-sync launch on `st` over the input ring `in` up to k1 (opting the instance in to `smem_max` bytes first); only the
// 4FSK-FM symbol sync with the external epilogue passes the epilogue's scratch, chunk bound, chunk capacity and header
template <class K>
int launch_symsync(qrl_rx* h, K* kern, int smem_max, int grid, int threads, size_t smem, cudaStream_t st, const Ring& in, long long k1,
                   int maxs, long long* nsoft_i, float* scratch = nullptr, int chunk_bound = 0, int chunk_cap = 0, int* hdr = nullptr)
{
    if (int rc = smem_opt_in(h, kern, smem_max)) return rc;
    kern<<<grid, threads, smem, st>>>(
        h->ssp, h->d_ss, h->C, static_cast<const float*>(in.d), in.mask, in.stride, k1,
        h->d_port1, h->port1_cap, h->d_port1_cnt, static_cast<int>(h->port1_cap),
        static_cast<unsigned char*>(h->r5.d), h->r5.mask, h->r5.stride, maxs, nsoft_i, scratch, chunk_bound, chunk_cap, hdr);
    h->launches++;
    return QRL_OK;
}

// stage 5 on the FEC stream: Viterbi + descrambler over the slice's soft bits -> port 2; dual: a second decoder on the same soft
// stream behind delay(1) -> port 3
void launch_viterbi(qrl_rx* h, long long* nsoft_i, bool dual)
{
    constexpr int CPB = 4;    // 4 channels (8 warps) per CTA
    cudaEvent_t pe = h->prof.begin(4, h->s_fec);
    viterbi_k7_kernel<CPB><<<(h->C + CPB - 1) / CPB, 64 * CPB, 0, h->s_fec>>>(h->d_vs, nsoft_i, h->C,
        static_cast<const unsigned char*>(h->r5.d), h->r5.mask, h->r5.stride,
        h->d_port2, h->port2_cap, h->d_port2_cnt, static_cast<int>(h->port2_cap), 0);
    if (dual)
        viterbi_k7_kernel<CPB><<<(h->C + CPB - 1) / CPB, 64 * CPB, 0, h->s_fec>>>(h->d_vs2, nsoft_i, h->C,
            static_cast<const unsigned char*>(h->r5.d), h->r5.mask, h->r5.stride,
            h->d_port3, h->port2_cap, h->d_port3_cnt, static_cast<int>(h->port2_cap), 1);
    h->launches += dual ? 2 : 1;
    h->prof.end(pe);
}

// gr_demod_dsss: the whole chain in one kernel on the loop stream, then the two decoders
int slice_dsss(qrl_rx* h, const Slice& s)
{
    if (int rc = hand_off(h, h->ev_a[s.i], s.sp, h->s_loop)) return rc;
    cudaEvent_t pe = h->prof.begin(3, h->s_loop);
    dsss_chain_kernel<<<h->C, 256, 0, h->s_loop>>>(h->dsp, h->d_ds, static_cast<const float2*>(h->r1.d), h->r1.mask, h->r1.stride, s.k1,
        h->d_ds_arms, h->d_taps2, h->d_ds_taps,
        static_cast<float2*>(h->ds_a.d), static_cast<float2*>(h->ds_c.d), h->ds_a.mask, h->ds_a.stride,
        static_cast<float2*>(h->ds_d.d), h->ds_d.mask, h->ds_d.stride,
        h->d_port0, h->port0_cap, h->ds_o_call0,
        h->d_port1, h->port1_cap, h->d_port1_cnt, static_cast<int>(h->port1_cap),
        static_cast<unsigned char*>(h->r5.d), h->r5.mask, h->r5.stride, s.nsoft_i);
    h->launches++;
    h->prof.end(pe);
    if (int rc = hand_off(h, h->ev_b[s.i], h->s_loop, h->s_fec)) return rc;
    launch_viterbi(h, s.nsoft_i, true);
    return QRL_OK;
}

// SSB, FreeDV, AM, NBFM, WBFM: channel / side-band filter on the parallel stream (-> port 0), then the audio chain on the loop stream
// (NBFM: its de-emphasis on the second loop stream)
int slice_analog(qrl_rx* h, const Slice& s)
{
    cudaEvent_t pe;
    if (s.n_new > 0) {
        pe = h->prof.begin(1, s.sp);
        if (h->kind == QRL_DEMOD_NBFM || h->kind == QRL_DEMOD_WBFM) {
            if (int rc = launch_channel_filter(h, s, s.sp, h->r1, 0)) return rc;
        } else {
            fir_ccc_ring_kernel<<<s.gtile, kTileThreads, sizeof(float) * 2 * h->ntaps2, s.sp>>>(
                static_cast<const float2*>(h->r1.d), h->r1.mask, h->r1.stride,
                static_cast<float2*>(h->r2.d), h->r2.mask, h->r2.stride,
                h->d_taps2, h->ntaps2, 1.0f, s.k0, s.k1, h->d_port0, h->port0_cap, s.k_call0);
            h->launches++;
        }
        h->prof.end(pe);
    }
    if (int rc = hand_off(h, h->ev_a[s.i], s.sp, h->s_loop)) return rc;
    pe = h->prof.begin(3, h->s_loop);
    const size_t fat = h->nbfm_split ? 120 * 1024 : 0;       // one CTA per SM, and never next to a de-emphasis CTA
    switch (h->kind) {
    case QRL_DEMOD_SSB:
        ssb_audio_kernel<<<h->C, 128, 0, h->s_loop>>>(h->ssbp, h->d_ssb,
            static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, s.k1,
            static_cast<float2*>(h->rclip.d), h->rclip.mask, h->rclip.stride,
            static_cast<float*>(h->rstr.d), h->rstr.mask, h->rstr.stride,
            h->d_audio_taps, h->d_port1f, 2 * h->port1_cap, h->d_port1_cnt, static_cast<int>(2 * h->port1_cap));
        break;
    case QRL_DEMOD_FREEDV:
        freedv_rx_tail_kernel<<<h->C, 128, sizeof(float) * h->fdp.nt_audio, h->s_loop>>>(h->fdp, h->d_fdv,
            static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, s.k1,
            static_cast<float*>(h->rstr.d), h->rstr.mask, h->rstr.stride, h->d_audio_taps,
            reinterpret_cast<short*>(h->d_port1), 4 * h->port1_cap, h->d_port1_cnt, static_cast<int>(4 * h->port1_cap));
        break;
    default:    // AM, NBFM, WBFM (the de-emphasis ring and the CTCSS squelch ring only exist for NBFM; empty otherwise)
        if (h->nbfm_split) {
            int rc;
            if ((rc = smem_opt_in(h, nbfm_audio_kernel, 120 * 1024)) || (rc = smem_opt_in(h, nbfm_deemph_kernel, 120 * 1024))) return rc;
        }
        nbfm_audio_kernel<<<h->C, 128, fat, h->s_loop>>>(h->nbp, h->d_nb,
            static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, s.k1, h->d_env,
            static_cast<float2*>(h->rg.d), h->rg.mask, h->rg.stride,
            static_cast<float*>(h->rd.d), h->rd.mask, h->rd.stride,
            static_cast<float*>(h->rr.d), h->rr.mask, h->rr.stride,
            h->d_arm_taps, h->d_audio_taps, h->d_port1f, 2 * h->port1_cap, h->d_port1_cnt, static_cast<int>(2 * h->port1_cap),
            h->nbfm_split ? static_cast<float*>(h->raud.d) : nullptr, h->raud.mask, h->raud.stride, h->nbfm_split ? s.nsoft_i : nullptr,
            static_cast<float*>(h->rq.d), h->rq.mask, h->rq.stride, h->ctc, h->d_cenv);
    }
    h->launches++;
    h->prof.end(pe);
    if (h->nbfm_split) {
        if (int rc = hand_off(h, h->ev_b[s.i], h->s_loop, h->s_loop2)) return rc;
        pe = h->prof.begin(5, h->s_loop2);
        nbfm_deemph_kernel<<<h->C, 128, fat, h->s_loop2>>>(h->nbp.b0, h->nbp.b1, h->nbp.a1, h->nbp.out_gain, h->d_nb2,
            static_cast<const float*>(h->raud.d), h->raud.mask, h->raud.stride, s.nsoft_i,
            h->d_port1f, 2 * h->port1_cap, h->d_port1_cnt, static_cast<int>(2 * h->port1_cap));
        h->launches++;
        h->prof.end(pe);
    }
    return QRL_OK;
}

// BPSK, 2FSK, GMSK: FLL (not GMSK), channel filter / RRC and detector, agc2 (BPSK), symbol sync, all on the loop stream; then the
// two decoders
int slice_fll_bpsk_2fsk(qrl_rx* h, const Slice& s)
{
    const bool bpsk = h->kind == QRL_DEMOD_BPSK;
    if (int rc = hand_off(h, h->ev_a[s.i], s.sp, h->s_loop)) return rc;
    cudaEvent_t pe = h->prof.begin(1, h->s_loop);
    if (!h->gmsk) launch_fll(h, s);
    h->prof.end(pe);
    if (s.n_new > 0) {
        // ---- channel filter / RRC on the FLL output -> port 0 (+ ring: channel-major for 2FSK, interleaved for BPSK)
        pe = h->prof.begin(2, h->s_loop);
        if (int rc = launch_channel_filter(h, s, h->s_loop, h->gmsk ? h->r1 : h->rf, bpsk ? 1 : 0)) return rc;     // GMSK: no FLL
        if (!bpsk && h->flag) {
            if (int rc = launch_qdemod_fir(h, h->s_loop, static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride,
                                           static_cast<float*>(h->r4.d), h->r4.mask, h->r4.stride,
                                           h->d_taps3, h->ntaps3, h->qd_gain, s.k0, s.k1)) return rc;
        } else if (!bpsk) {
            fsk_bank_kernel<2><<<s.gtile, kTileThreads, sizeof(float) * 4 * h->nt_bank, h->s_loop>>>(
                static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, h->d_bank_taps, h->nt_bank, s.k0, s.k1,
                static_cast<float*>(h->rbank.d), h->rbank.mask, h->rbank.stride);
            fir_fff_ring_kernel<<<s.gtile, kTileThreads, sizeof(float) * h->nt_symf, h->s_loop>>>(
                static_cast<const float*>(h->rbank.d), h->rbank.mask, h->rbank.stride,
                static_cast<float*>(h->r4.d), h->r4.mask, h->r4.stride, h->d_symf_taps, h->nt_symf, s.k0, s.k1);
            h->launches += 2;
        }
        h->prof.end(pe);
    }
    pe = h->prof.begin(3, h->s_loop);
    if (bpsk) {
        {   // agc2_cc (Costas bypassed): r2 -> r3
            constexpr int CH = 128, NST = 2;
            const size_t smem = sizeof(float2) * (NST * CH + AC_NHB * (CH + 1)) * 32;      // every hand-off block + its padding row
            auto kern = agc_costas_kernel<CH, NST, 0, 0>;
            if (int rc = smem_opt_in(h, kern, 200 * 1024)) return rc;
            kern<<<s.groups, 96, smem, h->s_loop>>>(h->acp, h->d_ac, h->C,
                static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, s.k1,
                static_cast<float2*>(h->r3.d), h->r3.mask, h->r3.stride);
            h->launches++;
        }
        // clock_recovery_mm_cc: its window bound is (CH + 1) / min_period symbols
        constexpr int CH = 128, NST = 3, NEPI = 1;
        const int maxs = static_cast<int>((CH + 1) / (h->ssp.min_period) + 3);
        const size_t smem = sizeof(float) * (NST * CH * 64 + SYMSYNC_TAB_FLOATS + 2 * maxs * 64) + sizeof(int) * 64;
        if (int rc = launch_symsync(h, symsync_kernel<2, SL_BPSK, EPI_BPSK, CH, NST, NEPI, LOOP_CRMM>, 200 * 1024, s.groups, 64 + 32 * NEPI,
                                    smem, h->s_loop, h->r3, s.k1, maxs, s.nsoft_i)) return rc;
    } else {
        constexpr int CH = 256, NST = 3, NEPI = 2;
        const int maxs = symsync_maxs(h->ssp, CH);
        const size_t smem = sizeof(float) * (NST * CH * 32 + SYMSYNC_TAB_FLOATS + 2 * maxs * 32) + sizeof(int) * 64;
        if (int rc = launch_symsync(h, symsync_kernel<1, SL_BPSK, EPI_REAL1, CH, NST, NEPI>, 200 * 1024, s.groups, 64 + 32 * NEPI,
                                    smem, h->s_loop, h->r4, s.k1, maxs, s.nsoft_i)) return rc;
    }
    h->prof.end(pe);
    if (int rc = hand_off(h, h->ev_b[s.i], h->s_loop, h->s_fec)) return rc;
    launch_viterbi(h, s.nsoft_i, true);
    return QRL_OK;
}

// 4FSK-FM symbol sync with CH-row windows and NST input stages: lean recurrence on the loop stream + external epilogue (symbols leave
// the SM by TMA bulk store; the phase modulator / soft-bit stores run on the wide partition behind it, on s_epi when there is one)
template <int CH, int NST>
int symsync_4fsk_ext(qrl_rx* h, const Slice& s)
{
    cudaEvent_t pe = h->prof.begin(3, h->s_loop);
    const int maxs = symsync_maxs(h->ssp, CH);
    const bool rep = symsync_ext_smem(h->ssp, CH, NST, true) <= 220 * 1024 && !h->dmr;
    // gr_demod_dmr: TED_MUELLER_AND_MULLER instead of the modified detector -> generic recurrence, variant 3
    auto kern = h->dmr ? symsync_kernel<1, SL_RECT4, EPI_EXT_4FSK_FM, CH, NST, 1, LOOP_SYMSYNC, 3>
              : rep ? symsync_kernel<1, SL_RECT4, EPI_EXT_4FSK_FM, CH, NST, 1, LOOP_SYMSYNC, 2>
                    : symsync_kernel<1, SL_RECT4, EPI_EXT_4FSK_FM, CH, NST, 1, LOOP_SYMSYNC, 1>;
    // overlapped calls: the previous call's Viterbi of slice i still reads d_nsoft[i], its epilogue scratch region i
    if (h->overlap) QRL_CK(cudaStreamWaitEvent(h->s_loop, h->ev_v[s.i], 0));
    // every slice of a call gets its own scratch region and header (the epilogue of slice i overlaps symsync i+1)
    if (s.i == 0) h->ss_chunk_off = 0;
    const int chunk_bound = static_cast<int>(std::min<long long>(h->ss_chunk_cap - h->ss_chunk_off, s.n_new / symsync_stride(CH, h->ssp.lookahead) + 3));
    float* scratch_i = h->d_ss_scratch + static_cast<size_t>(h->ss_chunk_off) * (maxs + 2) * 32;
    int* hdr_i = h->d_ss_hdr + static_cast<size_t>(s.i) * s.groups * 128;
    h->ss_chunk_off += chunk_bound;
    if (int rc = launch_symsync(h, kern, 224 * 1024, s.groups, 96, symsync_ext_smem(h->ssp, CH, NST, rep), h->s_loop, h->r4, s.k1, maxs,
                                s.nsoft_i, scratch_i, chunk_bound, static_cast<int>(h->ss_chunk_cap), hdr_i)) return rc;
    h->prof.end(pe);
    cudaStream_t se = h->s_epi ? h->s_epi : h->s_loop;
    if (se != h->s_loop || h->overlap) QRL_CK(cudaEventRecord(h->ev_c[s.i], h->s_loop));
    if (se != h->s_loop) QRL_CK(cudaStreamWaitEvent(se, h->ev_c[s.i], 0));
    pe = h->prof.begin(5, se);
    auto epi = h->dmr ? symsync_ext_epilogue_kernel<1> : symsync_ext_epilogue_kernel<0>;
    if (chunk_bound > 0)        // (counted in h->launches with the symbol sync it finishes)
        epi<<<dim3(chunk_bound, s.groups), dim3(32, 8), 0, se>>>(
            h->ssp, h->C, scratch_i, static_cast<int>(h->ss_chunk_cap), maxs, hdr_i,
            h->d_port1, h->port1_cap, static_cast<int>(h->port1_cap),
            static_cast<unsigned char*>(h->r5.d), h->r5.mask, h->r5.stride,
            h->m17 ? h->d_port2 : nullptr, h->port2_cap, static_cast<int>(h->port2_cap), h->d_port2_cnt, h->d_port1_cnt);
    h->prof.end(pe);
    QRL_CK(cudaEventRecord(h->ev_b[s.i], se));
    return QRL_OK;
}

// 4FSK (FM discriminator or band-pass bank), M17, DMR: channel filter and detector on the parallel stream, symbol sync on the loop
// stream, then the decoder (M17: none)
int slice_4fsk(qrl_rx* h, const Slice& s)
{
    cudaEvent_t pe;
    if (s.n_new > 0) {
        // ---- stage 2: channel filter -> ring + port 0
        pe = h->prof.begin(1, s.sp);
        if (int rc = launch_channel_filter(h, s, s.sp, h->r1, 0)) return rc;
        h->prof.end(pe);
        // ---- stage 3: quadrature demod + RRC   |   band-pass bank + discriminator + symbol filter
        // overlapped calls: this slice overwrites ring slots the previous call's symbol sync (slices i, i+1) read
        if (h->overlap && h->prev_nsub > 0) {
            // the slots [k0, k1) overwrite the samples cap older; the previous call's symbol sync of slice q has
            // consumed everything up to prev_k1[q] - lookahead
            const long long must = s.k1 - (static_cast<long long>(h->r4.mask) + 1) + 64;
            int q = -1;
            for (int j = 0; j < h->prev_nsub; j++) if (h->prev_k1[j] - 64 < must) q = j;      // not yet safe after slice j alone
            if (q >= 0) QRL_CK(cudaStreamWaitEvent(s.sp, h->ev_c[std::min(q + 1, h->prev_nsub - 1)], 0));
        }
        pe = h->prof.begin(2, s.sp);
        if (h->flag) {
            if (int rc = launch_qdemod_fir(h, s.sp, static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride,
                                           static_cast<float*>(h->r4.d), h->r4.mask, h->r4.stride,
                                           h->d_taps3, h->ntaps3, h->qd_gain, s.k0, s.k1)) return rc;
            if (h->dmr) {      // gr_demod_dmr.cpp:103: the symbol filter output is port 3
                ring_to_port_f32_kernel<<<dim3(static_cast<unsigned>((s.k1 - s.k0 + 31) / 32), s.groups), dim3(32, 8), 0, s.sp>>>(
                    static_cast<const float*>(h->r4.d), h->r4.mask, h->r4.stride, h->C, s.k0, s.k1,
                    h->d_port3f, h->port0_cap, s.k0 - s.k_call0);
                h->launches++;
            }
        } else {
            fsk_bank_kernel<4><<<s.gtile, kTileThreads, sizeof(float) * 8 * h->nt_bank, s.sp>>>(
                static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, h->d_bank_taps, h->nt_bank, s.k0, s.k1,
                static_cast<float*>(h->rbank.d), h->rbank.mask, h->rbank.stride);
            h->launches++;
            if (int rc = launch_fir_ccf(h, s.sp, static_cast<const float2*>(h->rbank.d), h->rbank.mask, h->rbank.stride,
                                        static_cast<float2*>(h->r3.d), h->r3.mask, h->r3.stride,
                                        h->d_symf_taps, h->nt_symf, s.k0, s.k1, nullptr, 0, 0, 1)) return rc;
        }
        h->prof.end(pe);
    }
    // ---- stage 4: symbol sync (+ phase mod + soft bits) on the loop stream
    if (int rc = hand_off(h, h->ev_a[s.i], s.sp, h->s_loop)) return rc;
    if (h->flag) {
        const int rc = h->ss_ch == 512 ? symsync_4fsk_ext<512, 2>(h, s) : symsync_4fsk_ext<256, 3>(h, s);
        if (rc) return rc;
    } else {
        pe = h->prof.begin(3, h->s_loop);
        constexpr int CH = 128, NST = 3, NEPI = 2;
        const int maxs = symsync_maxs(h->ssp, CH);
        const size_t smem = sizeof(float) * (NST * CH * 64 + SYMSYNC_TAB_FLOATS + 2 * maxs * 64) + sizeof(int) * 64;
        if (int rc = launch_symsync(h, symsync_kernel<2, SL_RECT4, EPI_CPLX, CH, NST, NEPI>, 200 * 1024, s.groups, 64 + 32 * NEPI,
                                    smem, h->s_loop, h->r3, s.k1, maxs, s.nsoft_i)) return rc;
        h->prof.end(pe);
        QRL_CK(cudaEventRecord(h->ev_b[s.i], h->s_loop));
    }
    // ---- stage 5: Viterbi + descrambler on the FEC stream
    QRL_CK(cudaStreamWaitEvent(h->s_fec, h->ev_b[s.i], 0));
    // gr_demod_m17 has no FEC: the epilogue wrote the hard bits of port 2 (s_fec joins it at the end)
    if (!h->m17) launch_viterbi(h, s.nsoft_i, false);
    if (h->overlap) QRL_CK(cudaEventRecord(h->ev_v[s.i], h->s_fec));
    return QRL_OK;
}

// QPSK agc2 + Costas "PLL" on the loop stream (r2 -> r3): CH-row windows, 2 input stages + the hand-off blocks (164 KB at CH = 128)
template <int CH>
int qpsk_agc_costas(qrl_rx* h, const Slice& s)
{
    constexpr int NST = 2;
    const size_t smem = sizeof(float2) * (NST * CH + AC_NHB * (CH + 1)) * 32;      // every hand-off block + its padding row
    auto kern = (h->acp.order == 4 && h->acp.use_snr) ? agc_costas_kernel<CH, NST, 4, 1> : agc_costas_kernel<CH, NST>;
    int rc;                                 // both instantiations, whichever this call takes
    if ((rc = smem_opt_in(h, agc_costas_kernel<CH, NST, 4, 1>, 200 * 1024)) || (rc = smem_opt_in(h, agc_costas_kernel<CH, NST>, 200 * 1024))) return rc;
    kern<<<s.groups, 96, smem, h->s_loop>>>(h->acp, h->d_ac, h->C,
        static_cast<const float2*>(h->r2.d), h->r2.mask, h->r2.stride, s.k1,
        static_cast<float2*>(h->r3.d), h->r3.mask, h->r3.stride);
    h->launches++;
    return QRL_OK;
}

// QPSK symbol sync + second Costas + diff phasor + soft bits on the second loop stream.  LEAN: the prefetching complex recurrence
// (symbol-sync variant 2, replicated tap bank) with the epilogue split into a Costas warp and a feed-forward warp over a 3-deep symbol
// ring (NEPI = 2); else the generic recurrence, one epilogue warp
template <int CH, int NST, bool LEAN>
int qpsk_symsync(qrl_rx* h, const Slice& s)
{
    constexpr int NEPI = LEAN ? 2 : 1, NB = LEAN ? 3 : 2;
    const int maxs = symsync_maxs(h->ssp, CH);
    const size_t smem = sizeof(float) * (NST * CH * 64 + SYMSYNC_TAB_FLOATS + NB * maxs * 64) + sizeof(int) * 32 * (NB == 2 ? 2 : 4) +
                        (LEAN ? 129 * 512 : 0);
    if (smem > 224 * 1024) { set_err(h, "QPSK symbol sync: window does not fit shared memory"); return QRL_EINVAL; }
    return launch_symsync(h, symsync_kernel<2, SL_DQPSK, EPI_QPSK, CH, NST, NEPI, LOOP_SYMSYNC, LEAN ? 2 : 0>, 224 * 1024, s.groups,
                          64 + 32 * NEPI, smem, h->s_loop2, h->r3, s.k1, maxs, s.nsoft_i);
}

// QPSK: FLL (sps > 4) on the loop stream, RRC shaping filter on the parallel stream, agc2 + Costas on the loop stream, symbol sync on
// the second loop stream, then the decoder
int slice_qpsk(qrl_rx* h, const Slice& s)
{
    if (h->d_fll) {     // sps > 4: fll_band_edge_cc between resampler and shaping filter (sequential, on the loop stream)
        if (int rc = hand_off(h, h->ev_a[s.i], s.sp, h->s_loop)) return rc;
        launch_fll(h, s);
        if (int rc = hand_off(h, h->ev_c[s.i], h->s_loop, s.sp)) return rc;
    }
    cudaEvent_t pe;
    if (s.n_new > 0) {
        // ---- stage 2: RRC shaping filter -> interleaved ring + port 0
        pe = h->prof.begin(1, s.sp);
        if (int rc = launch_channel_filter(h, s, s.sp, h->d_fll ? h->rf : h->r1, 1)) return rc;
        h->prof.end(pe);
    }
    // ---- stage 3: agc2 + costas "PLL" per sample on the loop stream
    if (int rc = hand_off(h, h->ev_a[s.i], s.sp, h->s_loop)) return rc;
    pe = h->prof.begin(2, h->s_loop);
    // many channels: 32-row windows (41 KB of shared memory, five CTAs per SM) instead of 128-row ones (164 KB)
    if (int rc = h->many ? qpsk_agc_costas<32>(h, s) : qpsk_agc_costas<128>(h, s)) return rc;
    h->prof.end(pe);
    // ---- stage 4: symbol sync on the second loop stream
    if (int rc = hand_off(h, h->ev_c[s.i], h->s_loop, h->s_loop2)) return rc;
    pe = h->prof.begin(3, h->s_loop2);
    // many channels: 64-row windows, two stages (~55 KB, four CTAs per SM) instead of 128-row ones
    const bool small_win = h->many && symsync_stride(64, h->ssp.lookahead) >= 32;
    static const bool lean_env = [] { const char* e = getenv("QRL_QPSK_LEAN_SS"); return !(e && e[0] == '0'); }();
    // the lean recurrence needs the in-lock window proof (kernel: lean_ok && window_sure) -- true for every QPSK instance of
    // gr_demod_base.cpp; the kernel itself falls back to the generic loop when it does not hold
    const int rc = small_win ? qpsk_symsync<64, 2, false>(h, s) : lean_env ? qpsk_symsync<128, 2, true>(h, s) : qpsk_symsync<128, 3, false>(h, s);
    if (rc) return rc;
    h->prof.end(pe);
    // ---- stage 5: Viterbi + descrambler on the FEC stream
    if (int rc2 = hand_off(h, h->ev_b[s.i], h->s_loop2, h->s_fec)) return rc2;
    launch_viterbi(h, s.nsoft_i, false);
    return QRL_OK;
}

}  // namespace

extern "C" {

int qrl_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
const char* qrl_version(void) { return "qrl_b200 0.1 (sm_90a)"; }
const char* qrl_last_error(const void* handle)
{
    if (handle) return static_cast<const HandleBase*>(handle)->err.c_str();
    return thread_last_error().c_str();
}

// gr_demod_freedv / gr_mod_freedv factory arguments the reference does not check itself: the chain only holds together at 8 ksps
static int check_freedv_args(const char* who, int sps, int samp_rate, int filter_width, int low_cutoff)
{
    if (sps <= 0 || samp_rate / sps != 8000) { set_err(nullptr, std::string(who) + ": samp_rate / sps must be 8000 (the codec2 modem rate)"); return QRL_EINVAL; }
    if (low_cutoff < 0 || low_cutoff >= filter_width || filter_width > 4000) {
        set_err(nullptr, std::string(who) + ": need 0 <= low_cutoff < filter_width <= 4000 (the side band of an 8 ksps stream)");
        return QRL_EINVAL;
    }
    return QRL_OK;
}

static int rx_create(int kind, int sps, int samp_rate, int carrier_freq, int filter_width, int flag, int low_cutoff,
                     int n_channels, long max_samples, int device, qrl_rx** out);

int qrl_rx_create(int kind, int sps, int samp_rate, int carrier_freq, int filter_width, int flag,
                  int n_channels, long max_samples, int device, qrl_rx** out)
{
    if (kind == QRL_DEMOD_FREEDV) { set_err(nullptr, "qrl_rx_create: QRL_DEMOD_FREEDV takes a low cutoff: use qrl_rx_create_freedv"); return QRL_EINVAL; }
    return rx_create(kind, sps, samp_rate, carrier_freq, filter_width, flag, 0, n_channels, max_samples, device, out);
}

int qrl_rx_create_freedv(int sps, int samp_rate, int carrier_freq, int filter_width, int low_cutoff, int sb,
                         int n_channels, long max_samples, int device, qrl_rx** out)
{
    int rc = check_freedv_args("qrl_rx_create_freedv", sps, samp_rate, filter_width, low_cutoff);
    if (rc) return rc;
    return rx_create(QRL_DEMOD_FREEDV, sps, samp_rate, carrier_freq, filter_width, sb ? 1 : 0, low_cutoff, n_channels, max_samples, device, out);
}

static int rx_create(int kind, int sps, int samp_rate, int carrier_freq, int filter_width, int flag, int low_cutoff,
                     int n_channels, long max_samples, int device, qrl_rx** out)
{
    if (!out || n_channels <= 0 || max_samples <= 0) { set_err(nullptr, "qrl_rx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_rx_create", device)) return rc;
    // gr_demod_gmsk.cpp:30-134 is the 2FSK (fm) chain without the band-edge FLL, with a plain low-pass as symbol filter and its
    // own clock-loop constants: it runs through the 2FSK code path
    const bool gmsk = (kind == QRL_DEMOD_GMSK);
    if (gmsk) { kind = QRL_DEMOD_2FSK; flag = 1; }
    // gr_demod_m17.cpp:30-113 is the 4FSK (fm) chain behind a x3 / 125 rational resampler (24 ksps, 5 samples per symbol) with a
    // hard-decision bit tail instead of the FEC: it runs through the 4FSK code path
    // gr_demod_dmr.cpp:32-112 is that M17 chain again with its own stage-1 taps, no IF filter, a 0.2 roll-off symbol filter tapped as
    // (float) port 3, the PLAIN Mueller & Mueller detector in the symbol sync and x0.9 in front of the phase modulator
    const bool dmr = (kind == QRL_DEMOD_DMR);
    const bool m17 = (kind == QRL_DEMOD_M17) || dmr;
    if (m17) { kind = QRL_DEMOD_4FSK; flag = 1; }
    if (dmr) { carrier_freq = 0; filter_width = 5000; }
    qrl_rx* h = new qrl_rx();
    h->kind = kind; h->sps = sps; h->samp_rate = samp_rate; h->carrier_freq = carrier_freq;
    h->filter_width = filter_width; h->flag = flag; h->C = n_channels; h->Tmax = max_samples;
    h->gmsk = gmsk; h->m17 = m17; h->dmr = dmr;
    auto fail = [&](int rc) { return create_failed(h, qrl_rx_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (rc) return fail(rc);

    std::vector<float> taps1, taps2, taps3;
    int tsr = 0, sym_sps = 0;
    if (kind == QRL_DEMOD_4FSK) {
        // gr_demod_4fsk.cpp:46-84 (sps ladder), :98-107 (resampler), :108-109 (filter), :125-131 (demod, RRC, sync)
        int decimation = 1, interpolation = 1, nfilts = 0;
        if (dmr) { tsr = 24000; sym_sps = 5; decimation = 125; interpolation = 3; nfilts = 25 * sym_sps; }           // gr_demod_dmr.cpp:38-45
        else if (m17) { tsr = 24000; sym_sps = 5; decimation = 125; interpolation = 3; nfilts = 50 * sym_sps; }      // gr_demod_m17.cpp:37-48
        else if (sps == 1) { tsr = 80000; sym_sps = sps * 8; decimation = 25; interpolation = 2; nfilts = 32 * sym_sps; }
        else if (sps == 5) { tsr = 20000; sym_sps = sps * 2; decimation = 50; nfilts = 25 * sym_sps; }
        else if (sps == 10) { tsr = 10000; sym_sps = sps; decimation = 100; nfilts = 25 * sym_sps; }
        else if (sps == 2) { decimation = 2; sym_sps = 5; tsr = 500000; nfilts = 50 * sym_sps; }
        else { set_err(h, "make_gr_demod_4fsk: unsupported sps"); return fail(QRL_EINVAL); }
        if ((nfilts % 2) == 0) nfilts += 1;
        taps1 = dmr ? low_pass_2(3, 3.0 * samp_rate, 5000, 2000, 60, WIN_BLACKMAN_HARRIS)              // gr_demod_dmr.cpp:54-55
                    : low_pass(interpolation, static_cast<double>(interpolation) * samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = decimation; h->L1 = interpolation;
        taps2 = dmr ? std::vector<float>{ 1.0f }                // no IF filter in gr_demod_dmr: the stage runs as a 1-tap pass-through
              : m17 ? low_pass(1, tsr, filter_width, filter_width, WIN_BLACKMAN_HARRIS)                 // gr_demod_m17.cpp:58-59
                    : low_pass(1, tsr, filter_width, filter_width / 2, WIN_BLACKMAN_HARRIS);
        taps3 = dmr ? root_raised_cosine(1, tsr, tsr / sym_sps, 0.2, nfilts)                            // gr_demod_dmr.cpp:61-62
                    : root_raised_cosine(1.5, tsr, tsr / sym_sps, m17 ? 0.5 : 0.2, nfilts);
        const float m17_rate = static_cast<float>(tsr) / static_cast<float>(sym_sps);
        h->qd_gain = dmr ? static_cast<float>(tsr / (kPi / 2 * m17_rate))                               // gr_demod_dmr.cpp:71
                         : static_cast<float>(sym_sps / (1 * kPi));
        const float dev = dmr ? 0.06f : (m17 ? 500.0f / m17_rate : 0.05f);                              // gr_demod_m17.cpp:67-70, gr_demod_dmr.cpp:68
        clock_loop_gains(dmr ? static_cast<float>(2 * kPi / 100.0f)
                             : (m17 ? static_cast<float>(2 * kPi / (m17_rate / 50)) : static_cast<float>(2 * kPi / 200.0f)), 1.0f, 0.2869f,
                         h->ssp.alpha, h->ssp.beta);
        if (dmr) h->ssp.sym_scale = 0.9f;                                                               // gr_demod_dmr.cpp:72
        h->ssp.sps = static_cast<float>(sym_sps);
        h->ssp.max_period = h->ssp.sps + dev; h->ssp.min_period = h->ssp.sps - dev;
        h->ssp.lookahead = 8 + static_cast<int>(ceilf(h->ssp.max_period)) + 1;
        h->ssp.pm_sens = static_cast<float>(kPi / 2);
        h->ssp.soft_scale = 128.0f;
        h->ssp.n0 = static_cast<int>(floorf(h->ssp.min_period - fabsf(h->ssp.alpha)));
        h->ssp.fl0 = static_cast<float>(h->ssp.n0);
        h->nports = dmr ? 4 : 3;
        if (!flag) {     // gr_demod_4fsk.cpp:110-124: four complex band-pass filters + discriminator + symbol filter
            int rs = 0, bw = 0;
            if (sps == 1) { rs = 10000; bw = 4000; } else if (sps == 5) { rs = 2000; bw = 4000; } else if (sps == 10) { rs = 1000; bw = 2000; }
            else { set_err(h, "make_gr_demod_4fsk: non-FM variant needs sps 1, 5 or 10"); return fail(QRL_EINVAL); }
            const int fw = filter_width;
            const double lo[4] = { double(-fw), double(-fw + rs), 0.0, double(fw - rs) }, hi[4] = { double(-fw + rs), 0.0, double(fw - rs), double(fw) };
            std::vector<float> bank;
            for (int b = 0; b < 4; b++) {
                std::vector<float> t = complex_band_pass(1, tsr, lo[b], hi[b], bw, WIN_BLACKMAN_HARRIS);
                h->nt_bank = static_cast<int>(t.size() / 2);
                bank.insert(bank.end(), t.begin(), t.end());
            }
            if ((rc = upload_floats(h, &h->d_bank_taps, bank))) return fail(rc);
            std::vector<float> sf = low_pass(1.0, tsr, tsr / sym_sps, tsr / sym_sps / 20, WIN_BLACKMAN_HARRIS);
            h->nt_symf = static_cast<int>(sf.size());
            if ((rc = upload_floats(h, &h->d_symf_taps, sf))) return fail(rc);
        }
    } else if (kind == QRL_DEMOD_QPSK) {
        // gr_demod_qpsk.cpp:46-71 (sps ladder), :98-103 (resampler), :106-110 (RRC), :104,113-118 (agc, sync, costas)
        int decimation; float costas_bw = static_cast<float>(kPi / 200);
        if (sps > 4 && sps < 125) { decimation = 25; sym_sps = sps * 4 / 25; tsr = 40000; }
        else if (sps >= 125) { decimation = 100; sym_sps = sps / 25; tsr = 10000; }
        else { decimation = 2; sym_sps = sps; tsr = 500000; costas_bw = static_cast<float>(kPi / 400); }
        if (sps > 4) {      // gr_demod_qpsk.cpp:105,130-134: FLL between the resampler and the shaping filter
            h->fllp.N = 32;
            control_loop_gains(static_cast<float>(2 * kPi / 100), h->fllp.alpha, h->fllp.beta);
            h->fllp.max_freq = static_cast<float>(2.0 * kPi * (2.0 / sym_sps)); h->fllp.min_freq = -h->fllp.max_freq;
        }
        taps1 = low_pass_2(1, static_cast<double>(samp_rate), tsr / 2, tsr / 10, 60, WIN_BLACKMAN_HARRIS);
        h->D1 = decimation;
        taps2 = root_raised_cosine(sym_sps, sym_sps, 1, 0.35, 11 * sym_sps);
        h->acp.attack = 1.0f; h->acp.decay = 1e-1f; h->acp.ref = 1.0f; h->acp.max_gain = 65536.0f;
        control_loop_gains(static_cast<float>(kPi / 200 / sym_sps), h->acp.alpha, h->acp.beta);
        h->acp.order = 4; h->acp.use_snr = 1;
        const float symbol_rate = static_cast<float>(tsr) / static_cast<float>(sym_sps);
        const float sps_dev = 200.0f / symbol_rate;
        clock_loop_gains(static_cast<float>(2 * kPi / (symbol_rate / 10)), 1.0f, 0.2869f, h->ssp.alpha, h->ssp.beta);
        h->ssp.sps = static_cast<float>(sym_sps);
        h->ssp.max_period = h->ssp.sps + sps_dev; h->ssp.min_period = h->ssp.sps - sps_dev;
        h->ssp.lookahead = 8 + static_cast<int>(ceilf(h->ssp.max_period)) + 1;
        control_loop_gains(costas_bw, h->ssp.costas_alpha, h->ssp.costas_beta);
        const float th = static_cast<float>(-3 * kPi / 4);
        h->ssp.rot_r = cosf(th); h->ssp.rot_i = sinf(th);
        h->ssp.soft_scale = 48.0f;
        h->ssp.n0 = static_cast<int>(floorf(h->ssp.min_period - fabsf(h->ssp.alpha)));
        h->ssp.fl0 = static_cast<float>(h->ssp.n0);
        h->nports = 3;
    } else if (kind == QRL_DEMOD_2FSK) {
        // gr_demod_2fsk.cpp:39-130 (fm variant)
        int decim, nfilts, interp = 1;
        if (sps == 10) { tsr = 20000; sym_sps = sps; decim = 50; nfilts = 35 * sym_sps; }
        else if (sps >= 5) { tsr = 40000; sym_sps = sps * 2; decim = 25; nfilts = 35 * sym_sps; }
        else if (sps == 1) { tsr = 80000; sym_sps = 4; decim = 25; interp = 2; nfilts = 125 * sym_sps; }
        else { set_err(h, "make_gr_demod_2fsk: unsupported sps"); return fail(QRL_EINVAL); }
        h->L1 = interp;
        if ((nfilts % 2) == 0) nfilts += 1;
        if (!flag) {     // gr_demod_2fsk.cpp:88-100: upper (-fw,0) / lower (0,fw) band filters, ratio detector, symbol filter
            std::vector<float> bank = complex_band_pass(1, tsr, -filter_width, 0, filter_width, WIN_BLACKMAN_HARRIS);
            std::vector<float> lower = complex_band_pass(1, tsr, 0, filter_width, filter_width, WIN_BLACKMAN_HARRIS);
            h->nt_bank = static_cast<int>(bank.size() / 2);
            bank.insert(bank.end(), lower.begin(), lower.end());
            if ((rc = upload_floats(h, &h->d_bank_taps, bank))) return fail(rc);
            std::vector<float> sf = low_pass(1.0, tsr, tsr / sym_sps, tsr / sym_sps, WIN_HAMMING);
            h->nt_symf = static_cast<int>(sf.size());
            if ((rc = upload_floats(h, &h->d_symf_taps, sf))) return fail(rc);
        }
        taps1 = low_pass(interp, static_cast<double>(interp) * samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = decim;
        taps2 = low_pass(1, tsr, filter_width, filter_width, WIN_BLACKMAN_HARRIS);
        taps3 = gmsk ? low_pass(1, tsr, tsr / sym_sps, tsr / sym_sps, WIN_HAMMING)            // gr_demod_gmsk.cpp:88-90
                     : root_raised_cosine(1, tsr, tsr / sym_sps, 0.2, nfilts);
        h->qd_gain = static_cast<float>(sym_sps / (1 * kPi / 2));
        const float symbol_rate = static_cast<float>(tsr) / static_cast<float>(sym_sps);
        const float sps_dev = gmsk ? 0.05f : 200.0f / symbol_rate;                                    // gr_demod_gmsk.cpp:79-84
        clock_loop_gains(gmsk ? static_cast<float>(2 * kPi / 200.0f) : static_cast<float>(2 * kPi / (symbol_rate / 10)), 1.0f, 0.2869f,
                         h->ssp.alpha, h->ssp.beta);
        h->ssp.sps = static_cast<float>(sym_sps);
        h->ssp.max_period = h->ssp.sps + sps_dev; h->ssp.min_period = h->ssp.sps - sps_dev;
        h->ssp.lookahead = 8 + static_cast<int>(ceilf(h->ssp.max_period)) + 1;
        h->ssp.soft_scale = 128.0f;
        h->ssp.n0 = static_cast<int>(floorf(h->ssp.min_period - fabsf(h->ssp.alpha)));
        h->ssp.fl0 = static_cast<float>(h->ssp.n0);
        h->fllp.N = 16;
        control_loop_gains(static_cast<float>(24 * kPi / 100), h->fllp.alpha, h->fllp.beta);
        h->fllp.max_freq = static_cast<float>(2.0 * kPi * (2.0 / sym_sps)); h->fllp.min_freq = -h->fllp.max_freq;
        h->nports = 4;
    } else if (kind == QRL_DEMOD_BPSK) {
        // gr_demod_bpsk.cpp:40-76
        tsr = 20000; sym_sps = sps;
        taps1 = low_pass(1, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = 50;
        taps2 = root_raised_cosine(sps, sps, 1, 0.35, 15 * sps);
        h->acp.attack = 1e-1f; h->acp.decay = 1e-1f; h->acp.ref = 1.0f; h->acp.max_gain = 65536.0f; h->acp.order = 0;
        const float gain_mu = 0.05f, gain_omega = 0.005f;
        h->ssp.loop_kind = LOOP_CRMM;
        h->ssp.sps = static_cast<float>(sps);
        h->ssp.gain_omega = gain_omega * gain_omega; h->ssp.gain_mu = gain_mu;
        h->ssp.omega_mid = static_cast<float>(sps); h->ssp.omega_lim = 0.001f * static_cast<float>(sps);
        h->ssp.lookahead = 24;
        h->ssp.max_period = static_cast<float>(sps) + 1.0f; h->ssp.min_period = static_cast<float>(sps) - 1.0f;   // bounds for buffer sizing only
        h->ssp.alpha = 0.0f;
        control_loop_gains(static_cast<float>(2 * kPi / 200), h->ssp.costas_alpha, h->ssp.costas_beta);
        h->ssp.soft_scale = 64.0f;
        h->fllp.N = 32;
        control_loop_gains(static_cast<float>(8 * kPi / 100), h->fllp.alpha, h->fllp.beta);
        h->fllp.max_freq = static_cast<float>(2.0 * kPi * (2.0 / sps)); h->fllp.min_freq = -h->fllp.max_freq;
        h->nports = 4;
    } else if (kind == QRL_DEMOD_DSSS) {
        // gr_demod_dsss.cpp:32-124 (instance gr_demod_base.cpp:218: make_gr_demod_dsss(25, 1e6, 1700, 150)); sps = items per chip at 5200 sps
        tsr = 20000; sym_sps = 2;
        taps1 = low_pass(1, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = 50;
        const std::vector<float> tif = low_pass(1, 20000, 5200 / 2, 5200 / 2, WIN_BLACKMAN_HARRIS);       // rational_resampler_ccf(13, 50)
        taps2 = low_pass(1, 5200, filter_width, 1200, WIN_BLACKMAN_HARRIS);
        DsssParams& d = h->dsp;
        d.nt_arm = (static_cast<int>(tif.size()) + 12) / 13; d.nt2 = static_cast<int>(taps2.size());
        d.N = sps * 13; d.ntaps = d.N + 11 * sps;
        if (sps < 1 || d.nt_arm > 8 || d.nt2 > 64 || d.ntaps > 640 || d.N + d.ntaps - 1 > kDsssChunk) {
            set_err(h, "make_gr_demod_dsss: sps / filter_width outside what the chain kernel holds in shared memory"); return fail(QRL_EINVAL);
        }
        if ((rc = upload_floats(h, &h->d_ds_arms, make_arms(tif, 13, d.nt_arm)))) return fail(rc);
        {   // dsss_decoder_cc_impl.cc:60-96: reversed Barker-13, `sps` items per chip, shaped by RRC(1, sps, 1, 0.35f, 11 sps); the block's
            // fir_filter_ccc keeps the taps reversed (what is uploaded)
            static const int barker_13[13] = { 1, 1, 1, 1, 1, 0, 0, 1, 1, 0, 1, 0, 1 };
            const int extra = 11 * sps, total = d.N + 2 * extra;
            std::vector<float> cs(total, 0.0f);
            for (int i = 0; i < 13; i++) { const float cv = barker_13[13 - (i + 1)] == 0 ? -1.0f : 1.0f; for (int k = 0; k < sps; k++) cs[extra + i * sps + k] = cv; }
            const std::vector<float> rrc = root_raised_cosine(1, sps, 1.0, static_cast<double>(0.350f), extra);
            const int nr = static_cast<int>(rrc.size());
            std::vector<float> t(2 * static_cast<size_t>(d.ntaps));
            for (int i = 0; i < d.ntaps; i++) {
                float acc = 0.0f, acci = 0.0f;
                for (int k = 0; k < nr; k++) { acc = acc + cs[i + k] * rrc[nr - 1 - k]; acci = acci + 0.0f * rrc[nr - 1 - k]; }
                t[2 * (d.ntaps - 1 - i)] = acc; t[2 * (d.ntaps - 1 - i) + 1] = acci;
            }
            float* tp = nullptr;
            if ((rc = upload_floats(h, &tp, t))) return fail(rc);
            h->d_ds_taps = reinterpret_cast<float2*>(tp);
        }
        control_loop_gains(static_cast<float>(kPi / 200), d.pll_alpha, d.pll_beta);
        control_loop_gains(static_cast<float>(2 * kPi / 100), d.costas_alpha, d.costas_beta);
        d.agc_attack = 1e-1f; d.agc_decay = 1e-1f; d.agc_ref = 1.0f; d.agc_max = 65536.0f;
        const float gain_mu = 0.05f, gain_omega = 0.005f;
        d.gain_omega = gain_omega * gain_omega; d.gain_mu = gain_mu; d.omega_mid = 1.0f; d.omega_lim = 0.005f * 1.0f; d.soft_scale = 64.0f;
        h->ssp.lookahead = 0; h->ssp.sps = 2.0f;
        h->nports = 4;
    } else if (kind == QRL_DEMOD_SSB) {
        // gr_demod_ssb.cpp:37-61; flag = sb (0 USB, 1 LSB); sps = decimation (125)
        tsr = 8000; sym_sps = 2;
        taps1 = low_pass(1, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = sps;
        taps2 = flag ? complex_band_pass_2(1, tsr, -filter_width, -200, 200, 90, WIN_BLACKMAN_HARRIS)
                     : complex_band_pass_2(1, tsr, 200, filter_width, 200, 90, WIN_BLACKMAN_HARRIS);
        h->nports = 2;
    } else if (kind == QRL_DEMOD_FREEDV) {
        // gr_demod_freedv.cpp:40-54; flag = sb (0 USB, 1 LSB); sps = decimation to 8 ksps.  The stage-1 taps are low_pass(sps, ...): DC gain sps
        tsr = 8000; sym_sps = 2;
        taps1 = low_pass(sps, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = sps;
        taps2 = flag ? complex_band_pass_2(1, tsr, -filter_width, -low_cutoff, 200, 90, WIN_BLACKMAN_HARRIS)
                     : complex_band_pass_2(1, tsr, low_cutoff, filter_width, 200, 90, WIN_BLACKMAN_HARRIS);
        h->nports = 2;
    } else if (kind == QRL_DEMOD_WBFM) {
        // gr_demod_wbfm.cpp:35-54
        tsr = 200000; sym_sps = 2;
        taps1 = low_pass(1, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = 5;
        taps2 = low_pass_2(1, tsr, filter_width, 600, 90, WIN_BLACKMAN_HARRIS);
        h->qd_gain = static_cast<float>(tsr / (2 * kPi * filter_width));
        h->nports = 2;
    } else if (kind == QRL_DEMOD_AM) {
        // gr_demod_am.cpp:35-56
        tsr = 20000; sym_sps = 2;
        taps1 = low_pass(1, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = 50;
        taps2 = complex_band_pass_2(1, tsr, -filter_width, filter_width, 200, 90, WIN_BLACKMAN_HARRIS);
        h->nports = 2;
    } else if (kind == QRL_DEMOD_NBFM) {
        // gr_demod_nbfm.cpp:39-66
        tsr = 20000; sym_sps = 2;
        taps1 = low_pass(1, samp_rate, tsr / 2, tsr / 2, WIN_BLACKMAN_HARRIS);
        h->D1 = 50;
        taps2 = low_pass_2(1, tsr, filter_width, 3500, 60, WIN_BLACKMAN_HARRIS);
        h->qd_gain = static_cast<float>(tsr / (4 * kPi * filter_width));
        h->nports = 2;
    } else {
        set_err(h, "qrl_rx_create: demod kind " + std::to_string(kind) + " not built");
        return fail(QRL_EINVAL);
    }
    h->sym_sps = sym_sps; h->tsr = tsr;

    // ---- stage 1 buffers
    h->ntaps1 = static_cast<int>(taps1.size());
    h->Q1 = (h->ntaps1 + h->D1 - 1) / h->D1;
    int padded = std::max(h->Q1 * h->D1, h->D1 == 2 ? 56 : 0);
    std::vector<float> tp(padded, 0.0f);
    std::copy(taps1.begin(), taps1.end(), tp.begin());
    if (h->L1 == 2) {       // rational_resampler arms: arm[p][k] = taps[p + k L], 105 taps per arm
        const int nt = 105;
        tp.assign(2 * nt, 0.0f);
        for (int p = 0; p < 2; p++) for (int k = 0; k < nt; k++) { const size_t j = p + 2 * k; if (j < taps1.size()) tp[p * nt + k] = taps1[j]; }
        padded = 128;       // history samples kept
    } else if (h->L1 > 2) {   // shape-generic rational resampler: arm[p][k] = taps[p + k L]
        const int nt = (static_cast<int>(taps1.size()) + h->L1 - 1) / h->L1;
        tp.assign(static_cast<size_t>(h->L1) * nt, 0.0f);
        for (int p = 0; p < h->L1; p++) for (int k = 0; k < nt; k++) { const size_t j = p + static_cast<size_t>(k) * h->L1; if (j < taps1.size()) tp[p * nt + k] = taps1[j]; }
        h->nt_arm1 = nt;
        padded = nt + 8;
    }
    if ((rc = upload_floats(h, &h->d_taps1, tp))) return fail(rc);
    h->H = padded;
    if ((rc = dev_alloc(h, &h->d_hist[0], static_cast<size_t>(h->H) * h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_hist[1], static_cast<size_t>(h->H) * h->C))) return fail(rc);
    h->n1max = h->Tmax * h->L1 / h->D1 + 2;
    // ---- rings
    h->ntaps2 = static_cast<int>(taps2.size()) / ((kind == QRL_DEMOD_SSB || kind == QRL_DEMOD_AM || kind == QRL_DEMOD_FREEDV) ? 2 : 1);
    h->ntaps3 = static_cast<int>(taps3.size());
    {
        std::vector<float> t2(std::max<size_t>(taps2.size(), 512), 0.0f);     // room for set_filter_width redesigns
        std::copy(taps2.begin(), taps2.end(), t2.begin());
        if ((rc = upload_floats(h, &h->d_taps2, t2))) return fail(rc);
        h->taps2_cap = t2.size();
    }
    if (!taps3.empty() && (rc = upload_floats(h, &h->d_taps3, taps3))) return fail(rc);
    if ((rc = make_ring(h, &h->r1, sizeof(float2), h->n1max + std::max(512, static_cast<int>(taps2.size())) + 8))) return fail(rc);
    if (kind == QRL_DEMOD_SSB) {
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + 64))) return fail(rc);
        std::vector<float> audio_f = band_pass_2(1, tsr, 200, filter_width, 200, 90, WIN_BLACKMAN_HARRIS);
        if ((rc = upload_floats(h, &h->d_audio_taps, audio_f))) return fail(rc);
        h->ssbp.sq_alpha = 0.01; h->ssbp.sq_threshold = std::pow(10.0, -140 / 10.0);
        h->ssbp.attack = 1e-1f; h->ssbp.decay = 1e-1f; h->ssbp.ref = 0.25f; h->ssbp.max_gain = 65536.0f;
        h->ssbp.clip = 0.95f; h->ssbp.emax = static_cast<float>(1 / (std::sqrt(0.5) / 2)); h->ssbp.out_gain = 1.333f;
        h->ssbp.nt_audio = static_cast<int>(audio_f.size());
        if ((rc = make_ring(h, &h->rclip, sizeof(float2), h->n1max + 16))) return fail(rc);
        if ((rc = make_ring(h, &h->rstr, sizeof(float), h->n1max + h->ssbp.nt_audio + 16))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_ssb, h->C))) return fail(rc);
    } else if (kind == QRL_DEMOD_FREEDV) {
        // gr_demod_freedv.cpp:57-77: agc2_ff(1e-1, 1e-3, 0.5, 1) (max gain 65536) -> band_pass_2(1, 8000, 200, 3500, 200, 90, BH) -> x0.1 ->
        // float_to_short(1, 32768); the feedforward_agc_cc of :56 is never connected
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + 64))) return fail(rc);
        std::vector<float> audio_f = band_pass_2(1, tsr, 200, 3500, 200, 90, WIN_BLACKMAN_HARRIS);
        if ((rc = upload_floats(h, &h->d_audio_taps, audio_f))) return fail(rc);
        h->fdp.attack = 1e-1f; h->fdp.decay = 1e-3f; h->fdp.ref = 0.5f; h->fdp.max_gain = 65536.0f;
        h->fdp.nt_audio = static_cast<int>(audio_f.size());
        if ((rc = make_ring(h, &h->rstr, sizeof(float), h->n1max + h->fdp.nt_audio + 16))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_fdv, h->C))) return fail(rc);
    } else if (kind == QRL_DEMOD_WBFM) {
        // gr_demod_wbfm.cpp:39-64: the analog audio kernel in mode 2
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + 64))) return fail(rc);
        std::vector<float> audio_rs = low_pass(1, tsr, 4000, 2000, WIN_BLACKMAN_HARRIS);
        if ((rc = upload_floats(h, &h->d_audio_taps, audio_rs))) return fail(rc);
        if ((rc = upload_floats(h, &h->d_arm_taps, std::vector<float>{ 0.0f, 0.0f }))) return fail(rc);
        if ((rc = upload_floats(h, &h->d_env, std::vector<float>{ 1.0f, 1.0f }))) return fail(rc);
        double a[2], b[2];
        deemph_taps(8000, 50e-6, a, b);                        // the reference designs them for 8 kHz (:39) and runs them at 200 ksps
        h->nbp.sq_alpha = 0.01; h->nbp.sq_threshold = std::pow(10.0, -140 / 10.0); h->nbp.sq_ramp = 0; h->nbp.sq_gate = 1;
        h->nbp.qd_gain = h->qd_gain; h->nbp.nt_arm = 1; h->nbp.nt_audio = static_cast<int>(audio_rs.size());
        h->nbp.b0 = b[0]; h->nbp.b1 = b[1]; h->nbp.a1 = a[1]; h->nbp.out_gain = 1.0f;
        h->nbp.mode = 2; h->nbp.am_gain = 0.9f;
        if ((rc = make_ring(h, &h->rg, sizeof(float2), h->n1max + 16))) return fail(rc);
        if ((rc = make_ring(h, &h->rd, sizeof(float), h->n1max + 16))) return fail(rc);
        if ((rc = make_ring(h, &h->rr, sizeof(float), h->n1max + h->nbp.nt_audio + 16))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_nb, h->C))) return fail(rc);
    } else if (kind == QRL_DEMOD_AM) {
        // gr_demod_am.cpp:41-70: the NBFM audio kernel in detector mode 1
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + 64))) return fail(rc);
        std::vector<float> audio_rs = low_pass(2, 2 * tsr, 3600, 600, WIN_BLACKMAN_HARRIS);
        std::vector<float> audio_f = low_pass(1, 8000, 3600, 300, WIN_BLACKMAN_HARRIS);
        const int nt_arm = (static_cast<int>(audio_rs.size()) + 1) / 2;
        std::vector<float> arms(2 * nt_arm, 0.0f);
        for (int pp = 0; pp < 2; pp++)
            for (int k = 0; k < nt_arm; k++) { const size_t j = pp + 2 * k; arms[pp * nt_arm + k] = j < audio_rs.size() ? audio_rs[j] : 0.0f; }
        if ((rc = upload_floats(h, &h->d_arm_taps, arms))) return fail(rc);
        if ((rc = upload_floats(h, &h->d_audio_taps, audio_f))) return fail(rc);
        if ((rc = upload_floats(h, &h->d_env, std::vector<float>{ 1.0f, 1.0f }))) return fail(rc);
        h->nbp.sq_alpha = 0.01; h->nbp.sq_threshold = std::pow(10.0, -140 / 10.0); h->nbp.sq_ramp = 0; h->nbp.sq_gate = 1;
        h->nbp.qd_gain = 0.0f; h->nbp.nt_arm = nt_arm; h->nbp.nt_audio = static_cast<int>(audio_f.size());
        h->nbp.b0 = 1.0; h->nbp.b1 = -1.0; h->nbp.a1 = -0.9999; h->nbp.out_gain = 1.0f;      // iir_filter_ffd({1,-1},{0,0.9999}), old style
        h->nbp.mode = 1; h->nbp.agc_attack = 1e-1f; h->nbp.agc_decay = 1e-1f; h->nbp.agc_ref = 1.0f; h->nbp.agc_max = 65536.0f; h->nbp.am_gain = 0.99f;
        if ((rc = make_ring(h, &h->rg, sizeof(float2), 64))) return fail(rc);
        if ((rc = make_ring(h, &h->rd, sizeof(float), h->n1max + nt_arm + 16))) return fail(rc);
        if ((rc = make_ring(h, &h->rr, sizeof(float), h->n1max * 2 / 5 + h->nbp.nt_audio + 16))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_nb, h->C))) return fail(rc);
    } else if (kind == QRL_DEMOD_NBFM) {
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + 64))) return fail(rc);
        std::vector<float> audio_rs = low_pass_2(2, 2 * tsr, 3600, 250, 60, WIN_BLACKMAN_HARRIS);
        std::vector<float> audio_f = low_pass_2(1, 8000, 3500, 200, 35, WIN_BLACKMAN_HARRIS);
        const int nt_arm = (static_cast<int>(audio_rs.size()) + 1) / 2;
        std::vector<float> arms(2 * nt_arm, 0.0f);
        for (int pp = 0; pp < 2; pp++)
            for (int k = 0; k < nt_arm; k++) { const size_t j = pp + 2 * k; arms[pp * nt_arm + k] = j < audio_rs.size() ? audio_rs[j] : 0.0f; }
        if ((rc = upload_floats(h, &h->d_arm_taps, arms))) return fail(rc);
        if ((rc = upload_floats(h, &h->d_audio_taps, audio_f))) return fail(rc);
        const int ramp = 320;
        std::vector<float> env(ramp + 1);
        for (int k = 0; k <= ramp; k++) env[k] = static_cast<float>(0.5 - std::cos(kPi * k / ramp) / 2.0);
        if ((rc = upload_floats(h, &h->d_env, env))) return fail(rc);
        double a[2], b[2];
        deemph_taps(tsr, 50e-6, a, b);
        h->nbp.sq_alpha = 0.01; h->nbp.sq_threshold = std::pow(10.0, -140 / 10.0); h->nbp.sq_ramp = ramp; h->nbp.sq_gate = 1;
        h->nbp.qd_gain = h->qd_gain; h->nbp.nt_arm = nt_arm; h->nbp.nt_audio = static_cast<int>(audio_f.size());
        h->nbp.b0 = b[0]; h->nbp.b1 = b[1]; h->nbp.a1 = a[1]; h->nbp.out_gain = 2.0f;
        if ((rc = make_ring(h, &h->rg, sizeof(float2), h->n1max + 16))) return fail(rc);
        if ((rc = make_ring(h, &h->rd, sizeof(float), h->n1max + nt_arm + 16))) return fail(rc);
        if ((rc = make_ring(h, &h->rr, sizeof(float), h->n1max * 2 / 5 + h->nbp.nt_audio + 16))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_nb, h->C))) return fail(rc);
        if (kind == QRL_DEMOD_NBFM) {
            // analog::ctcss_squelch_ff::make(8000, 88.5, 0.01, 8000, 160, true) (gr_demod_nbfm.cpp:60), out of the graph until set_ctcss(f)
            if ((rc = make_ring(h, &h->rq, sizeof(float), h->n1max * 2 / 5 + h->nbp.nt_audio + 64))) return fail(rc);
            h->ctc.on = 0; h->ctc.len = 8000; h->ctc.ramp = 160; h->ctc.gate = 1; h->ctc.level = 0.01f;
            std::vector<double> ce(h->ctc.ramp + 1);
            for (int k = 0; k <= h->ctc.ramp; k++) ce[k] = 0.5 - std::cos(kPi * k / h->ctc.ramp) / 2.0;       // squelch_base_ff envelope (double)
            if ((rc = dev_alloc(h, &h->d_cenv, ce.size(), false))) return fail(rc);
            if (cudaMemcpy(h->d_cenv, ce.data(), sizeof(double) * ce.size(), cudaMemcpyHostToDevice) != cudaSuccess) { set_err(h, "envelope upload failed"); return fail(QRL_ECUDA); }
        }
        // (an FP64 instruction occupies an SM's FP64 pipe for ~64 cycles whatever its lane count, so two recurrences only overlap on
        // DIFFERENT SMs: both kernels then ask for more than half an SM's shared memory, which keeps their CTAs one per SM and apart, and
        // the split is used while each kernel's C CTAs fit the SMs at once -- on an H100 it is faster up to 128 channels, slower at 160)
        int n_sm = 0;
        if (cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, h->device) != cudaSuccess) { set_err(h, "SM count query failed"); return fail(QRL_ECUDA); }
        if (kind == QRL_DEMOD_NBFM && h->C <= n_sm && !getenv("QRL_NBFM_NO_SPLIT")) {
            if ((rc = make_ring(h, &h->raud, sizeof(float), h->n1max * 2 / 5 + 64))) return fail(rc);
            if ((rc = dev_alloc(h, &h->d_nb2, h->C))) return fail(rc);
            h->zero_list.emplace_back(h->d_nb2, sizeof(NbfmDeemphState) * h->C);
            h->nbfm_split = true;
        }
    } else if (kind == QRL_DEMOD_DSSS) {
        const long long n5 = h->n1max * 13 / 50 + 8;
        if ((rc = make_ring(h, &h->ds_a, sizeof(float2), n5 + 2048))) return fail(rc);
        if ((rc = make_ring(h, &h->ds_c, sizeof(float2), n5 + 2048))) return fail(rc);
        if ((rc = make_ring(h, &h->ds_d, sizeof(float2), n5 / h->dsp.N + 128))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_ds, h->C))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_vs2, h->C))) return fail(rc);
    } else if (kind == QRL_DEMOD_4FSK || kind == QRL_DEMOD_2FSK) {
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + h->ntaps3 + 64))) return fail(rc);
        // two calls deep when the block may run with overlapped calls (the producer of call k+1 must not wait for the
        // consumer of call k)
        if ((rc = make_ring(h, &h->r4, sizeof(float), (flag && kind == QRL_DEMOD_4FSK ? 2 : 1) * h->n1max + 600, true))) return fail(rc);
        if (flag && kind == QRL_DEMOD_4FSK) {
            // scratch of the external symbol-sync epilogue: [groups][chunks][maxs + 2][32] floats + a 128-int header per group
            // window size: 512 rows x 2 stages when the replicated interpolator bank still fits next to it, else 256 x 3
            h->ss_ch = symsync_ext_smem(h->ssp, 512, 2, true) <= 220 * 1024 ? 512 : 256;
            if (const char* e = getenv("QRL_SS_CH")) { const int v = atoi(e); if (v == 512 || v == 256) h->ss_ch = v; }
            const int maxs = symsync_maxs(h->ssp, h->ss_ch);
            h->ss_chunk_cap = h->n1max / symsync_stride(h->ss_ch, h->ssp.lookahead) + 4 + 3 * qrl_rx::kMaxSub;
            const size_t groups = (h->C + 31) / 32;
            if ((rc = dev_alloc(h, &h->d_ss_scratch, groups * h->ss_chunk_cap * (maxs + 2) * 32))) return fail(rc);
            if ((rc = dev_alloc(h, &h->d_ss_hdr, groups * 128 * qrl_rx::kMaxSub))) return fail(rc);
        }
        if (!flag) {
            if ((rc = make_ring(h, &h->rbank, kind == QRL_DEMOD_4FSK ? sizeof(float2) : sizeof(float), h->n1max + h->nt_symf + 16))) return fail(rc);
            if (kind == QRL_DEMOD_4FSK && (rc = make_ring(h, &h->r3, sizeof(float2), h->n1max + 600, true))) return fail(rc);
        }
    } else {   // QPSK / BPSK: shaping-filter output and loop output are channel-interleaved complex rings
        if ((rc = make_ring(h, &h->r2, sizeof(float2), h->n1max + 600, true))) return fail(rc);
        if ((rc = make_ring(h, &h->r3, sizeof(float2), h->n1max + 600, true))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_ac, h->C))) return fail(rc);
    }
    const bool has_fll = kind == QRL_DEMOD_BPSK || kind == QRL_DEMOD_2FSK || (kind == QRL_DEMOD_QPSK && sps > 4);
    if (has_fll) {
        const float fsps = static_cast<float>(sym_sps);
        std::vector<float> ft = fll_design(fsps, kind == QRL_DEMOD_2FSK ? 0.1f : 0.35f, h->fllp.N);
        if ((rc = upload_floats(h, &h->d_fll_taps, ft))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_fll, h->C))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_fll_hist, static_cast<size_t>(32) * h->C))) return fail(rc);
        h->zero_list.emplace_back(h->d_fll_hist, sizeof(float2) * 32 * h->C);
        h->zero_list.emplace_back(h->d_fll, sizeof(FllState) * h->C);
        if ((rc = make_ring(h, &h->rf, sizeof(float2), h->n1max + 512 + 8))) return fail(rc);
        if (kind != QRL_DEMOD_QPSK && (rc = dev_alloc(h, &h->d_vs2, h->C))) return fail(rc);
    }
    if ((rc = make_ring(h, &h->r5, 1, 2 * h->n1max + 1024))) return fail(rc);
    h->port0_cap = h->n1max;
    if ((rc = dev_alloc(h, &h->d_port0, static_cast<size_t>(h->port0_cap) * h->C))) return fail(rc);
    h->port1_cap = h->n1max / std::max(1, sym_sps - 1) + 64;
    if ((rc = dev_alloc(h, &h->d_port1, static_cast<size_t>(h->port1_cap) * h->C))) return fail(rc);
    h->d_port1f = reinterpret_cast<float*>(h->d_port1);
    if ((rc = dev_alloc(h, &h->d_port1_cnt, h->C))) return fail(rc);
    h->port2_cap = (h->m17 ? 2 : 1) * h->port1_cap + 160;      // M17: two hard bits per symbol, no rate-1/2 decoder behind them
    if ((rc = dev_alloc(h, &h->d_port2, static_cast<size_t>(h->port2_cap) * h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_port2_cnt, h->C))) return fail(rc);
    if (h->dmr) {
        if ((rc = dev_alloc(h, &h->d_port3f, static_cast<size_t>(h->port0_cap) * h->C))) return fail(rc);
    } else if (h->nports == 4) {
        if ((rc = dev_alloc(h, &h->d_port3, static_cast<size_t>(h->port2_cap) * h->C))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_port3_cnt, h->C))) return fail(rc);
    }
    if ((rc = dev_alloc(h, &h->d_ss, h->C))) return fail(rc);
    if (h->ssp.lookahead > 0 && symsync_stride(128, h->ssp.lookahead) < 32 &&
        (kind == QRL_DEMOD_QPSK || kind == QRL_DEMOD_BPSK || (kind == QRL_DEMOD_4FSK && !flag))) {
        set_err(h, "symbol-sync lookahead does not fit the 128-row window of the complex-symbol kernels");
        return fail(QRL_EINVAL);
    }
    if ((rc = dev_alloc(h, &h->d_vs, h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_nsoft, static_cast<size_t>(qrl_rx::kMaxSub) * h->C))) return fail(rc);
    {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        bool ok = true;
        // loop partition: one SM per big-shared-memory loop CTA (4FSK: symbol sync; QPSK: agc/costas + symbol sync)
        const int groups = (h->C + 31) / 32;
        // analog blocks: one CTA per channel whose thread 0 runs the double-precision recurrences (squelch power, de-emphasis): they want
        // an SM (its FP64 pipe) each, up to half the machine
        const bool analog_kind = kind == QRL_DEMOD_NBFM || kind == QRL_DEMOD_SSB || kind == QRL_DEMOD_AM || kind == QRL_DEMOD_WBFM ||
                                 kind == QRL_DEMOD_FREEDV;
        const int big_ctas = (kind == QRL_DEMOD_QPSK) ? 2 * groups : (analog_kind ? (h->nbfm_split ? 2 * h->C : std::min(h->C, 44)) : groups);
        unsigned loop_sms = static_cast<unsigned>(std::min(48, 8 * ((big_ctas + 4 + 7) / 8)));
        if (const char* e = getenv("QRL_LOOP_SMS")) { int v = atoi(e); if (v >= 8 && v <= 64) loop_sms = static_cast<unsigned>(v); }
        // Many channels (more loop CTAs than a 48-SM partition holds one per SM): the loop kernels have enough warps in flight to
        // hide their own latency, a private partition would only serialise them.  They then run with small windows (several CTAs
        // per SM) on all SMs, next to the parallel stages, on priority streams.
        h->many = big_ctas > 44 || (analog_kind && h->C > 64);
        if (const char* e = getenv("QRL_MANY_CHANNELS")) h->many = e[0] == '1';
        // QPSK (per-sample loops, 2 loop CTAs per 32 channels + a heavy Viterbi load): runs WITHOUT a private partition, so that the
        // decoder gets the whole machine and the loop CTAs spread over more SMs; QRL_QPSK_PARTITION=1 brings the partition back.
        bool want_partition = kind != QRL_DEMOD_QPSK;
        if (const char* e = getenv("QRL_QPSK_PARTITION")) { if (kind == QRL_DEMOD_QPSK) want_partition = e[0] == '1'; }
        if (h->many || !want_partition || !make_sm_partition(h, loop_sms, hi, !analog_kind && groups <= 2)) {
            h->s_par = nullptr; h->sm_loop = 0; h->sm_par = 0;
            if (h->s_loop == nullptr)
                ok = cudaStreamCreateWithPriority(&h->s_loop, cudaStreamNonBlocking, hi) == cudaSuccess;
            if (h->s_loop2 == nullptr)
                ok = ok && cudaStreamCreateWithPriority(&h->s_loop2, cudaStreamNonBlocking, hi) == cudaSuccess;
            if (h->s_fec == nullptr)
                ok = ok && cudaStreamCreateWithPriority(&h->s_fec, cudaStreamNonBlocking, hi) == cudaSuccess;
            if (h->s_epi == nullptr)
                ok = ok && cudaStreamCreateWithPriority(&h->s_epi, cudaStreamNonBlocking, hi) == cudaSuccess;
        }
        auto mk = [&](cudaEvent_t* e) { ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess; };
        mk(&h->ev_start); mk(&h->ev_loop_done); mk(&h->ev_loop2_done); mk(&h->ev_fec_done); mk(&h->ev_par_done);
        for (int i = 0; i < qrl_rx::kMaxSub; i++) { mk(&h->ev_a[i]); mk(&h->ev_b[i]); mk(&h->ev_c[i]); }
        if (!ok) { set_err(h, "stream/event creation failed"); return fail(QRL_ECUDA); }
    }
    // QPSK: the call ends with the symbol sync + Viterbi of the last slice behind the per-sample loop (no overlapped calls for this
    // chain): the finest slicing the event arrays allow keeps that tail short
    if (kind == QRL_DEMOD_QPSK) h->nsub = qrl_rx::kMaxSub;
    if (const char* e = getenv("QRL_NSUB")) { int v = atoi(e); if (v >= 1 && v <= qrl_rx::kMaxSub) { h->nsub = v; h->nsub_forced = true; } }
    if (const char* e = getenv("QRL_FIR_GROUP")) { int v = atoi(e); if (v >= 1 && v <= qrl_rx::kMaxSub) { h->fir_group = v; h->fir_group_forced = true; } }
    if ((rc = qrl_rx_reset(h))) return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}

// host-side wait for everything a handle has in flight on its internal streams
static int rx_join_host(qrl_rx* h)
{
    if (h->s_loop) QRL_CK(cudaStreamSynchronize(h->s_loop));
    if (h->s_fec) QRL_CK(cudaStreamSynchronize(h->s_fec));
    if (h->s_loop2) QRL_CK(cudaStreamSynchronize(h->s_loop2));
    if (h->s_epi) QRL_CK(cudaStreamSynchronize(h->s_epi));
    if (h->s_par) QRL_CK(cudaStreamSynchronize(h->s_par));
    return QRL_OK;
}

int qrl_rx_reset(qrl_rx* h)
{
    if (!h) return QRL_EINVAL;
    if (int rc = rx_join_host(h)) return rc;
    // all-zero history / rings; loop states at their constructor values
    std::vector<SymSyncState> ss(h->C);
    std::vector<ViterbiState> vs(h->C);
    for (int c = 0; c < h->C; c++) {
        std::memset(&ss[c], 0, sizeof(SymSyncState));
        ss[c].avg_period = h->ssp.sps; ss[c].inst_period = h->ssp.sps;
        ss[c].mu = (h->ssp.loop_kind == LOOP_CRMM) ? 0.5f : 0.0f;          // clock_recovery_mm_cc(omega, g_omega, mu = 0.5, ...)
        vs[c].rd = 0; vs[c].start_state = 0; vs[c].descr_reg = 0x7F;
    }
    QRL_CK(cudaMemcpyAsync(h->d_ss, ss.data(), sizeof(SymSyncState) * h->C, cudaMemcpyHostToDevice, h->stream));
    QRL_CK(cudaMemcpyAsync(h->d_vs, vs.data(), sizeof(ViterbiState) * h->C, cudaMemcpyHostToDevice, h->stream));
    if (h->d_vs2) QRL_CK(cudaMemcpyAsync(h->d_vs2, vs.data(), sizeof(ViterbiState) * h->C, cudaMemcpyHostToDevice, h->stream));
    if (h->d_port3_cnt) QRL_CK(cudaMemsetAsync(h->d_port3_cnt, 0, sizeof(int) * h->C, h->stream));
    QRL_CK(cudaMemsetAsync(h->d_hist[0], 0, sizeof(float2) * h->H * h->C, h->stream));
    QRL_CK(cudaMemsetAsync(h->d_hist[1], 0, sizeof(float2) * h->H * h->C, h->stream));
    for (auto& z : h->zero_list) QRL_CK(cudaMemsetAsync(z.first, 0, z.second, h->stream));
    if (h->d_ds) {
        std::vector<DsssState> ds(h->C);
        for (int c = 0; c < h->C; c++) {
            std::memset(&ds[c], 0, sizeof(DsssState));
            ds[c].agc = 10.0f;                        // agc2_cc::make(1e-1, 1e-1, 1, 10): initial gain 10 (gr_demod_dsss.cpp:66)
            ds[c].omega = 1.0f; ds[c].mu = 0.5f;      // clock_recovery_mm_cc(1, ..., 0.5, ...)
        }
        QRL_CK(cudaMemcpyAsync(h->d_ds, ds.data(), sizeof(DsssState) * h->C, cudaMemcpyHostToDevice, h->stream));
        QRL_CK(cudaStreamSynchronize(h->stream));
        h->ds_o_call0 = 0;
    }
    std::vector<SsbState> sb(h->C);
    if (h->d_ssb) {
        for (int c = 0; c < h->C; c++) { std::memset(&sb[c], 0, sizeof(SsbState)); sb[c].sq_state = SQ_MUTED; sb[c].gain = 1.0f; }
        QRL_CK(cudaMemcpyAsync(h->d_ssb, sb.data(), sizeof(SsbState) * h->C, cudaMemcpyHostToDevice, h->stream));
    }
    std::vector<FreedvRxState> fdv(h->C);
    if (h->d_fdv) {
        for (auto& f : fdv) { f.n_in = 0; f.gain = 1.0f; f.pad_ = 0; }           // agc2_ff::make(..., gain = 1)
        QRL_CK(cudaMemcpyAsync(h->d_fdv, fdv.data(), sizeof(FreedvRxState) * h->C, cudaMemcpyHostToDevice, h->stream));
    }
    std::vector<NbfmState> nb(h->C);
    if (h->d_nb) {
        for (int c = 0; c < h->C; c++) {
            std::memset(&nb[c], 0, sizeof(NbfmState));
            nb[c].sq_state = SQ_MUTED; nb[c].envelope = h->nbp.sq_ramp ? 0.0f : 1.0f; nb[c].agc_gain = 1.0f;
            nb[c].c_mute = 1; nb[c].c_state = SQ_MUTED; nb[c].c_env = h->ctc.ramp ? 0.0 : 1.0;      // ctcss_squelch_ff: d_mute(true), squelch_base_ff starts muted
        }
        QRL_CK(cudaMemcpyAsync(h->d_nb, nb.data(), sizeof(NbfmState) * h->C, cudaMemcpyHostToDevice, h->stream));
    }
    std::vector<AgcCostasState> ac(h->C);
    if (h->d_ac) {
        for (int c = 0; c < h->C; c++) { ac[c].pos = 0; ac[c].gain = 1.0f; ac[c].pll.phase = 0.0f; ac[c].pll.freq = 0.0f; }
        QRL_CK(cudaMemcpyAsync(h->d_ac, ac.data(), sizeof(AgcCostasState) * h->C, cudaMemcpyHostToDevice, h->stream));
    }
    QRL_CK(cudaMemsetAsync(h->d_port1_cnt, 0, sizeof(int) * h->C, h->stream));
    QRL_CK(cudaMemsetAsync(h->d_port2_cnt, 0, sizeof(int) * h->C, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));   // the staging vectors above go out of scope
    h->n_in = 0; h->n1 = 0; h->n_in_s = 0; h->n1_s = 0; h->hist_cur = 0; h->port0_n = 0; h->prev_nsub = 0; h->rssi_n = 0;
    return QRL_OK;
}

int qrl_rx_destroy(qrl_rx* h)
{
    if (!h) return QRL_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    rx_join_host(h);
    for (cudaStream_t s : { h->s_loop, h->s_fec, h->s_loop2, h->s_epi, h->s_par }) if (s) cudaStreamDestroy(s);
    // every stream is idle now: the events recorded on them can go
    auto ev_free = [](cudaEvent_t e) { if (e) cudaEventDestroy(e); };
    for (cudaEvent_t e : { h->ev_start, h->ev_loop_done, h->ev_loop2_done, h->ev_fec_done, h->ev_par_done }) ev_free(e);
    for (int i = 0; i < qrl_rx::kMaxSub; i++) { ev_free(h->ev_a[i]); ev_free(h->ev_b[i]); ev_free(h->ev_c[i]); ev_free(h->ev_v[i]); }
    for (int q = 0; q < 2; q++) for (int j = 0; j < 3; j++) ev_free(h->ev_tail[q][j]);
    if (h->g_loop || h->g_par) {
        auto pDestroy = drv<CUresult (*)(CUgreenCtx)>("cuGreenCtxDestroy");
        if (pDestroy) { if (h->g_loop) pDestroy(h->g_loop); if (h->g_par) pDestroy(h->g_par); }
    }
    return handle_close(h);
}

int qrl_rx_set_stream(qrl_rx* h, void* s)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, s);
}

int qrl_rx_set_param(qrl_rx* h, int channel, int key, double value)
{
    if (!h) return QRL_EINVAL;
    if (key == QRL_PARAM_RSSI) {
        if (value != 0.0 && !h->d_rssi_ring) {
            int rc;
            if ((rc = dev_alloc(h, &h->d_rssi_ring, static_cast<size_t>(4096) * h->C))) return rc;
            if ((rc = dev_alloc(h, &h->d_rssi_y, h->C))) return rc;
            if ((rc = dev_alloc(h, &h->d_rssi_db, h->C))) return rc;
            h->zero_list.emplace_back(h->d_rssi_ring, sizeof(float) * 4096 * h->C);
            h->zero_list.emplace_back(h->d_rssi_y, sizeof(float) * h->C);
            h->rssi_n = 0;
        }
        h->rssi_on = value != 0.0;
        return QRL_OK;
    }
    if (key == QRL_PARAM_OVERLAP_CALLS) {
        // only the path whose ring reuse is fenced for it: real-symbol 4FSK (external soft-bit epilogue)
        if (!(h->kind == QRL_DEMOD_4FSK && h->flag) || h->dmr) { set_err(h, "QRL_PARAM_OVERLAP_CALLS: not supported for this block"); return QRL_EINVAL; }
        QRL_CK(cudaStreamSynchronize(h->stream));
        { int rc = rx_join_host(h); if (rc) return rc; }
        const bool on = value != 0.0;
        if (on && !h->alt_port1) {
            int rc;
            if ((rc = dev_alloc(h, &h->alt_port0, static_cast<size_t>(h->port0_cap) * h->C))) return rc;
            if ((rc = dev_alloc(h, &h->alt_port1, static_cast<size_t>(h->port1_cap) * h->C))) return rc;
            if ((rc = dev_alloc(h, &h->alt_port2, static_cast<size_t>(h->port2_cap) * h->C))) return rc;
            if ((rc = dev_alloc(h, &h->alt_port1_cnt, h->C))) return rc;
            if ((rc = dev_alloc(h, &h->alt_port2_cnt, h->C))) return rc;
            if (h->d_port3) {
                if ((rc = dev_alloc(h, &h->alt_port3, static_cast<size_t>(h->port2_cap) * h->C))) return rc;
                if ((rc = dev_alloc(h, &h->alt_port3_cnt, h->C))) return rc;
            }
            for (int q = 0; q < 2; q++) for (int j = 0; j < 3; j++)
                if (!h->ev_tail[q][j]) QRL_CK(cudaEventCreateWithFlags(&h->ev_tail[q][j], cudaEventDisableTiming));
            for (int i = 0; i < qrl_rx::kMaxSub; i++)
                if (!h->ev_v[i]) QRL_CK(cudaEventCreateWithFlags(&h->ev_v[i], cudaEventDisableTiming));
            QRL_CK(cudaStreamSynchronize(h->stream));
        }
        h->overlap = on;
        return QRL_OK;
    }
    if (key == QRL_PARAM_CARRIER_OFFSET_HZ) {        // gr_demod_base::set_carrier_offset (:1220-1225): phase inc = 2 pi (-offset) / fs
        if (channel >= h->C) { set_err(h, "set_param: channel out of range"); return QRL_EINVAL; }
        if (h->rot.empty()) h->rot.assign(h->C, RotState{ 0u, 0u, 0 });
        const unsigned inc = static_cast<unsigned>(static_cast<int>(static_cast<long long>(std::rint(-value / h->samp_rate * 4294967296.0))));
        h->rot_active = retune(h->rot, channel, inc, h->n_in);
        if (!h->d_rot) { int rc = dev_alloc(h, &h->d_rot, h->C); if (rc) return rc; }
        QRL_CK(cudaStreamSynchronize(h->stream));
        if (h->overlap) { int rc = rx_join_host(h); if (rc) return rc; }
        QRL_CK(cudaMemcpy(h->d_rot, h->rot.data(), sizeof(RotState) * h->C, cudaMemcpyHostToDevice));
        return QRL_OK;
    }
    // ---- run-time setters of the analog blocks.  Kernel parameters travel by value with every launch, so a plain host-side update is
    // enough for scalars; new taps are uploaded after everything in flight has drained and meet the true sample history (the rings)
    // from the next qrl_rx_work on.
    const bool nbfm = h->kind == QRL_DEMOD_NBFM, ssb = h->kind == QRL_DEMOD_SSB, am = h->kind == QRL_DEMOD_AM, wbfm = h->kind == QRL_DEMOD_WBFM;
    auto quiesce = [&]() -> int { QRL_CK(cudaStreamSynchronize(h->stream)); return rx_join_host(h); };
    auto upload = [&](float* dst, const std::vector<float>& t) -> int {
        int rc = quiesce(); if (rc) return rc;
        QRL_CK(cudaMemcpy(dst, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
        return QRL_OK;
    };
    if (key == QRL_PARAM_SQUELCH_DB && (nbfm || ssb || am || wbfm)) {
        // gr_demod_nbfm::set_squelch (:92-95), gr_demod_ssb.cpp:103-106, gr_demod_am.cpp:104-107, gr_demod_wbfm.cpp:88-91: _squelch->set_threshold(dB)
        const double thr = std::pow(10.0, value / 10.0);
        if (ssb) h->ssbp.sq_threshold = thr; else h->nbp.sq_threshold = thr;
        return QRL_OK;
    }
    if (key == QRL_PARAM_AGC_ATTACK && (ssb || am)) {    // gr_demod_ssb::set_agc_attack (:108-111), gr_demod_am.cpp:94-97
        if (ssb) h->ssbp.attack = static_cast<float>(value); else h->nbp.agc_attack = static_cast<float>(value);
        return QRL_OK;
    }
    if (key == QRL_PARAM_AGC_DECAY && (ssb || am)) {     // gr_demod_ssb::set_agc_decay (:113-116), gr_demod_am.cpp:99-102
        if (ssb) h->ssbp.decay = static_cast<float>(value); else h->nbp.agc_decay = static_cast<float>(value);
        return QRL_OK;
    }
    if (key == QRL_PARAM_GAIN && ssb) { h->if_gain = static_cast<float>(value); return QRL_OK; }      // gr_demod_ssb::set_gain (:118-121): _if_gain->set_k
    if (h->kind == QRL_DEMOD_FREEDV) {
        // gr_demod_freedv::set_agc_attack / set_agc_decay (:85-93): the agc2_ff rates, from the next sample on
        if (key == QRL_PARAM_AGC_ATTACK) { h->fdp.attack = static_cast<float>(value); return QRL_OK; }
        if (key == QRL_PARAM_AGC_DECAY) { h->fdp.decay = static_cast<float>(value); return QRL_OK; }
        if (key == QRL_PARAM_SQUELCH_DB) {
            set_err(h, "qrl_rx_set_param: gr_demod_freedv::set_squelch is codec2's (freedv_rx_ss::set_squelch_thresh), behind port 1");
            return QRL_EINVAL;
        }
    }
    if (key == QRL_PARAM_CTCSS && nbfm) {
        // gr_demod_nbfm::set_ctcss (:97-121).  0: tone squelch out of the graph, low-pass audio filter (only when it was in: the first
        // disconnect of :101 throws otherwise and the rest is skipped).  f: ctcss_squelch_ff::set_frequency(f) (new Goertzel filters at
        // the tone and its table neighbours, the block's squelch state is kept), and on the first switch the block goes in front of a
        // band-pass audio filter.
        if (value == 0.0) {
            if (!h->ctc.on) return QRL_OK;
            h->ctc.on = 0;
            return upload(h->d_audio_taps, low_pass_2(1, 8000, 3500, 200, 35, WIN_BLACKMAN_HARRIS));
        }
        static const float tones[38] = { 67.0f, 71.9f, 74.4f, 77.0f, 79.7f, 82.5f, 85.4f, 88.5f, 91.5f, 94.8f, 97.4f, 100.0f, 103.5f, 107.2f,
                                         110.9f, 114.8f, 118.8f, 123.0f, 127.3f, 131.8f, 136.5f, 141.3f, 146.2f, 151.4f, 156.7f, 162.2f, 167.9f,
                                         173.8f, 179.9f, 186.2f, 192.8f, 203.5f, 210.7f, 218.1f, 225.7f, 233.6f, 241.8f, 250.3f };
        const float freq = static_cast<float>(value);
        int idx = -1;
        for (int i = 0; i < 38; i++) if (tones[i] == freq) idx = i;
        const float fl = (idx == -1 || idx == 0) ? static_cast<float>(freq * 0.98) : tones[idx - 1];
        const float fr = (idx == -1 || idx == 37) ? static_cast<float>(freq * 1.02) : tones[idx + 1];
        auto gz = [](float f, float& wr, float& wi) { const float w = static_cast<float>(2.0 * kPi * f / 8000); wr = static_cast<float>(2.0 * std::cos(w)); wi = std::sin(w); };
        gz(fl, h->ctc.wr_l, h->ctc.wi_l); gz(freq, h->ctc.wr_c, h->ctc.wi_c); gz(fr, h->ctc.wr_r, h->ctc.wi_r);
        int rc = quiesce(); if (rc) return rc;
        {   // set_frequency makes new Goertzel objects: their running sums restart (the squelch state machine keeps its state)
            std::vector<NbfmState> stv(h->C);
            QRL_CK(cudaMemcpy(stv.data(), h->d_nb, sizeof(NbfmState) * h->C, cudaMemcpyDeviceToHost));
            for (auto& x : stv) { x.gl1 = x.gl2 = x.gc1 = x.gc2 = x.gr1 = x.gr2 = 0.0f; x.g_processed = 0; }
            QRL_CK(cudaMemcpy(h->d_nb, stv.data(), sizeof(NbfmState) * h->C, cudaMemcpyHostToDevice));
        }
        if (!h->ctc.on) {
            h->ctc.on = 1;
            return upload(h->d_audio_taps, band_pass_2(1, 8000, 300, 3500, 200, 35, WIN_BLACKMAN_HARRIS));
        }
        return QRL_OK;
    }
    if (key == QRL_PARAM_FILTER_WIDTH && (nbfm || ssb || am || wbfm)) {
        const int fw = static_cast<int>(value);
        if (fw <= 0) { set_err(h, "set_filter_width: out of range"); return QRL_EINVAL; }
        std::vector<float> t;
        if (nbfm || wbfm) t = low_pass(1, h->tsr, fw, 1200, WIN_BLACKMAN_HARRIS);                       // gr_demod_nbfm.cpp:82-90, gr_demod_wbfm.cpp:77-85
        else if (am) t = complex_band_pass(1, h->tsr, -fw, fw, 1200, WIN_BLACKMAN_HARRIS);              // gr_demod_am.cpp:84-92
        else t = h->flag ? complex_band_pass_2(1, h->tsr, -fw, -200, 200, 90, WIN_BLACKMAN_HARRIS)      // gr_demod_ssb.cpp:89-101
                         : complex_band_pass_2(1, h->tsr, 200, fw, 200, 90, WIN_BLACKMAN_HARRIS);
        if (t.size() > h->taps2_cap) { set_err(h, "set_filter_width: out of range (filter longer than the block was sized for)"); return QRL_EINVAL; }
        int rc = upload(h->d_taps2, t); if (rc) return rc;
        h->ntaps2 = static_cast<int>(t.size()) / ((ssb || am) ? 2 : 1);
        h->filter_width = fw;
        if (nbfm) h->qd_gain = static_cast<float>(h->tsr / (4 * kPi * fw));
        if (wbfm) h->qd_gain = static_cast<float>(h->tsr / (2 * kPi * fw));
        h->nbp.qd_gain = h->qd_gain;
        if (ssb) {          // the audio band-pass follows the filter width (gain 2 here, 1 in the constructor: the reference's)
            std::vector<float> a = band_pass_2(2, h->tsr, 200, fw, 200, 90, WIN_BLACKMAN_HARRIS);
            if (static_cast<int>(a.size()) != h->ssbp.nt_audio) { set_err(h, "set_filter_width: audio filter length changed"); return QRL_EINVAL; }
            if ((rc = upload(h->d_audio_taps, a))) return rc;
        }
        return QRL_OK;
    }
    set_err(h, "qrl_rx_set_param: key " + std::to_string(key) + " not supported for this block");
    return QRL_EINVAL;
}

static int rx_work_impl(qrl_rx* h, const void* iq_any, long T, long stride, int on_device, int sc16, float sc16_scale);

int qrl_rx_work(qrl_rx* h, const float* iq, long T, long stride, int on_device)
{
    return rx_work_impl(h, iq, T, stride, on_device, 0, 0.0f);
}
int qrl_rx_work_sc16(qrl_rx* h, const short* iq, long T, long stride, float scale, int on_device)
{
    return rx_work_impl(h, iq, T, stride, on_device, 2, scale);
}
int qrl_rx_work_sc8(qrl_rx* h, const signed char* iq, long T, long stride, float scale, int on_device)
{
    return rx_work_impl(h, iq, T, stride, on_device, 1, scale);
}

// sc16: 0 = gr_complex input, 2 = int16 pairs, 1 = int8 pairs (bytes per component)
static int rx_work_impl(qrl_rx* h, const void* iq_any, long T, long stride, int on_device, int sc16, float sc16_scale)
{
    const float* iq = static_cast<const float*>(iq_any);
    if (!h || !iq || T < 0) return QRL_EINVAL;
    if (T > h->Tmax) { set_err(h, "qrl_rx_work: T exceeds max_samples given at create"); return QRL_ERANGE; }
    if (T == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    if (on_device) { int rc = check_device_ptr(h, iq, "qrl_rx_work"); if (rc) return rc; }
    const float2* x = reinterpret_cast<const float2*>(iq);
    long long xstride = stride;
    // stride 0: one stream feeds every channel; it is copied and converted once (one row of T samples), and only the rotation and
    // what follows it run per channel.  The staging is rewritten on the handle's stream, which every call ends waiting for stage 1.
    // Stage 1 is the per-row kernel with in_stride 0: its channels read the one stream mostly from L2.  A kernel that fetches each
    // strip once for a group of channels and rotates it into a second window per channel was slower at every register-tiled shape
    // (stage 1 of 64 ch x 2^22 on an H100: 1.20 against 1.04 ms at /50, 1.95 against 1.25 ms at /125): two windows per CTA halve
    // the occupancy, and the per-channel rotation, not the HBM read, is the cost.
    const bool shared = stride == 0;
    const int rows = shared ? 1 : h->C;
    float2*& staging = shared ? h->d_in1 : h->d_in_staging;
    if (!on_device || sc16) {
        if (!staging) {
            int rc = dev_alloc(h, &staging, static_cast<size_t>(h->Tmax) * rows, false);
            if (rc) return rc;
        }
    }
    if (sc16) {
        // the SDR's wire format (interleaved int16 I/Q, 4 B per sample: half the PCIe bytes of gr_complex); converted on the device
        // exactly like the host converter in front of the reference's source block: float(v) * scale, one rounding
        const short2* s = static_cast<const short2*>(iq_any);
        long long sstride = stride;
        const size_t isz = sc16 == 2 ? sizeof(short2) : sizeof(char2);
        if (!on_device) {
            short2*& wire = shared ? h->d_in1_sc16 : h->d_in_sc16;
            if (!wire) {
                int rc = dev_alloc(h, &wire, static_cast<size_t>(h->Tmax) * rows, false);
                if (rc) return rc;
            }
            if (shared) QRL_CK(cudaMemcpyAsync(wire, iq_any, isz * T, cudaMemcpyHostToDevice, h->stream));
            else QRL_CK(cudaMemcpy2DAsync(wire, isz * h->Tmax, iq_any, isz * stride, isz * T, h->C, cudaMemcpyHostToDevice, h->stream));
            s = wire; sstride = h->Tmax;
        }
        dim3 g(static_cast<unsigned>(std::min<long long>((T + 1023) / 1024, 65535)), rows);
        if (sc16 == 2) sc16_to_fc32_kernel<<<g, 256, 0, h->stream>>>(s, sstride, staging, h->Tmax, T, sc16_scale);
        else sc8_to_fc32_kernel<<<g, 256, 0, h->stream>>>(reinterpret_cast<const char2*>(s), sstride, staging, h->Tmax, T, sc16_scale);
        h->launches++;
        x = staging;
        xstride = shared ? 0 : h->Tmax;
    } else if (!on_device) {
        if (shared) QRL_CK(cudaMemcpyAsync(staging, iq, sizeof(float2) * T, cudaMemcpyHostToDevice, h->stream));
        else QRL_CK(cudaMemcpy2DAsync(staging, sizeof(float2) * h->Tmax, iq, sizeof(float2) * stride,
                                      sizeof(float2) * T, h->C, cudaMemcpyHostToDevice, h->stream));
        x = staging;
        xstride = shared ? 0 : h->Tmax;
    }
    // carrier offset: inside the stage-1 kernel where it can rotate its window, else a separate pass
    h->rot_fused = h->rot_active && stage1_fuses_rotator(h) && !getenv("QRL_ROTATOR_PASS");
    if (h->rot_active && !h->rot_fused) {
        if (!h->d_rot_buf) { int rc = dev_alloc(h, &h->d_rot_buf, static_cast<size_t>(h->Tmax) * h->C, false); if (rc) return rc; }
        dim3 g(static_cast<unsigned>(std::min<long long>((T + 255) / 256, 4096)), h->C);
        rotator_kernel<<<g, 256, 0, h->stream>>>(h->d_rot, x, xstride, h->d_rot_buf, h->Tmax, T, h->n_in);
        h->launches++;
        x = h->d_rot_buf; xstride = h->Tmax;
    }
    // A call of a different length moves the slice boundaries, the symbol-sync scratch regions and the number of slices; the
    // per-slice fences below (ev_v[i], ev_c[q]) pair slice i of this call with slice i of the previous one, so such a call joins the
    // previous call's tail first (no overlap across that one seam).
    const bool seam = h->overlap && h->prev_T != T && h->prev_T >= 0;
    // Overlapped 4FSK calls launch stage 1 of the whole call BEFORE waiting for the tail of call k-2.  Stage 1 writes only the
    // stage-1 ring and its history, which nothing behind the channel filter reads (the channel filter runs on the same stream), so it
    // does not touch the double-buffered ports that tail still owns.  Waiting first put the FIR (about 0.8 ms at 64 x 2^22) behind
    // call k-2's last Viterbi slice, on the loop that sets the step; now it runs under that tail.
    const bool early_fir = h->overlap && !h->fir_group_forced && h->kind == QRL_DEMOD_4FSK && !seam;
    if (h->overlap) {
        h->call_parity ^= 1;
        std::swap(h->d_port0, h->alt_port0); std::swap(h->d_port1, h->alt_port1); std::swap(h->d_port2, h->alt_port2);
        std::swap(h->d_port1_cnt, h->alt_port1_cnt); std::swap(h->d_port2_cnt, h->alt_port2_cnt);
        if (h->d_port3) { std::swap(h->d_port3, h->alt_port3); std::swap(h->d_port3_cnt, h->alt_port3_cnt); }
        h->d_port1f = reinterpret_cast<float*>(h->d_port1);
    }
    // The call is cut into nsub time slices.  Per slice the parallel stages (decimating FIR, channel filter,
    // demod + RRC) run on the caller's stream; the sequential loop stage of slice i runs on s_loop and the
    // FEC stage on s_fec, overlapping the parallel stages of slices i+1.. (channels stay independent).
    bool began = false;
    auto begin_call = [&]() -> int {
        began = true;
        if (h->overlap) {
            // this call writes the buffers call k-2 used: wait for that call's tail, then they are free
            for (int j = 0; j < 3; j++) QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_tail[h->call_parity][j], 0));
            if (seam) for (int j = 0; j < 3; j++) QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_tail[h->call_parity ^ 1][j], 0));
        }
        QRL_CK(cudaMemsetAsync(h->d_port1_cnt, 0, sizeof(int) * h->C, h->stream));
        QRL_CK(cudaMemsetAsync(h->d_port2_cnt, 0, sizeof(int) * h->C, h->stream));
        if (h->d_port3_cnt) QRL_CK(cudaMemsetAsync(h->d_port3_cnt, 0, sizeof(int) * h->C, h->stream));
        QRL_CK(cudaEventRecord(h->ev_start, h->stream));
        QRL_CK(cudaStreamWaitEvent(h->s_loop, h->ev_start, 0));
        QRL_CK(cudaStreamWaitEvent(h->s_loop2, h->ev_start, 0));
        QRL_CK(cudaStreamWaitEvent(h->s_fec, h->ev_start, 0));
        if (h->s_par) QRL_CK(cudaStreamWaitEvent(h->s_par, h->ev_start, 0));
        return QRL_OK;
    };
    if (early_fir) {
        // stage 1 still follows everything the caller queued on its stream before this call (its input)
        QRL_CK(cudaEventRecord(h->ev_start, h->stream));
        if (h->s_par) QRL_CK(cudaStreamWaitEvent(h->s_par, h->ev_start, 0));
    } else {
        int rc = begin_call(); if (rc) return rc;
    }
    cudaStream_t sp = h->par();
    // overlapped calls keep the pipeline full across calls: two big slices are enough and cost least (every symbol-sync launch pays
    // its own start-up)
    int nsub = (h->overlap && !h->nsub_forced) ? 2 : h->nsub;
    if (T < 32768L * nsub) nsub = static_cast<int>(std::max<long>(1, T / 32768));
    const long long k_call0 = h->n1;
    h->port0_n = 0;
    for (int i = 0; i < nsub; i++) {
        // slice boundaries on multiples of 2*D: the slice base stays 16-byte aligned (TMA bulk fill) and every slice
        // produces the same number of stage-1 outputs
        const long long q2d = 2LL * h->D1;
        auto cut = [&](int j) { return j >= nsub ? static_cast<long long>(T) : (static_cast<long long>(T) * j / nsub) / q2d * q2d; };
        const long long t0 = cut(i), t1 = cut(i + 1);
        if (t1 <= t0) continue;
        const long long Ti = t1 - t0;
        cudaEvent_t pe = nullptr;
        // ---- stage 1: decimating FIR, one launch per group of slices (outputs k with D k <= last absolute input index)
        // stage-1 launch schedule: slice 0 alone (the loop stage starts as early as possible), then fir_group slices
        // per launch (bigger launches run closer to the HBM roofline)
        // (overlapped calls: the pipeline is already full, one launch for the whole call)
        const bool fir_here = h->overlap && !h->fir_group_forced ? (i == 0) : ((i == 0) || ((i - 1) % h->fir_group == 0));
        if (fir_here) {
            const long long tg1 = cut(h->overlap && !h->fir_group_forced ? nsub : (i == 0 ? 1 : std::min(i + h->fir_group, nsub)));
            const long long Tg = tg1 - t0;
            const float2* xg = x + t0;
            const long long Ng = h->n_in + Tg;
            const long long kg0 = h->n1;
            const long long kg1 = (Ng * h->L1 + h->D1 - 1) / h->D1;       // outputs i with floor(i M / L) <= N - 1
            pe = h->prof.begin(0, sp);
            int rc = stage1(h, xg, xstride, Tg, kg0, kg1);
            if (!rc && h->kind == QRL_DEMOD_SSB && kg1 > kg0) {
                // gr_demod_ssb's multiply_const_cc(_if_gain) sits between the resampler and the side-band filter: the gain is applied
                // to the samples as they pass (8 ksps), so after set_gain the filter's history keeps the old gain, like the reference's
                dim3 gs(static_cast<unsigned>((kg1 - kg0 + 255) / 256), h->C);
                scale2_ring_kernel<<<gs, 256, 0, sp>>>(static_cast<float2*>(h->r1.d), h->r1.mask, h->r1.stride, kg0, kg1, h->if_gain, 1.0f);
                h->launches++;
            }
            h->prof.end(pe);
            if (rc) return rc;
            dim3 g((h->H + 127) / 128, h->C);
            if (h->rot_fused) frontend_hist_kernel<<<g, 128, 0, sp>>>(h->d_rot, xg, xstride, Tg, h->n_in, h->d_hist[h->hist_cur], h->d_hist[h->hist_cur ^ 1], h->H);
            else hist_update_kernel<<<g, 128, 0, sp>>>(xg, xstride, Tg, h->d_hist[h->hist_cur], h->d_hist[h->hist_cur ^ 1], h->H);
            h->launches++;
            h->hist_cur ^= 1;
            h->n_in = Ng; h->n1 = kg1;
        }
        if (!began) { int rc2 = begin_call(); if (rc2) return rc2; }
        // ---- the stages behind it advance slice by slice
        const long long N = h->n_in_s + Ti;
        const long long k0 = h->n1_s;
        const long long k1 = (N * h->L1 + h->D1 - 1) / h->D1;
        h->n_in_s = N; h->n1_s = k1;
        h->cur_k1[i] = k1;
        const long long n_new = k1 - k0;
        h->port0_n += static_cast<long>(n_new);
        const Slice s{ i, k0, k1, n_new, k_call0, h->d_nsoft + static_cast<size_t>(i) * h->C, sp,
                       dim3(static_cast<unsigned>((std::max<long long>(n_new, 1) + kTileThreads - 1) / kTileThreads), h->C), (h->C + 31) / 32 };
        int rc;
        switch (h->kind) {
        case QRL_DEMOD_DSSS: rc = slice_dsss(h, s); break;
        case QRL_DEMOD_SSB: case QRL_DEMOD_FREEDV: case QRL_DEMOD_AM: case QRL_DEMOD_NBFM: case QRL_DEMOD_WBFM: rc = slice_analog(h, s); break;
        case QRL_DEMOD_BPSK: case QRL_DEMOD_2FSK: rc = slice_fll_bpsk_2fsk(h, s); break;      // (GMSK runs as 2FSK)
        case QRL_DEMOD_4FSK: rc = slice_4fsk(h, s); break;                                    // (M17 and DMR run as 4FSK)
        default: rc = slice_qpsk(h, s); break;
        }
        if (rc) return rc;
    }
    if (!began) { int rc = begin_call(); if (rc) return rc; }     // every slice was empty
    if (h->kind == QRL_DEMOD_DSSS) {          // port 0 holds 5200 sps items (13 / 50 of the stage-1 items counted in the loop)
        const long long o_end = (h->n1_s * 13 + 49) / 50;
        h->port0_n = static_cast<long>(o_end - h->ds_o_call0);
        h->ds_o_call0 = o_end;
    }
    if (h->rssi_on && h->port0_n > 0) {
        // port 0 of this call is complete on the parallel stream: append to the |x|^2 ring, evaluate the latest RSSI value
        rssi_kernel<<<h->C, 256, 0, sp>>>(h->d_port0, h->port0_cap, static_cast<int>(std::min<long>(h->port0_n, h->port0_cap)),
                                          h->rssi_n, h->d_rssi_ring, h->d_rssi_y, h->d_rssi_db);
        h->launches++;
        h->rssi_n += std::min<long>(h->port0_n, h->port0_cap);
    }
    for (int i = 0; i < nsub; i++) h->prev_k1[i] = h->cur_k1[i];
    h->prev_nsub = nsub;
    h->prev_T = T;
    if (h->overlap) {
        // the caller's stream only waits for the parallel stages (the input has been consumed); the loop / FEC tail runs
        // on under the next call and is joined by qrl_rx_join / qrl_rx_sync / qrl_rx_read_port
        QRL_CK(cudaEventRecord(h->ev_tail[h->call_parity][0], h->s_loop));
        QRL_CK(cudaEventRecord(h->ev_tail[h->call_parity][1], h->s_fec));
        QRL_CK(cudaEventRecord(h->ev_tail[h->call_parity][2], h->s_epi ? h->s_epi : h->s_loop));
        if (h->s_par) { QRL_CK(cudaEventRecord(h->ev_par_done, h->s_par)); QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_par_done, 0)); }
        QRL_CK(cudaGetLastError());
        return QRL_OK;
    }
    QRL_CK(cudaEventRecord(h->ev_loop_done, h->s_loop));
    QRL_CK(cudaEventRecord(h->ev_loop2_done, h->s_loop2));
    QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_loop2_done, 0));
    QRL_CK(cudaEventRecord(h->ev_fec_done, h->s_fec));
    if (h->s_par) { QRL_CK(cudaEventRecord(h->ev_par_done, h->s_par)); QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_par_done, 0)); }
    QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_loop_done, 0));
    QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_fec_done, 0));
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}

int qrl_rx_join(qrl_rx* h)
{
    if (!h) return QRL_EINVAL;
    if (!h->overlap) return QRL_OK;
    for (int j = 0; j < 3; j++) QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_tail[h->call_parity][j], 0));
    return QRL_OK;
}

int qrl_rx_profile(qrl_rx* h, int enable)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    h->prof.reset(enable != 0);
    return QRL_OK;
}

int qrl_rx_profile_read(qrl_rx* h, int stage, double* ms_total, long* n_launches)
{
    if (!h || stage < 0 || stage >= h->prof.stages()) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (h->overlap) { int rc = rx_join_host(h); if (rc) return rc; }
    h->prof.read(stage, ms_total, n_launches);
    return QRL_OK;
}

int qrl_rx_sync(qrl_rx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (h->overlap) return rx_join_host(h);
    return QRL_OK;
}

int qrl_rx_rssi(qrl_rx* h, float level, float* rssi_db_host)
{
    if (!h || !rssi_db_host) return QRL_EINVAL;
    if (!h->rssi_on || !h->d_rssi_db) { set_err(h, "qrl_rx_rssi: enable QRL_PARAM_RSSI first"); return QRL_EINVAL; }
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (h->s_par) QRL_CK(cudaStreamSynchronize(h->s_par));
    QRL_CK(cudaMemcpy(rssi_db_host, h->d_rssi_db, sizeof(float) * h->C, cudaMemcpyDeviceToHost));
    for (int c = 0; c < h->C; c++) rssi_db_host[c] = (h->rssi_n > 0 ? rssi_db_host[c] : -180.0f) + level;      // add_const_ff(level)
    return QRL_OK;
}

int qrl_rx_num_ports(const qrl_rx* h) { return h ? h->nports : QRL_EINVAL; }
int qrl_rx_port_itemsize(const qrl_rx* h, int port)
{
    if (!h || port < 0 || port >= h->nports) return QRL_EINVAL;
    if (port == 0) return 8;
    if (port == 1 && h->kind == QRL_DEMOD_FREEDV) return 2;        // int16 modem samples
    if (port == 1) return (h->kind == QRL_DEMOD_NBFM || h->kind == QRL_DEMOD_SSB || h->kind == QRL_DEMOD_AM || h->kind == QRL_DEMOD_WBFM) ? 4 : 8;
    if (port == 3 && h->dmr) return 4;
    return 1;
}

int qrl_rx_port_device(qrl_rx* h, int port, void** data, long* cap, int** counts)
{
    if (!h || port < 0 || port >= h->nports) return QRL_EINVAL;
    if (port == 0) { *data = h->d_port0; *cap = h->port0_cap; *counts = nullptr; }
    else if (port == 1) {
        *data = h->d_port1; *counts = h->d_port1_cnt;
        *cap = (h->kind == QRL_DEMOD_NBFM || h->kind == QRL_DEMOD_SSB || h->kind == QRL_DEMOD_AM || h->kind == QRL_DEMOD_WBFM) ? 2 * h->port1_cap : h->port1_cap;      // float view of the same buffer
        if (h->kind == QRL_DEMOD_FREEDV) *cap = 4 * h->port1_cap;                                                                   // int16 view
    }
    else if (port == 2) { *data = h->d_port2; *cap = h->port2_cap; *counts = h->d_port2_cnt; }
    else if (h->dmr) { *data = h->d_port3f; *cap = h->port0_cap; *counts = nullptr; }      // one float per port-0 sample
    else { *data = h->d_port3; *cap = h->port2_cap; *counts = h->d_port3_cnt; }
    return QRL_OK;
}

int qrl_rx_read_port(qrl_rx* h, int port, void* dst, long cap, int* counts, int dst_on_device)
{
    if (!h || port < 0 || port >= h->nports || !counts) return QRL_EINVAL;
    void* src; long scap; int* dcnt;
    int rc = qrl_rx_port_device(h, port, &src, &scap, &dcnt);
    if (rc) return rc;
    const int isz = qrl_rx_port_itemsize(h, port);
    long maxn = 0;
    if (h->overlap) { QRL_CK(cudaStreamSynchronize(h->stream)); rc = rx_join_host(h); if (rc) return rc; }
    if (dcnt) {
        QRL_CK(cudaMemcpyAsync(counts, dcnt, sizeof(int) * h->C, cudaMemcpyDeviceToHost, h->stream));
        QRL_CK(cudaStreamSynchronize(h->stream));
        for (int c = 0; c < h->C; c++) { if (counts[c] > scap) counts[c] = static_cast<int>(scap); maxn = std::max<long>(maxn, counts[c]); }
    } else {
        for (int c = 0; c < h->C; c++) counts[c] = static_cast<int>(h->port0_n);
        maxn = h->port0_n;
    }
    if (dst && maxn > 0) {
        const long w = std::min(maxn, cap);
        QRL_CK(cudaMemcpy2DAsync(dst, static_cast<size_t>(cap) * isz, src, static_cast<size_t>(scap) * isz, static_cast<size_t>(w) * isz, h->C,
                             dst_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, h->stream));
    }
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}

long qrl_rx_launch_count(const qrl_rx* h) { return h ? h->launches : 0; }
int qrl_rx_sm_partition(const qrl_rx* h, int* loop_sms, int* parallel_sms)
{
    if (!h) return QRL_EINVAL;
    if (loop_sms) *loop_sms = h->sm_loop;
    if (parallel_sms) *parallel_sms = h->sm_par;
    return QRL_OK;
}

// ---------------------------------------------------------------------------------------------- TX
// gr_zero_idle_bursts (gr_zero_idle_bursts.cpp:47-86) as host-side bookkeeping: the "zero_samples" tags waiting per channel and the count
// still running at the end of the last call; a call turns them into {channel, first item, end item} ranges that one kernel clears
// (a tag loads the counter, a later one overrides what is left of it, one output is cleared per count).  Shared by gr_mod_dmr (delay
// 62) and the MMDVM modulators (delay 0).
struct ZeroIdle {
    std::vector<std::map<long long, unsigned long long>> tags;      // per channel: start item -> count (first registered wins)
    std::vector<unsigned long long> counter;                       // per channel: count still running at the end of the last call
    long long* d_ranges = nullptr; size_t ranges_cap = 0;
    void init(int C) { tags.assign(C, {}); counter.assign(C, 0); }
    // tag for item `start` (already corrected for the block's delay); `produced` = items the block has put out so far
    void add(int channel, int C, long long start, unsigned long long val, long long produced)
    {
        if (start < produced) {                                                  // late: clear what is left of the count
            const unsigned long long late = static_cast<unsigned long long>(produced - start);
            if (late >= val) return;
            val -= late; start = produced;
        }
        for (int c = (channel < 0 ? 0 : channel); c < (channel < 0 ? C : channel + 1); c++) tags[c].emplace(start, val);
    }
    // ranges of the items [m0, m1) this call produces, as {c, a0 - base, a1 - base} triples
    void collect(int C, long long m0, long long m1, long long base, std::vector<long long>& ranges)
    {
        for (int c = 0; c < C; c++) {
            auto& tg = tags[c];
            tg.erase(tg.begin(), tg.lower_bound(m0));
            unsigned long long cnt = counter[c];
            if (cnt == 0 && (tg.empty() || tg.begin()->first >= m1)) continue;
            long long cur = m0;
            auto it = tg.begin();
            while (true) {
                const long long next = (it != tg.end() && it->first < m1) ? it->first : m1;
                const long long z_end = cnt >= static_cast<unsigned long long>(next - cur) ? next : cur + static_cast<long long>(cnt);
                if (z_end > cur) { ranges.push_back(c); ranges.push_back(cur - base); ranges.push_back(z_end - base); }
                cnt -= static_cast<unsigned long long>(z_end - cur);
                if (next == m1) break;
                cnt = it->second; cur = next; it = tg.erase(it);
            }
            counter[c] = cnt;
        }
    }
    // upload the triples (growing the device buffer if needed); returns a CUDA error code
    cudaError_t upload(const std::vector<long long>& ranges, cudaStream_t stream)
    {
        if (ranges.size() > ranges_cap) {
            cudaError_t e = cudaStreamSynchronize(stream); if (e != cudaSuccess) return e;
            if (d_ranges) { e = cudaFree(d_ranges); if (e != cudaSuccess) return e; d_ranges = nullptr; }
            ranges_cap = 2 * ranges.size() + 48;
            e = cudaMalloc(&d_ranges, sizeof(long long) * ranges_cap); if (e != cudaSuccess) return e;
        }
        return cudaMemcpyAsync(d_ranges, ranges.data(), sizeof(long long) * ranges.size(), cudaMemcpyHostToDevice, stream);
    }
    void release() { if (d_ranges) cudaFree(d_ranges); d_ranges = nullptr; }
};

// the transmit chains (DESIGN.md section 5): tx_create picks one and designs its taps and rings, qrl_tx_work runs its work function
enum class TxChain { Fsk, Psk, M17, Dmr, Dsss, Nbfm, Ssb, Am, Freedv };
struct qrl_tx : HandleBase {
    TxChain chain = TxChain::Fsk;
    int txm = 0, sym_per_item = 0;  // the byte-fed chains: tx_bits_kernel mode (TXM_*), symbols (DSSS: chips) per input byte
    int samp_rate = 0, flag = 0, C = 0;
    long max_items = 0;
    int L1 = 1, nt1 = 0;            // first interpolation (RRC): L1 arms of nt1 taps
    int L2 = 1, nt2 = 0;            // final interpolation (4FSK: the x20 low-pass): L2 arms of nt2 taps
    float* d_arms1 = nullptr; float* d_arms2 = nullptr;
    float fm_sens = 0, amplif = 0, bb_gain = 1.0f, pulse_scale = 0.66666666f;
    int repeat_only = 0;
    int M2 = 1;                     // gr_mod_m17 / gr_mod_dmr: 4 symbols per byte, IF stage at 24 ksps, x L2 / M2 rational interpolator
    float am_dc = 0.0f;             // gr_mod_am: the carrier added to the audio
    // gr_mod_nbfm::set_ctcss: multiply_const_ff gain and the CTCSS tone source (fxpt_nco phase / increment, advanced per sample with the tone on)
    float audio_gain = 0.99f; bool tone_on = false; unsigned tone_phase = 0, tone_inc = 0;
    // gr_mod_dmr: the m17 path with gr_zero_idle_bursts in place of the IF low-pass (a delay of history - 1 items + "zero_samples" tags)
    long long zi_delay_items = 0; unsigned zi_tag_delay = 0;
    ZeroIdle zi;                                                      // gr_mod_dmr: gr_zero_idle_bursts(62)
    TxBitState* d_bits = nullptr;
    unsigned char* d_in = nullptr; size_t in_isz = 1;   // [C][max_items] staging of host input: bytes, float audio (NBFM / SSB / AM) or int16 (FreeDV)
    float* d_sym = nullptr; unsigned sym_mask = 0; long long sym_stride = 0;    // float (4FSK) / float2 (QPSK)
    float2* d_if = nullptr; unsigned if_mask = 0; long long if_stride = 0;
    float2* d_out = nullptr; long long out_stride = 0; long n_out_last = 0;
    long long n_sym = 0;           // symbols produced so far (absolute)
    TxAnalogState* d_an = nullptr;                                                 // analog modulators (NBFM / SSB / AM)
    float* d_ra = nullptr; unsigned ra_mask = 0; long long ra_stride = 0;          // audio ring
    float* d_rb = nullptr;                                                         // filtered audio ring (same geometry)
    float2* d_rc = nullptr; unsigned rc_mask = 0; long long rc_stride = 0;         // SSB clip ring / NBFM IF-filter ring
    float2* d_rs2 = nullptr;                                                       // SSB stretcher ring (same geometry as rc)
    float* d_lpf = nullptr; int nt_lpf = 0; float* d_cfilt = nullptr; int nt_cfilt = 0;
    double pe_b0 = 0, pe_b1 = 0, pe_a1 = 0;
    long long n_audio = 0, n_mid = 0;        // audio samples consumed / mid-rate items produced (host mirror of the device counters)
    // 4FSK: the three stages (bit chain, pulse shaping + FM scan, x20 interpolator) run slice by slice on three streams
    static constexpr int kTxSub = 8;
    cudaStream_t s_bits = nullptr, s_shape = nullptr;
    cudaEvent_t ev_start = nullptr, ev_bits[kTxSub] = { nullptr }, ev_shape[kTxSub] = { nullptr }, ev_shape_done = nullptr, ev_out_done = nullptr;
    // optional per-stage device timing (qrl_tx_profile): 0 = bit chain, 1 = pulse shaping / FM scan, 2 = final interpolator
    StageProfiler prof{ 4 };
};
namespace {
// the interpolator and resampler kernels stage a whole arm table (L arms of nt taps) in shared memory
bool arms_fit(int L, int nt) { return static_cast<size_t>(L) * nt * sizeof(float) <= 40 * 1024; }
int arms_nt(const std::vector<float>& taps, int L) { return (static_cast<int>(taps.size()) + L - 1) / L; }
// register-tiled interpolator shapes.  tx_create pads a shorter arm table to the instance's taps per arm, so the same predicate
// picks the instance in qrl_tx_work: interp_fir_ccf_rt_kernel<20, 35, 8, 16> (4FSK's final x20), interp_fir_ccf_kernel<4, 16, 8, 64> (QPSK)
constexpr int kFskRtL = 20, kFskRtNT = 35, kQpskRtL = 4, kQpskRtNT = 16;
bool fsk_rt(int L2, int nt2) { return L2 == kFskRtL && nt2 <= kFskRtNT; }
bool qpsk_rt(int L1, int nt1) { return L1 == kQpskRtL && nt1 <= kQpskRtNT; }
// what a chain's create function designs; tx_create uploads the tables and allocates the rings
struct TxDesign {
    std::vector<float> t1, t2, lpf, cfilt;     // prototypes of d_arms1 (L1 arms of nt1) and d_arms2 (L2 arms of nt2); d_lpf, d_cfilt as given
    long long sym = 0, if_ = 0, rc = 0, ra = 0, out = 0;      // items each ring must hold (0: the chain has no such ring); out_stride
    int sym_floats = 1;                                       // 2: complex symbols
    bool rb = false, rs2 = false;                             // d_rb in d_ra's geometry, d_rs2 in d_rc's
};
// a [C][capacity] ring of at least min_items items, each `per_item` Ts
extern "C++" template <class T> int tx_ring(qrl_tx* h, T** d, unsigned* mask, long long* stride, long long min_items, int per_item = 1)
{
    const unsigned cap = pow2_at_least(min_items); *mask = cap - 1; *stride = cap;
    return dev_alloc(h, d, static_cast<size_t>(cap) * h->C * per_item);
}
void create_fsk(qrl_tx* h, TxDesign& d, int kind, int sps, int samp_rate, int fw)
{
    if (kind == QRL_MOD_4FSK) {
        // gr_mod_4fsk.cpp:55-92
        int sym_sps = sps, nfilts = sym_sps * 10, second_interp = 20;
        if (sps == 2) { sym_sps = 5; second_interp = 2; nfilts = 256; }
        int spacing = 2; h->amplif = 0.8f;
        if (h->flag) { h->amplif = 0.9f; spacing = 1; }
        h->repeat_only = h->flag ? 0 : 1;
        h->txm = TXM_4FSK; h->sym_per_item = 8;
        d.t1 = root_raised_cosine(sym_sps, sym_sps, 1, 0.2, nfilts);
        h->L1 = sym_sps;
        h->fm_sens = static_cast<float>((spacing * kPi) / sym_sps);
        h->L2 = second_interp;
    } else if (kind == QRL_MOD_GMSK) {
        // gr_mod_gmsk.cpp:30-100: the 2FSK (fm) modulator path with a Gaussian pulse (BT 0.3), sensitivity (pi/2)/sps and a
        // x5 (x1 for the 10k mode) final interpolation; instances gr_mod_base.cpp:160-162
        int nfilts = 35, second_interp = 5;
        if (sps == 10) { sps = 50; second_interp = 1; nfilts = 55; }
        if (sps == 50) nfilts = 55;
        if (sps == 100) nfilts = 35;
        if ((nfilts % 2) == 0) nfilts += 1;
        h->flag = 1;
        h->amplif = 0.9f; h->repeat_only = 0; h->pulse_scale = 1.0f;
        h->txm = TXM_2FSK; h->sym_per_item = 16;
        d.t1 = gaussian(sps, sps, 0.3, nfilts);
        h->L1 = sps;
        h->fm_sens = static_cast<float>((kPi / 2) / sps);
        h->L2 = second_interp;
    } else {
        // gr_mod_2fsk.cpp:43-76
        int nfilts = 25 * sps, spacing = 2; h->amplif = 0.8f;
        if (h->flag) { spacing = 1; h->amplif = 0.9f; }
        if (sps == 5) nfilts = nfilts * 5;
        if ((nfilts % 2) == 0) nfilts += 1;
        h->repeat_only = h->flag ? 0 : 1;
        h->pulse_scale = 1.0f;
        h->txm = TXM_2FSK; h->sym_per_item = 16;
        d.t1 = root_raised_cosine(sps, sps, 1, 0.2, nfilts);
        h->L1 = sps;
        h->fm_sens = static_cast<float>((spacing * kPi / 2) / sps);
        h->L2 = 10;
    }
    d.t2 = low_pass(h->L2, samp_rate, fw, fw, WIN_HAMMING);
    h->nt1 = arms_nt(d.t1, h->L1); h->nt2 = arms_nt(d.t2, h->L2);
    if (fsk_rt(h->L2, h->nt2)) h->nt2 = kFskRtNT;
    const long long max_sym = static_cast<long long>(h->sym_per_item) * h->max_items;
    d.sym = max_sym + 64; d.if_ = max_sym * h->L1 + 128; d.out = max_sym * h->L1 * h->L2;
}
void create_psk(qrl_tx* h, TxDesign& d, int kind, int sps)
{
    if (kind == QRL_MOD_QPSK) {
        // gr_mod_qpsk.cpp:58-75
        const int nfilts = sps > 120 ? 11 : (sps > 10 ? 13 : 15);
        d.t1 = root_raised_cosine(sps, sps, 1, 0.35, nfilts * sps);
        h->txm = TXM_QPSK; h->sym_per_item = 8;
    } else {
        // gr_mod_bpsk.cpp:44-56
        d.t1 = root_raised_cosine(sps, sps, 1, 0.35, 11 * sps);
        h->txm = TXM_BPSK; h->sym_per_item = 16;
    }
    h->L1 = sps; h->nt1 = arms_nt(d.t1, sps);
    if (h->txm == TXM_QPSK && qpsk_rt(h->L1, h->nt1)) h->nt1 = kQpskRtNT;
    h->amplif = 0.6f;
    const long long max_sym = static_cast<long long>(h->sym_per_item) * h->max_items;
    d.sym = max_sym + 64; d.sym_floats = 2; d.out = max_sym * h->L1;
}
int create_m17_dmr(qrl_tx* h, TxDesign& d, bool dmr, int sps, int samp_rate, int fw)
{
    h->amplif = 0.9f; h->repeat_only = 0;
    h->txm = TXM_M17; h->sym_per_item = 4;
    if (!dmr) {
        // gr_mod_m17.cpp:30-95: pulse shaping x5 (RRC 0.5, 250 + 1 taps) -> x0.66666666 -> frequency modulator (pi / 5) -> low-pass at
        // 24 ksps -> x0.9 -> bb gain -> rational_resampler_ccf(sps = 125, 3)
        d.t1 = root_raised_cosine(5, 5, 1, 0.5, 250);
        h->fm_sens = static_cast<float>(kPi / 5);
        d.cfilt = low_pass(1, 24000, fw, fw, WIN_BLACKMAN_HARRIS);
        h->nt_cfilt = static_cast<int>(d.cfilt.size());
        d.t2 = low_pass(sps, 3.0 * samp_rate, 12000, 12000, WIN_BLACKMAN_HARRIS);
    } else {
        // gr_mod_dmr.cpp:27-93: pulse shaping x5 (RRC(5, 24000, 4800, 0.2, 125 taps)) -> x0.66666666 -> frequency modulator
        // (pi * 4800 * 0.85 / 24000) -> gr_zero_idle_bursts(62) -> x0.9 -> bb gain -> rational_resampler_ccf(sps, 3, low_pass_2(sps, 3 fs,
        // fw, 2000, 60, BH)); the fft_filter_ccf of :72-73 is never connected
        const float if_samp_rate = 24000, symbol_rate = if_samp_rate / 5.0f;
        d.t1 = root_raised_cosine(5, if_samp_rate, symbol_rate, 0.2, 25 * 5);
        h->zi_tag_delay = static_cast<unsigned>((d.t1.size() - 1) / 2);                      // gr_mod_dmr.cpp:58
        h->zi_delay_items = h->zi_tag_delay > 0 ? 2 * 720 - 1 : 0;                             // gr_zero_idle_bursts.cpp:35-38, bursttimer.h:30
        h->fm_sens = static_cast<float>((kPi * symbol_rate * 0.85) / if_samp_rate);
        d.t2 = low_pass_2(sps, 3.0 * samp_rate, fw, 2000, 60, WIN_BLACKMAN_HARRIS);
    }
    h->L1 = 5; h->nt1 = arms_nt(d.t1, 5);
    h->L2 = sps; h->M2 = 3; h->nt2 = arms_nt(d.t2, sps);
    if (sps <= 3 || !arms_fit(h->L2, h->nt2)) { set_err(h, dmr ? "make_gr_mod_dmr: unsupported sps" : "make_gr_mod_m17: unsupported sps"); return QRL_EINVAL; }
    if (dmr) h->zi.init(h->C);
    const long long max_sym = 8LL * h->max_items;      // the symbol and IF rings have room for 8 symbols per byte
    d.sym = max_sym + 64; d.if_ = max_sym * h->L1 + 128 + h->zi_delay_items;
    d.rc = max_sym * h->L1 + 512 + h->nt2;             // behind the IF low-pass / delay
    d.out = (static_cast<long long>(h->sym_per_item) * h->max_items * h->L1 * h->L2 + h->M2 - 1) / h->M2 + 8;
    return QRL_OK;
}
// gr_mod_dsss.cpp:27-93: scrambler -> cc_encoder -> Barker-13 spreading -> {-1, +1} -> rational_resampler_ccf(sps, 1, RRC(sps, sps, 1,
// 0.35, 11 sps)) -> x0.65 -> bb gain -> rational_resampler_ccf(50, 13, low_pass(50, 5200 * 50, fw, 5 fw)) ->
// rational_resampler_ccf(50, 1, low_pass(50, fs, fw, 5 fw)); one input byte = 208 chips = 10^6 output samples (sps = 25)
int create_dsss(qrl_tx* h, TxDesign& d, int sps, int samp_rate, int fw)
{
    h->amplif = 0.65f;
    h->txm = TXM_DSSS; h->sym_per_item = 16 * 13;
    d.t1 = root_raised_cosine(sps, sps, 1, 0.35, 11 * sps);
    h->L1 = sps; h->nt1 = arms_nt(d.t1, sps);
    const std::vector<float> tif = low_pass(50.0, 5200.0 * 50, fw, fw * 5, WIN_HAMMING);
    h->nt_cfilt = arms_nt(tif, 50);
    d.t2 = low_pass(50, samp_rate, fw, fw * 5, WIN_HAMMING);
    h->L2 = 50; h->nt2 = arms_nt(d.t2, 50);
    if (!arms_fit(50, std::max(h->nt2, h->nt_cfilt)) || !arms_fit(h->L1, h->nt1)) {
        set_err(h, "make_gr_mod_dsss: filter_width too small for the shared-memory arm tables"); return QRL_EINVAL;
    }
    d.cfilt = make_arms(tif, 50, h->nt_cfilt);
    const long long max_sym = static_cast<long long>(h->sym_per_item) * h->max_items;         // chips per call
    const long long n20 = (max_sym * h->L1 * 50 + 12) / 13;                                    // 20 ksps items per call
    d.sym = max_sym + 64; d.sym_floats = 2;                                                    // complex chips
    d.if_ = max_sym * h->L1 + h->nt_cfilt + 128; d.rc = n20 + 8 + h->nt2 + 512; d.out = (n20 + 1) * 50;
    return QRL_OK;
}
// gr_mod_nbfm.cpp:35-63 (sps = final interpolation, 20)
void create_nbfm(qrl_tx* h, TxDesign& d, int sps, int samp_rate, int fw)
{
    double a[2], b[2];
    preemph_taps(8000, 50e-6, -1.0, a, b);
    h->pe_b0 = b[0]; h->pe_b1 = b[1]; h->pe_a1 = a[1];
    d.lpf = low_pass_2(1, 8000, 3500, 200, 35, WIN_BLACKMAN_HARRIS);
    d.t1 = low_pass_2(25, 50000 * 4, fw, 3500, 60, WIN_BLACKMAN_HARRIS);          // 25/4 resampler arms
    h->L1 = 25; h->nt1 = arms_nt(d.t1, 25);
    h->fm_sens = static_cast<float>(4 * kPi * fw / 50000.0f);
    d.cfilt = low_pass_2(1, 50000, fw, 3500, 60, WIN_BLACKMAN_HARRIS);
    h->nt_cfilt = static_cast<int>(d.cfilt.size());
    d.t2 = low_pass_2(sps, samp_rate, fw, 3500, 60, WIN_BLACKMAN_HARRIS);
    h->L2 = sps; h->nt2 = arms_nt(d.t2, sps);
    h->amplif = 0.8f;
    const long long max_mid = h->max_items * 25 / 4 + 8;                                       // 50 ksps items per call
    d.ra = h->max_items + 512; d.rb = true;
    d.rc = max_mid + 512; d.sym = max_mid + 64; d.if_ = max_mid + 128; d.out = max_mid * h->L2;
}
// gr_mod_ssb.cpp:40-58 (sps = final interpolation, 125; flag = sb)
void create_ssb(qrl_tx* h, TxDesign& d, int sps, int samp_rate, int fw)
{
    d.lpf = band_pass_2(1, 8000, 300, fw, 200, 90, WIN_BLACKMAN_HARRIS);
    d.cfilt = h->flag ? complex_band_pass_2(1, 8000, -fw, -200, 200, 90, WIN_BLACKMAN_HARRIS)
                      : complex_band_pass_2(1, 8000, 200, fw, 200, 90, WIN_BLACKMAN_HARRIS);
    h->nt_cfilt = static_cast<int>(d.cfilt.size() / 2);
    d.t2 = low_pass_2(sps, samp_rate, fw, fw, 90, WIN_BLACKMAN_HARRIS);
    h->L2 = sps; h->nt2 = arms_nt(d.t2, sps);
    h->amplif = 0.9f;
    const long long max_mid = h->max_items + 8;                                                // 8 ksps complex items per call
    d.ra = h->max_items + 512; d.rc = max_mid + 512; d.rs2 = true; d.if_ = max_mid + 128; d.out = max_mid * h->L2;
}
// gr_mod_am.cpp:25-72: agc2_ff -> rail -> x0.95 -> band_pass_2(1, 8000, 300, 3000, 200, 60, Hamming) -> + 0.5 cos(0) -> float_to_complex ->
// rational_resampler_ccf(sps, 1, low_pass(sps, fs, fw, fw)) -> x0.5 -> bb gain -> fft_filter_ccc(complex_band_pass_2(1, fs, -fw, fw, 1200,
// 120, BH)).  The band is symmetric, so the complex taps are the low-pass prototype times e^{j0}: imaginary parts exactly 0 and the
// filter is the real-tap ring FIR (same accumulation, see oracle fircc_work with hi = 0).
int create_am(qrl_tx* h, TxDesign& d, int sps, int samp_rate, int fw)
{
    h->amplif = 0.5f;
    d.lpf = band_pass_2(1, 8000, 300, 3000, 200, 60, WIN_HAMMING);
    d.t2 = low_pass(sps, samp_rate, fw, fw, WIN_HAMMING);
    h->L2 = sps; h->nt2 = arms_nt(d.t2, sps);
    const std::vector<float> cb = complex_band_pass_2(1, samp_rate, -fw, fw, 1200, 120, WIN_BLACKMAN_HARRIS);
    d.cfilt.resize(cb.size() / 2);
    for (size_t i = 0; i < d.cfilt.size(); i++) {
        if (cb[2 * i + 1] != 0.0f) { set_err(h, "make_gr_mod_am: output filter taps are not real"); return QRL_EINVAL; }
        d.cfilt[i] = cb[2 * i];
    }
    h->nt_cfilt = static_cast<int>(d.cfilt.size());
    if (!arms_fit(h->L2, h->nt2) || h->nt_cfilt > 8192) { set_err(h, "make_gr_mod_am: unsupported sps / filter_width"); return QRL_EINVAL; }
    { const std::vector<float> st_ = fxpt_sine_table(); const unsigned uc = 0x40000000u; const int ci = uc >> 22;
      const float c0 = st_[2 * ci] * static_cast<float>(uc >> 1) + st_[2 * ci + 1];
      h->am_dc = static_cast<float>(static_cast<double>(c0) * 0.5); }
    d.ra = h->max_items + static_cast<long long>(d.lpf.size()) + 64;
    d.rc = static_cast<long long>(h->max_items) * h->L2 + h->nt_cfilt + 64; d.rs2 = true;
    d.if_ = 8LL * h->max_items + 128;                                                          // 8 ksps, room for 8 items per input sample
    d.out = static_cast<long long>(h->max_items) * h->L2;
    return QRL_OK;
}
// gr_mod_freedv.cpp:34-85 (sps = final interpolation, 125; flag = sb): side-band filter complex_band_pass_2(1, 8000, lo, fw, 250, 90, BH)
// (LSB: (-fw, -lo)), feedforward_agc_cc(512, 1), rational_resampler_ccf(sps, 1, low_pass(sps, fs, fw, 1200)) (Hamming), x0.98, x bb gain
int create_freedv(qrl_tx* h, TxDesign& d, int sps, int samp_rate, int fw, int low_cutoff)
{
    h->amplif = 0.98f;
    d.cfilt = h->flag ? complex_band_pass_2(1, 8000, -fw, -low_cutoff, 250, 90, WIN_BLACKMAN_HARRIS)
                      : complex_band_pass_2(1, 8000, low_cutoff, fw, 250, 90, WIN_BLACKMAN_HARRIS);
    h->nt_cfilt = static_cast<int>(d.cfilt.size() / 2);
    d.t2 = low_pass(sps, samp_rate, fw, 1200, WIN_HAMMING);
    h->L2 = sps; h->nt2 = arms_nt(d.t2, sps);
    if (h->L2 != 125 || h->nt2 != 17) {     // the register-tiled x125 instance (2007 taps, 17 per arm) is the one built
        set_err(h, "make_gr_mod_freedv: interpolator shape not built (sps " + std::to_string(sps) + ", " + std::to_string(d.t2.size()) + " taps)"); return QRL_EINVAL;
    }
    // three 8 ksps complex rings of one geometry: the 512-item AGC window and the filters' history stay behind the newest call
    d.rc = d.if_ = h->max_items + 1024; d.rs2 = true; d.out = static_cast<long long>(h->max_items) * h->L2;
    return QRL_OK;
}
int tx_create(int kind, int sps, int samp_rate, int fw, int flag, int low_cutoff, int n_channels, long max_items, int device, qrl_tx** out)
{
    if (!out || n_channels <= 0 || max_items <= 0) { set_err(nullptr, "qrl_tx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_tx_create", device)) return rc;
    qrl_tx* h = new qrl_tx();
    h->samp_rate = samp_rate; h->flag = flag;
    h->C = n_channels; h->max_items = max_items;
    auto fail = [&](int rc) { return create_failed(h, qrl_tx_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (!rc) rc = dev_alloc(h, &h->d_bits, h->C);
    if (rc) return fail(rc);
    TxDesign d;
    switch (kind) {
    case QRL_MOD_4FSK: case QRL_MOD_2FSK: case QRL_MOD_GMSK: h->chain = TxChain::Fsk; create_fsk(h, d, kind, sps, samp_rate, fw); break;
    case QRL_MOD_QPSK: case QRL_MOD_BPSK: h->chain = TxChain::Psk; create_psk(h, d, kind, sps); break;
    case QRL_MOD_M17: case QRL_MOD_DMR:
        h->chain = kind == QRL_MOD_DMR ? TxChain::Dmr : TxChain::M17; rc = create_m17_dmr(h, d, kind == QRL_MOD_DMR, sps, samp_rate, fw); break;
    case QRL_MOD_DSSS: h->chain = TxChain::Dsss; rc = create_dsss(h, d, sps, samp_rate, fw); break;
    case QRL_MOD_NBFM: h->chain = TxChain::Nbfm; create_nbfm(h, d, sps, samp_rate, fw); break;
    case QRL_MOD_SSB: h->chain = TxChain::Ssb; create_ssb(h, d, sps, samp_rate, fw); break;
    case QRL_MOD_AM: h->chain = TxChain::Am; rc = create_am(h, d, sps, samp_rate, fw); break;
    case QRL_MOD_FREEDV: h->chain = TxChain::Freedv; rc = create_freedv(h, d, sps, samp_rate, fw, low_cutoff); break;
    default: set_err(h, "qrl_tx_create: mod kind " + std::to_string(kind) + " not built"); rc = QRL_EINVAL;
    }
    h->nt_lpf = static_cast<int>(d.lpf.size());
    h->in_isz = h->chain == TxChain::Freedv ? sizeof(short) : d.ra ? sizeof(float) : 1;      // int16 modem samples, float audio, bytes
    if (!rc && !d.t1.empty()) rc = upload_floats(h, &h->d_arms1, make_arms(d.t1, h->L1, h->nt1));
    if (!rc && !d.t2.empty()) rc = upload_floats(h, &h->d_arms2, make_arms(d.t2, h->L2, h->nt2));
    if (!rc && !d.lpf.empty()) rc = upload_floats(h, &h->d_lpf, d.lpf);
    if (!rc && !d.cfilt.empty()) rc = upload_floats(h, &h->d_cfilt, d.cfilt);
    if (!rc) rc = dev_alloc(h, &h->d_in, h->in_isz * h->max_items * h->C);
    if (!rc && d.sym) rc = tx_ring(h, &h->d_sym, &h->sym_mask, &h->sym_stride, d.sym, d.sym_floats);
    if (!rc && d.if_) rc = tx_ring(h, &h->d_if, &h->if_mask, &h->if_stride, d.if_);
    if (!rc && d.rc) rc = tx_ring(h, &h->d_rc, &h->rc_mask, &h->rc_stride, d.rc);
    if (!rc && d.rs2) rc = dev_alloc(h, &h->d_rs2, static_cast<size_t>(h->rc_stride) * h->C);
    if (!rc && d.ra) {      // the audio chains: audio ring and [C] states (AM: agc2_ff::make(1e-2, 1e-4, 1, 1), initial gain 1)
        std::vector<TxAnalogState> an(h->C);
        for (auto& a : an) { std::memset(&a, 0, sizeof a); a.agc = h->chain == TxChain::Am ? 1.0f : 0.0f; }
        rc = tx_ring(h, &h->d_ra, &h->ra_mask, &h->ra_stride, d.ra);
        if (!rc && d.rb) rc = dev_alloc(h, &h->d_rb, static_cast<size_t>(h->ra_stride) * h->C);
        if (!rc) rc = dev_alloc(h, &h->d_an, h->C);
        if (!rc) rc = upload_state(h, h->d_an, an.data(), sizeof(TxAnalogState) * h->C);
    }
    h->out_stride = d.out;
    if (!rc) rc = dev_alloc(h, &h->d_out, static_cast<size_t>(h->out_stride) * h->C, false);
    std::vector<TxBitState> st(h->C);
    for (auto& x : st) { x.scr_reg = 0x7F; x.enc_state = 0; x.diff_prev = 0; x.phase_q = 0; }
    if (!rc) rc = upload_state(h, h->d_bits, st.data(), sizeof(TxBitState) * h->C);
    if (rc) return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}
}  // namespace
int qrl_tx_create(int kind, int sps, int samp_rate, int /*carrier_freq*/, int filter_width, int flag,
                  int n_channels, long max_items, int device, qrl_tx** out)
{
    if (kind == QRL_MOD_FREEDV) { set_err(nullptr, "qrl_tx_create: QRL_MOD_FREEDV takes a low cutoff: use qrl_tx_create_freedv"); return QRL_EINVAL; }
    return tx_create(kind, sps, samp_rate, filter_width, flag, 0, n_channels, max_items, device, out);
}
int qrl_tx_create_freedv(int sps, int samp_rate, int /*carrier_freq*/, int filter_width, int low_cutoff, int sb,
                         int n_channels, long max_items, int device, qrl_tx** out)
{
    int rc = check_freedv_args("qrl_tx_create_freedv", sps, samp_rate, filter_width, low_cutoff);
    if (rc) return rc;
    return tx_create(QRL_MOD_FREEDV, sps, samp_rate, filter_width, sb ? 1 : 0, low_cutoff, n_channels, max_items, device, out);
}
int qrl_tx_destroy(qrl_tx* h)
{
    if (!h) return QRL_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->s_bits) { cudaStreamSynchronize(h->s_bits); cudaStreamDestroy(h->s_bits); }
    if (h->s_shape) { cudaStreamSynchronize(h->s_shape); cudaStreamDestroy(h->s_shape); }
    for (cudaEvent_t e : { h->ev_start, h->ev_shape_done, h->ev_out_done }) if (e) cudaEventDestroy(e);
    for (int i = 0; i < qrl_tx::kTxSub; i++) { if (h->ev_bits[i]) cudaEventDestroy(h->ev_bits[i]); if (h->ev_shape[i]) cudaEventDestroy(h->ev_shape[i]); }
    h->zi.release();
    return handle_close(h);
}
int qrl_tx_set_stream(qrl_tx* h, void* s)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, s);
}
namespace {
// set_param: the handle's stream drains, then the new tables replace the old ones once every upload succeeded
int swap_tables(qrl_tx* h, std::initializer_list<std::pair<float**, std::vector<float>>> tables)
{
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaStreamSynchronize(h->stream));
    std::vector<float*> d;
    for (const auto& t : tables) { d.push_back(nullptr); if (int rc = upload_floats(h, &d.back(), t.second)) return rc; }
    for (size_t i = 0; i < d.size(); i++) *tables.begin()[i].first = d[i];
    return QRL_OK;
}
// gr_mod_nbfm::set_filter_width (gr_mod_nbfm.cpp:78-93): new taps for the 25/4 resampler, the 50 ksps filter and the final
// interpolator, new sensitivity.  The rings keep the stream's true history, which the longer filters read from their next output on.
int nbfm_set_filter_width(qrl_tx* h, int fw)
{
    if (fw <= 0) { set_err(h, "qrl_tx_set_param: filter width must be positive"); return QRL_EINVAL; }
    const float if_samp_rate = 50000;
    const std::vector<float> t1 = low_pass_2(25, if_samp_rate * 4, fw, fw, 60, WIN_BLACKMAN_HARRIS);
    const std::vector<float> tc = low_pass_2(1, if_samp_rate, fw, 1200, 60, WIN_BLACKMAN_HARRIS);
    const std::vector<float> t2 = low_pass_2(h->L2, h->samp_rate, fw, fw, 60, WIN_BLACKMAN_HARRIS);
    const int nt1 = arms_nt(t1, 25), nt2 = arms_nt(t2, h->L2);
    if (nt1 > 256 || static_cast<int>(tc.size()) > 400 || nt2 > 400 || !arms_fit(h->L2, nt2)) {
        set_err(h, "qrl_tx_set_param: filter width too small for the rings' history"); return QRL_EINVAL;
    }
    if (int rc = swap_tables(h, { { &h->d_arms1, make_arms(t1, 25, nt1) }, { &h->d_cfilt, tc }, { &h->d_arms2, make_arms(t2, h->L2, nt2) } })) return rc;
    h->nt1 = nt1; h->nt_cfilt = static_cast<int>(tc.size()); h->nt2 = nt2;
    h->fm_sens = static_cast<float>(4 * kPi * fw / if_samp_rate);
    return QRL_OK;
}
// gr_mod_nbfm::set_ctcss (gr_mod_nbfm.cpp:101-139)
int nbfm_set_ctcss(qrl_tx* h, double value)
{
    std::vector<float> lp;
    if (value == 0) { h->audio_gain = 0.98f; h->tone_on = false; lp = low_pass_2(1, 8000, 3500, 200, 35, WIN_BLACKMAN_HARRIS); }
    else {
        h->audio_gain = 0.85f; h->tone_on = true;
        lp = band_pass_2(1, 8000, 300, 3500, 200, 35, WIN_BLACKMAN_HARRIS);
        float x = static_cast<float>(2 * kPi * static_cast<double>(static_cast<float>(value)) / 8000.0);      // fxpt::float_to_fixed
        const int d = static_cast<int>(std::floor(x / static_cast<float>(2.0 * kPi) + 0.5));
        x -= d * static_cast<float>(2.0 * kPi);
        h->tone_inc = static_cast<unsigned>(static_cast<int>(static_cast<float>(x) * 2147483648.0f / static_cast<float>(kPi)));
    }
    if (static_cast<int>(lp.size()) > 400) { set_err(h, "qrl_tx_set_param: audio filter too long"); return QRL_EINVAL; }
    if (int rc = swap_tables(h, { { &h->d_lpf, lp } })) return rc;
    h->nt_lpf = static_cast<int>(lp.size());
    return QRL_OK;
}
// gr_mod_ssb::set_filter_width (gr_mod_ssb.cpp:85-100) / gr_mod_am::set_filter_width (gr_mod_am.cpp:75-85)
int ssb_am_set_filter_width(qrl_tx* h, int fw)
{
    if (fw <= 0) { set_err(h, "qrl_tx_set_param: filter width must be positive"); return QRL_EINVAL; }
    const bool am = h->chain == TxChain::Am;
    std::vector<float> t2, cf;
    if (am) {
        t2 = low_pass(h->L2, h->samp_rate, fw, fw, WIN_HAMMING);
        const std::vector<float> cb = complex_band_pass_2(1, h->samp_rate, -fw, fw, 1200, 120, WIN_BLACKMAN_HARRIS);
        cf.resize(cb.size() / 2);
        for (size_t i = 0; i < cf.size(); i++) cf[i] = cb[2 * i];
    } else {
        t2 = low_pass_2(h->L2, h->samp_rate, fw, fw, 90, WIN_BLACKMAN_HARRIS);
        cf = h->flag ? complex_band_pass_2(1, 8000, -fw, -300, 250, 90, WIN_BLACKMAN_HARRIS) : complex_band_pass_2(1, 8000, 300, fw, 250, 90, WIN_BLACKMAN_HARRIS);
    }
    const int nt2 = arms_nt(t2, h->L2), ntc = static_cast<int>(am ? cf.size() : cf.size() / 2);
    if (nt2 > 60 || !arms_fit(h->L2, nt2) || ntc > (am ? 8192 : 500)) {
        set_err(h, "qrl_tx_set_param: filter width too small for the rings' history"); return QRL_EINVAL;
    }
    if (int rc = swap_tables(h, { { &h->d_arms2, make_arms(t2, h->L2, nt2) }, { &h->d_cfilt, cf } })) return rc;
    h->nt2 = nt2; h->nt_cfilt = ntc;
    return QRL_OK;
}
// launch helpers of the transmit chains: each writes one kernel's grid / shared-memory formula; the callers count the launches
dim3 grid256(const qrl_tx* h, long long n) { return dim3(static_cast<unsigned>((n + 255) / 256), h->C); }
void launch_tx_bits(qrl_tx* h, cudaStream_t st, const unsigned char* b, long n, long long stride, long long sym0)
{
    const dim3 g((h->C + 31) / 32);
    switch (h->txm) {
    case TXM_4FSK: tx_bits_kernel<TXM_4FSK><<<g, 32, 0, st>>>(h->d_bits, h->C, b, n, stride, h->d_sym, h->sym_mask, h->sym_stride, sym0); break;
    case TXM_QPSK: tx_bits_kernel<TXM_QPSK><<<g, 32, 0, st>>>(h->d_bits, h->C, b, n, stride, h->d_sym, h->sym_mask, h->sym_stride, sym0); break;
    case TXM_BPSK: tx_bits_kernel<TXM_BPSK><<<g, 32, 0, st>>>(h->d_bits, h->C, b, n, stride, h->d_sym, h->sym_mask, h->sym_stride, sym0); break;
    case TXM_2FSK: tx_bits_kernel<TXM_2FSK><<<g, 32, 0, st>>>(h->d_bits, h->C, b, n, stride, h->d_sym, h->sym_mask, h->sym_stride, sym0); break;
    case TXM_M17: tx_bits_kernel<TXM_M17><<<g, 32, 0, st>>>(h->d_bits, h->C, b, n, stride, h->d_sym, h->sym_mask, h->sym_stride, sym0); break;
    case TXM_DSSS: tx_bits_kernel<TXM_DSSS><<<g, 32, 0, st>>>(h->d_bits, h->C, b, n, stride, h->d_sym, h->sym_mask, h->sym_stride, sym0); break;
    }
}
// pulse shaping + FM scan: symbol ring -> IF ring
void launch_shape_fm(qrl_tx* h, cudaStream_t st, long long sym0, long long nsym, int L, int nt, int repeat_only, float pulse_scale, float g1, float g2)
{
    tx_shape_fm_kernel<1024, 2><<<h->C, 1024, 0, st>>>(h->d_bits, h->d_sym, h->sym_mask, h->sym_stride, sym0, nsym,
        L, nt, h->d_arms1, repeat_only, pulse_scale, h->fm_sens, g1, g2, h->d_if, h->if_mask, h->if_stride);
}
// xL interpolator, ring items [m0, m1) -> d_out from output m0 L on
void launch_interp_generic(qrl_tx* h, const float2* in, unsigned mask, long long stride, long long m0, long long m1, const float* arms,
                           int L, int NT, float g1, float g2, int apply)
{
    const int MT = std::max(1, 4096 / L);
    const size_t smem = sizeof(float) * ((L * NT + 1) & ~1) + sizeof(float2) * (MT + NT);
    interp_fir_ccf_generic_kernel<<<dim3(static_cast<unsigned>((m1 - m0 + MT - 1) / MT), h->C), 256, smem, h->stream>>>(
        in, mask, stride, m0, m1, arms, L, NT, MT, g1, g2, apply, h->d_out, h->out_stride, m0 * L);
}
// the FSK chains' final interpolator, IF items [m0, m1) -> d_out from output m0 L2 - out_base on
void launch_fsk_interp(qrl_tx* h, long long m0, long long m1, long long out_base)
{
    if (!fsk_rt(h->L2, h->nt2)) return launch_interp_generic(h, h->d_if, h->if_mask, h->if_stride, m0, m1, h->d_arms2, h->L2, h->nt2, 1.0f, 1.0f, 0);
    constexpr int L = kFskRtL, NT = kFskRtNT, R = 8, G = 16;
    interp_fir_ccf_rt_kernel<L, NT, R, G><<<dim3(static_cast<unsigned>((m1 - m0 + R * G - 1) / (R * G)), h->C), L * G, 0, h->stream>>>(
        h->d_if, h->if_mask, h->if_stride, m0, m1, h->d_arms2, 1.0f, 1.0f, 0, h->d_out, h->out_stride, out_base);
}
// rational resampler xL / M, ring to ring: outputs [o0, o1)
void launch_resamp(qrl_tx* h, const float2* in, unsigned in_mask, long long in_stride, const float* arms, int L, int M, int nt,
                   long long o0, long long o1, float g1, float g2, int apply, float2* out, unsigned out_mask, long long out_stride)
{
    resamp_ring_to_ring_ccf_kernel<<<grid256(h, o1 - o0), 256, sizeof(float) * L * nt, h->stream>>>(
        in, in_mask, in_stride, arms, L, M, nt, o0, o1, g1, g2, apply, out, out_mask, out_stride);
}
// real-tap filter d_cfilt, IF ring -> ring d_rc (NBFM's 50 ksps filter, M17's IF low-pass)
void launch_if_filter(qrl_tx* h, long long a0, long long a1)
{
    fir_ccf_ring_kernel<<<grid256(h, a1 - a0), 256, sizeof(float) * h->nt_cfilt, h->stream>>>(h->d_if, h->if_mask, h->if_stride,
        h->d_rc, h->rc_mask, h->rc_stride, h->d_cfilt, h->nt_cfilt, a0, a1, nullptr, 0, 0, 0);
}
// complex side-band filter d_cfilt, ring d_rs2 -> `out` (SSB, FreeDV)
void launch_sideband_filter(qrl_tx* h, float2* out, unsigned mask, long long stride, long long a0, long long a1)
{
    fir_ccc_ring_kernel<<<grid256(h, a1 - a0), 256, sizeof(float) * 2 * h->nt_cfilt, h->stream>>>(h->d_rs2, h->rc_mask, h->rc_stride,
        out, mask, stride, h->d_cfilt, h->nt_cfilt, 1.0f, a0, a1, nullptr, 0, 0);
}
void launch_gains(qrl_tx* h, float2* ring, unsigned mask, long long stride, long long a0, long long a1)
{
    scale2_ring_kernel<<<grid256(h, a1 - a0), 256, 0, h->stream>>>(ring, mask, stride, a0, a1, h->amplif, h->bb_gain);
}
// 4FSK: bit chain / pulse shaping + FM scan / x20 interpolator are pipelined slice by slice on three streams (the first two are
// one-CTA-per-channel recurrences that leave most SMs idle; the interpolator fills them)
int tx_work_4fsk_pipelined(qrl_tx* h, const unsigned char* b, long n, long long stride)
{
    if (!h->s_bits) {
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        bool ok = cudaStreamCreateWithPriority(&h->s_bits, cudaStreamNonBlocking, hi) == cudaSuccess &&
                  cudaStreamCreateWithPriority(&h->s_shape, cudaStreamNonBlocking, hi) == cudaSuccess;
        auto mk = [&](cudaEvent_t* e) { ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess; };
        mk(&h->ev_start); mk(&h->ev_shape_done); mk(&h->ev_out_done);
        for (int i = 0; i < qrl_tx::kTxSub; i++) { mk(&h->ev_bits[i]); mk(&h->ev_shape[i]); }
        if (!ok) { set_err(h, "qrl_tx_work: stream/event creation failed"); return QRL_ECUDA; }
    }
    constexpr int S = qrl_tx::kTxSub;
    const long long sym0 = h->n_sym, nsym = static_cast<long long>(h->sym_per_item) * n, out_base = sym0 * h->L1 * h->L2;
    QRL_CK(cudaEventRecord(h->ev_start, h->stream));
    QRL_CK(cudaStreamWaitEvent(h->s_bits, h->ev_start, 0));
    QRL_CK(cudaStreamWaitEvent(h->s_bits, h->ev_shape_done, 0));      // previous call: symbol ring consumed
    QRL_CK(cudaStreamWaitEvent(h->s_shape, h->ev_out_done, 0));       // previous call: IF ring consumed
    for (int j = 0; j < S; j++) {
        const long b0 = n * j / S, b1 = n * (j + 1) / S;
        if (b1 <= b0) continue;
        const long long symA = sym0 + h->sym_per_item * b0, nsym_j = h->sym_per_item * (b1 - b0);
        cudaEvent_t pe = h->prof.begin(0, h->s_bits);
        launch_tx_bits(h, h->s_bits, b + b0, b1 - b0, stride, symA);
        h->prof.end(pe);
        QRL_CK(cudaEventRecord(h->ev_bits[j], h->s_bits));
        QRL_CK(cudaStreamWaitEvent(h->s_shape, h->ev_bits[j], 0));
        pe = h->prof.begin(1, h->s_shape);
        launch_shape_fm(h, h->s_shape, symA, nsym_j, h->L1, h->nt1, h->repeat_only, h->pulse_scale, h->amplif, h->bb_gain);
        h->prof.end(pe);
        QRL_CK(cudaEventRecord(h->ev_shape[j], h->s_shape));
        QRL_CK(cudaStreamWaitEvent(h->stream, h->ev_shape[j], 0));
        pe = h->prof.begin(2, h->stream);
        launch_fsk_interp(h, symA * h->L1, (symA + nsym_j) * h->L1, out_base);
        h->prof.end(pe);
        h->launches += 3;
    }
    QRL_CK(cudaEventRecord(h->ev_shape_done, h->s_shape));
    QRL_CK(cudaEventRecord(h->ev_out_done, h->stream));
    h->n_out_last = static_cast<long>(nsym * h->L1 * h->L2);
    return QRL_OK;
}
// 4FSK (pipelined from 8 bytes per slice on when the final interpolator is the register-tiled x20), 2FSK, GMSK
int tx_work_fsk(qrl_tx* h, const unsigned char* b, long n, long long stride)
{
    if (h->txm == TXM_4FSK && fsk_rt(h->L2, h->nt2) && n >= 8 * qrl_tx::kTxSub) return tx_work_4fsk_pipelined(h, b, n, stride);
    const long long sym0 = h->n_sym, nsym = static_cast<long long>(h->sym_per_item) * n, m0 = sym0 * h->L1, m1 = (sym0 + nsym) * h->L1;
    launch_tx_bits(h, h->stream, b, n, stride, sym0);
    launch_shape_fm(h, h->stream, sym0, nsym, h->L1, h->nt1, h->repeat_only, h->pulse_scale, h->amplif, h->bb_gain);
    launch_fsk_interp(h, m0, m1, m0 * h->L2);
    h->launches += 3;
    h->n_out_last = static_cast<long>((m1 - m0) * h->L2);
    return QRL_OK;
}
// QPSK, BPSK: complex symbols -> xL1 RRC interpolator (x amplif x bb gain) -> d_out
void tx_work_psk(qrl_tx* h, const unsigned char* b, long n, long long stride)
{
    const long long sym0 = h->n_sym, nsym = static_cast<long long>(h->sym_per_item) * n;
    launch_tx_bits(h, h->stream, b, n, stride, sym0);
    const float2* sym = reinterpret_cast<const float2*>(h->d_sym);
    if (h->txm == TXM_QPSK && qpsk_rt(h->L1, h->nt1)) {
        constexpr int L = kQpskRtL, NT = kQpskRtNT, MB = 8, MLEN = 64;
        interp_fir_ccf_kernel<L, NT, MB, MLEN><<<dim3(static_cast<unsigned>((nsym + MB * MLEN - 1) / (MB * MLEN)), h->C), L * MB, 0, h->stream>>>(
            sym, h->sym_mask, h->sym_stride, sym0, sym0 + nsym, h->d_arms1, h->amplif, h->bb_gain, 1, h->d_out, h->out_stride, sym0 * L);
    } else {
        launch_interp_generic(h, sym, h->sym_mask, h->sym_stride, sym0, sym0 + nsym, h->d_arms1, h->L1, h->nt1, h->amplif, h->bb_gain, 1);
    }
    h->launches += 2;
    h->n_out_last = static_cast<long>(nsym * h->L1);
}
// M17, DMR: pulse shaping + FM scan (gains of 1: x0.9 and the bb gain sit behind the IF filter here), IF low-pass (DMR: the
// zero-idle delay), gains, x125 / 3
int tx_work_m17_dmr(qrl_tx* h, const unsigned char* b, long n, long long stride)
{
    const long long sym0 = h->n_sym, nsym = static_cast<long long>(h->sym_per_item) * n, m0 = sym0 * h->L1, m1 = (sym0 + nsym) * h->L1;
    launch_tx_bits(h, h->stream, b, n, stride, sym0);
    h->launches++;
    launch_shape_fm(h, h->stream, sym0, nsym, h->L1, h->nt1, 0, h->pulse_scale, 1.0f, 1.0f);
    if (h->chain == TxChain::Dmr) {
        tx_delay_ring_kernel<<<grid256(h, m1 - m0), 256, 0, h->stream>>>(h->d_if, h->if_mask, h->if_stride, h->d_rc, h->rc_mask, h->rc_stride,
                                                                          m0, m1, h->zi_delay_items);
        // the "zero_samples" counters of this call as item ranges (gr_zero_idle_bursts.cpp:61-79: a tag loads the counter, a later
        // one overrides what is left of it, one output is cleared per count)
        std::vector<long long> ranges;
        h->zi.collect(h->C, m0, m1, 0, ranges);
        if (!ranges.empty()) {
            QRL_CK(h->zi.upload(ranges, h->stream));
            tx_zero_ranges_kernel<<<static_cast<unsigned>(ranges.size() / 3), 256, 0, h->stream>>>(h->d_rc, h->rc_mask, h->rc_stride, h->zi.d_ranges);
            h->launches++;
        }
    } else {
        launch_if_filter(h, m0, m1);
    }
    launch_gains(h, h->d_rc, h->rc_mask, h->rc_stride, m0, m1);
    const long long o0 = (m0 * h->L2 + h->M2 - 1) / h->M2, o1 = (m1 * h->L2 + h->M2 - 1) / h->M2;   // outputs i with floor(i M / L) < m1
    if (o1 - o0 > h->out_stride) { set_err(h, "qrl_tx_work: output buffer too small"); return QRL_ERANGE; }
    resamp_ring_ccf_generic_kernel<<<grid256(h, o1 - o0), 256, sizeof(float) * h->L2 * h->nt2, h->stream>>>(h->d_rc, h->rc_mask, h->rc_stride,
        h->d_arms2, h->L2, h->M2, h->nt2, o0, o1, h->d_out, h->out_stride);
    h->launches += 4;
    h->n_out_last = static_cast<long>(o1 - o0);
    return QRL_OK;
}
// DSSS: chips -> x sps pulse shaping + the two gains (5200 sps ring) -> x50 / 13 (20 ksps ring: outputs i with floor(13 i / 50) < a1) -> x50
int tx_work_dsss(qrl_tx* h, const unsigned char* b, long n, long long stride)
{
    const long long sym0 = h->n_sym, nsym = static_cast<long long>(h->sym_per_item) * n, a0 = sym0 * h->L1, a1 = (sym0 + nsym) * h->L1;
    const long long o0 = (a0 * 50 + 12) / 13, o1 = (a1 * 50 + 12) / 13;
    launch_tx_bits(h, h->stream, b, n, stride, sym0);
    launch_resamp(h, reinterpret_cast<const float2*>(h->d_sym), h->sym_mask, h->sym_stride, h->d_arms1, h->L1, 1, h->nt1, a0, a1,
                  h->amplif, h->bb_gain, 1, h->d_if, h->if_mask, h->if_stride);
    launch_resamp(h, h->d_if, h->if_mask, h->if_stride, h->d_cfilt, 50, 13, h->nt_cfilt, o0, o1, 1.0f, 1.0f, 0, h->d_rc, h->rc_mask, h->rc_stride);
    if ((o1 - o0) * 50 > h->out_stride) { set_err(h, "qrl_tx_work: output buffer too small"); return QRL_ERANGE; }
    launch_interp_generic(h, h->d_rc, h->rc_mask, h->rc_stride, o0, o1, h->d_arms2, h->L2, h->nt2, 1.0f, 1.0f, 0);
    h->launches += 4;
    h->n_out_last = static_cast<long>((o1 - o0) * 50);
    return QRL_OK;
}
void tx_work_nbfm(qrl_tx* h, const float* au, long n, long long stride)
{
    tx_nbfm_front_kernel<<<h->C, 128, 0, h->stream>>>(h->d_an, au, n, stride, h->d_ra, h->ra_mask, h->ra_stride,
        h->d_rb, h->ra_mask, h->ra_stride, h->d_lpf, h->nt_lpf, h->pe_b0, h->pe_b1, h->pe_a1, h->d_arms1, h->nt1,
        h->d_sym, h->sym_mask, h->sym_stride, h->audio_gain, h->tone_on ? 1 : 0, h->tone_phase, h->tone_inc);
    if (h->tone_on) h->tone_phase += h->tone_inc * static_cast<unsigned>(n);
    const long long r0 = h->n_mid, r1 = ((h->n_audio + n) * 25 + 3) / 4;
    // frequency modulator (Q32 scan) on the 50 ksps stream: "RRC" stage degenerated to a pass-through arm {1}
    launch_shape_fm(h, h->stream, r0, r1 - r0, 1, 1, 1, 1.0f, 1.0f, 1.0f);
    if (r1 > r0) {
        launch_if_filter(h, r0, r1);
        launch_gains(h, h->d_rc, h->rc_mask, h->rc_stride, r0, r1);
        launch_interp_generic(h, h->d_rc, h->rc_mask, h->rc_stride, r0, r1, h->d_arms2, h->L2, h->nt2, 1.0f, 1.0f, 0);
    }
    h->launches += 5;
    h->n_out_last = static_cast<long>((r1 - r0) * h->L2);
    h->n_mid = r1;
}
void tx_work_ssb(qrl_tx* h, const float* au, long n, long long stride)
{
    tx_ssb_front_kernel<<<h->C, 128, 0, h->stream>>>(h->d_an, au, n, stride, h->d_ra, h->ra_mask, h->ra_stride,
        h->d_rc, h->rc_mask, h->rc_stride, h->d_lpf, h->nt_lpf, 0.95f, static_cast<float>(1 / (std::sqrt(0.5) / 2)),
        h->d_rs2, h->rc_mask, h->rc_stride);
    const long long s0 = h->n_mid, s1 = std::max<long long>(s0, h->n_audio + n - 2);
    if (s1 > s0) {
        launch_sideband_filter(h, h->d_if, h->if_mask, h->if_stride, s0, s1);
        launch_gains(h, h->d_if, h->if_mask, h->if_stride, s0, s1);
        launch_interp_generic(h, h->d_if, h->if_mask, h->if_stride, s0, s1, h->d_arms2, h->L2, h->nt2, 1.0f, 1.0f, 0);
    }
    h->launches += 4;
    h->n_out_last = static_cast<long>((s1 - s0) * h->L2);
    h->n_mid = s1;
}
// AM: audio ring d_ra -> 8 ksps complex ring d_if -> x sps (ring d_rc at the output rate) -> output filter (taps d_cfilt) -> d_out
int tx_work_am(qrl_tx* h, const float* au, long n, long long stride)
{
    const long long o0 = h->n_audio * h->L2, o1 = (h->n_audio + n) * h->L2;
    tx_am_front_kernel<<<h->C, 128, 0, h->stream>>>(h->d_an, au, n, stride, 1e-2f, 1e-4f, 1.0f, 1.0f,
        h->d_ra, h->ra_mask, h->ra_stride, h->d_lpf, h->nt_lpf, h->am_dc, h->d_if, h->if_mask, h->if_stride);
    launch_resamp(h, h->d_if, h->if_mask, h->if_stride, h->d_arms2, h->L2, 1, h->nt2, o0, o1, h->amplif, h->bb_gain, 1,
                  h->d_rc, h->rc_mask, h->rc_stride);
    h->launches += 2;
    if (int rc = launch_fir_ccf_c(h, h->C, h->stream, h->d_rc, h->rc_mask, h->rc_stride, h->d_rs2, h->rc_mask, h->rc_stride,
                                  h->d_cfilt, h->nt_cfilt, o0, o1, h->d_out, h->out_stride, o0, 0)) return rc;
    h->n_out_last = static_cast<long>(o1 - o0);
    return QRL_OK;
}
// FreeDV: int16 modem samples at 8 ksps -> ring d_rs2 -> side-band filter -> ring d_rc -> feedforward AGC -> ring d_if -> x sps -> d_out;
// every stage is one item per thread (no recurrence), all on the handle's stream
void tx_work_freedv(qrl_tx* h, const short* s, long n, long long stride)
{
    const long long a0 = h->n_audio, a1 = h->n_audio + n;
    cudaEvent_t pe = h->prof.begin(0, h->stream);
    short_to_complex_ring_kernel<<<dim3(static_cast<unsigned>(std::min<long long>((n + 255) / 256, 1024)), h->C), 256, 0, h->stream>>>(
        s, stride, n, static_cast<float>(1.0 / 32765.0), h->d_rs2, h->rc_mask, h->rc_stride, a0);
    launch_sideband_filter(h, h->d_rc, h->rc_mask, h->rc_stride, a0, a1);
    h->prof.end(pe);
    constexpr int AN = 512, ATILE = 3584, ANT = 256;
    pe = h->prof.begin(1, h->stream);
    ffagc_kernel<AN, ATILE, ANT><<<dim3(static_cast<unsigned>((n + ATILE - 1) / ATILE), h->C), ANT, 0, h->stream>>>(
        h->d_rc, h->rc_mask, h->rc_stride, a0, a1, 1.0f, h->d_if, h->if_mask, h->if_stride);
    h->prof.end(pe);
    // the HBM-write-bound stage (8 B per output sample): register-tiled, x0.98 and x bb_gain fused (the one shape tx_create accepts)
    constexpr int L = 125, NT = 17, R = 8, G = 4;
    pe = h->prof.begin(2, h->stream);
    interp_fir_ccf_rt_kernel<L, NT, R, G><<<dim3(static_cast<unsigned>((n + R * G - 1) / (R * G)), h->C), L * G, 0, h->stream>>>(
        h->d_if, h->if_mask, h->if_stride, a0, a1, h->d_arms2, h->amplif, h->bb_gain, 1, h->d_out, h->out_stride, a0 * L);
    h->prof.end(pe);
    h->launches += 4;
    h->n_out_last = static_cast<long>(n * h->L2);
}
}  // namespace
int qrl_tx_set_param(qrl_tx* h, int, int key, double value)
{
    if (!h) return QRL_EINVAL;
    if (key == QRL_PARAM_BB_GAIN) { h->bb_gain = static_cast<float>(value); return QRL_OK; }   // gr_mod_4fsk::set_bb_gain
    if (key == QRL_PARAM_FILTER_WIDTH && h->chain == TxChain::Nbfm) return nbfm_set_filter_width(h, static_cast<int>(value));
    if (key == QRL_PARAM_CTCSS && h->chain == TxChain::Nbfm) return nbfm_set_ctcss(h, value);
    if (key == QRL_PARAM_FILTER_WIDTH && (h->chain == TxChain::Ssb || h->chain == TxChain::Am)) return ssb_am_set_filter_width(h, static_cast<int>(value));
    set_err(h, "qrl_tx_set_param: unsupported key");
    return QRL_EINVAL;
}
int qrl_tx_work(qrl_tx* h, const void* in, long n, long stride, int on_device)
{
    if (!h || !in || n < 0) return QRL_EINVAL;
    if (n > h->max_items) { set_err(h, "qrl_tx_work: n exceeds max_items given at create"); return QRL_ERANGE; }
    h->n_out_last = 0;
    if (n == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    long long s = stride;
    if (on_device) { if (int rc = check_device_ptr(h, in, "qrl_tx_work")) return rc; }
    else {                  // [C][n] items of in_isz bytes at row stride `stride` -> the [C][max_items] staging buffer
        const size_t isz = h->in_isz;
        QRL_CK(cudaMemcpy2DAsync(h->d_in, isz * h->max_items, in, isz * stride, isz * n, h->C, cudaMemcpyHostToDevice, h->stream));
        in = h->d_in; s = h->max_items;
    }
    const unsigned char* b = static_cast<const unsigned char*>(in);
    const float* au = static_cast<const float*>(in);
    int rc = QRL_OK;
    switch (h->chain) {
    case TxChain::Fsk: rc = tx_work_fsk(h, b, n, s); break;
    case TxChain::Psk: tx_work_psk(h, b, n, s); break;
    case TxChain::M17: case TxChain::Dmr: rc = tx_work_m17_dmr(h, b, n, s); break;
    case TxChain::Dsss: rc = tx_work_dsss(h, b, n, s); break;
    case TxChain::Nbfm: tx_work_nbfm(h, au, n, s); break;
    case TxChain::Ssb: tx_work_ssb(h, au, n, s); break;
    case TxChain::Am: rc = tx_work_am(h, au, n, s); break;
    case TxChain::Freedv: tx_work_freedv(h, static_cast<const short*>(in), n, s); break;
    }
    if (rc) return rc;
    if (h->sym_per_item) h->n_sym += static_cast<long long>(h->sym_per_item) * n;     // symbols, or audio / modem samples consumed
    else h->n_audio += n;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_tx_zero_samples(qrl_tx* h, int channel, long long byte_offset, long n_samples)
{
    if (!h || channel < -1 || channel >= h->C || byte_offset < 0 || n_samples < 0) return QRL_EINVAL;
    if (h->chain != TxChain::Dmr) { set_err(h, "qrl_tx_zero_samples: only gr_mod_dmr has a zero-idle stage"); return QRL_EINVAL; }
    // the tag rides through packed_to_unpacked (x8), pack_k_bits(2) (/2) and the x5 pulse shaper: item 20 * byte_offset at the block
    const long long item = byte_offset * 4 * h->L1;
    if (item < static_cast<long long>(h->zi_tag_delay)) return QRL_OK;          // gr_zero_idle_bursts.cpp:63 can never match
    h->zi.add(channel, h->C, item - static_cast<long long>(h->zi_tag_delay), static_cast<unsigned long long>(n_samples), h->n_sym * h->L1);
    return QRL_OK;
}
int qrl_tx_sync(qrl_tx* h)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}
int qrl_tx_profile(qrl_tx* h, int enable)
{
    if (!h) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    h->prof.reset(enable != 0);
    return QRL_OK;
}
int qrl_tx_profile_read(qrl_tx* h, int stage, double* ms_total, long* n_launches)
{
    if (!h || stage < 0 || stage >= h->prof.stages()) return QRL_EINVAL;
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (h->s_bits) QRL_CK(cudaStreamSynchronize(h->s_bits));
    if (h->s_shape) QRL_CK(cudaStreamSynchronize(h->s_shape));
    h->prof.read(stage, ms_total, n_launches);
    return QRL_OK;
}
int qrl_tx_read(qrl_tx* h, float* dst, long cap, long* n_out, int dst_on_device)
{
    if (!h || !n_out) return QRL_EINVAL;
    *n_out = h->n_out_last;
    if (dst && h->n_out_last > 0) {
        const long w = std::min(cap, h->n_out_last);
        QRL_CK(cudaMemcpy2DAsync(dst, static_cast<size_t>(cap) * 8, h->d_out, static_cast<size_t>(h->out_stride) * 8, static_cast<size_t>(w) * 8, h->C,
                             dst_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, h->stream));
    }
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}
int qrl_tx_out_device(qrl_tx* h, float** data, long* stride, long* n_out)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = reinterpret_cast<float*>(h->d_out);
    if (stride) *stride = static_cast<long>(h->out_stride);
    if (n_out) *n_out = h->n_out_last;
    return QRL_OK;
}
long qrl_tx_launch_count(const qrl_tx* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------- front end (device rate >= 2 Msps)
namespace {
// frontend_shared_kernel: outputs per work item (odd: conflict-free window loads), taps per register chunk, threads per CTA; it
// serves D <= FESH_DMAX, where THE FIR order's slots are single branches.  Above, a shared stream runs frontend_fir_kernel with
// in_stride = 0.  The shared-memory budget keeps two CTAs on an SM.
constexpr int FESH_K = 9, FESH_KC = 8, FESH_NT = 256, FESH_DMAX = 32, FESH_SMEM = 113 * 1024;
size_t fesh_smem(int D, int QP, int Qmax, int NB)
{
    const int NOUT = NB * FESH_K, MW = NOUT + Qmax - 1;
    return sizeof(float) * D * QP + sizeof(float2) * D * (MW + (MW | 1) + NOUT);
}
// frontend_fir_kernel (per-channel calls, and shared calls above FESH_DMAX): the taps (rounded up to even) and the window of 128
// outputs.  Both grow with the rate, and FEFIR_SMEM_MAX caps it: 107 Msps needs 162 416 B (4475 taps), 108 Msps 163 936 B.
constexpr size_t FEFIR_SMEM_MAX = 160 * 1024;
size_t fefir_smem(int D, int ntaps) { return sizeof(float) * ((ntaps + 1) & ~1) + sizeof(float2) * (127 * static_cast<size_t>(D) + ntaps); }
}  // namespace

struct qrl_frontend : HandleBase {
    int samp_rate = 0, D = 1, C = 0, ntaps = 0, H = 0, hist_cur = 0;
    long max_in = 0;
    float* d_taps = nullptr;
    float2* d_hist[2] = { nullptr, nullptr };
    float2* d_in = nullptr; float2* d_out = nullptr; long long out_stride = 0; long n_out_last = 0;
    long long n_in = 0, n1 = 0;
    std::vector<RotState> rot; RotState* d_rot = nullptr; bool rot_active = false;
    // shared stream (stride 0): [max_in] host staging, and frontend_shared_kernel's chain-order taps [D][QP] and strip shape
    float2* d_in1 = nullptr;
    float* d_ht = nullptr; int QP = 0, Qmax = 0, NB = 0, n_sm = 0; size_t fs_smem = 0;
    size_t fir_smem = 0;                // frontend_fir_kernel's dynamic shared memory
};

int qrl_frontend_destroy(qrl_frontend* h) { return h ? handle_close(h) : QRL_OK; }
int qrl_frontend_create(int samp_rate, int n_channels, long max_in, int device, qrl_frontend** out)
{
    if (!out || n_channels <= 0 || max_in <= 0 || samp_rate < 2000000 || samp_rate % 1000000) { set_err(nullptr, "qrl_frontend_create: bad argument (samp_rate must be a multiple of 1e6, >= 2e6)"); return QRL_EINVAL; }
    *out = nullptr;
    // gr_demod_base.cpp:1329-1333: low_pass(1, samp_rate, 480000, 100000, BLACKMAN_HARRIS) in rational_resampler_ccf(1, samp_rate / 1e6)
    std::vector<float> taps = low_pass(1, samp_rate, 480000, 100000, WIN_BLACKMAN_HARRIS);
    const size_t fir_smem = fefir_smem(samp_rate / 1000000, static_cast<int>(taps.size()));
    if (fir_smem > FEFIR_SMEM_MAX) {
        set_err(nullptr, "qrl_frontend_create: samp_rate above 107 Msps (the decimating FIR's " + std::to_string(taps.size()) +
                             " taps and window need " + std::to_string(fir_smem) + " B of shared memory, the limit is 160 KiB)");
        return QRL_EINVAL;
    }
    if (int rc = check_device("qrl_frontend_create", device)) return rc;
    qrl_frontend* h = new qrl_frontend();
    h->samp_rate = samp_rate; h->D = samp_rate / 1000000; h->C = n_channels; h->max_in = max_in; h->fir_smem = fir_smem;
    auto fail = [&](int rc) { return create_failed(h, qrl_frontend_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (rc) return fail(rc);
    h->ntaps = static_cast<int>(taps.size());
    h->H = h->ntaps + h->D;
    if ((rc = upload_floats(h, &h->d_taps, taps))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_hist[0], static_cast<size_t>(h->H) * h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_hist[1], static_cast<size_t>(h->H) * h->C))) return fail(rc);
    h->out_stride = max_in / h->D + 2;
    if ((rc = dev_alloc(h, &h->d_out, static_cast<size_t>(h->out_stride) * h->C, false))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_rot, h->C))) return fail(rc);
    h->rot.assign(h->C, RotState{ 0u, 0u, 0 });
    if (h->D <= FESH_DMAX) {
        h->Qmax = (h->ntaps - 1) / h->D + 1;
        h->QP = (h->Qmax + 3) & ~3;
        std::vector<float> ht(static_cast<size_t>(h->D) * h->QP, 0.0f);
        for (int r = 0; r < h->D; r++) {
            const int Qr = (h->ntaps - 1 - r) / h->D + 1;
            for (int s = 0; s < Qr; s++) ht[static_cast<size_t>(r) * h->QP + s] = taps[static_cast<size_t>(h->D) * (Qr - 1 - s) + r];
        }
        if ((rc = upload_floats(h, &h->d_ht, ht))) return fail(rc);
        // strip of NB K outputs: the most useful work per CTA, i.e. the share of busy item slots (D NB items over whole rounds of
        // FESH_NT threads) times the share of the window that is not overlap with the next strip (NOUT / (NOUT + Qmax - 1))
        double best = -1.0;
        for (int nb = 1; fesh_smem(h->D, h->QP, h->Qmax, nb) <= FESH_SMEM; nb++) {
            const int items = h->D * nb, nout = nb * FESH_K;
            const double score = items / (static_cast<double>(FESH_NT) * ((items + FESH_NT - 1) / FESH_NT)) * nout / (nout + h->Qmax - 1.0);
            if (score > best + 1e-9) { best = score; h->NB = nb; }
        }
        h->fs_smem = fesh_smem(h->D, h->QP, h->Qmax, h->NB);
        if (cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, h->device) != cudaSuccess) { set_err(h, "SM count query failed"); return fail(QRL_ECUDA); }
    }
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}
int qrl_frontend_set_stream(qrl_frontend* h, void* s)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, s);
}
int qrl_frontend_set_carrier_offset(qrl_frontend* h, int channel, double offset_hz)
{
    // gr_demod_base::set_carrier_offset (:1220-1225): rotator phase increment 2 pi (-offset) / samp_rate at the DEVICE rate
    if (!h || channel >= h->C) return QRL_EINVAL;
    const unsigned inc = static_cast<unsigned>(static_cast<int>(static_cast<long long>(std::rint(-offset_hz / h->samp_rate * 4294967296.0))));
    h->rot_active = retune(h->rot, channel, inc, h->n_in);
    QRL_CK(cudaStreamSynchronize(h->stream));
    QRL_CK(cudaMemcpy(h->d_rot, h->rot.data(), sizeof(RotState) * h->C, cudaMemcpyHostToDevice));
    return QRL_OK;
}
int qrl_frontend_work(qrl_frontend* h, const float* iq, long T, long stride, int on_device, long* n_out)
{
    if (!h || !iq || T < 0) return QRL_EINVAL;
    if (T > h->max_in) { set_err(h, "qrl_frontend_work: T exceeds max_in given at create"); return QRL_ERANGE; }
    h->n_out_last = 0;
    if (n_out) *n_out = 0;
    if (T == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    const float2* x = reinterpret_cast<const float2*>(iq);
    long long xstride = stride;
    const bool shared = stride == 0;                                     // one stream for every channel
    if (!on_device && shared) {
        if (!h->d_in1) { int rc = dev_alloc(h, &h->d_in1, static_cast<size_t>(h->max_in), false); if (rc) return rc; }
        QRL_CK(cudaMemcpyAsync(h->d_in1, iq, sizeof(float2) * T, cudaMemcpyHostToDevice, h->stream));
        x = h->d_in1;
    } else if (!on_device) {
        if (!h->d_in) { int rc = dev_alloc(h, &h->d_in, static_cast<size_t>(h->max_in) * h->C, false); if (rc) return rc; }
        QRL_CK(cudaMemcpy2DAsync(h->d_in, sizeof(float2) * h->max_in, iq, sizeof(float2) * stride, sizeof(float2) * T, h->C, cudaMemcpyHostToDevice, h->stream));
        x = h->d_in; xstride = h->max_in;
    }
    const long long N = h->n_in + T;
    const long long k0 = h->n1, k1 = (N + h->D - 1) / h->D;              // outputs k with D k <= N - 1
    const RotState* rs = h->rot_active ? h->d_rot : nullptr;
    if (k1 > k0 && shared && h->D <= FESH_DMAX) {
        auto kern = frontend_shared_kernel<FESH_K, FESH_KC>;
        if (int rc = smem_opt_in(h, kern, FESH_SMEM)) return rc;
        // channel groups: enough CTAs for two per SM (a short call splits the channels), else one group, one raw load per strip
        const long long strips = (k1 - k0 + h->NB * FESH_K - 1) / (h->NB * FESH_K);
        const long long groups = std::min<long long>(h->C, (2LL * h->n_sm + strips - 1) / strips);
        const int CG = static_cast<int>((h->C + groups - 1) / groups);
        dim3 g(static_cast<unsigned>(strips), static_cast<unsigned>((h->C + CG - 1) / CG));
        kern<<<g, FESH_NT, h->fs_smem, h->stream>>>(rs, x, T, h->n_in, h->d_hist[h->hist_cur], h->H, h->d_ht, h->QP, h->ntaps, h->D, h->Qmax,
                                                    h->NB, h->C, CG, h->d_out, h->out_stride, k0, k1);
        h->launches++;
    } else if (k1 > k0) {
        if (int rc = smem_opt_in(h, frontend_fir_kernel, static_cast<int>(FEFIR_SMEM_MAX))) return rc;       // create checked fir_smem
        dim3 g(static_cast<unsigned>((k1 - k0 + 127) / 128), h->C);
        frontend_fir_kernel<<<g, 128, h->fir_smem, h->stream>>>(rs, x, xstride, T, h->n_in, h->d_hist[h->hist_cur], h->H, h->d_taps,
                                                                h->ntaps, h->D, h->d_out, h->out_stride, k0, k1);
        h->launches++;
    }
    dim3 gh((h->H + 127) / 128, h->C);
    frontend_hist_kernel<<<gh, 128, 0, h->stream>>>(rs, x, xstride, T, h->n_in, h->d_hist[h->hist_cur], h->d_hist[h->hist_cur ^ 1], h->H);
    h->launches++;
    h->hist_cur ^= 1;
    h->n_in = N; h->n1 = k1;
    h->n_out_last = static_cast<long>(k1 - k0);
    if (n_out) *n_out = h->n_out_last;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_frontend_out_device(qrl_frontend* h, float** data, long* stride, long* n_out)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = reinterpret_cast<float*>(h->d_out);
    if (stride) *stride = static_cast<long>(h->out_stride);
    if (n_out) *n_out = h->n_out_last;
    return QRL_OK;
}
int qrl_frontend_read(qrl_frontend* h, float* dst, long cap)
{
    if (!h || !dst) return QRL_EINVAL;
    const long w = std::min(cap, h->n_out_last);
    if (w > 0) QRL_CK(cudaMemcpy2DAsync(dst, static_cast<size_t>(cap) * 8, h->d_out, static_cast<size_t>(h->out_stride) * 8, static_cast<size_t>(w) * 8, h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}
long qrl_frontend_launch_count(const qrl_frontend* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------- transmit front end (x N to the device rate)
namespace {
// tx_frontend_interp_kernel: taps per register chunk, outputs per thread.  R = 18 puts the windows of consecutive groups 144 B apart,
// so the groups of one warp (16 at N = 2) read different banks; R = 16 (128 B) puts them all on one bank: 0.33 of FP32 issue at
// N = 2 against 0.56 with R = 18 (64 channels, H100 SXM at 700 W; R = 14 / 16 / 17 / 18 measured at N = 2 ... 32, 18 the best or
// within 2 % at every N)
constexpr int TXFE_KC = 10, TXFE_R = 18;

// gr_mod_base.cpp:211-259: rational_resampler_ccf(N, 1, low_pass(N, samp_rate, 480000, 20000, BLACKMAN_HARRIS)) as the arm table of
// the interpolating kernels ([NTP][N], the taps zero-padded to NTP N, NTP a multiple of kc), and G, the groups of N threads of a CTA
struct TxInterp { std::vector<float> arms; int ntaps = 0, NTP = 0, G = 0; };
TxInterp tx_interp_design(int samp_rate, int kc)
{
    const int N = samp_rate / 1000000;
    TxInterp d;
    d.arms = low_pass(N, samp_rate, 480000, 20000, WIN_BLACKMAN_HARRIS);
    d.ntaps = static_cast<int>(d.arms.size());
    const int nt = (d.ntaps + N - 1) / N;
    d.NTP = (nt + kc - 1) / kc * kc;
    d.arms.resize(static_cast<size_t>(d.NTP) * N, 0.0f);
    // threads per CTA = N G: whole warps where possible, near 256
    double best = -1.0;
    for (int g = (128 + N - 1) / N; g * N <= 512; g++) {
        const int t = g * N;
        const double eff = t / (32.0 * ((t + 31) / 32)) - std::abs(t - 256) * 1e-6;
        if (eff > best) { best = eff; d.G = g; }
    }
    return d;
}
}  // namespace

struct qrl_tx_frontend : HandleBase {
    int samp_rate = 0, N = 1, C = 0, ntaps = 0, NTP = 0, G = 0, H = 0, hist_cur = 0;
    long max_in = 0;
    float* d_arms = nullptr;                    // [NTP][N]: the taps, zero-padded to NTP N
    float2* d_hist[2] = { nullptr, nullptr };
    float2* d_in = nullptr; float2* d_out = nullptr; long long out_stride = 0; long n_out_last = 0;
    long long n_in = 0;
    std::vector<RotState> rot; RotState* d_rot = nullptr; bool rot_active = false;
};

int qrl_tx_frontend_destroy(qrl_tx_frontend* h) { return h ? handle_close(h) : QRL_OK; }
int qrl_tx_frontend_create(int samp_rate, int n_channels, long max_in, int device, qrl_tx_frontend** out)
{
    if (!out || n_channels <= 0 || max_in <= 0 || samp_rate < 1000000 || samp_rate > 32000000 || samp_rate % 1000000) {
        set_err(nullptr, "qrl_tx_frontend_create: bad argument (samp_rate must be a multiple of 1e6 in [1e6, 32e6])");
        return QRL_EINVAL;
    }
    *out = nullptr;
    if (int rc = check_device("qrl_tx_frontend_create", device)) return rc;
    qrl_tx_frontend* h = new qrl_tx_frontend();
    h->samp_rate = samp_rate; h->N = samp_rate / 1000000; h->C = n_channels; h->max_in = max_in;
    auto fail = [&](int rc) { return create_failed(h, qrl_tx_frontend_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (rc) return fail(rc);
    if (h->N >= 2) {
        const TxInterp d = tx_interp_design(samp_rate, TXFE_KC);
        h->ntaps = d.ntaps; h->NTP = d.NTP; h->G = d.G;
        h->H = h->NTP - 1;
        if ((rc = upload_floats(h, &h->d_arms, d.arms))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_hist[0], static_cast<size_t>(h->H) * h->C))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_hist[1], static_cast<size_t>(h->H) * h->C))) return fail(rc);
    }
    h->out_stride = static_cast<long long>(max_in) * h->N;
    if ((rc = dev_alloc(h, &h->d_out, static_cast<size_t>(h->out_stride) * h->C, false))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_rot, h->C))) return fail(rc);
    h->rot.assign(h->C, RotState{ 0u, 0u, 0 });
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}
int qrl_tx_frontend_set_stream(qrl_tx_frontend* h, void* s)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, s);
}
int qrl_tx_frontend_set_carrier_offset(qrl_tx_frontend* h, int channel, double offset_hz)
{
    // gr_mod_base::set_carrier_offset (:799-805): rotator_cc(2 pi offset / 1e6) at the modulators' 1 Msps, whatever the device rate
    if (!h || channel >= h->C) return QRL_EINVAL;
    const unsigned inc = static_cast<unsigned>(static_cast<int>(static_cast<long long>(std::rint(offset_hz / 1e6 * 4294967296.0))));
    h->rot_active = retune(h->rot, channel, inc, h->n_in);
    QRL_CK(cudaStreamSynchronize(h->stream));
    QRL_CK(cudaMemcpy(h->d_rot, h->rot.data(), sizeof(RotState) * h->C, cudaMemcpyHostToDevice));
    return QRL_OK;
}
int qrl_tx_frontend_work(qrl_tx_frontend* h, const float* iq, long n, long stride, int on_device, long* n_out)
{
    if (!h || !iq || n < 0 || stride < n) return QRL_EINVAL;
    if (n > h->max_in) { set_err(h, "qrl_tx_frontend_work: n exceeds max_in given at create"); return QRL_ERANGE; }
    if (on_device) { int rc = check_device_ptr(h, iq, "qrl_tx_frontend_work"); if (rc) return rc; }
    h->n_out_last = 0;
    if (n_out) *n_out = 0;
    if (n == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    const float2* x = reinterpret_cast<const float2*>(iq);
    long long xstride = stride;
    const RotState* rs = h->rot_active ? h->d_rot : nullptr;
    if (h->N == 1) {
        // the reference has no resampler at 1 Msps (gr_mod_base.cpp:260-293): the rotator alone, or a copy
        if (!rs) {
            QRL_CK(cudaMemcpy2DAsync(h->d_out, sizeof(float2) * h->out_stride, iq, sizeof(float2) * stride, sizeof(float2) * n, h->C,
                                     on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
        } else {
            if (!on_device) {
                if (!h->d_in) { int rc = dev_alloc(h, &h->d_in, static_cast<size_t>(h->max_in) * h->C, false); if (rc) return rc; }
                QRL_CK(cudaMemcpy2DAsync(h->d_in, sizeof(float2) * h->max_in, iq, sizeof(float2) * stride, sizeof(float2) * n, h->C, cudaMemcpyHostToDevice, h->stream));
                x = h->d_in; xstride = h->max_in;
            }
            dim3 g(static_cast<unsigned>(std::min<long long>((n + 255) / 256, 4096)), h->C);
            rotator_kernel<<<g, 256, 0, h->stream>>>(rs, x, xstride, h->d_out, h->out_stride, n, h->n_in);
            h->launches++;
        }
    } else {
        if (!on_device) {
            if (!h->d_in) { int rc = dev_alloc(h, &h->d_in, static_cast<size_t>(h->max_in) * h->C, false); if (rc) return rc; }
            QRL_CK(cudaMemcpy2DAsync(h->d_in, sizeof(float2) * h->max_in, iq, sizeof(float2) * stride, sizeof(float2) * n, h->C, cudaMemcpyHostToDevice, h->stream));
            x = h->d_in; xstride = h->max_in;
        }
        auto kern = tx_frontend_interp_kernel<TXFE_KC, TXFE_R>;
        const int TM = h->G * TXFE_R;
        const size_t smem = sizeof(float) * ((h->NTP * h->N + 3) & ~3) + sizeof(float2) * (TM + h->NTP - 1);
        if (int rc = smem_opt_in(h, kern, 96 * 1024)) return rc;
        if (smem > 96 * 1024) { set_err(h, "qrl_tx_frontend_work: arm table too large for this kernel"); return QRL_EINVAL; }
        dim3 g(static_cast<unsigned>((n + TM - 1) / TM), h->C);
        kern<<<g, h->G * h->N, smem, h->stream>>>(rs, x, xstride, n, h->n_in, h->d_hist[h->hist_cur], h->H, h->d_arms, h->N, h->NTP, h->G,
                                                  h->d_out, h->out_stride);
        h->launches++;
        dim3 gh((h->H + 127) / 128, h->C);
        frontend_hist_kernel<<<gh, 128, 0, h->stream>>>(rs, x, xstride, n, h->n_in, h->d_hist[h->hist_cur], h->d_hist[h->hist_cur ^ 1], h->H);
        h->launches++;
        h->hist_cur ^= 1;
    }
    h->n_in += n;
    h->n_out_last = n * h->N;
    if (n_out) *n_out = h->n_out_last;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_tx_frontend_out_device(qrl_tx_frontend* h, float** data, long* stride, long* n_out)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = reinterpret_cast<float*>(h->d_out);
    if (stride) *stride = static_cast<long>(h->out_stride);
    if (n_out) *n_out = h->n_out_last;
    return QRL_OK;
}
int qrl_tx_frontend_read(qrl_tx_frontend* h, float* dst, long cap)
{
    if (!h || !dst) return QRL_EINVAL;
    const long w = std::min(cap, h->n_out_last);
    if (w > 0) QRL_CK(cudaMemcpy2DAsync(dst, static_cast<size_t>(cap) * 8, h->d_out, static_cast<size_t>(h->out_stride) * 8, static_cast<size_t>(w) * 8, h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}
long qrl_tx_frontend_launch_count(const qrl_tx_frontend* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------- transmit combiner (N modulators -> one SDR stream)
namespace {
// tx_combiner_kernel: taps per register chunk, outputs per thread (tx_frontend_interp_kernel's bank argument: R = 18 keeps the groups
// of an N = 2 warp on different banks)
constexpr int TXC_KC = 10, TXC_R = 18;
// bound on the block partial sums: a call is cut into input ranges whose partials fit in this many bytes
constexpr long long TXC_SCRATCH_BYTES = 64ll << 20;
}  // namespace

struct qrl_tx_combiner : HandleBase {
    int samp_rate = 0, N = 1, C = 0, nblk = 1, NTP = 0, G = 0, H = 0, hist_cur = 0;
    long max_in = 0;
    long long range = 0;                        // input positions per launch range
    float gain = 1.0f;
    float* d_arms = nullptr;                    // [NTP][N]
    float2* d_hist[2] = { nullptr, nullptr };   // [C][H]: the raw inputs' tail
    float2* d_in = nullptr;                     // [C][max_in]: host rows staged
    float2* d_y = nullptr; long n_out_last = 0; // [max_in N]: the summed stream
    float2* d_part = nullptr;                   // [nblk][range N]: block partial sums (nblk > 1)
    const float2** d_rows = nullptr; std::vector<const float2*> rows;
    long long n_out = 0;                        // absolute device-rate index of the next output
    std::vector<RotState> rot; RotState* d_rot = nullptr;
};

int qrl_tx_combiner_destroy(qrl_tx_combiner* h) { return h ? handle_close(h) : QRL_OK; }
int qrl_tx_combiner_create(int samp_rate, int n_channels, long max_in, int device, qrl_tx_combiner** out)
{
    if (!out || n_channels <= 0 || max_in <= 0 || samp_rate < 1000000 || samp_rate > 32000000 || samp_rate % 1000000) {
        set_err(nullptr, "qrl_tx_combiner_create: bad argument (samp_rate must be a multiple of 1e6 in [1e6, 32e6])");
        return QRL_EINVAL;
    }
    *out = nullptr;
    if (int rc = check_device("qrl_tx_combiner_create", device)) return rc;
    qrl_tx_combiner* h = new qrl_tx_combiner();
    h->samp_rate = samp_rate; h->N = samp_rate / 1000000; h->C = n_channels; h->max_in = max_in;
    h->nblk = (n_channels + TXC_BLOCK - 1) / TXC_BLOCK;
    auto fail = [&](int rc) { return create_failed(h, qrl_tx_combiner_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (rc) return fail(rc);
    long long tile = 256;
    if (h->N >= 2) {
        const TxInterp d = tx_interp_design(samp_rate, TXC_KC);
        h->NTP = d.NTP; h->G = d.G; h->H = h->NTP - 1;
        tile = static_cast<long long>(h->G) * TXC_R;
        if ((rc = upload_floats(h, &h->d_arms, d.arms))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_hist[0], static_cast<size_t>(h->H) * h->C))) return fail(rc);
        if ((rc = dev_alloc(h, &h->d_hist[1], static_cast<size_t>(h->H) * h->C))) return fail(rc);
    }
    h->range = max_in;
    if (h->nblk > 1) {
        const long long fit = TXC_SCRATCH_BYTES / (static_cast<long long>(h->nblk) * h->N * 8) / tile * tile;
        h->range = std::min<long long>(max_in, std::max(fit, tile));
        if ((rc = dev_alloc(h, &h->d_part, static_cast<size_t>(h->nblk) * h->range * h->N, false))) return fail(rc);
    }
    if ((rc = dev_alloc(h, &h->d_y, static_cast<size_t>(max_in) * h->N, false))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_rows, h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_rot, h->C))) return fail(rc);
    h->rows.assign(h->C, nullptr);
    h->rot.assign(h->C, RotState{ 0u, 0u, 0 });
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}
int qrl_tx_combiner_set_stream(qrl_tx_combiner* h, void* s)
{
    if (!h) return QRL_EINVAL;
    return handle_set_stream(h, s);
}
int qrl_tx_combiner_set_carrier_offset(qrl_tx_combiner* h, int channel, double offset_hz)
{
    // gr_mod_mmdvm_multi.cpp:53-125: rotator_cc(2 pi offset / samp_rate) behind each channel's resampler, at the device rate
    if (!h || channel < -1 || channel >= h->C || !(std::abs(offset_hz) <= 0.5 * h->samp_rate)) {
        set_err(h, "qrl_tx_combiner_set_carrier_offset: bad channel or |offset| > samp_rate / 2");
        return QRL_EINVAL;
    }
    const unsigned inc = static_cast<unsigned>(static_cast<int>(static_cast<long long>(std::rint(offset_hz / h->samp_rate * 4294967296.0))));
    retune(h->rot, channel, inc, h->n_out);
    QRL_CK(cudaStreamSynchronize(h->stream));
    QRL_CK(cudaMemcpy(h->d_rot, h->rot.data(), sizeof(RotState) * h->C, cudaMemcpyHostToDevice));
    return QRL_OK;
}
int qrl_tx_combiner_set_gain(qrl_tx_combiner* h, float bb_gain)
{
    if (!h) return QRL_EINVAL;
    h->gain = bb_gain;
    return QRL_OK;
}
int qrl_tx_combiner_work(qrl_tx_combiner* h, const float* const* rows, long n, int on_device, long* n_out)
{
    if (!h || !rows || n < 0) return QRL_EINVAL;
    for (int c = 0; c < h->C; c++) {
        if (!rows[c] || (reinterpret_cast<uintptr_t>(rows[c]) & 7)) {
            set_err(h, "qrl_tx_combiner_work: row " + std::to_string(c) + " is NULL or not 8-byte aligned");
            return QRL_EINVAL;
        }
    }
    if (n > h->max_in) { set_err(h, "qrl_tx_combiner_work: n exceeds max_in given at create"); return QRL_ERANGE; }
    if (on_device)
        for (int c = 0; c < h->C; c++) { int rc = check_device_ptr(h, rows[c], "qrl_tx_combiner_work"); if (rc) return rc; }
    h->n_out_last = 0;
    if (n_out) *n_out = 0;
    if (n == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    if (!on_device && !h->d_in) { int rc = dev_alloc(h, &h->d_in, static_cast<size_t>(h->max_in) * h->C, false); if (rc) return rc; }
    for (int c = 0; c < h->C; c++) {
        if (on_device) { h->rows[c] = reinterpret_cast<const float2*>(rows[c]); continue; }
        h->rows[c] = h->d_in + static_cast<long long>(c) * h->max_in;
        QRL_CK(cudaMemcpyAsync(h->d_in + static_cast<long long>(c) * h->max_in, rows[c], sizeof(float2) * n, cudaMemcpyHostToDevice, h->stream));
    }
    QRL_CK(cudaMemcpyAsync(h->d_rows, h->rows.data(), sizeof(float2*) * h->C, cudaMemcpyHostToDevice, h->stream));
    const float g1 = 1.0f / static_cast<float>(h->C), g2 = h->gain;
    const int final = h->nblk == 1;
    const size_t smem = h->N >= 2 ? sizeof(float) * ((h->NTP * h->N + 3) & ~3) + sizeof(float2) * 2 * ((h->G * TXC_R + h->NTP + 1) & ~1) : 0;
    auto kern = tx_combiner_kernel<TXC_KC, TXC_R>;
    if (h->N >= 2) {
        if (int rc = smem_opt_in(h, kern, 96 * 1024)) return rc;
        if (smem > 96 * 1024) { set_err(h, "qrl_tx_combiner_work: arm table too large for this kernel"); return QRL_EINVAL; }
    }
    for (long long lo = 0; lo < n; lo += h->range) {
        const long long hi = std::min<long long>(n, lo + h->range);
        float2* dst = final ? h->d_y + lo * h->N : h->d_part;
        const long long pstride = h->range * h->N;
        if (h->N == 1) {
            dim3 g(static_cast<unsigned>(std::min<long long>((hi - lo + 255) / 256, 4096)), h->nblk);
            tx_combiner_direct_kernel<<<g, 256, 0, h->stream>>>(h->d_rows, h->C, h->d_rot, lo, hi, h->n_out, dst, pstride, final, g1, g2);
        } else {
            const long long TM = static_cast<long long>(h->G) * TXC_R;
            dim3 g(static_cast<unsigned>((hi - lo + TM - 1) / TM), h->nblk);
            kern<<<g, h->G * h->N, smem, h->stream>>>(h->d_rows, h->C, h->d_rot, n, lo, hi, h->n_out, h->d_hist[h->hist_cur],
                                                      hi == n ? h->d_hist[h->hist_cur ^ 1] : nullptr, h->H, h->d_arms, h->N, h->NTP, h->G,
                                                      dst, pstride, final, g1, g2);
        }
        h->launches++;
        if (!final) {
            const long long m = (hi - lo) * h->N;
            tx_combiner_sum_kernel<<<static_cast<unsigned>(std::min<long long>((m + 255) / 256, 4096)), 256, 0, h->stream>>>(
                h->d_part, pstride, h->nblk, m, h->d_y + lo * h->N, g1, g2);
            h->launches++;
        }
    }
    if (h->N >= 2) h->hist_cur ^= 1;
    h->n_out += static_cast<long long>(n) * h->N;
    h->n_out_last = n * h->N;
    if (n_out) *n_out = h->n_out_last;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_tx_combiner_out_device(qrl_tx_combiner* h, float** data, long* n_out)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = reinterpret_cast<float*>(h->d_y);
    if (n_out) *n_out = h->n_out_last;
    return QRL_OK;
}
int qrl_tx_combiner_read(qrl_tx_combiner* h, float* dst, long cap)
{
    if (!h || !dst) return QRL_EINVAL;
    const long w = std::min(cap, h->n_out_last);
    if (w > 0) QRL_CK(cudaMemcpyAsync(dst, h->d_y, static_cast<size_t>(w) * 8, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}
long qrl_tx_combiner_launch_count(const qrl_tx_combiner* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------- design helpers
static int copy_out(const std::vector<float>& v, float* out, int cap, int per_item = 1)
{
    const int n = static_cast<int>(v.size()) / per_item;
    if (n > cap) return -n;
    if (out) std::memcpy(out, v.data(), v.size() * sizeof(float));
    return n;
}
int qrl_firdes_low_pass(double gain, double fs, double fc, double tw, int window, float* out, int cap)
{ return copy_out(low_pass(gain, fs, fc, tw, window), out, cap); }
int qrl_firdes_low_pass_2(double gain, double fs, double fc, double tw, double att, int window, float* out, int cap)
{ return copy_out(low_pass_2(gain, fs, fc, tw, att, window), out, cap); }
int qrl_firdes_band_pass(double gain, double fs, double lo, double hi, double tw, int window, float* out, int cap)
{ return copy_out(band_pass(gain, fs, lo, hi, tw, window), out, cap); }
int qrl_firdes_complex_band_pass(double gain, double fs, double lo, double hi, double tw, int window, float* out, int cap)
{ return copy_out(complex_band_pass(gain, fs, lo, hi, tw, window), out, cap, 2); }
int qrl_firdes_root_raised_cosine(double gain, double fs, double symrate, double alpha, int ntaps, float* out, int cap)
{ return copy_out(root_raised_cosine(gain, fs, symrate, alpha, ntaps), out, cap); }
int qrl_firdes_gaussian(double gain, double spb, double bt, int ntaps, float* out, int cap)
{ return copy_out(gaussian(gain, spb, bt, ntaps), out, cap); }
int qrl_design_table(const char* name, float* out, int cap)
{
    std::string n(name ? name : "");
    if (n == "atan") return copy_out(atan_table(), out, cap);
    if (n == "tanh") return copy_out(tanh_table(), out, cap);
    if (n == "mmse") return copy_out(mmse_table(), out, cap);
    if (n == "fxpt_sine") return copy_out(fxpt_sine_table(), out, cap);
    return QRL_EINVAL;
}
int qrl_design_deemph(int fs, double tau, double* a2, double* b2) { deemph_taps(fs, tau, a2, b2); return QRL_OK; }

int qrl_fir_decim_ccf_device(const float* taps, int ntaps, int D, const float* x_dev, long T, long x_stride,
                             float* y_dev, long y_stride, int C, void* cuda_stream)
{
    if (!taps || ntaps < 1 || ntaps > 65536 || D < 1 || !x_dev || !y_dev || T < 0 || C < 1) { set_err(nullptr, "qrl_fir_decim_ccf_device: bad argument"); return QRL_EINVAL; }
    if (qrl_device_count() < 1) { set_err(nullptr, "qrl_fir_decim_ccf_device: no CUDA device (this library has no CPU fallback)"); return QRL_ENODEV; }
    const long long nout = (static_cast<long long>(T) + D - 1) / D;
    if (nout == 0) return QRL_OK;
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    float* d_taps = nullptr;
    HandleBase* h = nullptr;
    QRL_CK(cudaMalloc(&d_taps, sizeof(float) * ntaps));
    cudaError_t e = cudaMemcpyAsync(d_taps, taps, sizeof(float) * ntaps, cudaMemcpyHostToDevice, st);
    int dev = 0, n_sm = 0;
    if (e == cudaSuccess) e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) {
        dim3 g(static_cast<unsigned>(std::min<long long>((nout + 7) / 8, n_sm * 16LL)), static_cast<unsigned>(C));
        fir_decim_generic_kernel<<<g, 256, 0, st>>>(d_taps, ntaps, D, reinterpret_cast<const float2*>(x_dev), T, x_stride,
                                                    reinterpret_cast<float2*>(y_dev), y_stride, nout);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);          // the tap buffer is released below
    cudaFree(d_taps);
    if (e != cudaSuccess) { set_err(nullptr, std::string("qrl_fir_decim_ccf_device: ") + cudaGetErrorString(e)); return QRL_ECUDA; }
    return QRL_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------- MMDVM channel chains
// gr_demod_mmdvm_multi2.cpp:56-126 behind the channelizer (qrl_pfb): per channel rational_resampler_ccf(24, 25) -> low-pass -> RSSI tags ->
// quadrature_demod_cf -> x level -> float_to_short; gr_mod_mmdvm_multi2.cpp:47-126 in front of the synthesizer: short_to_float -> x level ->
// frequency_modulator_fc -> low-pass -> x0.8 -> rational_resampler_ccf(25, 24) [-> synthesizer -> x 1 / num_channels -> x bb_gain].
struct qrl_mmdvm_rx : HandleBase {
    int C = 0, n_rows = 0, nt_arm = 0, nt2 = 0;
    long max_in = 0;
    int* d_rows = nullptr; float* d_arms = nullptr; float* d_taps2 = nullptr;
    float2 *d_r25 = nullptr, *d_r24 = nullptr, *d_rf = nullptr, *d_in = nullptr;
    unsigned m25 = 0, m24 = 0; long long s25 = 0, s24 = 0;
    short* d_out = nullptr; long long out_stride = 0; long n_out_last = 0;
    float* d_rssi = nullptr; long long rssi_stride = 0; int n_rssi_last = 0; long long rssi_b0_last = 0;
    long long n_in = 0, n24 = 0, n_blocks = 0;
    float qd_gain = 0, level = 1.0f, cal = 0.0f;
    int L = 24, M = 25; bool single = false;       // single: gr_demod_mmdvm (250 ksps in, x12 / 125, RSSI in front of the filter, 10 kHz discriminator)
};
struct qrl_mmdvm_tx : HandleBase {
    int C = 0, n_rows = 0, num_channels = 0, nt_arm = 0, nt2 = 0;
    long max_in = 0;
    int* d_rows = nullptr; float* d_arms = nullptr; float* d_taps2 = nullptr; float* d_one = nullptr;
    TxBitState* d_bits = nullptr;
    short* d_in = nullptr;
    float* d_sym = nullptr; unsigned sym_mask = 0; long long sym_stride = 0;
    float2 *d_if = nullptr, *d_rf = nullptr; unsigned if_mask = 0; long long if_stride = 0;
    float2* d_lin = nullptr; long long lin_stride = 0;
    float2* d_out = nullptr; long long out_stride = 0; long n_out_last = 0;
    long long n_in = 0, n25 = 0;
    float fm_sens = 0, level = 1.0f, bb_gain = 1.0f;
    int L = 25, M = 24; bool single = false;       // single: gr_mod_mmdvm (x125 / 12 to 250 ksps, bb_gain in front of the resampler)
    ZeroIdle zi;                                   // gr_zero_idle_bursts(0): behind the FM modulator (single) / behind the resampler (multi2)
};

static int mmdvm_rows(HandleBase* h, int** d_rows, const int* rows, int C, int n_rows)
{
    std::vector<int> r(C);
    for (int c = 0; c < C; c++) {
        r[c] = rows ? rows[c] : c;
        if (r[c] < 0 || r[c] >= n_rows) { set_err(h, "mmdvm: row index outside the slab"); return QRL_EINVAL; }
    }
    int rc = dev_alloc(h, d_rows, static_cast<size_t>(C), false);
    if (rc) return rc;
    if (cudaMemcpy(*d_rows, r.data(), sizeof(int) * C, cudaMemcpyHostToDevice) != cudaSuccess) { set_err(h, "mmdvm: row upload failed"); return QRL_ECUDA; }
    return QRL_OK;
}

extern "C" {

int qrl_mmdvm_rx_destroy(qrl_mmdvm_rx* h) { return h ? handle_close(h) : QRL_OK; }
int qrl_mmdvm_rx_set_stream(qrl_mmdvm_rx* h, void* s) { return h ? handle_set_stream(h, s) : QRL_EINVAL; }
int qrl_mmdvm_rx_create(int variant, int n_channels, const int* rows, int n_rows, int filter_width, long max_in, int device, qrl_mmdvm_rx** out)
{
    if (!out || variant < 0 || variant > 1 || n_channels <= 0 || n_rows < n_channels || max_in <= 0 || filter_width <= 0) { set_err(nullptr, "qrl_mmdvm_rx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_mmdvm_rx_create", device)) return rc;
    qrl_mmdvm_rx* h = new qrl_mmdvm_rx();
    h->C = n_channels; h->n_rows = n_rows; h->max_in = max_in;
    auto fail = [&](int rc) { return create_failed(h, qrl_mmdvm_rx_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (rc) return fail(rc);
    if ((rc = mmdvm_rows(h, &h->d_rows, rows, h->C, n_rows))) return fail(rc);
    // gr_demod_mmdvm_multi2.cpp:58-62,66,71,76 | gr_demod_mmdvm.cpp:43-52
    h->single = variant == 1;
    h->L = h->single ? 12 : 24; h->M = h->single ? 125 : 25;
    const std::vector<float> ti = h->single ? low_pass_2(12, 12 * 250000.0, filter_width, 2000, 60, WIN_BLACKMAN_HARRIS)
                                            : low_pass_2(1, 600000.0, filter_width, 2000, 60, WIN_BLACKMAN_HARRIS);
    const std::vector<float> tf = low_pass_2(1, 24000.0, filter_width, 2000, 60, WIN_BLACKMAN_HARRIS);
    h->nt_arm = (static_cast<int>(ti.size()) + h->L - 1) / h->L; h->nt2 = static_cast<int>(tf.size());
    if (static_cast<size_t>(h->L) * h->nt_arm * sizeof(float) > 40 * 1024 || h->nt2 > kMaxTapsSmem) { set_err(h, "qrl_mmdvm_rx_create: filter_width too small"); return fail(QRL_EINVAL); }
    if ((rc = upload_floats(h, &h->d_arms, make_arms(ti, h->L, h->nt_arm)))) return fail(rc);
    if ((rc = upload_floats(h, &h->d_taps2, tf))) return fail(rc);
    h->qd_gain = static_cast<float>(24000.0f / (2 * kPi * (h->single ? 10000.0f : 12500.0f)));
    const unsigned c25 = pow2_at_least(max_in + h->nt_arm + 64), c24 = pow2_at_least(max_in + h->nt2 + 400);
    h->m25 = c25 - 1; h->s25 = c25; h->m24 = c24 - 1; h->s24 = c24;
    if ((rc = dev_alloc(h, &h->d_r25, static_cast<size_t>(c25) * h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_r24, static_cast<size_t>(c24) * h->C))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_rf, static_cast<size_t>(c24) * h->C))) return fail(rc);
    h->out_stride = max_in * h->L / h->M + 2;
    if ((rc = dev_alloc(h, &h->d_out, static_cast<size_t>(h->out_stride) * h->C, false))) return fail(rc);
    h->rssi_stride = h->out_stride / 300 + 2;
    if ((rc = dev_alloc(h, &h->d_rssi, static_cast<size_t>(h->rssi_stride) * h->C, false))) return fail(rc);
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}
int qrl_mmdvm_rx_calibrate_rssi(qrl_mmdvm_rx* h, float level) { if (!h) return QRL_EINVAL; h->cal = level; return QRL_OK; }   // rssi_tag_block::calibrate_rssi
int qrl_mmdvm_rx_work(qrl_mmdvm_rx* h, const float* iq, long n, long stride, int on_device, long* n_out)
{
    if (!h || !iq || n < 0) return QRL_EINVAL;
    if (n > h->max_in) { set_err(h, "qrl_mmdvm_rx_work: n exceeds max_in given at create"); return QRL_ERANGE; }
    h->n_out_last = 0; h->n_rssi_last = 0;
    if (n_out) *n_out = 0;
    if (n == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    const float2* x = reinterpret_cast<const float2*>(iq);
    long long xstride = stride;
    if (on_device) { int rc = check_device_ptr(h, iq, "qrl_mmdvm_rx_work"); if (rc) return rc; }
    else {
        if (!h->d_in) { int rc = dev_alloc(h, &h->d_in, static_cast<size_t>(h->max_in) * h->n_rows, false); if (rc) return rc; }
        QRL_CK(cudaMemcpy2DAsync(h->d_in, sizeof(float2) * h->max_in, iq, sizeof(float2) * stride, sizeof(float2) * n, h->n_rows, cudaMemcpyHostToDevice, h->stream));
        x = h->d_in; xstride = h->max_in;
    }
    const int TB = 256;
    mmdvm_gather_kernel<<<dim3(static_cast<unsigned>(std::min<long long>((n + TB - 1) / TB, 4096)), h->C), TB, 0, h->stream>>>(
        x, xstride, h->d_rows, n, h->d_r25, h->m25, h->s25, h->n_in);
    const long long N = h->n_in + n;
    const long long o0 = h->n24, o1 = (N * h->L + h->M - 1) / h->M;    // outputs o whose newest input floor(M o / L) has arrived
    h->launches++;
    if (o1 > o0) {
        dim3 g(static_cast<unsigned>((o1 - o0 + TB - 1) / TB), h->C);
        if (!h->single && h->nt_arm == 35) {       // the reference's filter width (5000 Hz: 819 taps): tiled instance
            const int span_cap = 256 * 25 / 24 + 35 + 4;
            const size_t smem = sizeof(float) * ((24 * 35 + 1) & ~1) + sizeof(float2) * span_cap;
            resamp_ring_to_ring_tiled_kernel<35><<<g, 256, smem, h->stream>>>(h->d_r25, h->m25, h->s25, h->d_arms, 24, 25, o0, o1, h->d_r24, h->m24, h->s24, span_cap);
        } else {
            resamp_ring_to_ring_ccf_kernel<<<g, TB, sizeof(float) * h->L * h->nt_arm, h->stream>>>(h->d_r25, h->m25, h->s25, h->d_arms, h->L, h->M, h->nt_arm, o0, o1,
                                                                                                    1.0f, 1.0f, 0, h->d_r24, h->m24, h->s24);
        }
        { int rc = launch_fir_ccf_c(h, h->C, h->stream, h->d_r24, h->m24, h->s24, h->d_rf, h->m24, h->s24, h->d_taps2, h->nt2, o0, o1, nullptr, 0, 0, 0); if (rc) return rc; h->launches--; }
        mmdvm_demod_short_kernel<<<g, TB, 0, h->stream>>>(h->d_rf, h->m24, h->s24, o0, o1, h->qd_gain, h->level, h->d_out, h->out_stride);
        h->launches += 3;
        const long long b1 = o1 / 300;                                   // complete 300-item blocks so far
        if (b1 > h->n_blocks) {
            const int nb = static_cast<int>(b1 - h->n_blocks);
            // gr_demod_mmdvm tags the resampler's output, gr_demod_mmdvm_multi2 the channel filter's
            mmdvm_rssi_kernel<<<dim3((nb + 63) / 64, h->C), 64, 0, h->stream>>>(h->single ? h->d_r24 : h->d_rf, h->m24, h->s24, h->n_blocks, nb, h->cal, h->d_rssi, h->rssi_stride);
            h->launches++;
            h->n_rssi_last = nb; h->rssi_b0_last = h->n_blocks; h->n_blocks = b1;
        }
    }
    h->n_in = N; h->n24 = o1;
    h->n_out_last = static_cast<long>(o1 - o0);
    if (n_out) *n_out = h->n_out_last;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_mmdvm_rx_out_device(qrl_mmdvm_rx* h, short** data, long* stride, long* n_out, float** rssi_db, long* rssi_stride, int* n_rssi, long long* first_rssi_item)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = h->d_out;
    if (stride) *stride = static_cast<long>(h->out_stride);
    if (n_out) *n_out = h->n_out_last;
    if (rssi_db) *rssi_db = h->d_rssi;
    if (rssi_stride) *rssi_stride = static_cast<long>(h->rssi_stride);
    if (n_rssi) *n_rssi = h->n_rssi_last;
    if (first_rssi_item) *first_rssi_item = h->rssi_b0_last * 300 + 299;
    return QRL_OK;
}
int qrl_mmdvm_rx_read(qrl_mmdvm_rx* h, short* dst, long dst_stride, float* rssi_db, long rssi_cap, int* n_rssi, long long* first_rssi_item)
{
    if (!h || !dst) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    if (h->n_out_last > 0)
        QRL_CK(cudaMemcpy2DAsync(dst, sizeof(short) * dst_stride, h->d_out, sizeof(short) * h->out_stride, sizeof(short) * h->n_out_last, h->C, cudaMemcpyDeviceToHost, h->stream));
    const int nr = static_cast<int>(std::min<long>(h->n_rssi_last, rssi_cap));
    if (rssi_db && nr > 0)
        QRL_CK(cudaMemcpy2DAsync(rssi_db, sizeof(float) * rssi_cap, h->d_rssi, sizeof(float) * h->rssi_stride, sizeof(float) * nr, h->C, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (n_rssi) *n_rssi = nr;
    if (first_rssi_item) *first_rssi_item = h->rssi_b0_last * 300 + 299;
    return QRL_OK;
}
long qrl_mmdvm_rx_launch_count(qrl_mmdvm_rx* h) { return h ? h->launches : 0; }

int qrl_mmdvm_tx_destroy(qrl_mmdvm_tx* h)
{
    if (!h) return QRL_OK;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    h->zi.release();
    return handle_close(h);
}
int qrl_mmdvm_tx_set_stream(qrl_mmdvm_tx* h, void* s) { return h ? handle_set_stream(h, s) : QRL_EINVAL; }
int qrl_mmdvm_tx_create(int variant, int n_channels, const int* rows, int n_rows, int filter_width, long max_in, int device, qrl_mmdvm_tx** out)
{
    if (!out || variant < 0 || variant > 1 || n_channels <= 0 || n_rows < n_channels || max_in <= 0 || filter_width <= 0) { set_err(nullptr, "qrl_mmdvm_tx_create: bad argument"); return QRL_EINVAL; }
    *out = nullptr;
    if (int rc = check_device("qrl_mmdvm_tx_create", device)) return rc;
    qrl_mmdvm_tx* h = new qrl_mmdvm_tx();
    h->C = n_channels; h->n_rows = n_rows; h->num_channels = n_channels; h->max_in = max_in;
    h->zi.init(h->C);
    auto fail = [&](int rc) { return create_failed(h, qrl_mmdvm_tx_destroy, rc); };
    int rc = handle_open(h, device);
    if (!rc) rc = upload_tables(h);
    if (rc) return fail(rc);
    if ((rc = mmdvm_rows(h, &h->d_rows, rows, h->C, n_rows))) return fail(rc);
    // gr_mod_mmdvm_multi2.cpp:47-50,64,72,80 | gr_mod_mmdvm.cpp:36-45
    h->single = variant == 1;
    h->L = h->single ? 125 : 25; h->M = h->single ? 12 : 24;
    const std::vector<float> ti = h->single ? low_pass_2(125, 125 * 24000.0, filter_width, 2000, 60, WIN_BLACKMAN_HARRIS)
                                            : low_pass_2(25, 600000.0, filter_width, 2000, 60, WIN_BLACKMAN_HARRIS);
    const std::vector<float> tf = low_pass_2(1, 24000.0, filter_width, 2000, 60, WIN_BLACKMAN_HARRIS);
    h->nt_arm = (static_cast<int>(ti.size()) + h->L - 1) / h->L; h->nt2 = static_cast<int>(tf.size());
    if (static_cast<size_t>(h->L) * h->nt_arm * sizeof(float) > 40 * 1024 || h->nt2 > kMaxTapsSmem) { set_err(h, "qrl_mmdvm_tx_create: filter_width too small"); return fail(QRL_EINVAL); }
    if ((rc = upload_floats(h, &h->d_arms, make_arms(ti, h->L, h->nt_arm)))) return fail(rc);
    if ((rc = upload_floats(h, &h->d_taps2, tf))) return fail(rc);
    if ((rc = upload_floats(h, &h->d_one, std::vector<float>{ 1.0f }))) return fail(rc);
    h->fm_sens = static_cast<float>(2 * kPi * 12500.0f / 24000.0f);
    if ((rc = dev_alloc(h, &h->d_bits, h->C))) return fail(rc);
    { std::vector<TxBitState> st(h->C); for (auto& x : st) { x.scr_reg = 0x7F; x.enc_state = 0; x.diff_prev = 0; x.phase_q = 0; }
      if ((rc = upload_state(h, h->d_bits, st.data(), sizeof(TxBitState) * h->C))) return fail(rc); }
    { const unsigned cap = pow2_at_least(max_in + 64); h->sym_mask = cap - 1; h->sym_stride = cap;
      if ((rc = dev_alloc(h, &h->d_sym, static_cast<size_t>(cap) * h->C))) return fail(rc); }
    { const unsigned cap = pow2_at_least(max_in + std::max(h->nt2, h->nt_arm) + 128); h->if_mask = cap - 1; h->if_stride = cap;
      if ((rc = dev_alloc(h, &h->d_if, static_cast<size_t>(cap) * h->C))) return fail(rc);
      if ((rc = dev_alloc(h, &h->d_rf, static_cast<size_t>(cap) * h->C))) return fail(rc); }
    h->lin_stride = max_in * h->L / h->M + 4; h->out_stride = h->lin_stride;
    if ((rc = dev_alloc(h, &h->d_lin, static_cast<size_t>(h->lin_stride) * h->C, false))) return fail(rc);
    if ((rc = dev_alloc(h, &h->d_out, static_cast<size_t>(h->out_stride) * h->n_rows))) return fail(rc);      // unused rows stay zero (null_source)
    if (cudaStreamSynchronize(h->stream) != cudaSuccess) { set_err(h, "create sync failed"); return fail(QRL_ECUDA); }
    *out = h;
    return QRL_OK;
}
int qrl_mmdvm_tx_set_bb_gain(qrl_mmdvm_tx* h, float g) { if (!h) return QRL_EINVAL; h->bb_gain = g; return QRL_OK; }      // gr_mod_mmdvm_multi2::set_bb_gain
int qrl_mmdvm_tx_zero_samples(qrl_mmdvm_tx* h, int channel, long long item_offset, long n_samples)
{
    if (!h || channel < -1 || channel >= h->C || item_offset < 0 || n_samples < 0) return QRL_EINVAL;
    h->zi.add(channel, h->C, item_offset, static_cast<unsigned long long>(n_samples), h->single ? h->n_in : h->n25);
    return QRL_OK;
}
int qrl_mmdvm_tx_work(qrl_mmdvm_tx* h, const short* in, long n, long stride, int on_device, long* n_out)
{
    if (!h || !in || n < 0) return QRL_EINVAL;
    if (n > h->max_in) { set_err(h, "qrl_mmdvm_tx_work: n exceeds max_in given at create"); return QRL_ERANGE; }
    h->n_out_last = 0;
    if (n_out) *n_out = 0;
    if (n == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    const short* s = in; long long sstride = stride;
    if (on_device) { int rc = check_device_ptr(h, in, "qrl_mmdvm_tx_work"); if (rc) return rc; }
    else {
        if (!h->d_in) { int rc = dev_alloc(h, &h->d_in, static_cast<size_t>(h->max_in) * h->C, false); if (rc) return rc; }
        QRL_CK(cudaMemcpy2DAsync(h->d_in, sizeof(short) * h->max_in, in, sizeof(short) * stride, sizeof(short) * n, h->C, cudaMemcpyHostToDevice, h->stream));
        s = h->d_in; sstride = h->max_in;
    }
    const int TB = 256;
    const long long a0 = h->n_in, a1 = h->n_in + n;
    mmdvm_short_float_kernel<<<dim3(static_cast<unsigned>(std::min<long long>((n + TB - 1) / TB, 4096)), h->C), TB, 0, h->stream>>>(
        s, sstride, n, h->level, h->d_sym, h->sym_mask, h->sym_stride, a0);
    // frequency_modulator_fc: the FM scan kernel with a one-tap "pulse" (x * 1.0 is exact), Q32 phase carried in the state
    tx_shape_fm_kernel<1024, 2><<<h->C, 1024, 0, h->stream>>>(h->d_bits, h->d_sym, h->sym_mask, h->sym_stride, a0, n,
        1, 1, h->d_one, 0, 1.0f, h->fm_sens, 1.0f, 1.0f, h->d_if, h->if_mask, h->if_stride);
    if (h->single) {
        // gr_mod_mmdvm.cpp:51-58: gr_zero_idle_bursts(0) between the FM modulator and the filter (items of the 24 ksps stream)
        std::vector<long long> ranges;
        h->zi.collect(h->C, a0, a1, 0, ranges);
        if (!ranges.empty()) {
            QRL_CK(h->zi.upload(ranges, h->stream));
            tx_zero_ranges_kernel<<<static_cast<unsigned>(ranges.size() / 3), 256, 0, h->stream>>>(h->d_if, h->if_mask, h->if_stride, h->zi.d_ranges);
            h->launches++;
        }
    }
    dim3 g(static_cast<unsigned>((n + TB - 1) / TB), h->C);
    { int rc = launch_fir_ccf_c(h, h->C, h->stream, h->d_if, h->if_mask, h->if_stride, h->d_rf, h->if_mask, h->if_stride, h->d_taps2, h->nt2, a0, a1, nullptr, 0, 0, 0); if (rc) return rc; h->launches--; }
    scale2_ring_kernel<<<g, TB, 0, h->stream>>>(h->d_rf, h->if_mask, h->if_stride, a0, a1, 0.8f, h->single ? h->bb_gain : 1.0f);   // gr_mod_mmdvm: bb_gain here
    const long long o0 = h->n25, o1 = (a1 * h->L + h->M - 1) / h->M;     // outputs i with floor(M i / L) < a1
    if (o1 - o0 > h->lin_stride) { set_err(h, "qrl_mmdvm_tx_work: output buffer too small"); return QRL_ERANGE; }
    if (o1 > o0) {
        dim3 go(static_cast<unsigned>((o1 - o0 + 255) / 256), h->C);
        resamp_ring_ccf_generic_kernel<<<go, 256, sizeof(float) * h->L * h->nt_arm, h->stream>>>(h->d_rf, h->if_mask, h->if_stride, h->d_arms, h->L, h->M, h->nt_arm, o0, o1,
                                                                                               h->d_lin, h->lin_stride);
        if (!h->single) {
            // gr_mod_mmdvm_multi2.cpp:88,108-117: gr_zero_idle_bursts(0) between the x25/24 resampler and the synthesizer (items of the
            // 25 ksps stream; the linear buffer holds items o0 .. o1 of this call)
            std::vector<long long> ranges;
            h->zi.collect(h->C, o0, o1, o0, ranges);
            if (!ranges.empty()) {
                QRL_CK(h->zi.upload(ranges, h->stream));
                tx_zero_ranges_kernel<<<static_cast<unsigned>(ranges.size() / 3), 256, 0, h->stream>>>(h->d_lin, 0xffffffffu, h->lin_stride, h->zi.d_ranges);
                h->launches++;
            }
        }
        mmdvm_scatter_kernel<<<dim3(static_cast<unsigned>(std::min<long long>((o1 - o0 + TB - 1) / TB, 4096)), h->C), TB, 0, h->stream>>>(
            h->d_lin, h->lin_stride, h->d_rows, o1 - o0, h->d_out, h->out_stride);
    }
    h->launches += 6;
    h->n_in = a1; h->n25 = o1;
    h->n_out_last = static_cast<long>(o1 - o0);
    if (n_out) *n_out = h->n_out_last;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_mmdvm_tx_out_device(qrl_mmdvm_tx* h, float** data, long* stride, long* n_out)
{
    if (!h) return QRL_EINVAL;
    if (data) *data = reinterpret_cast<float*>(h->d_out);
    if (stride) *stride = static_cast<long>(h->out_stride);
    if (n_out) *n_out = h->n_out_last;
    return QRL_OK;
}
int qrl_mmdvm_tx_read(qrl_mmdvm_tx* h, float* dst, long dst_stride)
{
    if (!h || !dst) return QRL_EINVAL;
    QRL_CK(cudaSetDevice(h->device));
    if (h->n_out_last > 0)
        QRL_CK(cudaMemcpy2DAsync(dst, sizeof(float2) * dst_stride, h->d_out, sizeof(float2) * h->out_stride, sizeof(float2) * h->n_out_last, h->n_rows, cudaMemcpyDeviceToHost, h->stream));
    QRL_CK(cudaStreamSynchronize(h->stream));
    return QRL_OK;
}
// behind the synthesizer (gr_mod_mmdvm_multi2.cpp:94-96,123-125): multiply_const_cc(1 / num_channels) -> multiply_const_cc(bb_gain), in place
int qrl_mmdvm_tx_finish(qrl_mmdvm_tx* h, float* wideband_dev, long n)
{
    if (!h || !wideband_dev || n < 0) return QRL_EINVAL;
    if (n == 0) return QRL_OK;
    QRL_CK(cudaSetDevice(h->device));
    int rc = check_device_ptr(h, wideband_dev, "qrl_mmdvm_tx_finish"); if (rc) return rc;
    scale2_linear_kernel<<<static_cast<unsigned>(std::min<long>((n + 255) / 256, 4096)), 256, 0, h->stream>>>(
        reinterpret_cast<float2*>(wideband_dev), n, 1.0f / static_cast<float>(h->num_channels), h->bb_gain);
    h->launches++;
    QRL_CK(cudaGetLastError());
    return QRL_OK;
}
int qrl_mmdvm_rx_sync(qrl_mmdvm_rx* h) { if (!h) return QRL_EINVAL; QRL_CK(cudaStreamSynchronize(h->stream)); return QRL_OK; }
int qrl_mmdvm_tx_sync(qrl_mmdvm_tx* h) { if (!h) return QRL_EINVAL; QRL_CK(cudaStreamSynchronize(h->stream)); return QRL_OK; }
long qrl_mmdvm_tx_launch_count(qrl_mmdvm_tx* h) { return h ? h->launches : 0; }

}  // extern "C"

#ifdef QRL_SS_PROF
// profiling build only (tools/ss_prof.py): read and clear the symbol-sync loop warp's cycle counters
extern "C" int qrl_debug_ss_prof(long long* out16)
{
    if (cudaMemcpyFromSymbol(out16, qrl::d_ss_prof, sizeof(long long) * 16) != cudaSuccess) return -1;
    long long z[16] = { 0 };
    return cudaMemcpyToSymbol(qrl::d_ss_prof, z, sizeof(z)) == cudaSuccess ? 0 : -1;
}
#endif
