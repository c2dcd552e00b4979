// dmr_rx_harness.cpp -- the part of the DMR receive chain behind the resampler (gr_demod_dmr.cpp:60-112) on host threads: the CUDA
// kernels extracted from qrl_kernels.cuh (quadrature demod + symbol filter, port-3 copy, symbol sync variant 3 = generic recurrence
// with the plain Mueller & Mueller detector incl. its TMA producer / drain warps, external epilogue with the x0.9 scaling) wired like
// the QRL_DEMOD_DMR path of qrl_rx_create / qrl_rx_work in qradiolink_b200/csrc/qrl_b200.cu, one slice per call.
// TEST INFRASTRUCTURE (see cuda_emu.hpp): input is the oracle's port 0 (the 24 ksps resampler output), outputs are ports 1, 2, 3.
//   usage: dmr_rx_harness <in.bin: C x n float2> <C> <n> <out prefix> cut1 cut2 ...      (cuts = call boundaries in 24 ksps samples)
#include "qrl_tma_emu.hpp"

#include "../../qradiolink_b200/csrc/qrl_design.hpp"

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace qrl {
#include "kernels_extracted.inc"
}
using namespace qrl;

static unsigned pow2_at_least(long long n) { unsigned long long c = 64; while (c < (unsigned long long)n) c <<= 1; return (unsigned)c; }

int main(int argc, char** argv)
{
    if (argc < 5) return 2;
    const int C = atoi(argv[2]); const long n_total = atol(argv[3]);
    std::vector<float2> x((size_t)C * n_total);
    FILE* f = fopen(argv[1], "rb"); if (!f || fread(x.data(), sizeof(float2), x.size(), f) != x.size()) return 3; fclose(f);
    std::vector<long> edges{ 0 };
    for (int i = 5; i < argc; i++) edges.push_back(atol(argv[i]));
    edges.push_back(n_total);
    long n1max = 2;
    for (size_t e = 0; e + 1 < edges.size(); e++) n1max = std::max(n1max, edges[e + 1] - edges[e] + 2);

    // ---- tables and parameters: qrl_rx_create, QRL_DEMOD_DMR
    { auto t = atan_table(); std::copy(t.begin(), t.end(), d_atan_tab); }
    { auto t = tanh_table(); std::copy(t.begin(), t.end(), d_tanh_tab); }
    { auto t = mmse_table(); std::copy(t.begin(), t.end(), d_mmse_tab); }
    const int tsr = 24000, sym_sps = 5, groups = (C + 31) / 32;
    std::vector<float> taps3 = root_raised_cosine(1, tsr, tsr / sym_sps, 0.2, 25 * sym_sps);
    const int ntaps3 = (int)taps3.size();
    const float rate = (float)tsr / (float)sym_sps;
    const float qd_gain = (float)(tsr / (kPi / 2 * rate));
    SymSyncParams ssp{};
    clock_loop_gains((float)(2 * kPi / 100.0f), 1.0f, 0.2869f, ssp.alpha, ssp.beta);
    ssp.sps = (float)sym_sps; ssp.max_period = ssp.sps + 0.06f; ssp.min_period = ssp.sps - 0.06f;
    ssp.lookahead = 8 + (int)ceilf(ssp.max_period) + 1;
    ssp.pm_sens = (float)(kPi / 2); ssp.soft_scale = 128.0f;
    ssp.n0 = (int)floorf(ssp.min_period - fabsf(ssp.alpha)); ssp.fl0 = (float)ssp.n0;
    ssp.sym_scale = 0.9f;
    constexpr int CH = 256, NST = 3;
    const int maxs = (int)((CH + 1) / (ssp.min_period - fabsf(ssp.alpha)) + 3);
    const long long ss_chunk_cap = n1max / symsync_stride(CH, ssp.lookahead) + 4 + 3 * 16;
    const unsigned r2_cap = pow2_at_least(n1max + ntaps3 + 64), r4_cap = pow2_at_least(2 * n1max + 600);
    std::vector<float2> r2((size_t)r2_cap * C, float2{ 0, 0 });
    std::vector<float> r4((size_t)r4_cap * groups * 32, 0.0f);
    const Ring<float2> r2_ring{ r2.data(), r2_cap - 1, r2_cap };
    const Ring<float> r4_ring{ r4.data(), r4_cap - 1, r4_cap };
    std::vector<float> scratch((size_t)groups * ss_chunk_cap * (maxs + 2) * 32, 0.0f);
    std::vector<int> hdr((size_t)groups * 128, 0);
    const long port0_cap = n1max, port1_cap = n1max / std::max(1, sym_sps - 1) + 64, port2_cap = 2 * port1_cap + 160;
    std::vector<float2> port1((size_t)port1_cap * C);
    std::vector<unsigned char> port2((size_t)port2_cap * C), soft(64);
    std::vector<float> port3((size_t)port0_cap * C);
    std::vector<int> port1_cnt(C), port2_cnt(C);
    const Ring<unsigned char> soft_ring{ soft.data(), 63, 64 };
    std::vector<long long> nsoft(C);
    std::vector<SymSyncState> ss(C);
    for (auto& s : ss) { memset(&s, 0, sizeof s); s.avg_period = ssp.sps; s.inst_period = ssp.sps; s.mu = 0.0f; }

    std::vector<std::vector<float2>> o1(C); std::vector<std::vector<unsigned char>> o2(C); std::vector<std::vector<float>> o3(C);
    long long k1 = 0;
    for (size_t e = 0; e + 1 < edges.size(); e++) {
        const long long k0 = k1; k1 = edges[e + 1];
        const long long n_new = k1 - k0;
        std::fill(port1_cnt.begin(), port1_cnt.end(), 0); std::fill(port2_cnt.begin(), port2_cnt.end(), 0);
        // stage 2 stand-in: this call's resampler output enters the channel-major ring
        for (int c = 0; c < C; c++) for (long long a = k0; a < k1; a++) r2[(size_t)c * r2_cap + (a & (r2_cap - 1))] = x[(size_t)c * n_total + a];
        if (n_new > 0) {
            const int TB = 256;
            dim3 gtile((unsigned)((n_new + TB - 1) / TB), C);
            emu::launch(gtile, dim3(TB), sizeof(float) * (2 * ntaps3 + TB), [&] {
                qdemod_fir_fff_kernel(r2_ring, r4_ring, taps3.data(), ntaps3, qd_gain, k0, k1); });
            emu::launch(dim3((unsigned)((n_new + 31) / 32), groups), dim3(32, 8), 0, [&] {
                ring_to_port_f32_kernel(r4_ring, C, k0, k1, port3.data(), port0_cap, 0); });
        }
        const size_t smem = sizeof(float) * (NST * CH * 32 + SYMSYNC_TAB_FLOATS + 2 * (maxs + 2) * 32) + sizeof(int) * 64;
        const int chunk_bound = (int)std::min<long long>(ss_chunk_cap, n_new / symsync_stride(CH, ssp.lookahead) + 3);
        emu::launch(dim3(groups), dim3(96), smem, [&] {
            symsync_kernel<1, SL_RECT4, EPI_EXT_4FSK_FM, CH, NST, 1, LOOP_SYMSYNC, 3>(
                ssp, ss.data(), C, r4_ring, k1, port1.data(), port1_cap, port1_cnt.data(), (int)port1_cap,
                soft_ring, maxs, nsoft.data(), scratch.data(), chunk_bound, (int)ss_chunk_cap, hdr.data()); });
        if (chunk_bound > 0)
            emu::launch(dim3(chunk_bound, groups), dim3(32, 8), 0, [&] {
                symsync_ext_epilogue_kernel<1>(ssp, C, scratch.data(), (int)ss_chunk_cap, maxs, hdr.data(), port1.data(), port1_cap, (int)port1_cap,
                                               soft.data(), 63, 64, port2.data(), port2_cap, (int)port2_cap, port2_cnt.data(), port1_cnt.data()); });
        for (int c = 0; c < C; c++) {
            o1[c].insert(o1[c].end(), port1.begin() + (size_t)c * port1_cap, port1.begin() + (size_t)c * port1_cap + port1_cnt[c]);
            o2[c].insert(o2[c].end(), port2.begin() + (size_t)c * port2_cap, port2.begin() + (size_t)c * port2_cap + port2_cnt[c]);
            o3[c].insert(o3[c].end(), port3.begin() + (size_t)c * port0_cap, port3.begin() + (size_t)c * port0_cap + n_new);
        }
    }
    const std::string pre = argv[4];
    for (int c = 0; c < C; c++) {
        char name[512];
        snprintf(name, sizeof name, "%s.p1.%d.bin", pre.c_str(), c); f = fopen(name, "wb"); fwrite(o1[c].data(), sizeof(float2), o1[c].size(), f); fclose(f);
        snprintf(name, sizeof name, "%s.p2.%d.bin", pre.c_str(), c); f = fopen(name, "wb"); fwrite(o2[c].data(), 1, o2[c].size(), f); fclose(f);
        snprintf(name, sizeof name, "%s.p3.%d.bin", pre.c_str(), c); f = fopen(name, "wb"); fwrite(o3[c].data(), sizeof(float), o3[c].size(), f); fclose(f);
    }
    printf("OK\n");
    return 0;
}
