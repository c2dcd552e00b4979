// m17_tx_harness.cpp -- runs the M17 modulator's CUDA kernels (extracted from qrl_kernels.cuh into kernels_extracted.inc by
// tests/test_kernel_emulation.py) on host threads, wired exactly like the QRL_MOD_M17 branches of qrl_tx_create / qrl_tx_work in
// qradiolink_b200/csrc/qrl_b200.cu.  TEST INFRASTRUCTURE: checks kernel arithmetic, ring indexing and the output-count formulas
// against the oracle where no GPU exists; the host wiring in qrl_b200.cu itself is only confirmed by the GPU tier.
//   usage: m17_tx_harness <in.bin: C x n bytes> <C> <n> <out.bin: C x n_out float2> cut1 cut2 ...   (cuts = call boundaries in bytes)
#include "cuda_emu.hpp"

#include "../../qradiolink_b200/csrc/qrl_design.hpp"

#include <cstdio>
#include <cstdlib>
#include <vector>

namespace qrl {
#include "kernels_extracted.inc"
}
using namespace qrl;

static unsigned pow2_at_least(long long n) { unsigned long long c = 64; while (c < (unsigned long long)n) c <<= 1; return (unsigned)c; }
static std::vector<float> make_arms(const std::vector<float>& taps, int L, int nt)
{
    std::vector<float> a((size_t)L * nt, 0.0f);
    for (int p = 0; p < L; p++) for (int k = 0; k < nt; k++) { size_t j = p + (size_t)k * L; if (j < taps.size()) a[p * nt + k] = taps[j]; }
    return a;
}

int main(int argc, char** argv)
{
    if (argc < 5) return 2;
    const int C = atoi(argv[2]); const long max_items = atol(argv[3]);
    std::vector<unsigned char> data((size_t)C * max_items);
    FILE* f = fopen(argv[1], "rb"); if (!f || fread(data.data(), 1, data.size(), f) != data.size()) return 3; fclose(f);
    std::vector<long> edges{ 0 };
    for (int i = 5; i < argc; i++) edges.push_back(atol(argv[i]));
    edges.push_back(max_items);

    // ---- qrl_tx_create, QRL_MOD_M17 (sps 125, samp_rate 1e6, filter_width 9000)
    const int sps = 125, samp_rate = 1000000, filter_width = 9000;
    auto sn = fxpt_sine_table(); std::copy(sn.begin(), sn.end(), d_sine_tab);
    std::vector<float> t1 = root_raised_cosine(5, 5, 1, 0.5, 250);
    const int L1 = 5, nt1 = ((int)t1.size() + 4) / 5;
    const float fm_sens = (float)(kPi / 5), pulse_scale = 0.66666666f, amplif = 0.9f, bb_gain = 1.0f;
    std::vector<float> cfilt = low_pass(1, 24000, filter_width, filter_width, WIN_BLACKMAN_HARRIS);
    const int nt_cfilt = (int)cfilt.size();
    std::vector<float> t2 = low_pass(sps, 3.0 * samp_rate, 12000, 12000, WIN_BLACKMAN_HARRIS);
    const int L2 = sps, M2 = 3, nt2 = ((int)t2.size() + sps - 1) / sps;
    std::vector<float> arms1 = make_arms(t1, L1, nt1), arms2 = make_arms(t2, L2, nt2);
    const long long max_sym = 8LL * max_items;
    const unsigned sym_cap = pow2_at_least(max_sym + 64), if_cap = pow2_at_least(max_sym * L1 + 128), rc_cap = pow2_at_least(max_sym * L1 + 512 + nt2);
    std::vector<float> sym((size_t)sym_cap * C, 0.0f);
    std::vector<float2> ifr((size_t)if_cap * C, float2{ 0, 0 }), rc((size_t)rc_cap * C, float2{ 0, 0 });
    const Ring<float> sym_ring{ sym.data(), sym_cap - 1, sym_cap };
    const Ring<float2> if_ring{ ifr.data(), if_cap - 1, if_cap }, rc_ring{ rc.data(), rc_cap - 1, rc_cap };
    const long long out_stride = (4LL * max_items * L1 * L2 + M2 - 1) / M2 + 8;
    std::vector<float2> out((size_t)out_stride * C), all((size_t)out_stride * C);
    std::vector<TxBitState> st(C, TxBitState{ 0x7F, 0, 0, 0 });
    long long n_sym = 0, total_out = 0;

    // ---- qrl_tx_work, M17 branch, once per call
    for (size_t e = 0; e + 1 < edges.size(); e++) {
        const long n = edges[e + 1] - edges[e];
        if (n <= 0) continue;
        const unsigned char* b = data.data() + edges[e];
        const long long sym0 = n_sym, nsym = 4LL * n;
        emu::launch(dim3((C + 31) / 32), dim3(32), 0, [&] {
            tx_bits_kernel<TXM_M17>(st.data(), C, b, n, max_items, sym_ring, sym0); });
        emu::launch(dim3(C), dim3(1024), 0, [&] {
            tx_shape_fm_kernel<1024, 2>(st.data(), sym_ring, sym0, nsym, L1, nt1, arms1.data(), 0, pulse_scale, fm_sens,
                                        1.0f, 1.0f, if_ring); });
        const long long m0 = sym0 * L1, m1 = (sym0 + nsym) * L1;
        const int TB = 256;
        dim3 g((unsigned)((m1 - m0 + TB - 1) / TB), C);
        emu::launch(g, dim3(TB), sizeof(float) * nt_cfilt, [&] {
            fir_ccf_ring_kernel(if_ring, rc_ring, cfilt.data(), nt_cfilt, m0, m1, nullptr, 0, 0, 0); });
        emu::launch(g, dim3(TB), 0, [&] { scale2_ring_kernel(rc_ring, m0, m1, amplif, bb_gain); });
        const long long o0 = (m0 * L2 + M2 - 1) / M2, o1 = (m1 * L2 + M2 - 1) / M2;
        if (o1 - o0 > out_stride) return 4;
        emu::launch(dim3((unsigned)((o1 - o0 + 255) / 256), C), dim3(256), sizeof(float) * L2 * nt2, [&] {
            resamp_ring_ccf_generic_kernel(rc_ring, arms2.data(), L2, M2, nt2, o0, o1, out.data(), out_stride); });
        for (int c = 0; c < C; c++)
            for (long long i = 0; i < o1 - o0; i++) all[(size_t)c * out_stride + total_out + i] = out[(size_t)c * out_stride + i];
        total_out += o1 - o0;
        n_sym += nsym;
    }
    f = fopen(argv[4], "wb"); if (!f) return 5;
    for (int c = 0; c < C; c++) fwrite(all.data() + (size_t)c * out_stride, sizeof(float2), total_out, f);
    fclose(f);
    printf("%lld\n", total_out);
    return 0;
}
