// C++ host-side test of the FreeDV factories of include/qrl_b200_gr.hpp on the GPU: int16 modem samples (a multi-tone stand-in for what
// freedv_tx_ss produces) -> make_gr_mod_freedv -> make_gr_demod_freedv, USB, 3 channels; the tones come back on port 0 (IQ at 8 ksps) at
// their frequencies, and port 1 delivers int16 modem samples, one per port-0 sample.
#include <cmath>
#include <complex>
#include <cstdio>
#include <vector>
#include "qrl_b200_gr.hpp"

using namespace qrl_gr;

int main()
{
    const int C = 3, N = 16000;                  // 2 s at 8 ksps
    const double tones[C] = { 700.0, 1100.0, 1900.0 };
    std::vector<short> in(static_cast<size_t>(C) * N);
    for (int c = 0; c < C; c++)
        for (int i = 0; i < N; i++) in[c * N + i] = static_cast<short>(std::lrint(8000.0 * std::sin(2 * M_PI * tones[c] * i / 8000.0)));
    try {
        auto mod = make_gr_mod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, C, N);
        std::vector<gr_complex> iq; long n_out = 0;
        if (mod->work(in.data(), N, N, iq, &n_out) < 0 || n_out != 125L * N) { std::printf("FAIL tx work (%ld outputs)\n", n_out); return 1; }
        auto demod = make_gr_demod_freedv(125, 1000000, 1700, 2500, 200, 0, 0, C, n_out);
        if (demod->work(iq.data(), static_cast<int>(n_out), n_out) < 0) { std::printf("FAIL rx work: %s\n", demod->last_error()); return 1; }
        for (int c = 0; c < C; c++) {
            int n0 = 0, n1 = 0;
            const gr_complex* y = demod->port<gr_complex>(0, c, &n0);
            const short* s = demod->port<short>(1, c, &n1);
            if (n0 != N || n1 != N || !y || !s) { std::printf("FAIL counts %d %d\n", n0, n1); return 1; }
            // strongest DFT bin of the last second, 1 Hz grid over 0..4000 Hz
            double best = 0; int fbest = -1;
            for (int f = 0; f < 4000; f++) {
                std::complex<double> acc = 0;
                for (int i = N / 2; i < N; i++) acc += std::complex<double>(y[i].real(), y[i].imag()) * std::polar(1.0, -2 * M_PI * f * i / 8000.0);
                if (std::abs(acc) > best) { best = std::abs(acc); fbest = f; }
            }
            int peak = 0;
            for (int i = N / 2; i < N; i++) peak = std::max(peak, std::abs(static_cast<int>(s[i])));
            std::printf("channel %d: tone %.0f Hz -> %d Hz, port-1 peak %d\n", c, tones[c], fbest, peak);
            if (std::abs(fbest - tones[c]) > 2 || peak < 100) { std::printf("FAIL\n"); return 1; }
        }
        bool threw = false;
        try { make_gr_demod_freedv(125, 1000000, 1700, 2500, 2500); } catch (const std::runtime_error&) { threw = true; }
        if (!threw) { std::printf("FAIL: low_cutoff >= filter_width did not throw\n"); return 1; }
    } catch (const std::exception& e) { std::printf("FAIL exception: %s\n", e.what()); return 1; }
    std::printf("OK\n");
    return 0;
}
