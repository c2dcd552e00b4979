// ring_to_port_harness.cpp -- ring_to_port_f32_kernel (gr_demod_dmr port 3 copy) on host threads: every (channel, sample) of a slice
// must land at port[c][port_off + a - a0], nothing else may be written.  TEST INFRASTRUCTURE (see cuda_emu.hpp).
#include "cuda_emu.hpp"

#include <cstdio>
#include <vector>

namespace qrl {
#include "kernels_extracted.inc"
}

int main()
{
    const int C = 37, groups = (C + 31) / 32;
    const unsigned cap = 256;                         // ring slots per group
    const long long port_stride = 300;
    std::vector<float> ring((size_t)groups * cap * 32);
    auto val = [](int c, long long a) { return (float)(c * 100000 + a); };
    int bad = 0;
    const long long cases[][3] = { { 0, 70, 0 }, { 70, 71, 70 }, { 200, 290, 5 }, { 290, 290, 0 }, { 1000, 1256, 40 } };   // a0, a1, port_off
    for (auto& cs : cases) {
        const long long a0 = cs[0], a1 = cs[1], off = cs[2];
        for (int c = 0; c < groups * 32; c++)
            for (long long a = a1 - cap; a < a1; a++) if (a >= 0) ring[((size_t)(c >> 5) * cap + (a & (cap - 1))) * 32 + (c & 31)] = val(c, a);
        std::vector<float> port((size_t)C * port_stride, -1.0f);
        if (a1 > a0)
            emu::launch(dim3((unsigned)((a1 - a0 + 31) / 32), groups), dim3(32, 8), 0, [&] {
                qrl::ring_to_port_f32_kernel(qrl::Ring<const float>{ ring.data(), cap - 1, cap }, C, a0, a1, port.data(), port_stride, off); });
        for (int c = 0; c < C; c++)
            for (long long i = 0; i < port_stride; i++) {
                const long long a = a0 + (i - off);
                const float want = (i >= off && a < a1) ? val(c, a) : -1.0f;
                if (port[(size_t)c * port_stride + i] != want) bad++;
            }
    }
    printf(bad ? "FAIL %d\n" : "OK\n", bad);
    return bad ? 1 : 0;
}
