// qrl_golay.cuh -- the (23,12) Golay code's check bits from its generator polynomial g(x) = 0xC75, shared by the M17 LICH
// (qrl_m17.cu) and the DMR AMBE FEC (qrl_dmr.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// the 12 check bits of data d of the extended (24,12) code: ((d(x) x^11 mod g(x)) << 1) | the parity of the 23-bit codeword
__host__ __device__ constexpr uint16_t golay_check(uint32_t d)
{
    uint32_t r = d << 11;
    for (int b = 22; b >= 11; b--)
        if (r >> b & 1u) r ^= 0xC75u << (b - 11);
    int par = 0;
    for (int b = 0; b < 12; b++) par += static_cast<int>((d >> b) & 1u) + static_cast<int>((r >> b) & 1u);
    return static_cast<uint16_t>((r << 1) | (par & 1));
}
