// lone_warp.cu -- what does a LONE warp pay per dependent instruction on sm_90a (H100)?
// (measurement tool behind DESIGN.md's latency floors: the symbol-sync and Costas recurrences run one warp per 32 channels,
// so their time is (items per channel) x (cycles of the loop-carried chain))
//   build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -fmad=false -I../../qradiolink_b200/csrc
//          -o lone_warp lone_warp.cu
//   run  : ./lone_warp            (prints cycles per operation / per Costas item for a few occupancy shapes)
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <cuda_runtime.h>
#include "qrl_kernels.cuh"

using namespace qrl;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

// mode: 0 = dependent FFMA chain, 1 = two interleaved FFMA chains, 2 = dependent FMNMX chain (alu pipe),
//       3 = FMUL -> FMNMX alternating (cross pipe), 4 = FFMA chain with one independent IADD between links,
//       5 = dependent FMUL -> FADD chain (non-fused, what -fmad=false code mostly is), 6 = LDS pointer chase
template <int MODE>
__global__ void chain_kernel(float a0, float b0, int iters, long long* __restrict__ cyc, float* __restrict__ sink, unsigned warp_mask)
{
    __shared__ int chase[1024];
    for (int i = threadIdx.x; i < 1024; i += blockDim.x) chase[i] = ((i + 33) & 1023) * 4;
    __syncthreads();
    const int warp = threadIdx.x >> 5;
    if (!((warp_mask >> warp) & 1)) return;
    float a = a0 + threadIdx.x * 1e-7f, b = b0, c = a0 * 0.5f, d = 0.25f;
    int k = threadIdx.x;
    unsigned p = (threadIdx.x & 31) * 4;
    const long long t0 = clock64();
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int u = 0; u < 64; u++) {
            if (MODE == 0) a = fmaf(a, b, d);
            if (MODE == 1) { a = fmaf(a, b, d); c = fmaf(c, b, d); }
            if (MODE == 2) a = fminf(fmaxf(a, -b), b + u);
            if (MODE == 3) { a = a * b; a = fminf(a, 3.0f + u); }
            if (MODE == 4) { a = fmaf(a, b, d); k += u; }
            if (MODE == 5) { a = a * b; a = a + d; }
            if (MODE == 6) { p = __float_as_uint(lds_f32<0>(smem_u32(chase) + p)); }
        }
    }
    const long long t1 = clock64();
    if ((threadIdx.x & 31) == 0) cyc[blockIdx.x * 32 + warp] = t1 - t0;
    sink[blockIdx.x * blockDim.x + threadIdx.x] = a + c + k + p;
}

// the Costas recurrence of agc_costas_kernel / symsync_kernel's QPSK epilogue, alone: items in shared memory, n per pass
__global__ void costas_kernel(int n, int passes, long long* __restrict__ cyc, float* __restrict__ sink, unsigned warp_mask)
{
    extern __shared__ __align__(128) float2 items[];          // [warps][n + 1][32]
    __shared__ float tanh_s[259];
    __shared__ volatile int opaque_zero;
    for (int i = threadIdx.x; i < 259; i += blockDim.x) tanh_s[i] = i < 257 ? tanhf((i < 256 ? i : 255) / 64.0f - 2.0f) : (i == 257 ? 1.0f : -1.0f);
    if (threadIdx.x == 0) opaque_zero = 0;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float2* mine = items + static_cast<size_t>(warp) * (n + 1) * 32;
    unsigned s = 12345u + threadIdx.x * 7919u + blockIdx.x * 104729u;
    for (int i = 0; i <= n; i++) {
        s = s * 1664525u + 1013904223u; const float re = ((s >> 8) & 0xffff) / 65536.0f - 0.5f;
        s = s * 1664525u + 1013904223u; const float im = ((s >> 8) & 0xffff) / 65536.0f - 0.5f;
        mine[i * 32 + lane] = make_float2(re * 2.0f, im * 2.0f);
    }
    __syncthreads();
    if (!((warp_mask >> warp) & 1)) return;
    LoopState st{ 0.1f * lane, 0.001f };
    const uint32_t tanh_m = smem_u32(tanh_s) - (0x4B000000u << 2) + static_cast<uint32_t>(opaque_zero);
    const long long t0 = clock64();
    for (int p = 0; p < passes; p++)
        qrl_costas4_snr_chunk(st, 0.0222f, 0.00025f, smem_u32(mine + lane), 256u, n, tanh_m);
    const long long t1 = clock64();
    if (lane == 0) cyc[blockIdx.x * 32 + warp] = t1 - t0;
    sink[blockIdx.x * blockDim.x + threadIdx.x] = st.phase + st.freq;
}

static double run_chain(int mode, int grid, int block, unsigned mask, int iters, long long* d_cyc, float* d_sink)
{
    CK(cudaMemset(d_cyc, 0, 4096 * sizeof(long long)));
    for (int rep = 0; rep < 2; rep++) {
        switch (mode) {
        case 0: chain_kernel<0><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        case 1: chain_kernel<1><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        case 2: chain_kernel<2><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        case 3: chain_kernel<3><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        case 4: chain_kernel<4><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        case 5: chain_kernel<5><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        case 6: chain_kernel<6><<<grid, block>>>(0.999f, 0.9999f, iters, d_cyc, d_sink, mask); break;
        }
        CK(cudaDeviceSynchronize());
    }
    std::vector<long long> h(4096);
    CK(cudaMemcpy(h.data(), d_cyc, 4096 * sizeof(long long), cudaMemcpyDeviceToHost));
    long long mx = 0;
    for (long long v : h) mx = v > mx ? v : mx;
    return static_cast<double>(mx) / (static_cast<double>(iters) * 64.0);
}

int main()
{
    long long* d_cyc; float* d_sink;
    CK(cudaMalloc(&d_cyc, 4096 * sizeof(long long)));
    CK(cudaMalloc(&d_sink, 1 << 20));
    const char* names[] = { "dependent FFMA", "2 interleaved FFMA chains (per pair)", "FMNMX+FMNMX (per pair)", "FMUL->FMNMX (per pair)",
                            "FFMA + independent IADD (per pair)", "FMUL->FADD (per pair)", "LDS pointer chase" };
    printf("# cycles per unrolled step, max over warps (clock64)\n");
    for (int mode = 0; mode < 7; mode++) {
        const double lone = run_chain(mode, 1, 32, 0x1, 256, d_cyc, d_sink);
        const double lone8 = run_chain(mode, 8, 32, 0x1, 256, d_cyc, d_sink);
        const double w4 = run_chain(mode, 1, 128, 0xf, 256, d_cyc, d_sink);       // one warp on each SMSP
        const double w2same = run_chain(mode, 1, 256, 0x11, 256, d_cyc, d_sink);  // warps 0 and 4: same SMSP
        const double w8 = run_chain(mode, 1, 256, 0xff, 256, d_cyc, d_sink);      // two per SMSP
        printf("%-40s lone %.2f | 8 CTAs x lone %.2f | 4 warps (1/SMSP) %.2f | 2 warps same SMSP %.2f | 8 warps %.2f\n",
               names[mode], lone, lone8, w4, w2same, w8);
    }
    // Costas recurrence
    const int n = 100, passes = 80;
    struct Shape { const char* name; int grid, block; unsigned mask; } shapes[] = {
        { "lone warp, 1 CTA", 1, 32, 0x1 }, { "lone warp, 8 CTAs", 8, 32, 0x1 }, { "warp 2 of a 96-thread CTA (as in agc_costas_kernel)", 8, 96, 0x4 },
        { "4 warps, one per SMSP", 1, 128, 0xf }, { "2 warps on the same SMSP", 1, 256, 0x11 }, { "8 warps, two per SMSP", 1, 256, 0xff },
    };
    CK(cudaFuncSetAttribute(costas_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    for (const Shape& sh : shapes) {
        const size_t smem = static_cast<size_t>(sh.block / 32) * (n + 1) * 32 * sizeof(float2);
        CK(cudaMemset(d_cyc, 0, 4096 * sizeof(long long)));
        for (int rep = 0; rep < 2; rep++) { costas_kernel<<<sh.grid, sh.block, smem>>>(n, passes, d_cyc, d_sink, sh.mask); CK(cudaDeviceSynchronize()); }
        std::vector<long long> h(4096);
        CK(cudaMemcpy(h.data(), d_cyc, 4096 * sizeof(long long), cudaMemcpyDeviceToHost));
        long long mx = 0; for (long long v : h) mx = v > mx ? v : mx;
        printf("costas4_snr recurrence, %-52s %.1f cycles per item\n", sh.name, static_cast<double>(mx) / (n * passes));
    }
    return 0;
}
