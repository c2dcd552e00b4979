// qrl_tma.cuh -- TMA 1-D bulk copy (cp.async.bulk -> UBLKCP), mbarrier and shared-memory address helpers (sm_90a).
// Header-only, shared by the translation units of libqrl_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace qrl {

// ------------------------------------------------------------------------------------------------
// TMA 1-D bulk copy (cp.async.bulk -> UBLKCP) + mbarrier helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
// shared-memory access by 32-bit shared address + immediate offset (keeps the recurrence's address math in one IMAD)
template <int OFF> __device__ __forceinline__ float lds_f32(uint32_t a)
{
    float v; asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(a), "n"(OFF)); return v;
}
template <int OFF> __device__ __forceinline__ float4 lds_f32x4(uint32_t a)
{
    float4 v; asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4+%5];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a), "n"(OFF));
    return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
template <int OFF> __device__ __forceinline__ float2 lds_f32x2(uint32_t a)
{
    float2 v; asm volatile("ld.shared.v2.f32 {%0,%1}, [%2+%3];" : "=f"(v.x), "=f"(v.y) : "r"(a), "n"(OFF)); return v;
}
__device__ __forceinline__ void sts_f32x2(uint32_t a, float x, float y) { asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(a), "f"(x), "f"(y) : "memory"); }
// FP32 pair FMA: acc.x = fma(s, v.x, acc.x), acc.y = fma(s, v.y, acc.y), a complex sample times a real tap.  sm_90 has no
// packed FP32 FMA, so this is two correctly rounded single FFMAs (the numerics contract asks for exactly these roundings).
__device__ __forceinline__ void ffma2(float2& acc, float s, float2 v)
{
    acc.x = fmaf(s, v.x, acc.x);
    acc.y = fmaf(s, v.y, acc.y);
}
// acc.x = fma(s, p.x, acc.x), acc.y = fma(s, p.y, acc.y) with a per-half multiplier pair p (DFT butterflies: s * (wr, wi))
__device__ __forceinline__ void ffma2_sp(float2& acc, float s, float px, float py)
{
    ffma2(acc, s, make_float2(px, py));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t done;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    } while (!done);
}

// nanosecond wall clock of the device (profiling build only: tools/ss_prof.py)
__device__ __forceinline__ unsigned long long globaltimer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

}  // namespace qrl
