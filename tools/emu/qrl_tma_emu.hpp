// qrl_tma_emu.hpp -- host-thread stand-ins for qradiolink_b200/csrc/qrl_tma.cuh (same names, same signatures) on top of cuda_emu.hpp:
// mbarrier = arrival count + pending transaction bytes + phase, cp.async.bulk = memcpy (+ complete_tx), shared-memory "addresses" =
// offsets from a static arena that also holds the dynamic shared memory.  TEST INFRASTRUCTURE ONLY (see cuda_emu.hpp).
#pragma once
#include "cuda_emu.hpp"

#include <atomic>
#include <map>
#include <mutex>

struct float4 { float x, y, z, w; };

namespace emu {
// shared-memory "addresses" are offsets from 64 MB below cuda_emu.hpp's static arena (which holds the dynamic shared memory): the
// function-local statics that stand in for __shared__ variables live in the same data segment, within 32-bit reach
inline uintptr_t arena_base() { return reinterpret_cast<uintptr_t>(smem_arena) - (64u << 20); }
struct MBar { int expected = 0, pending = 0; long long tx = 0; unsigned long long phase = 0; };
inline std::mutex mbar_mu;
inline std::map<const void*, MBar> mbars;
inline void mbar_check(MBar& b) { if (b.pending == 0 && b.tx == 0) { b.phase++; b.pending = b.expected; } }
}  // namespace emu

namespace qrl {
inline uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(reinterpret_cast<uintptr_t>(p) - emu::arena_base()); }
inline void* smem_ptr(uint32_t a) { return reinterpret_cast<void*>(emu::arena_base() + a); }
template <int OFF> inline float lds_f32(uint32_t a) { return *static_cast<const float*>(smem_ptr(a + OFF)); }
template <int OFF> inline float4 lds_f32x4(uint32_t a) { return *static_cast<const float4*>(smem_ptr(a + OFF)); }
inline void sts_f32(uint32_t a, float v) { *static_cast<float*>(smem_ptr(a)) = v; }
template <int OFF> inline float2 lds_f32x2(uint32_t a) { return *static_cast<const float2*>(smem_ptr(a + OFF)); }
inline void sts_f32x2(uint32_t a, float x, float y) { *static_cast<float2*>(smem_ptr(a)) = make_float2(x, y); }
inline void mbar_init(uint64_t* bar, int count)
{
    std::lock_guard<std::mutex> lk(emu::mbar_mu);
    emu::MBar b; b.expected = count; b.pending = count;
    emu::mbars[bar] = b;
}
inline void mbar_fence_init() {}
inline void fence_proxy_async() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    std::lock_guard<std::mutex> lk(emu::mbar_mu);
    emu::MBar& b = emu::mbars.at(bar); b.tx += bytes; b.pending--; emu::mbar_check(b);
}
inline void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    std::memcpy(dst, src, bytes);
    std::lock_guard<std::mutex> lk(emu::mbar_mu);
    emu::MBar& b = emu::mbars.at(bar); b.tx -= bytes; emu::mbar_check(b);
}
inline void bulk_s2g(void* dst, const void* src, uint32_t bytes) { std::memcpy(dst, src, bytes); }
inline void bulk_commit() {}
inline void bulk_wait_read0() {}
inline void bulk_wait_all0() {}
inline void mbar_arrive(uint64_t* bar)
{
    std::lock_guard<std::mutex> lk(emu::mbar_mu);
    emu::MBar& b = emu::mbars.at(bar); b.pending--; emu::mbar_check(b);
}
inline void mbar_wait(uint64_t* bar, uint32_t parity)
{
    for (;;) {
        { std::lock_guard<std::mutex> lk(emu::mbar_mu); if ((emu::mbars.at(bar).phase & 1) != parity) return; }
        std::this_thread::yield();
    }
}
inline unsigned long long globaltimer_ns() { return 0; }   // profiling build only

// (a >= b) ? 1.0f : 0.0f  (set.ge.f32.f32 in qrl_kernels.cuh)
inline float qrl_ge1(float a, float b) { return a >= b ? 1.0f : 0.0f; }
// (x >= t) ? a : b  (setp.ge.f32 + selp.f32 in qrl_kernels.cuh)
inline float qrl_sel_ge(float x, float t, float a, float b) { return x >= t ? a : b; }
// (a >= b) ? 0xffffffff : 0  (set.ge.u32.f32 in qrl_kernels.cuh)
inline uint32_t qrl_ge_mask(float a, float b) { return a >= b ? 0xffffffffu : 0u; }
}  // namespace qrl
