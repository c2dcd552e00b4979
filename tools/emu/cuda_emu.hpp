// cuda_emu.hpp -- "CUDA on host threads" for CPU-tier tests (tests/test_kernel_emulation.py, tests/test_emulated_library.py).
//
// TEST INFRASTRUCTURE ONLY (like oracle/): nothing under qradiolink_b200/ includes this, and it is no fallback -- it exists so that
// the library's kernels and host code can be exercised against the oracle in a container that has no GPU.  One OS thread per CUDA
// thread, the blocks of a grid run one after the other, __shared__ becomes a function-local static (shared by the block's threads),
// dynamic shared memory is a static arena.  Warp collectives are rendezvous among the lanes named by their mask (lanes that already
// left the kernel are not waited for); __activemask() returns the lanes of the warp that are at it once every other lane is blocked
// in a collective or gone.  Not emulated: anything about timing, the memory model, or hardware limits.
#pragma once
#include <barrier>
#include <cmath>
#include <condition_variable>
#include <cstdint>
#include <cstdlib>
#include <cfenv>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>
#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/asan_interface.h>
#endif

struct float2 { float x, y; };
struct uint2 { unsigned x, y; };
struct short2 { short x, y; };
struct char2 { signed char x, y; };
struct uint4 { unsigned x, y, z, w; };
static inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{ x, y }; }
static inline float2 make_float2(float x, float y) { return float2{ x, y }; }
namespace qrl {
// qrl_tma.cuh's ffma2 helpers = two independent correctly rounded fma
inline void ffma2(float2& acc, float s, float2 v) { acc.x = std::fmaf(s, v.x, acc.x); acc.y = std::fmaf(s, v.y, acc.y); }
inline void ffma2_sp(float2& acc, float s, float px, float py) { acc.x = std::fmaf(s, px, acc.x); acc.y = std::fmaf(s, py, acc.y); }
}
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };

namespace emu {
inline thread_local dim3 t_idx, b_idx;
inline dim3 b_dim, g_dim;
inline std::barrier<>* blk_bar = nullptr;
inline void* dyn_smem = nullptr;
alignas(128) inline unsigned char smem_arena[256 << 10];     // dynamic shared memory of the running block (static: see qrl_tma_emu.hpp)
inline unsigned lin_tid() { return t_idx.x + b_dim.x * (t_idx.y + b_dim.y * t_idx.z); }

enum { RUNNING = 0, BLOCKED = 1, EXITED = 2, AT_ACTIVEMASK = 3 };
struct Rendezvous { unsigned arrived = 0; unsigned long long gen = 0; unsigned long long buf[2][32]; };
struct WarpCtl {
    std::mutex m;
    std::condition_variable cv;
    unsigned existing = 0, exited = 0;
    int state[32] = { 0 };
    std::map<unsigned, Rendezvous> rv;
    unsigned am_mask = 0; int am_left = 0;                    // a published __activemask() result still being picked up
};
inline std::vector<std::unique_ptr<WarpCtl>> warps;

// every lane of `mask` (minus the lanes that have left the kernel) deposits a value; returns the snapshot of all of them
inline const unsigned long long* gather(unsigned mask, unsigned long long v)
{
    const unsigned t = lin_tid(), l = t & 31;
    WarpCtl& w = *warps[t >> 5];
    std::unique_lock<std::mutex> lk(w.m);
    mask &= w.existing;
    Rendezvous& r = w.rv[mask];
    const unsigned long long gen = r.gen;
    r.buf[gen & 1][l] = v;
    r.arrived |= 1u << l;
    auto complete = [&] { return (r.arrived & ~w.exited) == (mask & ~w.exited); };
    if (complete()) { r.arrived = 0; r.gen++; w.cv.notify_all(); }
    else {
        w.state[l] = BLOCKED;
        w.cv.notify_all();
        w.cv.wait(lk, [&] {
            if (r.gen != gen) return true;
            if (complete()) { r.arrived = 0; r.gen++; w.cv.notify_all(); return true; }      // the missing lanes left the kernel meanwhile
            return false;
        });
        w.state[l] = RUNNING;
    }
    return r.buf[gen & 1];
}
inline unsigned activemask()
{
    const unsigned t = lin_tid(), l = t & 31;
    WarpCtl& w = *warps[t >> 5];
    std::unique_lock<std::mutex> lk(w.m);
    w.state[l] = AT_ACTIVEMASK;
    w.cv.notify_all();
    for (;;) {
        if (w.am_left > 0 && (w.am_mask >> l & 1)) break;
        bool quiet = w.am_left == 0;
        for (int i = 0; i < 32 && quiet; i++) if ((w.existing >> i & 1) && w.state[i] == RUNNING) quiet = false;
        if (quiet) {
            unsigned mk = 0;
            for (int i = 0; i < 32; i++) if ((w.existing >> i & 1) && w.state[i] == AT_ACTIVEMASK) mk |= 1u << i;
            w.am_mask = mk; w.am_left = __builtin_popcount(mk);
            w.cv.notify_all();
            break;
        }
        w.cv.wait(lk);
    }
    const unsigned mk = w.am_mask;
    w.am_left--;
    w.state[l] = RUNNING;
    w.cv.notify_all();
    return mk;
}
inline void set_state(int s)
{
    const unsigned t = lin_tid();
    WarpCtl& w = *warps[t >> 5];
    std::lock_guard<std::mutex> lk(w.m);
    w.state[t & 31] = s;
    if (s == EXITED) w.exited |= 1u << (t & 31);
    w.cv.notify_all();
}

template <class F>
void launch(dim3 grid, dim3 block, size_t smem_bytes, F&& kernel_call)
{
    const unsigned nt = block.x * block.y * block.z;
    b_dim = block; g_dim = grid;
    if (smem_bytes > sizeof(smem_arena)) std::abort();
    dyn_smem = smem_arena;
#if defined(__SANITIZE_ADDRESS__)
    // AddressSanitizer build (QRL_EMU_ASAN=1): everything behind this launch's dynamic shared memory is poisoned
    __asan_unpoison_memory_region(smem_arena, sizeof(smem_arena));
    __asan_poison_memory_region(smem_arena + ((smem_bytes + 7) & ~size_t(7)), sizeof(smem_arena) - ((smem_bytes + 7) & ~size_t(7)));
#endif
    for (unsigned bz = 0; bz < grid.z; bz++) for (unsigned by = 0; by < grid.y; by++) for (unsigned bx = 0; bx < grid.x; bx++) {
        std::barrier<> bar(nt);
        blk_bar = &bar;
        warps.clear();
        for (unsigned w = 0; w < (nt + 31) / 32; w++) {
            warps.emplace_back(new WarpCtl());
            const unsigned lanes = std::min(32u, nt - 32 * w);
            warps.back()->existing = lanes == 32 ? 0xffffffffu : ((1u << lanes) - 1);
        }
        std::vector<std::thread> th;
        th.reserve(nt);
        for (unsigned t = 0; t < nt; t++)
            th.emplace_back([&, t]() {
                t_idx = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
                b_idx = dim3(bx, by, bz);
                kernel_call();
                set_state(EXITED);                   // a thread that returned early must not be waited for at later barriers
                blk_bar->arrive_and_drop();
            });
        for (auto& x : th) x.join();
    }
}
}  // namespace emu

#define threadIdx (emu::t_idx)
#define blockIdx (emu::b_idx)
#define blockDim (emu::b_dim)
#define gridDim (emu::g_dim)
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define EMU_DYN_SMEM(type, name) type* name = static_cast<type*>(emu::dyn_smem)

static inline void __syncthreads() { emu::set_state(emu::BLOCKED); emu::blk_bar->arrive_and_wait(); emu::set_state(emu::RUNNING); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::gather(mask, 0); }
template <class T> static inline unsigned long long emu_raw(T v) { static_assert(sizeof(T) <= 8); unsigned long long r = 0; std::memcpy(&r, &v, sizeof(T)); return r; }
template <class T> static inline T emu_unraw(unsigned long long r) { T v; std::memcpy(&v, &r, sizeof(T)); return v; }
template <class T> static inline T __shfl_sync(unsigned mask, T v, int src) { return emu_unraw<T>(emu::gather(mask, emu_raw(v))[src & 31]); }
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int off) { return emu_unraw<T>(emu::gather(mask, emu_raw(v))[((emu::lin_tid() & 31) ^ off) & 31]); }
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, int off)
{
    const unsigned l = emu::lin_tid() & 31; const unsigned long long* s = emu::gather(mask, emu_raw(v));
    return static_cast<int>(l) >= off ? emu_unraw<T>(s[l - off]) : v;
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, int off)
{
    const unsigned l = emu::lin_tid() & 31; const unsigned long long* s = emu::gather(mask, emu_raw(v));
    return l + off < 32 ? emu_unraw<T>(s[l + off]) : v;
}
static inline unsigned __ballot_sync(unsigned mask, int pred)
{
    const unsigned long long* s = emu::gather(mask, pred ? 1 : 0);
    const unsigned t = emu::lin_tid(); const unsigned alive = emu::warps[t >> 5]->existing & mask;
    unsigned m = 0;
    for (int l = 0; l < 32; l++) if ((alive >> l & 1) && s[l]) m |= 1u << l;
    return m;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __reduce_min_sync(unsigned mask, int v)
{
    const unsigned long long* s = emu::gather(mask, emu_raw(v));
    const unsigned t = emu::lin_tid(); const unsigned alive = emu::warps[t >> 5]->existing & mask;
    int r = v;
    for (int l = 0; l < 32; l++) if (alive >> l & 1) { const int o = emu_unraw<int>(s[l]); r = o < r ? o : r; }
    return r;
}
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) { return static_cast<unsigned>(__reduce_min_sync(mask, static_cast<int>(v))); }   // keys < 2^31
static inline unsigned __activemask() { return emu::activemask(); }
// __byte_perm(x, y, s): result byte i = byte (nibble i of s) of the 8-byte value y:x
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s)
{
    const unsigned long long v = (static_cast<unsigned long long>(y) << 32) | x;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) r |= static_cast<unsigned>((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
static inline unsigned __viaddmin_u32(unsigned a, unsigned b, unsigned c) { const unsigned t = a + b; return t < c ? t : c; }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline unsigned __brev(unsigned v)
{
    v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1); v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
    v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4); v = ((v >> 8) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8);
    return (v >> 16) | (v << 16);
}
static inline float __fadd_rd(float a, float b)
{
    const int old = std::fegetround(); std::fesetround(FE_DOWNWARD);
    volatile float x = a, y = b; volatile float r = x + y;
    std::fesetround(old);
    return r;
}
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline void sincospif(float x, float* s, float* c) { *s = static_cast<float>(std::sin(3.14159265358979323846 * static_cast<double>(x))); *c = static_cast<float>(std::cos(3.14159265358979323846 * static_cast<double>(x))); }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline long long __double_as_longlong(double d) { long long v; std::memcpy(&v, &d, 8); return v; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline unsigned __float_as_uint(float f) { unsigned i; std::memcpy(&i, &f, 4); return i; }
