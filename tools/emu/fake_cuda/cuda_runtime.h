// fake cuda_runtime.h -- the slice of the CUDA runtime API that qradiolink_b200/csrc/*.cu uses, executed synchronously on the host,
// for the emulated TEST build of the library (tools/emu/build_emulated_lib.py).  Kernel launches were rewritten to emu::launch by
// that script, so every launch runs to completion where the host issues it: issue order is a valid order of the stream / event
// graph (an event can only be waited on after it was recorded), so streams and events need no behaviour here.
// TEST INFRASTRUCTURE ONLY: never shipped, never loaded by the qradiolink_b200 package.
#pragma once
#include "../qrl_tma_emu.hpp"

#include <cfenv>
#include <cstdio>
#include <cstdlib>
#include <cstring>

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2 };
struct emuStream { int dummy; };
struct emuEvent { int dummy; };
typedef emuStream* cudaStream_t;
typedef emuEvent* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaEnableDefault = 0 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
enum cudaDriverEntryPointQueryResult { cudaDriverEntryPointSuccess = 0, cudaDriverEntryPointSymbolNotFound = 1 };

static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr, int) { *v = 132; return cudaSuccess; }
static inline cudaError_t cudaDeviceGetStreamPriorityRange(int* lo, int* hi) { *lo = 0; *hi = -1; return cudaSuccess; }
static inline cudaError_t cudaMalloc(void** p, size_t n)
{
    *p = std::aligned_alloc(256, (n + 255) & ~size_t(255));
    // device memory is not zeroed by cudaMalloc: QRL_EMU_POISON=1 fills it with 0xFF (NaN as float) so that a kernel reading memory
    // nobody initialised shows up as a mismatch instead of a lucky zero
    if (*p && std::getenv("QRL_EMU_POISON")) std::memset(*p, 0xFF, (n + 255) & ~size_t(255));
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc(reinterpret_cast<void**>(p), n); }
static inline cudaError_t cudaFree(void* p) { std::free(p); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* p, int v, size_t n) { std::memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t = nullptr) { std::memset(p, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { std::memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { std::memcpy(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dpitch, const void* s, size_t spitch, size_t width, size_t height, cudaMemcpyKind,
                                            cudaStream_t = nullptr)
{
    for (size_t r = 0; r < height; r++) std::memcpy(static_cast<char*>(d) + r * dpitch, static_cast<const char*>(s) + r * spitch, width);
    return cudaSuccess;
}
#define cudaMemcpyToSymbol(sym, src, n) (std::memcpy(&(sym), (src), (n)), cudaSuccess)
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = new emuStream{ 0 }; return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithPriority(cudaStream_t* s, unsigned, int) { *s = new emuStream{ 0 }; return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new emuEvent{ 0 }; return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = new emuEvent{ 0 }; return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void* devicePointer; void* hostPointer; };
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes* a, const void* p)
{
    *a = cudaPointerAttributes{ cudaMemoryTypeUnregistered, 0, const_cast<void*>(p), const_cast<void*>(p) };
    return cudaSuccess;
}
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, int, int) { return cudaSuccess; }
static inline cudaError_t cudaGetDriverEntryPoint(const char*, void** fn, int, cudaDriverEntryPointQueryResult* st)
{
    *fn = nullptr; if (st) *st = cudaDriverEntryPointSymbolNotFound; return cudaSuccess;      // no green contexts: the library falls back to plain streams
}

// ---- device intrinsics beyond cuda_emu.hpp / qrl_tma_emu.hpp
// (__ldg, __ffs, __brev, __fadd_rd live in cuda_emu.hpp: the kernel-extraction harnesses need them too)
static inline size_t __cvta_generic_to_shared(const void* p) { return qrl::smem_u32(p); }
// CUDA's global min / max overloads
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline long long min(long long a, long long b) { return a < b ? a : b; }
static inline long long max(long long a, long long b) { return a > b ? a : b; }
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
