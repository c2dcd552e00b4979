// qrl_handle.hpp -- the host plumbing every handle type of libqrl_b200.so shares (qrl_rx, qrl_tx, qrl_frontend, qrl_mmdvm_rx,
// qrl_mmdvm_tx, qrl_pfb, qrl_spectrum, qrl_deframer, qrl_dfbb): the common fields (one real base class, so that
// qrl_last_error(handle) reads `err` without a layout pun), error reporting, device buffers, stream ownership, create / destroy,
// the per-stage device profiler and the once-per-device setup (shared-memory opt-in, lookup tables).
// Host code only: the kernel launches stay in the .cu files.
#pragma once
#include "../../include/qrl_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>
#include <set>
#include <string>
#include <utility>
#include <vector>

struct QrlHandleBase {
    std::string err;
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    long launches = 0;
    std::vector<void*> allocs;
};

// ---- errors: every failure sets the calling thread's last error (qrl_last_error(NULL)) and, given a handle, the handle's own
inline std::string& thread_last_error()
{
    static thread_local std::string e;
    return e;
}

inline void set_err(QrlHandleBase* h, const std::string& s)
{
    thread_last_error() = s;
    if (h) h->err = s;
}

// a CUDA call that must succeed, inside a function with the handle (or nullptr) in scope as `h`
#define QRL_CK(call)                                                                                 \
    do {                                                                                             \
        cudaError_t e__ = (call);                                                                    \
        if (e__ != cudaSuccess) {                                                                    \
            set_err(h, std::string(#call) + ": " + cudaGetErrorString(e__));                         \
            return QRL_ECUDA;                                                                        \
        }                                                                                            \
    } while (0)

// ---- device buffers, owned by the handle (freed by handle_close)
template <class T>
int dev_alloc(QrlHandleBase* h, T** p, size_t n_items, bool zero = true)
{
    void* q = nullptr;
    size_t bytes = std::max<size_t>(n_items * sizeof(T), 16);
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e != cudaSuccess) { set_err(h, std::string("cudaMalloc: ") + cudaGetErrorString(e)); return QRL_ENOMEM; }
    if (zero) {
        e = cudaMemsetAsync(q, 0, bytes, h->stream);
        if (e != cudaSuccess) { set_err(h, std::string("cudaMemset: ") + cudaGetErrorString(e)); return QRL_ECUDA; }
    }
    h->allocs.push_back(q);
    *p = static_cast<T*>(q);
    return QRL_OK;
}

// initial state into a buffer dev_alloc zeroed: the zeroing memset is queued on the handle's (non-blocking) stream, so the copy goes
// on the same stream behind it -- a plain cudaMemcpy on the legacy stream is not ordered against it and can be overwritten by it
inline int upload_state(QrlHandleBase* h, void* dst, const void* src, size_t bytes)
{
    cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) { set_err(h, std::string("state upload: ") + cudaGetErrorString(e)); return QRL_ECUDA; }
    return QRL_OK;
}

inline int upload_floats(QrlHandleBase* h, float** p, const std::vector<float>& v)
{
    int rc = dev_alloc(h, p, v.size(), false);
    if (rc) return rc;
    cudaError_t e = cudaMemcpy(*p, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { set_err(h, std::string("tap upload: ") + cudaGetErrorString(e)); return QRL_ECUDA; }
    return QRL_OK;
}

// ---- lifecycle.  A create checks the device before it allocates anything, then handle_open()s the new handle and hands every later
// failure to create_failed; a destroy releases what only its type holds, then handle_close()s.
inline int check_device(const char* who, int device)
{
    if (qrl_device_count() > device) return QRL_OK;
    set_err(nullptr, std::string(who) + ": no CUDA device (this library has no CPU fallback)");
    return QRL_ENODEV;
}

// the handle's device and its own non-blocking stream
inline int handle_open(QrlHandleBase* h, int device)
{
    h->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { set_err(h, "cudaSetDevice failed"); return QRL_ECUDA; }
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) { set_err(h, "stream create failed"); return QRL_ECUDA; }
    h->own_stream = true;
    return QRL_OK;
}

// a create that failed half way: the type's destroy takes the handle down, its error stays the thread's last error
template <class H>
int create_failed(H* h, int (*destroy)(H*), int rc)
{
    const std::string e = h->err;
    destroy(h);
    set_err(nullptr, e);
    return rc;
}

template <class H>
int handle_close(H* h)
{
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    for (void* p : h->allocs) cudaFree(p);
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    delete h;
    return QRL_OK;
}

// a device pointer handed to a *_work call must live on the handle's device (a pointer from another GPU would fault inside a kernel
// long after the call returned)
inline int check_device_ptr(QrlHandleBase* h, const void* p, const char* who)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return QRL_OK; }
    if (a.type == cudaMemoryTypeDevice && a.device != h->device) {
        set_err(h, std::string(who) + ": the device pointer belongs to GPU " + std::to_string(a.device) + ", the handle to GPU " + std::to_string(h->device));
        return QRL_EINVAL;
    }
    return QRL_OK;
}

// *_set_stream: the handle's work so far drains, then it runs on the caller's stream; NULL = back to a stream of its own
inline int handle_set_stream(QrlHandleBase* h, void* s)
{
    QRL_CK(cudaSetDevice(h->device));
    QRL_CK(cudaStreamSynchronize(h->stream));
    if (h->own_stream && h->stream) { cudaStreamDestroy(h->stream); h->own_stream = false; }
    if (s) h->stream = static_cast<cudaStream_t>(s);
    else { QRL_CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true; }
    return QRL_OK;
}

// ---- optional per-stage device timing (qrl_rx_profile, qrl_tx_profile): an event pair around each profiled launch, summed per stage
// when read
class StageProfiler {
public:
    explicit StageProfiler(int n_stages) : ms_(n_stages, 0.0), n_(n_stages, 0) {}
    StageProfiler(const StageProfiler&) = delete;
    StageProfiler& operator=(const StageProfiler&) = delete;
    ~StageProfiler()
    {
        for (Rec& r : recs_) { if (r.a) cudaEventDestroy(r.a); if (r.b) cudaEventDestroy(r.b); }
    }
    int stages() const { return static_cast<int>(ms_.size()); }
    // start of a profiled launch on `s`: returns the event end() records behind it (nullptr while profiling is off)
    cudaEvent_t begin(int stage, cudaStream_t s)
    {
        stream_ = s;
        if (!on_) return nullptr;
        if (used_ == recs_.size()) {
            Rec r{ stage, nullptr, nullptr };
            cudaEventCreate(&r.a); cudaEventCreate(&r.b);
            recs_.push_back(r);
        }
        Rec& r = recs_[used_];
        r.stage = stage;
        cudaEventRecord(r.a, stream_);
        return r.b;
    }
    void end(cudaEvent_t b) { if (b) { cudaEventRecord(b, stream_); used_++; } }
    void reset(bool enable)
    {
        on_ = enable;
        used_ = 0;
        std::fill(ms_.begin(), ms_.end(), 0.0);
        std::fill(n_.begin(), n_.end(), 0L);
    }
    // folds the pairs recorded since the last read into the per-stage sums; the streams they were recorded on must have drained
    void read(int stage, double* ms_total, long* n_launches)
    {
        for (size_t i = 0; i < used_; i++) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, recs_[i].a, recs_[i].b) == cudaSuccess) { ms_[recs_[i].stage] += ms; n_[recs_[i].stage]++; }
        }
        used_ = 0;
        if (ms_total) *ms_total = ms_[stage];
        if (n_launches) *n_launches = n_[stage];
    }

private:
    struct Rec { int stage; cudaEvent_t a, b; };
    bool on_ = false;
    std::vector<Rec> recs_;
    size_t used_ = 0;
    std::vector<double> ms_;
    std::vector<long> n_;
    cudaStream_t stream_ = nullptr;
};

// ---- setup that belongs to a device's context (function attributes, __constant__ tables): done once per (key, device ordinal),
// under one lock, so any device ordinal and any number of host threads are safe.  A thread that finds the key done never runs ahead
// of the setup; a failed setup is retried by the next caller.
struct DeviceSetups {
    std::mutex mu;
    std::set<std::pair<const void*, int>> done;
};

inline DeviceSetups& device_setups()
{
    static DeviceSetups s;
    return s;
}

// setup() returns a QRL_* code
template <class F>
int once_per_device(const void* key, int device, F&& setup)
{
    DeviceSetups& s = device_setups();
    std::lock_guard<std::mutex> lk(s.mu);
    if (s.done.count({ key, device })) return QRL_OK;
    const int rc = setup();
    if (rc == QRL_OK) s.done.insert({ key, device });
    return rc;
}

// lets `kernel` launch with up to `bytes` of dynamic shared memory on the handle's device (the current device)
template <class K>
int smem_opt_in(QrlHandleBase* h, K* kernel, int bytes)
{
    return once_per_device(reinterpret_cast<const void*>(kernel), h->device, [&]() -> int {
        QRL_CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        return QRL_OK;
    });
}
