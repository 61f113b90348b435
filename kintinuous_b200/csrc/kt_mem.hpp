// kintinuous_b200 -- the one owner of CUDA memory, events and streams (host code only).
//
// Every cudaMalloc / cudaHostAlloc of the library is made here.  A refused allocation sets the error text (what was asked for, how
// many bytes), clears the runtime's "last error" -- a failed cudaMalloc records one, and the next KT_LAUNCH_CHECK on the thread would
// report it as a failed launch of an unrelated kernel -- returns KT_ERR_CUDA and leaves the pointer null.  Two owners release what they
// hold: DeviceBuffer (one growable device buffer) and Allocations (many allocations with one lifetime).
#pragma once
#include "kt_common.cuh"
#include "../../include/kintinuous_b200.h"
#include <memory>
#include <utility>
#include <vector>

namespace kt {

// the failure path of every allocation and creation below (bytes = 0: an event or a stream)
inline int refused(cudaError_t e, const char* call, const char* what, size_t bytes)
{
    cudaGetLastError();
    if (bytes) set_error("%s of %zu bytes for %s refused (%s)", call, bytes, what, cudaGetErrorString(e));
    else set_error("%s for %s refused (%s)", call, what, cudaGetErrorString(e));
    return KT_ERR_CUDA;
}

inline int device_malloc(void** p, size_t bytes, const char* what)
{
    const cudaError_t e = cudaMalloc(p, bytes);
    if (e == cudaSuccess) return 0;
    *p = nullptr;
    return refused(e, "cudaMalloc", what, bytes);
}

// page-locked host memory; flags cudaHostAllocMapped also maps it into the device's address space
inline int host_malloc(void** p, size_t bytes, const char* what, unsigned int flags = cudaHostAllocDefault)
{
    const cudaError_t e = cudaHostAlloc(p, bytes, flags);
    if (e == cudaSuccess) return 0;
    *p = nullptr;
    return refused(e, "cudaHostAlloc", what, bytes);
}

inline cudaError_t host_free(void* p) { return cudaFreeHost(p); }

// One device buffer that grows on demand.  Contents are not kept across a grow: the old buffer is freed before the new one is allocated.
template <class T> class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept { if (this != &o) { reset(); std::swap(p_, o.p_); std::swap(cap_, o.cap_); } return *this; }
    ~DeviceBuffer() { reset(); }
    T* get() const { return p_; }
    size_t capacity() const { return cap_; }
    // room for n elements: below that, free and allocate `want` (>= n) elements
    int grow(size_t n, size_t want, const char* what)
    {
        if (n <= cap_) return 0;
        reset();
        void* q = nullptr;
        if (int r = device_malloc(&q, want * sizeof(T), what)) return r;
        p_ = (T*)q; cap_ = want;
        return 0;
    }
    void reset() { if (p_) cudaFree(p_); p_ = nullptr; cap_ = 0; }
private:
    T* p_ = nullptr;
    size_t cap_ = 0;
};

// One owned event
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
using Event = std::unique_ptr<CUevent_st, EventDestroy>;
inline int make_event(Event* out, unsigned int flags, const char* what)
{
    cudaEvent_t e = nullptr;
    const cudaError_t s = cudaEventCreateWithFlags(&e, flags);
    if (s != cudaSuccess) return refused(s, "cudaEventCreate", what, 0);
    out->reset(e);
    return 0;
}

// Device, pinned and mapped-pinned memory, events and streams with one lifetime, released in reverse order.  Constructed with a stream,
// it is per-call scratch used on that stream: the stream is synchronised before anything is released.
class Allocations {
public:
    Allocations() = default;
    explicit Allocations(cudaStream_t s) : sync_(true), stream_(s) {}
    Allocations(Allocations&& o) noexcept : items_(std::move(o.items_)), sync_(o.sync_), stream_(o.stream_) { o.items_.clear(); }
    Allocations& operator=(Allocations&& o) noexcept
    {
        if (this != &o) { release(); items_ = std::move(o.items_); o.items_.clear(); sync_ = o.sync_; stream_ = o.stream_; }
        return *this;
    }
    ~Allocations() { release(); }

    // n elements of T; n = 0 gets one byte, so that a granted pointer is never null
    template <class T> int device(T** p, size_t n, const char* what)
    {
        void* q = nullptr;
        if (int r = device_malloc(&q, n ? n * sizeof(T) : 1, what)) { *p = nullptr; return r; }
        items_.push_back(Item{DEVICE, q}); *p = (T*)q;
        return 0;
    }
    template <class T> int pinned(T** p, size_t n, const char* what) { return host((void**)p, n * sizeof(T), cudaHostAllocDefault, what); }
    template <class T> int mapped(T** p, size_t n, const char* what) { return host((void**)p, n * sizeof(T), cudaHostAllocMapped, what); }
    int event(cudaEvent_t* e, unsigned int flags, const char* what)
    {
        const cudaError_t s = cudaEventCreateWithFlags(e, flags);
        if (s != cudaSuccess) { *e = nullptr; return refused(s, "cudaEventCreate", what, 0); }
        items_.push_back(Item{EVENT, (void*)*e});
        return 0;
    }
    int stream(cudaStream_t* q, const char* what)         // non-blocking
    {
        const cudaError_t s = cudaStreamCreateWithFlags(q, cudaStreamNonBlocking);
        if (s != cudaSuccess) { *q = nullptr; return refused(s, "cudaStreamCreate", what, 0); }
        items_.push_back(Item{STREAM, (void*)*q});
        return 0;
    }

private:
    enum Kind { DEVICE, HOST, EVENT, STREAM };
    struct Item { Kind kind; void* p; };
    std::vector<Item> items_;
    bool sync_ = false;
    cudaStream_t stream_ = nullptr;

    int host(void** p, size_t bytes, unsigned int flags, const char* what)
    {
        if (int r = host_malloc(p, bytes ? bytes : 1, what, flags)) return r;
        items_.push_back(Item{HOST, *p});
        return 0;
    }
    void release()
    {
        if (sync_) cudaStreamSynchronize(stream_);
        for (size_t i = items_.size(); i-- > 0;) {
            const Item& it = items_[i];
            switch (it.kind) {
            case DEVICE: cudaFree(it.p); break;
            case HOST: cudaFreeHost(it.p); break;
            case EVENT: cudaEventDestroy((cudaEvent_t)it.p); break;
            case STREAM: cudaStreamDestroy((cudaStream_t)it.p); break;
            }
        }
        items_.clear();
    }
};

} // namespace kt
