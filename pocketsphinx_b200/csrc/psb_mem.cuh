// psb_mem.cuh -- the owners of the library's device memory, pinned host memory, streams and events.
// Host C++ over the CUDA runtime API only: no device code, so that it also builds with a plain C++ compiler.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <atomic>

#include "../../include/psb200.h"

void psb_set_error(const char *fmt, ...);
extern std::atomic<long long> g_psb_bytes_live;   // device + pinned bytes held by the library (psb_device_bytes_live)

// Every allocation goes through here.  A failure is cleared from the runtime's last error, so that the next
// launch check does not report it a second time, and returns PSB_ERR_NOMEM with the size in the message.
static inline int psb_mem_alloc(void **p, size_t bytes, bool pinned)
{
    *p = nullptr;
    const cudaError_t e = pinned ? cudaMallocHost(p, bytes) : cudaMalloc(p, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        *p = nullptr;
        psb_set_error("%s of %zu bytes failed: %s", pinned ? "cudaMallocHost" : "cudaMalloc", bytes, cudaGetErrorString(e));
        return PSB_ERR_NOMEM;
    }
    g_psb_bytes_live.fetch_add((long long)bytes, std::memory_order_relaxed);
    return PSB_OK;
}

static inline void psb_mem_free(void *p, size_t bytes, bool pinned)
{
    if (!p) return;
    if (pinned) cudaFreeHost(p);
    else cudaFree(p);
    g_psb_bytes_live.fetch_sub((long long)bytes, std::memory_order_relaxed);
}

// A grow-only buffer of T in device memory or pinned host memory.  It converts to T * so that launches and
// copies take it like the raw pointer it owns.
template <class T, bool Pinned>
class PsbBuf {
public:
    PsbBuf() = default;
    PsbBuf(PsbBuf &&o) noexcept : p_(o.p_), cap_(o.cap_) { o.p_ = nullptr; o.cap_ = 0; }
    PsbBuf &operator=(PsbBuf &&o) noexcept
    {
        if (this != &o) {
            release();
            p_ = o.p_; cap_ = o.cap_;
            o.p_ = nullptr; o.cap_ = 0;
        }
        return *this;
    }
    PsbBuf(const PsbBuf &) = delete;
    PsbBuf &operator=(const PsbBuf &) = delete;
    ~PsbBuf() { release(); }

    // Room for at least `need` elements.  A smaller block is freed first and need + headroom elements are
    // allocated; after a failure the buffer is empty with capacity 0, so the next call tries again.
    int reserve(size_t need, size_t headroom = 0)
    {
        if (cap_ >= need) return PSB_OK;
        release();
        void *p;
        const int rc = psb_mem_alloc(&p, (need + headroom) * sizeof(T), Pinned);
        if (rc) return rc;
        p_ = static_cast<T *>(p);
        cap_ = need + headroom;
        return PSB_OK;
    }
    void release()
    {
        psb_mem_free(p_, cap_ * sizeof(T), Pinned);
        p_ = nullptr;
        cap_ = 0;
    }
    T *get() const { return p_; }
    operator T *() const { return p_; }
    size_t cap() const { return cap_; }

private:
    T *p_ = nullptr;
    size_t cap_ = 0;   // elements
};

template <class T> using DevBuf = PsbBuf<T, false>;
template <class T> using HostBuf = PsbBuf<T, true>;

class Stream {
public:
    Stream() = default;
    Stream(Stream &&o) noexcept : s_(o.s_) { o.s_ = nullptr; }
    Stream &operator=(Stream &&o) noexcept
    {
        if (this != &o) { reset(); s_ = o.s_; o.s_ = nullptr; }
        return *this;
    }
    Stream(const Stream &) = delete;
    Stream &operator=(const Stream &) = delete;
    ~Stream() { reset(); }

    cudaError_t create(unsigned flags = cudaStreamNonBlocking)
    {
        reset();
        const cudaError_t e = cudaStreamCreateWithFlags(&s_, flags);
        if (e != cudaSuccess) s_ = nullptr;
        return e;
    }
    void reset()
    {
        if (s_) cudaStreamDestroy(s_);
        s_ = nullptr;
    }
    operator cudaStream_t() const { return s_; }

private:
    cudaStream_t s_ = nullptr;
};

class Event {
public:
    Event() = default;
    Event(Event &&o) noexcept : e_(o.e_) { o.e_ = nullptr; }
    Event &operator=(Event &&o) noexcept
    {
        if (this != &o) { reset(); e_ = o.e_; o.e_ = nullptr; }
        return *this;
    }
    Event(const Event &) = delete;
    Event &operator=(const Event &) = delete;
    ~Event() { reset(); }

    cudaError_t create(unsigned flags = cudaEventDefault)
    {
        reset();
        const cudaError_t e = cudaEventCreateWithFlags(&e_, flags);
        if (e != cudaSuccess) e_ = nullptr;
        return e;
    }
    void reset()
    {
        if (e_) cudaEventDestroy(e_);
        e_ = nullptr;
    }
    operator cudaEvent_t() const { return e_; }

private:
    cudaEvent_t e_ = nullptr;
};
