// yb_cuda.h -- move-only owners of the CUDA runtime resources the engine holds (host code only).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <string>
#include <utility>

#include "yb_model.h"

namespace yb {

#define CUDA_OK(call)                                                                                   \
    do {                                                                                                \
        cudaError_t _e = (call);                                                                        \
        if (_e != cudaSuccess)                                                                          \
            fatal_throw(std::string("CUDA error: ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" + \
                        std::to_string(__LINE__) + " (" #call ")");                                     \
    } while (0)

// An array of T in device memory (DevBuf, cudaMalloc) or pinned host memory (PinnedBuf, cudaHostAlloc); empty until sized.
template <typename T, bool Pinned>
class CudaBuf {
public:
    CudaBuf() = default;
    explicit CudaBuf(size_t count) { ensure(count); }
    CudaBuf(CudaBuf &&o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
    CudaBuf &operator=(CudaBuf o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
    ~CudaBuf() { release(p_); }

    T *get() const { return p_; }
    size_t count() const { return n_; }
    explicit operator bool() const { return p_ != nullptr; }
    // Room for at least `count` elements; the contents are not kept.  The new block is allocated before the old one is
    // freed, and the size is recorded last, so a failed allocation leaves the buffer as it was.
    void ensure(size_t count) {
        if (count <= n_) return;
        void *q = nullptr;
        if (Pinned) CUDA_OK(cudaHostAlloc(&q, count * sizeof(T), cudaHostAllocDefault));
        else CUDA_OK(cudaMalloc(&q, count * sizeof(T)));
        release(p_);
        p_ = static_cast<T *>(q);
        n_ = count;
    }

private:
    static void release(T *p) {
        if (p && Pinned) cudaFreeHost(p);
        else if (p) cudaFree(p);
    }
    T *p_ = nullptr;
    size_t n_ = 0;
};
template <typename T> using DevBuf = CudaBuf<T, false>;
template <typename T> using PinnedBuf = CudaBuf<T, true>;

// One CUDA handle, released by Destroy; empty when default-constructed.  Converts to the raw handle for the runtime calls.
template <typename H, cudaError_t (*Destroy)(H)>
class CudaHandle {
public:
    CudaHandle() = default;
    explicit CudaHandle(H h) : h_(h) {}
    CudaHandle(CudaHandle &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    CudaHandle &operator=(CudaHandle o) noexcept { std::swap(h_, o.h_); return *this; }
    ~CudaHandle() { if (h_) Destroy(h_); }
    operator H() const { return h_; }

private:
    H h_ = nullptr;
};
using Event = CudaHandle<cudaEvent_t, cudaEventDestroy>;
using Stream = CudaHandle<cudaStream_t, cudaStreamDestroy>;
using GraphExec = CudaHandle<cudaGraphExec_t, cudaGraphExecDestroy>;

// events only order work unless timing is asked for
inline Event make_event(unsigned flags = cudaEventDisableTiming) {
    cudaEvent_t ev = nullptr;
    CUDA_OK(cudaEventCreateWithFlags(&ev, flags));
    return Event(ev);
}
inline Stream make_stream() {
    cudaStream_t s = nullptr;
    CUDA_OK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    return Stream(s);
}

}  // namespace yb
