// Move-only owners of the CUDA resources behind the C ABI's handles: device memory, pinned host memory, events and
// streams.  A handle's members release themselves, so its destroy function and every early return of its create
// function free exactly what was allocated.
#pragma once

#include <cuda_runtime.h>

#include <cstddef>
#include <utility>

namespace b200
{
// T[capacity] in device memory (cudaMalloc / cudaFree, which synchronises the device) or in page-locked host memory
// (cudaMallocHost or cudaHostAlloc / cudaFreeHost).  alloc and grow do not keep the contents, and they set the pointer
// and the capacity only when the allocation succeeds: after a failure the owner is empty.
template <typename T, bool Pinned>
class CudaBuffer
{
public:
    CudaBuffer() = default;
    CudaBuffer(CudaBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)) {}
    CudaBuffer& operator=(CudaBuffer&& o) noexcept
    {
        if (this != &o)
            {
                reset();
                p_ = std::exchange(o.p_, nullptr);
                cap_ = std::exchange(o.cap_, 0);
            }
        return *this;
    }
    ~CudaBuffer() { reset(); }

    operator T*() const { return p_; }
    T* operator->() const { return p_; }
    T* get() const { return p_; }
    size_t capacity() const { return cap_; }
    bool fits(size_t n) const { return n <= cap_; }

    cudaError_t reset()
    {
        const cudaError_t err = !p_ ? cudaSuccess : Pinned ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr;
        cap_ = 0;
        return err;
    }
    // n elements; host_flags: cudaHostAlloc flags of a pinned buffer (0 = cudaMallocHost)
    cudaError_t alloc(size_t n, unsigned int host_flags = 0)
    {
        cudaError_t err = reset();
        if (err != cudaSuccess) return err;
        void* q = nullptr;
        const size_t bytes = sizeof(T) * n;
        err = !Pinned ? cudaMalloc(&q, bytes) : host_flags ? cudaHostAlloc(&q, bytes, host_flags) : cudaMallocHost(&q, bytes);
        if (err == cudaSuccess)
            {
                p_ = static_cast<T*>(q);
                cap_ = n;
            }
        return err;
    }
    cudaError_t grow(size_t needed, size_t new_capacity) { return fits(needed) ? cudaSuccess : alloc(new_capacity); }

private:
    T* p_{nullptr};
    size_t cap_{0};
};

template <typename T>
using DevBuf = CudaBuffer<T, false>;
template <typename T>
using PinBuf = CudaBuffer<T, true>;

// An event or stream.  A borrowed handle (a stream the caller or another object owns) is used but never destroyed.
template <typename H, cudaError_t (*Create)(H*, unsigned int), cudaError_t (*Destroy)(H)>
class CudaHandle
{
public:
    CudaHandle() = default;
    CudaHandle(CudaHandle&& o) noexcept : h_(std::exchange(o.h_, nullptr)), owned_(std::exchange(o.owned_, false)) {}
    CudaHandle& operator=(CudaHandle&& o) noexcept
    {
        if (this != &o)
            {
                reset();
                h_ = std::exchange(o.h_, nullptr);
                owned_ = std::exchange(o.owned_, false);
            }
        return *this;
    }
    ~CudaHandle() { reset(); }

    operator H() const { return h_; }
    bool owned() const { return owned_; }

    void reset()
    {
        if (owned_) Destroy(h_);
        h_ = nullptr;
        owned_ = false;
    }
    cudaError_t create(unsigned int flags)
    {
        reset();
        H h = nullptr;
        const cudaError_t err = Create(&h, flags);
        if (err == cudaSuccess)
            {
                h_ = h;
                owned_ = true;
            }
        return err;
    }
    void borrow(H h)
    {
        reset();
        h_ = h;
    }

private:
    H h_{nullptr};
    bool owned_{false};
};

using CudaEvent = CudaHandle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
using CudaStream = CudaHandle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;
}  // namespace b200
