// host_mem.h — single owners of the host code's device blocks, pinned blocks and timing events (host code only)
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <utility>
#include <vector>

namespace jv {

// One device block, freed by its destructor. Moving hands the block over; copying is not allowed.
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(DeviceBuffer &&o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)) {}
    DeviceBuffer &operator=(DeviceBuffer &&o) noexcept { std::swap(p_, o.p_); std::swap(cap_, o.cap_); return *this; }
    ~DeviceBuffer() { reset(); }
    // exactly `bytes`; the old block is freed first
    cudaError_t alloc(size_t bytes)
    {
        reset();
        const cudaError_t e = cudaMalloc(&p_, bytes);
        if (e == cudaSuccess) cap_ = bytes;
        else p_ = nullptr;
        return e;
    }
    // staging: reallocated only when `bytes` does not fit, to bytes + bytes / 4 + 256. The old block is freed first, and
    // cudaFree waits for the device, so no queued work still reads it when it goes.
    cudaError_t grow(size_t bytes) { return bytes <= cap_ ? cudaSuccess : alloc(bytes + bytes / 4 + 256); }
    void reset() { if (p_) cudaFree(p_); abandon(); }
    void abandon() { p_ = nullptr; cap_ = 0; }  // forget the block without freeing it: the runtime is already gone at exit
    template <typename T = void> T *get() const { return static_cast<T *>(p_); }

private:
    void *p_ = nullptr;
    size_t cap_ = 0;
};

// a new block of `bytes` appended to `owners`, with `p` pointing at it (nullptr when the allocation fails)
template <typename T>
cudaError_t alloc_owned(std::vector<DeviceBuffer> &owners, T *&p, size_t bytes)
{
    owners.emplace_back();
    const cudaError_t e = owners.back().alloc(bytes);
    p = owners.back().get<T>();
    return e;
}

// One pinned, device-mapped host block, freed by its destructor.
class PinnedBuffer {
public:
    PinnedBuffer() = default;
    PinnedBuffer(const PinnedBuffer &) = delete;
    PinnedBuffer &operator=(const PinnedBuffer &) = delete;
    ~PinnedBuffer() { reset(); }
    // the rule of DeviceBuffer::grow; the caller makes sure that no queued work still uses the old block
    cudaError_t grow(size_t bytes)
    {
        if (bytes <= cap_) return cudaSuccess;
        reset();
        const size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaHostAlloc(&h_, want, cudaHostAllocMapped);
        if (e == cudaSuccess) e = cudaHostGetDevicePointer(&d_, h_, 0);
        if (e == cudaSuccess) cap_ = want;
        else reset();
        return e;
    }
    void reset() { if (h_) cudaFreeHost(h_); abandon(); }
    void abandon() { h_ = d_ = nullptr; cap_ = 0; }
    template <typename T = void> T *get() const { return static_cast<T *>(h_); }
    template <typename T = void> T *dev() const { return static_cast<T *>(d_); }
    size_t capacity() const { return cap_; }

private:
    void *h_ = nullptr, *d_ = nullptr;
    size_t cap_ = 0;
};

// Device time from start(s) to stop(s); the first start() creates the events. ms() is valid once the stream has passed stop().
class StreamTimer {
public:
    StreamTimer() = default;
    StreamTimer(const StreamTimer &) = delete;
    StreamTimer &operator=(const StreamTimer &) = delete;
    ~StreamTimer() { reset(); }
    cudaError_t start(cudaStream_t s)
    {
        for (cudaEvent_t *ev : {&e0_, &e1_}) {
            const cudaError_t e = *ev ? cudaSuccess : cudaEventCreate(ev);
            if (e != cudaSuccess) { *ev = nullptr; return e; }
        }
        return cudaEventRecord(e0_, s);
    }
    cudaError_t stop(cudaStream_t s) { return cudaEventRecord(e1_, s); }
    float ms() const { float t = 0.f; cudaEventElapsedTime(&t, e0_, e1_); return t; }
    void reset() { if (e0_) cudaEventDestroy(e0_); if (e1_) cudaEventDestroy(e1_); abandon(); }
    void abandon() { e0_ = e1_ = nullptr; }

private:
    cudaEvent_t e0_ = nullptr, e1_ = nullptr;
};

}  // namespace jv
