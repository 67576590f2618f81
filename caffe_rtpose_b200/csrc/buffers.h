// Owning buffers of device and pinned host memory (engine.cu).  Host-only: no kernels, no streams, only cudart's allocators.
#pragma once
#include <cuda_runtime_api.h>
#include <stddef.h>
#include <stdint.h>

namespace pe {

// One allocation, freed by the destructor.  Move-only; size() is 0 exactly when the buffer holds nothing.
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Release)(void*)>
class Buffer {
    void* p_ = nullptr;
    size_t n_ = 0;
public:
    Buffer() = default;
    Buffer(Buffer&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    Buffer& operator=(Buffer&& o) noexcept {   // frees what this buffer held, on the current device
        if (this != &o) { if (p_) Release(p_); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; }
        return *this;
    }
    ~Buffer() { if (p_) Release(p_); }
    // At least `need` bytes: a no-op when the buffer holds that many, else it frees and allocates `need`.  A failed allocation
    // leaves the buffer empty, so the next reserve allocates again whatever it asks for.
    cudaError_t reserve(size_t need) {
        if (need <= n_) return cudaSuccess;
        if (p_) Release(p_);
        n_ = 0;
        const cudaError_t err = Alloc(&p_, need);
        if (err == cudaSuccess) n_ = need; else p_ = nullptr;
        return err;
    }
    template <class T = uint8_t> T* get() const { return (T*)p_; }
    size_t size() const { return n_; }
};
using DeviceBuffer = Buffer<cudaMalloc, cudaFree>;
using PinnedBuffer = Buffer<cudaMallocHost, cudaFreeHost>;

// Consecutive ranges of one allocation, 256-byte aligned as separate cudaMalloc calls would be.  Over a null base it hands out
// null pointers and only counts, so the code that lays a group out also sizes its allocation.
class Carver {
    uint8_t* base_;
    size_t used_ = 0;
public:
    explicit Carver(void* base) : base_((uint8_t*)base) {}
    template <class T> T* take(size_t count) {
        T* p = base_ ? (T*)(base_ + used_) : nullptr;
        used_ += (count * sizeof(T) + 255) & ~(size_t)255;
        return p;
    }
    size_t used() const { return used_; }
};

// Reserves b for the ranges layout(Carver&) takes, then lays them out over it.  On failure b is empty and the ranges are null.
template <class B, class F>
cudaError_t reserve_carved(B& b, F layout) {
    Carver size(nullptr);
    layout(size);
    const cudaError_t err = b.reserve(size.used());
    Carver k(err == cudaSuccess ? b.get() : nullptr);
    layout(k);
    return err;
}

}  // namespace pe
