// Small CUDA runtime helpers shared by the XR-Linear and HNSW engines.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>

namespace pb200 {

inline void cuda_check(cudaError_t err, const char* what, const char* file, int line) {
    if (err != cudaSuccess) {
        throw std::runtime_error(std::string("pecos_b200: CUDA error '") + cudaGetErrorString(err) + "' in " + what +
                                 " (" + file + ":" + std::to_string(line) +
                                 "). This library has no CPU fallback: a working sm_90a (H100) GPU is required.");
    }
}
#define PB200_CUDA(call) ::pb200::cuda_check((call), #call, __FILE__, __LINE__)

// Owning device buffer (cudaMalloc / cudaFree).  reserve(n) beyond the capacity frees the allocation and makes a new one of
// exactly n elements: the address changes and the contents are dropped.
template <typename T>
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    DeviceBuffer(DeviceBuffer&& o) noexcept : ptr_(o.ptr_), cap_(o.cap_) { o.ptr_ = nullptr; o.cap_ = 0; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        if (this != &o) { release(); ptr_ = o.ptr_; cap_ = o.cap_; o.ptr_ = nullptr; o.cap_ = 0; }
        return *this;
    }
    ~DeviceBuffer() { release(); }

    void reserve(uint64_t n) {
        if (n <= cap_) return;
        release();
        PB200_CUDA(cudaMalloc(reinterpret_cast<void**>(&ptr_), n * sizeof(T)));
        cap_ = n;
    }
    void upload(const T* host, uint64_t n, cudaStream_t stream) {
        reserve(n);
        if (n) PB200_CUDA(cudaMemcpyAsync(ptr_, host, n * sizeof(T), cudaMemcpyHostToDevice, stream));
    }
    void release() {
        if (ptr_) cudaFree(ptr_);
        ptr_ = nullptr;
        cap_ = 0;
    }
    T* get() const { return ptr_; }
    uint64_t capacity() const { return cap_; }
    uint64_t bytes() const { return cap_ * sizeof(T); }

private:
    T* ptr_ = nullptr;
    uint64_t cap_ = 0;
};

// Owning pinned host buffer.
template <typename T>
class PinnedBuffer {
public:
    PinnedBuffer() = default;
    PinnedBuffer(const PinnedBuffer&) = delete;
    PinnedBuffer& operator=(const PinnedBuffer&) = delete;
    ~PinnedBuffer() { release(); }
    void reserve(uint64_t n) {
        if (n <= cap_) return;
        release();
        PB200_CUDA(cudaMallocHost(reinterpret_cast<void**>(&ptr_), n * sizeof(T)));
        cap_ = n;
    }
    void release() {
        if (ptr_) cudaFreeHost(ptr_);
        ptr_ = nullptr;
        cap_ = 0;
    }
    T* get() const { return ptr_; }

private:
    T* ptr_ = nullptr;
    uint64_t cap_ = 0;
};

}  // namespace pb200
