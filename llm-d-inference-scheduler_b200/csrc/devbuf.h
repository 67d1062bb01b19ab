// devbuf.h -- grow-only device and pinned host allocations used by the engine's host logic.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    ~DevBuf() { if (p) cudaFree(p); }
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    // Grows (never shrinks); contents are NOT preserved.
    cudaError_t reserve(size_t bytes, size_t *accounted) {
        if (bytes <= cap) return cudaSuccess;
        if (p) { cudaFree(p); if (accounted) *accounted -= cap; p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { want = bytes; e = cudaMalloc(&p, want); }
        if (e != cudaSuccess) { p = nullptr; return e; }
        cap = want;
        if (accounted) *accounted += cap;
        return cudaSuccess;
    }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// Pinned staging of asynchronous host-to-device copies.  The caller refills it only once the copy that last read it has
// run, so reserve may free the old allocation.
struct HostBuf {
    void *p = nullptr;
    size_t cap = 0;
    ~HostBuf() { if (p) cudaFreeHost(p); }
    HostBuf() = default;
    HostBuf(const HostBuf &) = delete;
    HostBuf &operator=(const HostBuf &) = delete;
    // Grows (never shrinks) to twice the request, at least 4 KiB; contents are NOT preserved.
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) {
            cudaError_t e = cudaFreeHost(p);
            p = nullptr;
            cap = 0;
            if (e != cudaSuccess) return e;
        }
        const size_t want = bytes * 2 > 4096 ? bytes * 2 : 4096;
        cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
        if (e != cudaSuccess) { p = nullptr; return e; }
        cap = want;
        return cudaSuccess;
    }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};
