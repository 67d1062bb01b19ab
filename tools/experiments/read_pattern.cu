// read_pattern.cu -- microbenchmark: HBM read bandwidth of the hash kernels' access pattern (R requests of 16 KiB, each
// CTA walks 32 requests 512 bytes at a time) against a linear sweep of the same 1 GiB, with no hashing at all.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/_build/read_pattern tools/experiments/read_pattern.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

// 32 bytes as two 128-bit loads (the widest global load of sm_90)
__device__ __forceinline__ void ld256(const uint8_t *p, uint64_t x[4]) {
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(x[0]), "=l"(x[1]) : "l"(p));
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(x[2]), "=l"(x[3]) : "l"(p + 16));
}

// linear sweep: thread reads 64 B at consecutive positions, grid-stride
__global__ void k_linear(const uint8_t *d, size_t n64, uint64_t *out) {
    uint64_t acc = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n64; i += (size_t)gridDim.x * blockDim.x) {
        uint64_t a[4], b[4];
        ld256(d + i * 64, a);
        ld256(d + i * 64 + 32, b);
        acc ^= a[0] ^ a[1] ^ a[2] ^ a[3] ^ b[0] ^ b[1] ^ b[2] ^ b[3];
    }
    if (acc == 0x1234567) out[0] = acc;
}

// tiled: CTA = 256 threads = 32 requests x 8 blocks; thread (r, j) reads block k*8+j of request r, k = 0..nwin-1;
// DEPTH windows are loaded before the first is consumed
template <int DEPTH>
__global__ void k_tiled(const uint8_t *d, int R, int row_bytes, int n_tiles, uint64_t *out) {
    const int t = threadIdx.x, r = t / 8, j = t % 8;
    const int nwin = row_bytes / 512;
    uint64_t acc = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint8_t *base = d + (size_t)(tile * 32 + r) * row_bytes + j * 64;
        for (int k0 = 0; k0 < nwin; k0 += DEPTH) {
            uint64_t a[DEPTH][4], b[DEPTH][4];
#pragma unroll
            for (int q = 0; q < DEPTH; q++) { ld256(base + (size_t)(k0 + q) * 512, a[q]); ld256(base + (size_t)(k0 + q) * 512 + 32, b[q]); }
#pragma unroll
            for (int q = 0; q < DEPTH; q++) acc ^= a[q][0] ^ a[q][1] ^ a[q][2] ^ a[q][3] ^ b[q][0] ^ b[q][1] ^ b[q][2] ^ b[q][3];
        }
    }
    if (acc == 0x1234567) out[0] = acc;
}

// request-major: CTA reads ONE request's 16 KiB at a time (256 threads x 64 B), like the v1 digest kernel
__global__ void k_request(const uint8_t *d, int R, int row_bytes, uint64_t *out) {
    uint64_t acc = 0;
    for (int r = blockIdx.x; r < R; r += gridDim.x) {
        const uint8_t *base = d + (size_t)r * row_bytes;
        for (int o = threadIdx.x * 64; o < row_bytes; o += blockDim.x * 64) {
            uint64_t a[4], b[4];
            ld256(base + o, a);
            ld256(base + o + 32, b);
            acc ^= a[0] ^ a[1] ^ a[2] ^ a[3] ^ b[0] ^ b[1] ^ b[2] ^ b[3];
        }
    }
    if (acc == 0x1234567) out[0] = acc;
}

template <typename F>
static void timeit(const char *name, size_t bytes, F launch) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int i = 0; i < 3; i++) launch();
    cudaEventRecord(e0);
    const int K = 10;
    for (int i = 0; i < K; i++) launch();
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    printf("%-40s %8.4f ms  %8.1f GB/s\n", name, ms / K, bytes / (ms / K * 1e-3) / 1e9);
}

int main() {
    const int R = 65536, row = 16384;
    const size_t bytes = (size_t)R * row;
    uint8_t *d; uint64_t *out;
    cudaMalloc(&d, bytes); cudaMalloc(&out, 64);
    cudaMemset(d, 1, bytes);
    const int sm = 132;
    timeit("linear sweep, 132x8 CTAs x 256", bytes, [&] { k_linear<<<sm * 8, 256>>>(d, bytes / 64, out); });
    timeit("request-major (v1 digest pattern)", bytes, [&] { k_request<<<sm * 8, 256>>>(d, R, row, out); });
    timeit("tiled 32 req x 512 B, depth 1, 4 CTA/SM", bytes, [&] { k_tiled<1><<<sm * 4, 256>>>(d, R, row, R / 32, out); });
    timeit("tiled 32 req x 512 B, depth 1, 8 CTA/SM", bytes, [&] { k_tiled<1><<<sm * 8, 256>>>(d, R, row, R / 32, out); });
    timeit("tiled 32 req x 512 B, depth 2, 4 CTA/SM", bytes, [&] { k_tiled<2><<<sm * 4, 256>>>(d, R, row, R / 32, out); });
    timeit("tiled 32 req x 512 B, depth 4, 4 CTA/SM", bytes, [&] { k_tiled<4><<<sm * 4, 256>>>(d, R, row, R / 32, out); });
    timeit("tiled 32 req x 512 B, depth 4, 8 CTA/SM", bytes, [&] { k_tiled<4><<<sm * 8, 256>>>(d, R, row, R / 32, out); });
    // same with a non-power-of-two row pitch (16 KiB + 512 B): is it the 16 KiB stride?
    {
        const int row2 = 16384 + 512;
        uint8_t *d2; cudaMalloc(&d2, (size_t)R * row2); cudaMemset(d2, 1, (size_t)R * row2);
        timeit("tiled, row pitch 16896, depth 2, 4 CTA/SM", bytes, [&] { k_tiled<2><<<sm * 4, 256>>>(d2, R, row2, R / 32, out); });
        cudaFree(d2);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
