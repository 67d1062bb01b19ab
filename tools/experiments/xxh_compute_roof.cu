// xxh_compute_roof.cu -- how many prompt bytes per second can the SMs DIGEST (XXH64 stripe rounds + merge per 64-byte
// block, xxh64.cuh) with the data already in registers?  The compute roof of a1, measured: no loads, no stores.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I llm-d-inference-scheduler_b200/csrc -o tools/_build/xxh_compute_roof tools/experiments/xxh_compute_roof.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include "xxh64.cuh"
using namespace epp;

template <int ILP>
__global__ void k_digest(uint64_t *out, int iters, uint64_t seed) {
    uint64_t x[ILP][8];
#pragma unroll
    for (int s = 0; s < ILP; s++)
#pragma unroll
        for (int c = 0; c < 8; c++) x[s][c] = seed * (threadIdx.x + 1) + (uint64_t)(s * 8 + c) * 0x9E3779B97F4A7C15ull + blockIdx.x;
    uint64_t acc = 0;
    for (int i = 0; i < iters; i++) {
#pragma unroll
        for (int s = 0; s < ILP; s++) {
            uint64_t v[4];
            xxh_init(v);
#pragma unroll
            for (int c = 0; c < 4; c++) v[c] = xxh_round(v[c], x[s][c]);
#pragma unroll
            for (int c = 0; c < 4; c++) v[c] = xxh_round(v[c], x[s][4 + c]);
            const uint64_t m = xxh_merge_all(v);
            acc ^= m;
            x[s][i & 7] += m;                 // next block's data depends on this digest: nothing can be hoisted
        }
    }
    if (acc == 0x1234567) out[0] = acc;
}

// the serial chain step alone, lane = request (ILP 1 per thread)
__global__ void k_chain(uint64_t *out, int iters, uint64_t seed) {
    uint64_t prev = seed + threadIdx.x, m = seed * 3 + blockIdx.x;
    for (int i = 0; i < iters; i++) { prev = xxh_chain_step32(m, 72, prev); m += 0x9E3779B97F4A7C15ull; }
    if (prev == 0x1234567) out[0] = prev;
}

template <typename F>
static float timeit(F launch) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    launch();
    cudaEventRecord(e0);
    launch();
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    return ms;
}

int main() {
    uint64_t *out; cudaMalloc(&out, 64);
    const int sm = 132, iters = 4096;
    printf("digest of 64-byte blocks from registers (rounds + merge), bytes/s the SMs can hash:\n");
    for (int wps : {4, 8, 16, 32, 48, 64}) {           // warps per SM
        const int threads = 128, ctas = sm * wps / 4;
        float m1 = timeit([&] { k_digest<1><<<ctas, threads>>>(out, iters, 7); });
        float m2 = timeit([&] { k_digest<2><<<ctas, threads>>>(out, iters, 7); });
        const double b1 = (double)ctas * threads * iters * 64, b2 = b1 * 2;
        printf("  %2d warps/SM: ILP1 %7.3f ms %8.1f GB/s | ILP2 %7.3f ms %8.1f GB/s\n", wps, m1, b1 / (m1 * 1e-3) / 1e9, m2, b2 / (m2 * 1e-3) / 1e9);
    }
    printf("chain step (serial per thread), block-steps/s (x64 B = bytes/s the chain can follow):\n");
    for (int wps : {1, 2, 4, 8, 16, 32}) {
        const int threads = 32, ctas = sm * wps;
        float ms = timeit([&] { k_chain<<<ctas, threads>>>(out, iters, 7); });
        const double steps = (double)ctas * threads * iters;
        printf("  %2d warps/SM: %7.3f ms  %8.2f Gsteps/s = %8.1f GB/s of prompt\n", wps, ms, steps / (ms * 1e-3) / 1e9, steps * 64 / (ms * 1e-3) / 1e9);
    }
    printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
