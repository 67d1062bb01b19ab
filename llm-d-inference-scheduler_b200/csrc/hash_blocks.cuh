// hash_blocks.cuh -- the parallel part of a1 shared by the hash kernels: the stripe rounds + merge of one FULL block
// (part A of xxh64.cuh), fed by register 128-bit global loads.
#pragma once
#include "xxh64.cuh"

namespace epp {

// One 32-byte XXH64 stripe -> four little-endian u64 lanes: two 128-bit loads (the widest global load of sm_90; both
// halves of a 32-byte-aligned stripe fall in one DRAM sector).
__device__ __forceinline__ void load_stripe(const uint8_t *p, uint64_t x[4]) {
    uint4 a = __ldg(reinterpret_cast<const uint4 *>(p)), c = __ldg(reinterpret_cast<const uint4 *>(p) + 1);
    x[0] = ((uint64_t)a.y << 32) | a.x; x[1] = ((uint64_t)a.w << 32) | a.z;
    x[2] = ((uint64_t)c.y << 32) | c.x; x[3] = ((uint64_t)c.w << 32) | c.z;
}

// Stripe rounds + merge of one full block (part A of xxh64.cuh).
__device__ __forceinline__ uint64_t block_digest(const uint8_t *src, int n_stripes) {
    uint64_t v[4];
    xxh_init(v);
    if (n_stripes == 2) {   // the default 64-byte block: both stripes in flight at once
        uint64_t x0[4], x1[4];
        load_stripe(src, x0);
        load_stripe(src + 32, x1);
#pragma unroll
        for (int q = 0; q < 4; q++) v[q] = xxh_round(v[q], x0[q]);
#pragma unroll
        for (int q = 0; q < 4; q++) v[q] = xxh_round(v[q], x1[q]);
    } else {
        for (int st = 0; st < n_stripes; st++) {
            uint64_t x[4];
            load_stripe(src + 32 * st, x);
#pragma unroll
            for (int q = 0; q < 4; q++) v[q] = xxh_round(v[q], x[q]);
        }
    }
    return xxh_merge_all(v);
}

}  // namespace epp
