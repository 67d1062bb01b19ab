// index.cuh -- device-side probe of the prefix-block table (shared by the match kernels).
#pragma once
#include "kernels.h"

namespace epp {

// Raw content of a hit slot: cnt and the five id words.
struct Hit {
    uint32_t cnt;
    uint32_t w[kInlineIds];
};

__device__ __forceinline__ void load_slot(const IndexSlot *p, uint64_t &key, Hit &h) {
    uint64_t a, b, c, d;   // the whole slot: two 128-bit loads (sm_90's widest) of the same 32-byte sector
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p));
    asm volatile("ld.global.nc.v2.u64 {%0,%1}, [%2];" : "=l"(c), "=l"(d) : "l"(reinterpret_cast<const uint8_t *>(p) + 16));
    key = a;
    h.cnt = (uint32_t)b;
    h.w[0] = (uint32_t)(b >> 32);
    h.w[1] = (uint32_t)c;
    h.w[2] = (uint32_t)(c >> 32);
    h.w[3] = (uint32_t)d;
    h.w[4] = (uint32_t)(d >> 32);
}

// indexer.Get (indexer.go:86-102): true iff some endpoint holds the block hash.
__device__ __forceinline__ bool probe(const IndexView &ix, uint64_t hash, Hit &h) {
    h.cnt = 0;
    if (hash == kEmptyKey) {
        h.cnt = ix.special.cnt;
#pragma unroll
        for (int q = 0; q < kInlineIds; q++) h.w[q] = ix.special.ids[q];
        return h.cnt != 0;
    }
    if (!ix.slots) return false;
    uint64_t i = hash & ix.mask;
    for (;;) {
        uint64_t key;
        load_slot(ix.slots + i, key, h);
        if (key == hash) return h.cnt != 0;               // cnt == 0: every holder was evicted (incremental patching)
        if (key == kEmptyKey) {                           // a never-used slot terminates the probe sequence
            h.cnt = 0;
            return false;
        }
        i = (i + 1) & ix.mask;
    }
}

// Presence bitmap of the read table: one bit per bucket of the key's top log2(bits) bits (shift = 64 - log2(bits);
// the table's `key & mask` uses the low bits).  A clear bit proves that no endpoint holds the key, a set bit means
// "maybe".  The all-ones key lives in the side record and always reads as present.
__device__ __forceinline__ bool presence_maybe(const uint32_t *bits, int shift, uint64_t h) {
    const uint32_t b = (uint32_t)(h >> shift);
    return h == kEmptyKey || ((__ldg(bits + (b >> 5)) >> (b & 31)) & 1u);
}
__device__ __forceinline__ void presence_set(uint32_t *bits, int shift, uint64_t h) {
    const uint32_t b = (uint32_t)(h >> shift);
    atomicOr(bits + (b >> 5), 1u << (b & 31));
}

// k-th endpoint of a hit (k < h.cnt).
__device__ __forceinline__ uint32_t posting(const IndexView &ix, const Hit &h, uint32_t k) {
    if (h.cnt > (uint32_t)kInlineIds) return ix.postings[h.w[0] + k];
    uint32_t e = h.w[0];
#pragma unroll
    for (int q = 1; q < kInlineIds; q++) e = (k == (uint32_t)q) ? h.w[q] : e;
    return e;
}

}  // namespace epp
