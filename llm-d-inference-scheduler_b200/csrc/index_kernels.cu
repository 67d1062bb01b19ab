// index_kernels.cu -- a2: the GPU-resident prefix-block index (inverted map  blockHash -> {endpoints}),
// the device counterpart of indexer.hashToPods (approximateprefix/indexer.go:32-37).
//
// Layout in HBM: one open-addressed table of 32-byte slots {key u64, count u32, 5 x endpoint u32} -- one sector,
// two 128-bit loads per probe -- linear probing from key & mask (XXH64 output is already uniformly mixed), load
// factor <= 0.5.  Lists longer than five endpoints spill to a contiguous u32 postings array.  Every list is
// sorted by endpoint id and duplicate-free (podSet is a set, indexer.go:78-82).
//
// Build (bulk, on the device, from a snapshot of (hash, endpoint) pairs):
//   k_index_clear -> k_index_insert (atomicCAS claim + count) -> k_index_alloc (posting ranges by atomic cursor)
//   -> k_index_fill (scatter endpoint ids) -> k_index_finalize (sort + dedupe, move short lists into the slot)
//   -> k_intern_* (equal spilled lists share one copy).
// Between bulk builds the table is kept up to date in place from the write side's change log (index_store.cu:
// k_patch_group / k_patch_apply): new keys claim free slots, lists are rewritten copy-on-write, a hash that loses its
// last endpoint keeps its slot with count 0 -- probe chains therefore end at FREE slots (key == sentinel), not at
// count == 0.
#include "index.cuh"

namespace epp {

__global__ void k_index_clear(IndexSlot *slots, uint32_t *fill, uint64_t capacity, uint32_t *cursor,
                              IndexSlot *special) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < capacity) {
        IndexSlot z;
        z.key = kEmptyKey;
        z.cnt = 0;
        for (int q = 0; q < kInlineIds; q++) z.ids[q] = 0;
        slots[i] = z;
        fill[i] = 0;
    }
    if (i == 0) {
        cursor[0] = 0;   // posting cursor
        cursor[1] = 0;   // special fill
        cursor[2] = 0;   // distinct hashes
        cursor[3] = 0;   // claimed keys of the interning table
        special->key = kEmptyKey;
        special->cnt = 0;
        for (int q = 0; q < kInlineIds; q++) special->ids[q] = 0;
    }
}

__device__ __forceinline__ uint64_t find_or_claim(IndexSlot *slots, uint64_t mask, uint64_t key, uint32_t *distinct) {
    uint64_t i = key & mask;
    for (;;) {
        unsigned long long *kp = reinterpret_cast<unsigned long long *>(&slots[i].key);
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(kp);
        if (cur == key) return i;
        if (cur == kEmptyKey) {
            unsigned long long old = atomicCAS(kp, (unsigned long long)kEmptyKey, (unsigned long long)key);
            if (old == kEmptyKey) { atomicAdd(distinct, 1u); return i; }
            if (old == key) return i;
        }
        i = (i + 1) & mask;
    }
}

__global__ void k_index_insert(const uint64_t *pair_hash, uint64_t n, IndexSlot *slots, uint64_t mask,
                               uint32_t *cursor, IndexSlot *special) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint64_t key = pair_hash[t];
    if (key == kEmptyKey) {
        atomicAdd(&special->cnt, 1u);
        return;
    }
    uint64_t i = find_or_claim(slots, mask, key, &cursor[2]);
    atomicAdd(&slots[i].cnt, 1u);
}

__global__ void k_index_alloc(IndexSlot *slots, uint64_t capacity, uint32_t *cursor, IndexSlot *special) {
    // one atomic per warp: the lanes' list lengths are prefix-summed with shuffles
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t cnt = i < capacity ? slots[i].cnt : 0u;
    uint32_t incl = cnt;
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
    }
    const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
    uint32_t base = 0;
    if (lane == 31 && total) base = atomicAdd(&cursor[0], total);
    base = __shfl_sync(0xffffffffu, base, 31);
    if (cnt) slots[i].ids[0] = base + incl - cnt;
    if (i == 0 && special->cnt) special->ids[0] = atomicAdd(&cursor[0], special->cnt);
}

__device__ __forceinline__ uint64_t find_slot(const IndexSlot *slots, uint64_t mask, uint64_t key) {
    uint64_t i = key & mask;
    while (slots[i].key != key) i = (i + 1) & mask;   // present by construction
    return i;
}

__global__ void k_index_fill(const uint64_t *pair_hash, const uint32_t *pair_ep, uint64_t n, IndexSlot *slots,
                             uint64_t mask, uint32_t *fill, uint32_t *postings, uint32_t *cursor,
                             IndexSlot *special) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint64_t key = pair_hash[t];
    if (key == kEmptyKey) {
        uint32_t pos = atomicAdd(&cursor[1], 1u);
        postings[special->ids[0] + pos] = pair_ep[t];
        return;
    }
    uint64_t i = find_slot(slots, mask, key);
    uint32_t pos = atomicAdd(&fill[i], 1u);
    postings[slots[i].ids[0] + pos] = pair_ep[t];
}

// In-place insertion sort + unique of one posting list; returns the new length.
__device__ inline uint32_t sort_unique(uint32_t *list, uint32_t cnt) {
    for (uint32_t a = 1; a < cnt; a++) {
        uint32_t e = list[a];
        uint32_t b = a;
        while (b > 0 && list[b - 1] > e) { list[b] = list[b - 1]; b--; }
        list[b] = e;
    }
    uint32_t w = 0;
    for (uint32_t a = 0; a < cnt; a++)
        if (w == 0 || list[w - 1] != list[a]) list[w++] = list[a];
    return w;
}

__device__ inline void finalize_slot(IndexSlot *sl, uint32_t *postings) {
    uint32_t off = sl->ids[0];
    uint32_t cnt = sort_unique(postings + off, sl->cnt);
    sl->cnt = cnt;
    if (cnt <= (uint32_t)kInlineIds) {
        uint32_t tmp[kInlineIds];
        for (uint32_t q = 0; q < (uint32_t)kInlineIds; q++) tmp[q] = q < cnt ? postings[off + q] : 0;
        for (int q = 0; q < kInlineIds; q++) sl->ids[q] = tmp[q];
    }
}

__global__ void k_index_finalize(IndexSlot *slots, uint64_t capacity, uint32_t *postings, IndexSlot *special) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < capacity && slots[i].cnt) finalize_slot(&slots[i], postings);
    if (i == 0 && special->cnt) finalize_slot(special, postings);
}

// ---- interning of spilled lists: blocks of one cached prefix carry the same endpoint set; pointing all of them at
// ONE copy of the list makes "same set" a comparison of (count, offset), which the match kernel's run detection uses.
__device__ __forceinline__ uint64_t list_hash(const uint32_t *list, uint32_t cnt) {
    uint64_t h = 0x9E3779B185EBCA87ULL ^ cnt;
    for (uint32_t k = 0; k < cnt; k++) {
        h ^= list[k];
        h *= 0xC2B2AE3D27D4EB4FULL;
        h ^= h >> 29;
    }
    return h == kEmptyKey ? 0 : h;
}

__global__ void k_intern_clear(uint64_t *ikeys, uint32_t *ivals, uint64_t capacity) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < capacity) { ikeys[i] = kEmptyKey; ivals[i] = 0xFFFFFFFFu; }
}

// keys_used (claim only): counts the keys this call claims, so that patches can bound the table's fill (index_store.cu)
__device__ __forceinline__ uint64_t intern_find_or_claim(uint64_t *ikeys, uint64_t mask, uint64_t key, bool claim,
                                                         uint32_t *keys_used = nullptr) {
    uint64_t i = key & mask;
    for (;;) {
        unsigned long long *kp = reinterpret_cast<unsigned long long *>(&ikeys[i]);
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(kp);
        if (cur == key) return i;
        if (cur == kEmptyKey) {
            if (!claim) return i;
            unsigned long long old = atomicCAS(kp, (unsigned long long)kEmptyKey, (unsigned long long)key);
            if (old == kEmptyKey) atomicAdd(keys_used, 1u);
            if (old == kEmptyKey || old == key) return i;
        }
        i = (i + 1) & mask;
    }
}

__global__ void k_intern_claim(const IndexSlot *slots, uint64_t capacity, const uint32_t *postings, uint64_t *ikeys,
                               uint32_t *ivals, uint32_t *cursor) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= capacity || slots[i].cnt <= (uint32_t)kInlineIds) return;
    uint32_t off = slots[i].ids[0];
    uint64_t j = intern_find_or_claim(ikeys, capacity - 1, list_hash(postings + off, slots[i].cnt), true, &cursor[3]);
    atomicMin(&ivals[j], (uint32_t)i);  // canonical copy = the list of the lowest slot among equal-hash lists
}

__global__ void k_intern_apply(IndexSlot *slots, uint64_t capacity, const uint32_t *postings, uint64_t *ikeys,
                               const uint32_t *ivals) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= capacity || slots[i].cnt <= (uint32_t)kInlineIds) return;
    uint32_t off = slots[i].ids[0], cnt = slots[i].cnt;
    uint64_t j = intern_find_or_claim(ikeys, capacity - 1, list_hash(postings + off, cnt), false);
    uint32_t cslot = ivals[j];
    if (cslot == (uint32_t)i || cslot == 0xFFFFFFFFu) return;     // the canonical slot itself is never rewritten
    // same list hash is only a hint: verify length and content (exactness)
    if (slots[cslot].cnt != cnt) return;
    uint32_t canon = slots[cslot].ids[0];
    for (uint32_t k = 0; k < cnt; k++)
        if (postings[canon + k] != postings[off + k]) return;
    slots[i].ids[0] = canon;
}

cudaError_t launch_index_build(const uint64_t *pair_hash, const uint32_t *pair_ep, uint64_t n, IndexSlot *slots,
                               uint64_t capacity, uint32_t *postings, uint32_t *scratch, uint32_t *cursor,
                               IndexSlot *special_dev, uint64_t *intern_keys, uint32_t *intern_vals,
                               cudaStream_t s, int *launches) {
    unsigned gc = (unsigned)((capacity + 255) / 256);
    if (gc == 0) gc = 1;
    k_index_clear<<<gc, 256, 0, s>>>(slots, scratch, capacity, cursor, special_dev);
    int nl = 1;
    if (n > 0) {
        unsigned gn = (unsigned)((n + 255) / 256);
        uint64_t mask = capacity - 1;
        k_index_insert<<<gn, 256, 0, s>>>(pair_hash, n, slots, mask, cursor, special_dev);
        k_index_alloc<<<gc, 256, 0, s>>>(slots, capacity, cursor, special_dev);
        k_index_fill<<<gn, 256, 0, s>>>(pair_hash, pair_ep, n, slots, mask, scratch, postings, cursor, special_dev);
        k_index_finalize<<<gc, 256, 0, s>>>(slots, capacity, postings, special_dev);
        k_intern_clear<<<gc, 256, 0, s>>>(intern_keys, intern_vals, capacity);
        k_intern_claim<<<gc, 256, 0, s>>>(slots, capacity, postings, intern_keys, intern_vals, cursor);
        k_intern_apply<<<gc, 256, 0, s>>>(slots, capacity, postings, intern_keys, intern_vals);
        nl += 7;
    }
    if (launches) *launches += nl;
    return cudaGetLastError();
}

// Presence bitmap of the table (index.cuh): cleared, then one bit per key that some endpoint holds.
__global__ void k_presence_build(const IndexSlot *slots, uint64_t capacity, uint32_t *bits, int shift) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= capacity) return;
    const uint64_t key = slots[i].key;
    if (key != kEmptyKey && slots[i].cnt) presence_set(bits, shift, key);
}

cudaError_t launch_presence_build(const IndexSlot *slots, uint64_t capacity, uint32_t *bits, int log2bits, cudaStream_t s,
                                  int *launches) {
    cudaError_t e = cudaMemsetAsync(bits, 0, ((size_t)1 << log2bits) / 8, s);
    if (e != cudaSuccess || !slots || !capacity) return e;
    k_presence_build<<<(unsigned)((capacity + 255) / 256), 256, 0, s>>>(slots, capacity, bits, 64 - log2bits);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

__global__ void k_index_get(IndexView ix, uint64_t hash, uint32_t *out_eps, int32_t cap, int32_t *out_n) {
    if (threadIdx.x || blockIdx.x) return;
    Hit h;
    probe(ix, hash, h);
    for (uint32_t k = 0; k < h.cnt && (int32_t)k < cap; k++) out_eps[k] = posting(ix, h, k);
    *out_n = (int32_t)h.cnt;
}

cudaError_t launch_index_get(const IndexView &ix, uint64_t hash, uint32_t *out_eps, int32_t cap, int32_t *out_n,
                             cudaStream_t s) {
    k_index_get<<<1, 32, 0, s>>>(ix, hash, out_eps, cap, out_n);
    return cudaGetLastError();
}

}  // namespace epp
