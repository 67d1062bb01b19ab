// index_store.cu -- kernels and host logic of the HBM-resident write side of the prefix index (see index_store.h).
#include "index.cuh"
#include "index_store.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <utility>

namespace epp {

namespace {

constexpr unsigned long long kLeakBit = 1ull << 63;   // log entry: evicting it leaves the pair in the inverted map
constexpr unsigned long long kTmpBit = 1ull << 62;    // scratch of k_store_leak
constexpr unsigned long long kSeqMask = ~(kLeakBit | kTmpBit);
constexpr int kCallChunk = 1024;                      // calls per ordering chunk (= threads of k_store_offsets)
enum { kCtrPtUsed = 0, kCtrTotalItems, kCtrNeedRepack, kCtrInMap, kCtrCursor, kCtrAlive, kCtrEvict, kCtrTouch,
       kCtrTouchLost, kCtrPatchFlag, kCtrPatchDirty, kCtrPatchClaims, kCtrPatchAdd, kCtrPatchDel, kCtrPatchIntern,
       kCtrPatchPost, kCtrN = 16 };

// One (hash, endpoint) pair of the write side: 32 bytes = one sector.
struct __align__(32) StoreEntry {
    unsigned long long hash;   // kEmptyKey = free slot
    unsigned long long seq;    // 0 = not in the endpoint's LRU, else sequence number of the latest Add of the pair
    uint32_t ep;               // kNoEp between the claim of `hash` and the publication of the endpoint
    uint32_t in_map;           // 1 = endpoint is in hashToPods[hash]
    unsigned long long pad;
};

}  // namespace

struct IndexStore::View {
    StoreEntry *pt;
    uint64_t pt_mask;
    unsigned long long *log_hash;
    unsigned long long *log_seq;
    uint32_t E;
    int32_t default_cap;
    uint32_t *cap, *live, *firstcall, *sp_in_map;
    unsigned long long *seg_off, *seg_cap, *head, *tail, *inc, *next_seq, *sp_seq, *cut;
    unsigned long long *ctr;
    // touch log: every (hash, endpoint) whose membership in the inverted map changed since the read table was last
    // brought up to date (consumed by patch_read_table)
    unsigned long long *touch_hash;
    uint32_t *touch_ep;
    unsigned long long touch_cap;
};

namespace {
using View = IndexStore::View;

struct EntryRef {
    unsigned long long *seq;
    uint32_t *in_map;
};

__device__ __forceinline__ uint64_t pt_home(uint64_t h, uint32_t e, uint64_t mask) {
    // XXH64 output is uniformly mixed; the endpoint term keeps the many endpoints of one hot hash off one probe chain
    return (h + (uint64_t)e * 0x9E3779B97F4A7C15ULL) & mask;
}

// Finds or creates the entry of (h, e).  Lock-free: a slot is claimed by CAS on its hash word; its endpoint word is
// then published by CAS as well, by the claimer or by any thread inserting the same hash (whoever wins owns the
// slot, the loser keeps probing) -- no thread ever waits for another.
__device__ __forceinline__ StoreEntry *pt_find_or_claim(const View &v, uint64_t h, uint32_t e, uint32_t &claimed) {
    uint64_t i = pt_home(h, e, v.pt_mask);
    for (;;) {
        StoreEntry *s = v.pt + i;
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(&s->hash);
        if (cur == kEmptyKey) {
            unsigned long long old = atomicCAS(&s->hash, (unsigned long long)kEmptyKey, (unsigned long long)h);
            if (old == kEmptyKey) {
                claimed++;                      // the caller adds its total to ctr[kCtrPtUsed] once
                cur = h;
            } else {
                cur = old;
            }
        }
        if (cur == h) {
            uint32_t ce = *reinterpret_cast<volatile uint32_t *>(&s->ep);
            if (ce == kNoEp) {
                uint32_t old = atomicCAS(&s->ep, kNoEp, e);
                ce = old == kNoEp ? e : old;
            }
            if (ce == e) return s;
        }
        i = (i + 1) & v.pt_mask;
    }
}

__device__ __forceinline__ StoreEntry *pt_find(const View &v, uint64_t h, uint32_t e) {
    uint64_t i = pt_home(h, e, v.pt_mask);
    for (;;) {
        StoreEntry *s = v.pt + i;
        unsigned long long cur = s->hash;
        if (cur == kEmptyKey) return nullptr;
        if (cur == h && s->ep == e) return s;
        i = (i + 1) & v.pt_mask;
    }
}

__device__ __forceinline__ EntryRef ref_claim(const View &v, uint64_t h, uint32_t e, uint32_t &claimed) {
    if (h == kEmptyKey) return {&v.sp_seq[e], &v.sp_in_map[e]};    // the one hash equal to the free-slot sentinel
    StoreEntry *s = pt_find_or_claim(v, h, e, claimed);
    return {&s->seq, &s->in_map};
}

__device__ __forceinline__ bool ref_find(const View &v, uint64_t h, uint32_t e, EntryRef &r) {
    if (h == kEmptyKey) {
        r = {&v.sp_seq[e], &v.sp_in_map[e]};
        return true;
    }
    StoreEntry *s = pt_find(v, h, e);
    if (!s) return false;
    r = {&s->seq, &s->in_map};
    return true;
}

// Appends this lane's (hash, endpoint) to the touch log; warp-aggregated, every lane of the warp must call it.
__device__ __forceinline__ void touch_append(const View &v, bool take, unsigned long long hsh, uint32_t ep) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, take);
    if (!ballot) return;
    unsigned long long base = 0;
    if (lane == (uint32_t)(__ffs(ballot) - 1)) base = atomicAdd(&v.ctr[kCtrTouch], (unsigned long long)__popc(ballot));
    base = __shfl_sync(0xFFFFFFFFu, base, __ffs(ballot) - 1);
    if (take) {
        const unsigned long long at = base + __popc(ballot & ((1u << lane) - 1u));
        if (at < v.touch_cap) {
            v.touch_hash[at] = hsh;
            v.touch_ep[at] = ep;
        } else {
            v.ctr[kCtrTouchLost] = 1;          // the log is incomplete: the next commit rebuilds the table instead
        }
    }
}

// ---- table / state initialisation ---------------------------------------------------------------------------------
__global__ void k_store_pt_clear(StoreEntry *pt, uint64_t capacity) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= capacity) return;
    StoreEntry z;
    z.hash = kEmptyKey;
    z.seq = 0;
    z.ep = kNoEp;
    z.in_map = 0;
    z.pad = 0;
    pt[i] = z;
}

__global__ void k_store_state_clear(View v) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < v.E) {
        v.cap[e] = 0;
        v.live[e] = 0;
        v.firstcall[e] = kNoEp;
        v.sp_in_map[e] = 0;
        v.seg_off[e] = 0;
        v.seg_cap[e] = 0;
        v.head[e] = 0;
        v.tail[e] = 0;
        v.inc[e] = 0;
        v.next_seq[e] = 1;
        v.sp_seq[e] = 0;
        v.cut[e] = 0;
    }
    if (e < kCtrN) v.ctr[e] = 0;
}

// ---- picks -> calls (plugin.go:164-200) -------------------------------------------------------------------------------
__global__ void k_store_calls_from_picks(const epp_decision *dec, const int32_t *nblocks, int64_t R, int32_t max_blocks,
                                         uint32_t E, uint32_t *call_ep, uint32_t *call_n, int32_t *call_nb,
                                         unsigned long long *call_src) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    epp_decision d = dec[r];
    const bool ok = d.status == 0 && d.pick != EPP_NO_ENDPOINT && d.pick < E;      // plugin.go:168-170
    const uint32_t n = ok ? (uint32_t)max(0, nblocks[r]) : 0u;
    call_ep[2 * r] = ok ? d.pick : kNoEp;
    call_n[2 * r] = n;
    call_nb[2 * r] = 0;
    call_src[2 * r] = (unsigned long long)r * (unsigned long long)max_blocks;
    const bool pf = ok && d.prefill_pick != EPP_NO_ENDPOINT && d.prefill_pick < E;   // plugin.go:176-178
    call_ep[2 * r + 1] = pf ? d.prefill_pick : kNoEp;
    call_n[2 * r + 1] = pf ? n : 0u;
    call_nb[2 * r + 1] = 0;
    call_src[2 * r + 1] = (unsigned long long)r * (unsigned long long)max_blocks;
}

// ---- sequencing: where in its endpoint's Add order does each call start? ---------------------------------------------
__global__ void k_store_batch_clear(View v, uint32_t *hist, uint64_t hist_n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < hist_n) hist[i] = 0;
    if (i < v.E) v.firstcall[i] = kNoEp;
    if (i == 0) {
        v.ctr[kCtrTotalItems] = 0;
        v.ctr[kCtrNeedRepack] = 0;
    }
}

__global__ void k_store_hist(View v, uint32_t M, const uint32_t *call_ep, const uint32_t *call_n, uint32_t *hist) {
    uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= M) return;
    uint32_t e = call_ep[c];
    if (e >= v.E) return;
    if (call_n[c]) atomicAdd(&hist[(uint64_t)(c / kCallChunk) * v.E + e], call_n[c]);
    atomicMin(&v.firstcall[e], c);
}

// Per endpoint: exclusive scan of its per-chunk item counts (hist becomes the chunk's starting offset), creation of
// the LRU by the endpoint's first call of the batch (indexer.go:57-69), room check of the log segment.
__global__ void k_store_plan(View v, uint32_t n_chunks, uint32_t *hist, const int32_t *call_nb) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v.E) return;
    unsigned long long run = 0;
    for (uint32_t ch = 0; ch < n_chunks; ch++) {
        uint32_t t = hist[(uint64_t)ch * v.E + e];
        hist[(uint64_t)ch * v.E + e] = (uint32_t)run;
        run += t;
    }
    v.inc[e] = run;
    uint32_t fc = v.firstcall[e];
    if (fc != kNoEp && v.cap[e] == 0) {
        int32_t nb = call_nb[fc];
        int32_t c = nb > 0 ? nb : v.default_cap;
        v.cap[e] = c > 0 ? (uint32_t)c : 1u;
    }
    if (run) atomicAdd(&v.ctr[kCtrTotalItems], run);
}

__global__ void __launch_bounds__(kCallChunk) k_store_offsets(View v, uint32_t M, const uint32_t *call_ep,
                                                               const uint32_t *call_n, const uint32_t *hist,
                                                               unsigned long long *call_off) {
    __shared__ uint32_t s_ep[kCallChunk];
    __shared__ uint32_t s_n[kCallChunk];
    const uint32_t t = threadIdx.x, c = blockIdx.x * kCallChunk + t;
    const uint32_t e = c < M ? call_ep[c] : kNoEp;
    s_ep[t] = e;
    s_n[t] = c < M ? call_n[c] : 0u;
    __syncthreads();
    if (e >= v.E) return;
    unsigned long long before = 0;
    for (uint32_t u = 0; u < t; u++) before += s_ep[u] == e ? s_n[u] : 0u;
    call_off[c] = hist[(uint64_t)blockIdx.x * v.E + e] + before;
}

// ---- Add: append to the endpoint's log, upsert the pair table (first loop + second loop of indexer.Add) ---------------
__global__ void k_store_upsert(View v, uint32_t M, const uint32_t *call_ep, const uint32_t *call_n,
                               const unsigned long long *call_src, const unsigned long long *call_off,
                               const unsigned long long *hashes) {
    const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
    uint32_t in_map_new = 0, claimed = 0;
    for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < M; c += warps) {
        const uint32_t e = call_ep[c], n = call_n[c];
        if (e >= v.E || n == 0) continue;
        uint32_t live_new = 0;
        const unsigned long long off = call_off[c];
        const unsigned long long seq0 = v.next_seq[e] + off;
        const unsigned long long pos0 = v.seg_off[e] + v.head[e] + off;
        const unsigned long long *src = hashes + call_src[c];
        for (uint32_t i0 = 0; i0 < n; i0 += 32) {
            const uint32_t i = i0 + lane;
            bool added = false;
            unsigned long long hsh = 0;
            if (i < n) {
                hsh = src[i];
                const unsigned long long seq = seq0 + i;
                v.log_hash[pos0 + i] = hsh;
                v.log_seq[pos0 + i] = seq;
                EntryRef r = ref_claim(v, hsh, e, claimed);
                if (atomicMax(r.seq, seq) == 0) live_new++;                  // lru.Add of an absent key
                added = *reinterpret_cast<volatile uint32_t *>(r.in_map) == 0 && atomicExch(r.in_map, 1u) == 0;
                if (added) in_map_new++;
            }
            touch_append(v, added, hsh, e);
        }
        for (int o = 16; o; o >>= 1) live_new += __shfl_xor_sync(0xFFFFFFFFu, live_new, o);
        if (lane == 0 && live_new) atomicAdd(&v.live[e], live_new);
    }
    for (int o = 16; o; o >>= 1) {
        in_map_new += __shfl_xor_sync(0xFFFFFFFFu, in_map_new, o);
        claimed += __shfl_xor_sync(0xFFFFFFFFu, claimed, o);
    }
    if (lane == 0 && in_map_new) atomicAdd(&v.ctr[kCtrInMap], (unsigned long long)in_map_new);
    if (lane == 0 && claimed) atomicAdd(&v.ctr[kCtrPtUsed], (unsigned long long)claimed);
}

// Calls longer than their endpoint's LRU: hash i of the call is evicted BY THE SAME CALL iff at least `cap` distinct
// hashes follow its last occurrence; indexer.go:76-83 then re-inserts it into the inverted map only (leak bit).
__global__ void k_store_leak(View v, uint32_t M, const uint32_t *call_ep, const uint32_t *call_n,
                             const unsigned long long *call_off) {
    for (uint32_t c = blockIdx.x; c < M; c += gridDim.x) {
        const uint32_t e = call_ep[c], n = call_n[c];
        if (e >= v.E || n <= v.cap[e]) continue;                    // uniform across the CTA
        const uint32_t cap = v.cap[e];
        const unsigned long long pos0 = v.seg_off[e] + v.head[e] + call_off[c];
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long hsh = v.log_hash[pos0 + i];
            bool last = true;
            for (uint32_t j = i + 1; j < n && last; j++) last = v.log_hash[pos0 + j] != hsh;
            if (last) v.log_seq[pos0 + i] |= kTmpBit;
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
            if (!(v.log_seq[pos0 + i] & kTmpBit)) continue;
            uint32_t after = 0;
            for (uint32_t j = i + 1; j < n && after < cap; j++) after += (v.log_seq[pos0 + j] & kTmpBit) ? 1u : 0u;
            if (after >= cap) v.log_seq[pos0 + i] |= kLeakBit;
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) v.log_seq[pos0 + i] &= ~kTmpBit;
        __syncthreads();
    }
}

// ---- eviction: per endpoint, drop the oldest live log entries until live <= cap (lru.Add overflow + callback) ----------
// A skewed batch can append millions of entries to ONE endpoint, so the walk from the tail is spread over CTAs:
//   k_evict_count  live entries per 256-entry block of every over-full endpoint's log window
//   k_evict_cut    per endpoint: the position right after the k-th oldest live entry (k = live - cap)
//   k_evict_apply  every live entry before the cut leaves the LRU (and the inverted map, unless it leaked)
//   k_evict_finish tail / live bookkeeping
constexpr int kEvictBlock = 256;

__device__ __forceinline__ bool log_entry_live(const View &v, uint32_t e, unsigned long long at, EntryRef &r, bool &leak) {
    const unsigned long long hsh = v.log_hash[at], sq = v.log_seq[at];
    leak = (sq & kLeakBit) != 0;
    return ref_find(v, hsh, e, r) && *r.seq == (sq & kSeqMask) && *r.seq != 0;
}

// Folds the batch into the endpoint's counters (head, next_seq) and lists the over-full endpoints with the range of
// 256-entry log blocks each contributes to ONE flat block index space (so a single endpoint that received millions of
// entries is spread over the whole grid).  One packed atomic orders (list position, first block) together.
constexpr int kEvictPackShift = 40;
__global__ void k_store_advance(View v, uint32_t *list_e, unsigned long long *list_start) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v.E) return;
    const unsigned long long inc = v.inc[e];
    if (inc) {
        v.head[e] += inc;
        v.next_seq[e] += inc;
        v.inc[e] = 0;
    }
    const unsigned long long tail = v.tail[e], head = v.head[e];
    v.cut[e] = tail;
    const uint32_t cap = v.cap[e];
    if (cap == 0 || v.live[e] <= cap) return;
    const unsigned long long nb = (head + kEvictBlock - 1) / kEvictBlock - tail / kEvictBlock;
    const unsigned long long old = atomicAdd(&v.ctr[kCtrEvict], (1ull << kEvictPackShift) | nb);
    list_e[old >> kEvictPackShift] = e;
    list_start[old >> kEvictPackShift] = old & ((1ull << kEvictPackShift) - 1);
}

// Flat block g -> (endpoint, block of its log).  list_start is increasing; n > 0.
__device__ __forceinline__ void evict_locate(const View &v, const uint32_t *list_e, const unsigned long long *list_start,
                                             uint32_t n, unsigned long long g, uint32_t &e, unsigned long long &b) {
    uint32_t lo = 0, hi = n;                      // last j with list_start[j] <= g
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (list_start[mid] <= g) lo = mid; else hi = mid;
    }
    e = list_e[lo];
    b = v.tail[e] / kEvictBlock + (g - list_start[lo]);
}

__global__ void __launch_bounds__(kEvictBlock) k_evict_count(View v, const uint32_t *list_e,
                                                              const unsigned long long *list_start, uint32_t *blockcnt) {
    const unsigned long long packed = v.ctr[kCtrEvict];
    const uint32_t n = (uint32_t)(packed >> kEvictPackShift);
    const unsigned long long total = packed & ((1ull << kEvictPackShift) - 1);
    for (unsigned long long g = blockIdx.x; g < total; g += gridDim.x) {
        uint32_t e;
        unsigned long long b;
        evict_locate(v, list_e, list_start, n, g, e, b);
        const unsigned long long seg = v.seg_off[e], tail = v.tail[e], head = v.head[e];
        const unsigned long long idx = b * kEvictBlock + threadIdx.x;
        bool is_live = false, leak;
        EntryRef r;
        if (idx >= tail && idx < head) is_live = log_entry_live(v, e, seg + idx, r, leak);
        const int cnt = __syncthreads_count(is_live);
        if (threadIdx.x == 0) blockcnt[seg / kEvictBlock + b] = (uint32_t)cnt;
    }
}

__global__ void k_evict_cut(View v, const uint32_t *blockcnt) {
    const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < v.E; e += warps) {
        const uint32_t cap = v.cap[e], live = v.live[e];
        if (cap == 0 || live <= cap) continue;
        unsigned long long k = live - cap;
        const unsigned long long seg = v.seg_off[e], tail = v.tail[e], head = v.head[e];
        const unsigned long long b0 = tail / kEvictBlock, b1 = (head + kEvictBlock - 1) / kEvictBlock;
        // 1. the block holding the k-th oldest live entry (each lane sums kPer consecutive block counts per step)
        constexpr int kPer = 8;
        const uint32_t *bc = blockcnt + seg / kEvictBlock;
        unsigned long long b = b0;
        bool found = false;
        while (b < b1 && !found) {
            const unsigned long long mine = b + (unsigned long long)lane * kPer;
            uint32_t c[kPer], sum = 0;
#pragma unroll
            for (int q = 0; q < kPer; q++) {
                c[q] = mine + q < b1 ? bc[mine + q] : 0u;
                sum += c[q];
            }
            uint32_t incl = sum;
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                if (lane >= (uint32_t)o) incl += t;
            }
            const uint32_t hit = __ballot_sync(0xFFFFFFFFu, incl >= k);
            if (hit) {
                const int l = __ffs(hit) - 1;
                // inside lane l's strip
                unsigned long long before = incl - sum, bb = mine;
                if ((int)lane == l) {
#pragma unroll
                    for (int q = 0; q < kPer; q++) {
                        if (before + c[q] >= k) break;
                        before += c[q];
                        bb++;
                    }
                }
                before = __shfl_sync(0xFFFFFFFFu, before, l);
                bb = __shfl_sync(0xFFFFFFFFu, bb, l);
                k -= before;
                b = bb;
                found = true;
            } else {
                k -= __shfl_sync(0xFFFFFFFFu, incl, 31);
                b += 32 * kPer;
            }
        }
        unsigned long long pos = head;
        if (found) {
            // 2. inside that block: right after its k-th live entry
            pos = b * kEvictBlock;
            for (int w = 0; w < kEvictBlock / 32 && k > 0; w++) {
                const unsigned long long idx = pos + lane;
                bool is_live = false, leak;
                EntryRef r;
                if (idx >= tail && idx < head) is_live = log_entry_live(v, e, seg + idx, r, leak);
                const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, is_live);
                const uint32_t n_live = __popc(ballot);
                if (n_live >= k) {
                    uint32_t bb = ballot;
                    for (uint32_t q = 1; q < k; q++) bb &= bb - 1;
                    pos += (uint32_t)__ffs(bb);
                    k = 0;
                } else {
                    k -= n_live;
                    pos += 32;
                }
            }
        }
        if (lane == 0) v.cut[e] = pos < head ? pos : head;
    }
}

__global__ void __launch_bounds__(kEvictBlock) k_evict_apply(View v, const uint32_t *list_e,
                                                              const unsigned long long *list_start) {
    const unsigned long long packed = v.ctr[kCtrEvict];
    const uint32_t n = (uint32_t)(packed >> kEvictPackShift);
    const unsigned long long total = packed & ((1ull << kEvictPackShift) - 1);
    unsigned long long removed = 0;
    for (unsigned long long g = blockIdx.x; g < total; g += gridDim.x) {
        uint32_t e;
        unsigned long long b;
        evict_locate(v, list_e, list_start, n, g, e, b);
        const unsigned long long idx = b * kEvictBlock + threadIdx.x;
        bool gone = false;
        unsigned long long hsh = 0;
        if (idx >= v.tail[e] && idx < v.cut[e]) {
            bool leak;
            EntryRef r;
            hsh = v.log_hash[v.seg_off[e] + idx];
            if (log_entry_live(v, e, v.seg_off[e] + idx, r, leak)) {
                *r.seq = 0;                              // out of the LRU ...
                if (!leak) {                             // ... and, through the eviction callback, out of the map
                    *r.in_map = 0;
                    removed++;
                    gone = true;
                }
            }
        }
        touch_append(v, gone, hsh, e);
    }
    for (int o = 16; o; o >>= 1) removed += __shfl_xor_sync(0xFFFFFFFFu, removed, o);
    if ((threadIdx.x & 31) == 0 && removed) atomicAdd(&v.ctr[kCtrInMap], (unsigned long long)(0ull - removed));
}

__global__ void k_evict_finish(View v) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v.E) return;
    if (v.cut[e] > v.tail[e]) {
        v.tail[e] = v.cut[e];
        v.live[e] = v.cap[e];
    }
}

// Log compaction for endpoints whose segment cannot take the batch's entries (head + inc > cap): the LIVE entries of
// [tail, head) move, in order, to the front of the segment.  The logs are append-only (a re-Add of a cached pair appends
// a new entry and kills the old one), and one skewed batch can hand millions of entries to ONE endpoint, so the walk is a
// flat space of 256-entry blocks spread over the whole grid, like the eviction (k_evict_*): list the endpoints and their
// block ranges -> per block: liveness mask + count -> per endpoint: exclusive scan of the counts -> per block: scatter
// into the spare log buffers -> copy the compacted prefix back -> new head / tail.  If the segment is still too small
// the whole log space is re-allocated afterwards (k_store_repack).
__device__ __forceinline__ bool needs_compaction(const View &v, uint32_t e) {
    const unsigned long long inc = v.inc[e];
    return inc != 0 && v.head[e] + inc > v.seg_cap[e];
}
__global__ void k_compact_list(View v, uint32_t *list_e, unsigned long long *list_start) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v.E || !needs_compaction(v, e)) return;
    const unsigned long long tail = v.tail[e], head = v.head[e];
    const unsigned long long nb = (head + kEvictBlock - 1) / kEvictBlock - tail / kEvictBlock;
    const unsigned long long old = atomicAdd(&v.ctr[kCtrEvict], (1ull << kEvictPackShift) | nb);
    list_e[old >> kEvictPackShift] = e;
    list_start[old >> kEvictPackShift] = old & ((1ull << kEvictPackShift) - 1);
}
// blockcnt[b] = live entries of block b, blockmask[8 b + w] = liveness of its entries 32 w .. 32 w + 31.
__global__ void __launch_bounds__(kEvictBlock) k_compact_count(View v, const uint32_t *list_e, const unsigned long long *list_start,
                                                                uint32_t *blockcnt, uint32_t *blockmask) {
    const unsigned long long packed = v.ctr[kCtrEvict];
    const uint32_t n = (uint32_t)(packed >> kEvictPackShift);
    const unsigned long long total = packed & ((1ull << kEvictPackShift) - 1);
    for (unsigned long long g = blockIdx.x; g < total; g += gridDim.x) {
        uint32_t e;
        unsigned long long b;
        evict_locate(v, list_e, list_start, n, g, e, b);
        const unsigned long long seg = v.seg_off[e], tail = v.tail[e], head = v.head[e];
        const unsigned long long idx = b * kEvictBlock + threadIdx.x;
        bool is_live = false, leak;
        EntryRef r;
        if (idx >= tail && idx < head) is_live = log_entry_live(v, e, seg + idx, r, leak);
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, is_live);
        if ((threadIdx.x & 31) == 0) blockmask[(seg / kEvictBlock + b) * (kEvictBlock / 32) + (threadIdx.x >> 5)] = m;
        const int cnt = __syncthreads_count(is_live);
        if (threadIdx.x == 0) blockcnt[seg / kEvictBlock + b] = (uint32_t)cnt;
    }
}
// Per compacted endpoint: blockcnt -> exclusive prefix (position of the block's first live entry in the compacted log);
// new_head[e] = number of live entries.
__global__ void k_compact_scan(View v, uint32_t *blockcnt, unsigned long long *new_head) {
    const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < v.E; e += warps) {
        if (!needs_compaction(v, e)) continue;
        const unsigned long long seg = v.seg_off[e], tail = v.tail[e], head = v.head[e];
        const unsigned long long b0 = tail / kEvictBlock, b1 = (head + kEvictBlock - 1) / kEvictBlock;
        uint32_t *bc = blockcnt + seg / kEvictBlock;
        unsigned long long run = 0;
        for (unsigned long long b = b0; b < b1; b += 32) {
            const uint32_t c = b + lane < b1 ? bc[b + lane] : 0u;
            uint32_t incl = c;
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                if ((int)lane >= o) incl += t;
            }
            if (b + lane < b1) bc[b + lane] = (uint32_t)(run + incl - c);      // fits: a segment holds < 2^32 entries
            run += __shfl_sync(0xFFFFFFFFu, incl, 31);
        }
        if (lane == 0) new_head[e] = run;
    }
}
__global__ void __launch_bounds__(kEvictBlock) k_compact_scatter(View v, const uint32_t *list_e, const unsigned long long *list_start,
                                                                  const uint32_t *blockoff, const uint32_t *blockmask,
                                                                  unsigned long long *spare_hash, unsigned long long *spare_seq) {
    const unsigned long long packed = v.ctr[kCtrEvict];
    const uint32_t n = (uint32_t)(packed >> kEvictPackShift);
    const unsigned long long total = packed & ((1ull << kEvictPackShift) - 1);
    const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (unsigned long long g = blockIdx.x; g < total; g += gridDim.x) {
        uint32_t e;
        unsigned long long b;
        evict_locate(v, list_e, list_start, n, g, e, b);
        const unsigned long long seg = v.seg_off[e];
        const uint32_t *bm = blockmask + (seg / kEvictBlock + b) * (kEvictBlock / 32);
        const uint32_t mine = bm[w];
        if (!((mine >> lane) & 1u)) continue;
        uint32_t rank = __popc(mine & ((1u << lane) - 1u));
        for (uint32_t k = 0; k < w; k++) rank += __popc(bm[k]);
        const unsigned long long src = seg + b * kEvictBlock + threadIdx.x, dst = seg + blockoff[seg / kEvictBlock + b] + rank;
        spare_hash[dst] = v.log_hash[src];
        spare_seq[dst] = v.log_seq[src];
    }
}
// The compacted prefix [0, new_head) back into the log (the flat block space of the OLD range covers it).
__global__ void __launch_bounds__(kEvictBlock) k_compact_copyback(View v, const uint32_t *list_e, const unsigned long long *list_start,
                                                                   const unsigned long long *new_head,
                                                                   const unsigned long long *spare_hash, const unsigned long long *spare_seq) {
    const unsigned long long packed = v.ctr[kCtrEvict];
    const uint32_t n = (uint32_t)(packed >> kEvictPackShift);
    const unsigned long long total = packed & ((1ull << kEvictPackShift) - 1);
    for (unsigned long long g = blockIdx.x; g < total; g += gridDim.x) {
        uint32_t e;
        unsigned long long b;
        evict_locate(v, list_e, list_start, n, g, e, b);
        const unsigned long long idx = (b - v.tail[e] / kEvictBlock) * kEvictBlock + threadIdx.x;
        if (idx >= new_head[e]) continue;
        const unsigned long long at = v.seg_off[e] + idx;
        v.log_hash[at] = spare_hash[at];
        v.log_seq[at] = spare_seq[at];
    }
}
__global__ void k_compact_finish(View v, const unsigned long long *new_head) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v.E || !needs_compaction(v, e)) return;
    const unsigned long long w = new_head[e];
    const bool still_short = w + v.inc[e] > v.seg_cap[e];
    v.head[e] = w;
    v.tail[e] = 0;
    if (still_short) atomicOr(&v.ctr[kCtrNeedRepack], 1ull);
}

// RemovePod (indexer.go:167-182): every key of the endpoint's LRU goes through the eviction callback, the LRU is
// deleted (the next Add of the endpoint creates a new one, possibly with another size).
__device__ __forceinline__ void remove_endpoint_warp(const View &v, uint32_t e, uint32_t lane) {
    const unsigned long long head = v.head[e], seg = v.seg_off[e];
    unsigned long long removed = 0;
    for (unsigned long long pos = v.tail[e]; pos < head; pos += 32) {
        const unsigned long long idx = pos + lane;
        bool gone = false;
        unsigned long long hsh = 0;
        if (idx < head) {
            EntryRef r;
            bool leak;
            hsh = v.log_hash[seg + idx];
            if (log_entry_live(v, e, seg + idx, r, leak)) {
                *r.seq = 0;
                *r.in_map = 0;
                removed++;
                gone = true;
            }
        }
        touch_append(v, gone, hsh, e);
    }
    for (int o = 16; o; o >>= 1) removed += __shfl_xor_sync(0xFFFFFFFFu, removed, o);
    __syncwarp();
    if (lane == 0) {
        v.head[e] = 0;
        v.tail[e] = 0;
        v.live[e] = 0;
        v.cap[e] = 0;
        if (removed) atomicAdd(&v.ctr[kCtrInMap], (unsigned long long)(0ull - removed));
    }
}

__global__ void k_store_remove_endpoint(View v, uint32_t e) { remove_endpoint_warp(v, e, threadIdx.x & 31); }

// CleanUpInactivePods (plugin.go:99-122): RemovePod for every endpoint that has an LRU and is not in the active set.
__global__ void k_store_retain(View v, const uint8_t *active) {
    const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < v.E; e += warps)
        if (v.cap[e] != 0 && !active[e]) remove_endpoint_warp(v, e, lane);
}

// ---- housekeeping: log compaction into fresh segments, pair-table rehash ------------------------------------------------
__global__ void k_store_repack(View v, const unsigned long long *new_off, const unsigned long long *new_cap,
                               unsigned long long *new_hash, unsigned long long *new_seq) {
    const uint32_t lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < v.E; e += warps) {
        const unsigned long long head = v.head[e], seg = v.seg_off[e], dst = new_off[e];
        unsigned long long w = 0;
        for (unsigned long long pos = v.tail[e]; pos < head; pos += 32) {
            const unsigned long long idx = pos + lane;
            bool is_live = false;
            unsigned long long hsh = 0, sq = 0;
            if (idx < head) {
                hsh = v.log_hash[seg + idx];
                sq = v.log_seq[seg + idx];
                EntryRef r;
                if (ref_find(v, hsh, e, r)) is_live = *r.seq == (sq & kSeqMask) && *r.seq != 0;
            }
            const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, is_live);
            if (is_live) {
                const unsigned long long at = dst + w + __popc(ballot & ((1u << lane) - 1u));
                new_hash[at] = hsh;
                new_seq[at] = sq;
            }
            w += __popc(ballot);
        }
        __syncwarp();
        if (lane == 0) {
            v.seg_off[e] = dst;
            v.seg_cap[e] = new_cap[e];
            v.head[e] = w;
            v.tail[e] = 0;
        }
    }
}

__global__ void k_store_count_alive(const StoreEntry *pt, uint64_t capacity, unsigned long long *ctr) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool alive = i < capacity && pt[i].hash != kEmptyKey && (pt[i].seq != 0 || pt[i].in_map != 0);
    uint32_t b = __ballot_sync(0xFFFFFFFFu, alive);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(&ctr[kCtrAlive], (unsigned long long)__popc(b));
}

__global__ void k_store_rehash(const StoreEntry *old_pt, uint64_t old_capacity, View v) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= old_capacity) return;
    StoreEntry o = old_pt[i];
    if (o.hash == kEmptyKey || (o.seq == 0 && o.in_map == 0)) return;       // free slot or tombstone
    uint32_t claimed = 0;
    StoreEntry *s = pt_find_or_claim(v, o.hash, o.ep, claimed);
    s->seq = o.seq;
    s->in_map = o.in_map;
    if (claimed) atomicAdd(&v.ctr[kCtrPtUsed], (unsigned long long)claimed);
}

// Scan of the pair table: kExportPer slots per thread, all loads issued before any is used (the scan is pure
// streaming: loads in flight set its rate).
constexpr int kExportPer = 4;
__global__ void k_store_export(View v, uint64_t capacity, unsigned long long *out_hash, uint32_t *out_ep) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t base = (uint64_t)blockIdx.x * (blockDim.x * kExportPer) + threadIdx.x;
    ulonglong2 lo[kExportPer];
    uint2 mid[kExportPer];
#pragma unroll
    for (int k = 0; k < kExportPer; k++) {
        const uint64_t i = base + (uint64_t)k * blockDim.x;
        lo[k] = make_ulonglong2(kEmptyKey, 0);
        mid[k] = make_uint2(0, 0);
        if (i < capacity) {
            const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(v.pt + i);      // {hash, seq}
            lo[k] = __ldcs(p);
            mid[k] = __ldcs(reinterpret_cast<const uint2 *>(p + 1));                    // {ep, in_map}
        }
    }
#pragma unroll
    for (int k = 0; k < kExportPer; k++) {
        const uint64_t i = base + (uint64_t)k * blockDim.x;
        bool take = false;
        unsigned long long hsh = lo[k].x;
        uint32_t ep = mid[k].x;
        if (i < capacity) {
            take = hsh != kEmptyKey && mid[k].y != 0;
        } else if (i - capacity < v.E) {                                     // tail threads: the sentinel-hash records
            ep = (uint32_t)(i - capacity);
            take = v.sp_in_map[ep] != 0;
            hsh = kEmptyKey;
        }
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, take);
        if (!ballot) continue;
        unsigned long long at0 = 0;
        if (lane == 0) at0 = atomicAdd(&v.ctr[kCtrCursor], (unsigned long long)__popc(ballot));
        at0 = __shfl_sync(0xFFFFFFFFu, at0, 0);
        if (take) {
            const unsigned long long at = at0 + __popc(ballot & ((1u << lane) - 1u));
            out_hash[at] = hsh;
            out_ep[at] = ep;
        }
    }
}

// ---- incremental maintenance of the READ table (index_kernels.cu layout) from the touch log ---------------------------
// The log names every (hash, endpoint) whose membership changed; the pair table holds the FINAL membership, so applying
// the log is idempotent and order-free:  for every touched hash, new list = (old list U touched endpoints that are
// in the map) \ (touched endpoints that are not).  Lists never change in place when spilled: the new list is written to
// fresh posting space (other slots may share the old one through interning), the old space becomes garbage until the
// next bulk build.  A hash whose last endpoint leaves keeps its slot with cnt = 0 (a tombstone: probes continue past
// it, and finding it means "nobody holds the block").
constexpr uint32_t kNil = 0xFFFFFFFFu;
constexpr int kPatchLocal = 16;

struct PatchView {
    IndexSlot *slots;
    uint64_t mask;
    uint32_t *postings;
    unsigned long long post_cap;
    unsigned long long *post_cursor;   // posting entries used (64-bit: failed allocations must not wrap)
    uint32_t *head;              // [capacity] pending-list head per slot (kNil when idle)
    uint32_t *next;              // [n_touch]
    uint32_t *dirty;             // [n_touch] slots with pending entries
    uint64_t *intern_keys;       // interning table of the last bulk build (capacity entries)
    uint32_t *intern_vals;
    unsigned long long *intern_claims;   // keys this patch claimed in it
    uint32_t *presence;          // presence bitmap of the read table; a key that loses its last endpoint keeps its bit
    int32_t presence_shift;
};

__device__ __forceinline__ uint64_t rt_find_or_claim(const PatchView &pv, uint64_t key, uint32_t &claimed) {
    uint64_t i = key & pv.mask;
    for (;;) {
        unsigned long long *kp = reinterpret_cast<unsigned long long *>(&pv.slots[i].key);
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(kp);
        if (cur == key) return i;
        if (cur == kEmptyKey) {
            unsigned long long old = atomicCAS(kp, (unsigned long long)kEmptyKey, (unsigned long long)key);
            if (old == kEmptyKey) { claimed++; return i; }
            if (old == key) return i;
        }
        i = (i + 1) & pv.mask;
    }
}

// Same list hash as index_kernels.cu (interning).
__device__ __forceinline__ uint64_t patch_list_hash(const uint32_t *list, uint32_t cnt) {
    uint64_t h = 0x9E3779B185EBCA87ULL ^ cnt;
    for (uint32_t k = 0; k < cnt; k++) {
        h ^= list[k];
        h *= 0xC2B2AE3D27D4EB4FULL;
        h ^= h >> 29;
    }
    return h == kEmptyKey ? 0 : h;
}

__global__ void k_patch_group(View v, PatchView pv, unsigned long long n_touch) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_touch) return;
    const unsigned long long hsh = v.touch_hash[t];
    if (hsh == kEmptyKey) {                       // the sentinel hash lives in the side record: bulk build handles it
        v.ctr[kCtrPatchFlag] = 1;
        return;
    }
    uint32_t claimed = 0;
    const uint64_t slot = rt_find_or_claim(pv, hsh, claimed);
    if (claimed) atomicAdd(&v.ctr[kCtrPatchClaims], 1ull);
    const uint32_t old = atomicExch(&pv.head[slot], (uint32_t)t);
    pv.next[t] = old;
    if (old == kNil) pv.dirty[atomicAdd(&v.ctr[kCtrPatchDirty], 1ull)] = (uint32_t)slot;
}

// Sorted-list helpers on a small array / a posting range.
__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t *a, uint32_t n, uint32_t x) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t list_apply(uint32_t *a, uint32_t n, uint32_t ep, bool member) {
    const uint32_t p = lower_bound_u32(a, n, ep);
    const bool present = p < n && a[p] == ep;
    if (member && !present) {
        for (uint32_t k = n; k > p; k--) a[k] = a[k - 1];
        a[p] = ep;
        return n + 1;
    }
    if (!member && present) {
        for (uint32_t k = p; k + 1 < n; k++) a[k] = a[k + 1];
        return n - 1;
    }
    return n;
}

__global__ void k_patch_apply(View v, PatchView pv, unsigned long long n_dirty) {
    const unsigned long long d = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_dirty) return;
    const uint32_t si = pv.dirty[d];
    IndexSlot *sl = &pv.slots[si];
    const uint64_t hsh = sl->key;
    const uint32_t cnt = sl->cnt;
    uint32_t k = 0;
    for (uint32_t t = pv.head[si]; t != kNil; t = pv.next[t]) k++;
    const bool was_spilled = cnt > (uint32_t)kInlineIds;
    const uint32_t old_off = sl->ids[0];
    uint32_t n_new;
    if (!was_spilled && cnt + k <= (uint32_t)kPatchLocal) {
        // ---- short list: registers / local memory, no posting space unless it outgrows the slot
        uint32_t a[kPatchLocal];
        for (uint32_t q = 0; q < cnt; q++) a[q] = sl->ids[q];
        n_new = cnt;
        for (uint32_t t = pv.head[si]; t != kNil; t = pv.next[t]) {
            const uint32_t ep = v.touch_ep[t];
            const StoreEntry *pe = pt_find(v, hsh, ep);
            n_new = list_apply(a, n_new, ep, pe && pe->in_map != 0);
        }
        if (n_new <= (uint32_t)kInlineIds) {
            for (uint32_t q = 0; q < (uint32_t)kInlineIds; q++) sl->ids[q] = q < n_new ? a[q] : 0u;
        } else {
            const unsigned long long off = atomicAdd(pv.post_cursor, (unsigned long long)n_new);
            if (off + n_new > pv.post_cap) { v.ctr[kCtrPatchFlag] = 1; pv.head[si] = kNil; return; }
            for (uint32_t q = 0; q < n_new; q++) pv.postings[off + q] = a[q];
            sl->ids[0] = (uint32_t)off;
            for (uint32_t q = 1; q < (uint32_t)kInlineIds; q++) sl->ids[q] = 0u;
        }
    } else {
        // ---- long list: copy-on-write into fresh posting space sized for the worst case
        const unsigned long long need = (unsigned long long)cnt + k;
        const unsigned long long off = atomicAdd(pv.post_cursor, need);
        if (off + need > pv.post_cap) { v.ctr[kCtrPatchFlag] = 1; pv.head[si] = kNil; return; }
        uint32_t *a = pv.postings + off;
        if (was_spilled) {
            // if this slot is the interning canonical of its old list, retire it so that a later equal list can register
            const uint64_t j0 = patch_list_hash(pv.postings + old_off, cnt) & pv.mask;
            for (uint64_t j = j0;; j = (j + 1) & pv.mask) {
                const uint64_t key = pv.intern_keys[j];
                if (key == kEmptyKey) break;
                if (pv.intern_vals[j] == si) { pv.intern_vals[j] = kNil; break; }
                if (((j + 1) & pv.mask) == j0) break;
            }
            for (uint32_t q = 0; q < cnt; q++) a[q] = pv.postings[old_off + q];
        } else {
            for (uint32_t q = 0; q < cnt; q++) a[q] = sl->ids[q];
        }
        n_new = cnt;
        for (uint32_t t = pv.head[si]; t != kNil; t = pv.next[t]) {
            const uint32_t ep = v.touch_ep[t];
            const StoreEntry *pe = pt_find(v, hsh, ep);
            n_new = list_apply(a, n_new, ep, pe && pe->in_map != 0);
        }
        if (n_new <= (uint32_t)kInlineIds) {
            uint32_t tmp[kInlineIds];
            for (uint32_t q = 0; q < (uint32_t)kInlineIds; q++) tmp[q] = q < n_new ? a[q] : 0u;
            for (uint32_t q = 0; q < (uint32_t)kInlineIds; q++) sl->ids[q] = tmp[q];
        } else {
            sl->ids[0] = (uint32_t)off;
            for (uint32_t q = 1; q < (uint32_t)kInlineIds; q++) sl->ids[q] = 0u;
        }
    }
    sl->cnt = n_new;
    pv.head[si] = kNil;
    if (n_new) presence_set(pv.presence, pv.presence_shift, hsh);
    if (n_new > cnt) atomicAdd(&v.ctr[kCtrPatchAdd], (unsigned long long)(n_new - cnt));
    if (n_new < cnt) atomicAdd(&v.ctr[kCtrPatchDel], (unsigned long long)(cnt - n_new));
}

// ---- interning of the lists a patch wrote (same table and rule as the bulk build: the lowest slot index among equal
// lists is canonical, everyone else points at its copy; equality is verified on the contents, the hash is a hint)
__device__ __forceinline__ uint64_t patch_intern_slot(const PatchView &pv, uint64_t key, bool claim) {
    uint64_t i = key & pv.mask;
    for (;;) {
        unsigned long long *kp = reinterpret_cast<unsigned long long *>(&pv.intern_keys[i]);
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long *>(kp);
        if (cur == key) return i;
        if (cur == kEmptyKey) {
            if (!claim) return i;
            unsigned long long old = atomicCAS(kp, (unsigned long long)kEmptyKey, (unsigned long long)key);
            if (old == kEmptyKey) atomicAdd(pv.intern_claims, 1ull);
            if (old == kEmptyKey || old == key) return i;
        }
        i = (i + 1) & pv.mask;
    }
}

__global__ void k_patch_intern_claim(PatchView pv, unsigned long long n_dirty) {
    const unsigned long long d = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_dirty) return;
    const uint32_t si = pv.dirty[d];
    const IndexSlot &sl = pv.slots[si];
    if (sl.cnt <= (uint32_t)kInlineIds) return;
    const uint64_t j = patch_intern_slot(pv, patch_list_hash(pv.postings + sl.ids[0], sl.cnt), true);
    atomicMin(&pv.intern_vals[j], si);
}

__global__ void k_patch_intern_apply(PatchView pv, unsigned long long n_dirty) {
    const unsigned long long d = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= n_dirty) return;
    const uint32_t si = pv.dirty[d];
    IndexSlot &sl = pv.slots[si];
    const uint32_t cnt = sl.cnt, off = sl.ids[0];
    if (cnt <= (uint32_t)kInlineIds) return;
    const uint64_t j = patch_intern_slot(pv, patch_list_hash(pv.postings + off, cnt), false);
    const uint32_t c = pv.intern_vals[j];
    if (c == si || c == kNil) return;                         // canonical slots are never rewritten
    if (pv.slots[c].cnt != cnt) return;
    const uint32_t canon = pv.slots[c].ids[0];
    for (uint32_t k = 0; k < cnt; k++)
        if (pv.postings[canon + k] != pv.postings[off + k]) return;
    sl.ids[0] = canon;
}

inline unsigned blocks_for(uint64_t n, unsigned per) { return (unsigned)std::max<uint64_t>(1, (n + per - 1) / per); }

}  // namespace

#define ST_TRY(expr)                         \
    do {                                     \
        cudaError_t _e = (expr);             \
        if (_e != cudaSuccess) return _e;    \
    } while (0)

void IndexStore::fill_view(View &v) const {
    v.pt = pt_.as<StoreEntry>();
    v.pt_mask = pt_cap_ ? pt_cap_ - 1 : 0;
    v.log_hash = log_hash_.as<unsigned long long>();
    v.log_seq = log_seq_.as<unsigned long long>();
    v.E = E_;
    v.default_cap = default_cap_;
    v.cap = cap_.as<uint32_t>();
    v.live = live_.as<uint32_t>();
    v.firstcall = firstcall_.as<uint32_t>();
    v.sp_in_map = sp_in_map_.as<uint32_t>();
    v.seg_off = seg_off_.as<unsigned long long>();
    v.seg_cap = seg_cap_.as<unsigned long long>();
    v.head = head_.as<unsigned long long>();
    v.tail = tail_.as<unsigned long long>();
    v.inc = inc_.as<unsigned long long>();
    v.next_seq = next_seq_.as<unsigned long long>();
    v.sp_seq = sp_seq_.as<unsigned long long>();
    v.cut = cut_.as<unsigned long long>();
    v.ctr = ctr_.as<unsigned long long>();
    v.touch_hash = touch_hash_.as<unsigned long long>();
    v.touch_ep = touch_ep_.as<uint32_t>();
    v.touch_cap = touch_disabled_ ? 0 : touch_cap_;
}

cudaError_t IndexStore::ensure_init(cudaStream_t s) {
    if (init_) return cudaSuccess;
    const size_t E = std::max<uint32_t>(E_, kCtrN);
    for (DevBuf *b : {&cap_, &live_, &firstcall_, &sp_in_map_}) ST_TRY(b->reserve(sizeof(uint32_t) * E, &bytes_));
    for (DevBuf *b : {&seg_off_, &seg_cap_, &head_, &tail_, &inc_, &next_seq_, &sp_seq_, &new_off_, &new_cap_, &cut_})
        ST_TRY(b->reserve(sizeof(unsigned long long) * E, &bytes_));
    ST_TRY(ctr_.reserve(sizeof(unsigned long long) * kCtrN, &bytes_));
    if (!ctr_host_) ST_TRY(cudaHostAlloc(reinterpret_cast<void **>(&ctr_host_), sizeof(unsigned long long) * kCtrN, cudaHostAllocDefault));
    pt_cap_ = 1024;
    ST_TRY(pt_.reserve(sizeof(StoreEntry) * pt_cap_, &bytes_));
    ST_TRY(log_hash_.reserve(sizeof(unsigned long long) * 64, &bytes_));
    ST_TRY(log_seq_.reserve(sizeof(unsigned long long) * 64, &bytes_));
    log_cap_ = 0;
    View v;
    fill_view(v);
    k_store_pt_clear<<<blocks_for(pt_cap_, 256), 256, 0, s>>>(v.pt, pt_cap_);
    k_store_state_clear<<<blocks_for(E, 256), 256, 0, s>>>(v);
    ST_TRY(cudaGetLastError());
    init_ = true;
    in_map_ = 0;
    pt_used_ = 0;
    return cudaSuccess;
}

cudaError_t IndexStore::clear(cudaStream_t s) {
    if (!init_) return cudaSuccess;
    ST_TRY(cudaStreamSynchronize(s));
    init_ = false;
    used_ = false;
    dirty_ = true;
    touch_upper_ = 0;
    touch_disabled_ = false;
    return ensure_init(s);
}

// Rebuilds the pair table (dropping tombstones) so that `incoming` more pairs keep the load factor under one half.
cudaError_t IndexStore::grow_pair_table(uint64_t incoming, cudaStream_t s) {
    View v;
    fill_view(v);
    ST_TRY(cudaMemsetAsync(&v.ctr[kCtrAlive], 0, sizeof(unsigned long long), s));
    k_store_count_alive<<<blocks_for(pt_cap_, 256), 256, 0, s>>>(v.pt, pt_cap_, v.ctr);
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    const uint64_t alive = ctr_host_[kCtrAlive];
    uint64_t want = 1024;
    while (want < (alive + incoming) * 5 / 2) want <<= 1;
    DevBuf &fresh = pt_spare_;
    ST_TRY(fresh.reserve(sizeof(StoreEntry) * want, &bytes_));
    k_store_pt_clear<<<blocks_for(want, 256), 256, 0, s>>>(fresh.as<StoreEntry>(), want);
    ST_TRY(cudaMemsetAsync(&v.ctr[kCtrPtUsed], 0, sizeof(unsigned long long), s));
    View nv = v;
    nv.pt = fresh.as<StoreEntry>();
    nv.pt_mask = want - 1;
    k_store_rehash<<<blocks_for(pt_cap_, 256), 256, 0, s>>>(v.pt, pt_cap_, nv);
    ST_TRY(cudaGetLastError());
    ST_TRY(cudaStreamSynchronize(s));
    std::swap(pt_.p, fresh.p);
    std::swap(pt_.cap, fresh.cap);
    pt_cap_ = want;
    pt_used_ = alive;
    last_launches += 3;
    last_rehashed = true;
    return cudaSuccess;
}

// Moves every endpoint's live log entries, in order, into a fresh segment sized for four times (live + incoming).
cudaError_t IndexStore::repack_logs(cudaStream_t s) {
    View v;
    fill_view(v);
    std::vector<uint32_t> live(E_), cap(E_);
    h_inc_.resize(E_);
    ST_TRY(cudaMemcpyAsync(live.data(), v.live, sizeof(uint32_t) * E_, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaMemcpyAsync(cap.data(), v.cap, sizeof(uint32_t) * E_, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaMemcpyAsync(h_inc_.data(), v.inc, sizeof(unsigned long long) * E_, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    h_off_.resize(E_);
    h_cap_.resize(E_);
    uint64_t total = 0;
    for (uint32_t e = 0; e < E_; e++) {
        uint64_t need = (uint64_t)live[e] + h_inc_[e];
        uint64_t c = need ? ((4 * need + 256 + 255) & ~255ull) : 0;      // whole eviction blocks; room for three more batches
                                                                           // of this size before the next compaction
        h_off_[e] = total;
        h_cap_[e] = c;
        total += c;
    }
    ST_TRY(cudaMemcpyAsync(new_off_.p, h_off_.data(), sizeof(unsigned long long) * E_, cudaMemcpyHostToDevice, s));
    ST_TRY(cudaMemcpyAsync(new_cap_.p, h_cap_.data(), sizeof(unsigned long long) * E_, cudaMemcpyHostToDevice, s));
    DevBuf &nh = log_hash_spare_, &ns = log_seq_spare_;
    ST_TRY(nh.reserve(sizeof(unsigned long long) * std::max<uint64_t>(total, 64), &bytes_));
    ST_TRY(ns.reserve(sizeof(unsigned long long) * std::max<uint64_t>(total, 64), &bytes_));
    k_store_repack<<<blocks_for((uint64_t)E_ * 32, 256), 256, 0, s>>>(v, new_off_.as<unsigned long long>(), new_cap_.as<unsigned long long>(),
                                                                     nh.as<unsigned long long>(), ns.as<unsigned long long>());
    ST_TRY(cudaGetLastError());
    ST_TRY(cudaStreamSynchronize(s));
    std::swap(log_hash_.p, nh.p);
    std::swap(log_hash_.cap, nh.cap);
    std::swap(log_seq_.p, ns.p);
    std::swap(log_seq_.cap, ns.cap);
    log_cap_ = total;
    last_launches += 1;
    last_repacked = true;
    return cudaSuccess;
}

namespace {
// EPP_STORE_TIMING=1: per-kernel CUDA-event times of every apply() on stderr (profiling aid).
struct StoreTimer {
    bool on;
    cudaStream_t s;
    std::vector<std::pair<const char *, cudaEvent_t>> marks;
    explicit StoreTimer(cudaStream_t st) : on(getenv("EPP_STORE_TIMING") != nullptr), s(st) { mark("start"); }
    void mark(const char *name) {
        if (!on) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, s);
        marks.emplace_back(name, e);
    }
    ~StoreTimer() {
        if (!on) return;
        cudaStreamSynchronize(s);
        for (size_t i = 1; i < marks.size(); i++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, marks[i - 1].second, marks[i].second);
            fprintf(stderr, "[store] %-10s %8.3f ms\n", marks[i].first, ms);
        }
        for (auto &m : marks) cudaEventDestroy(m.second);
    }
};
}  // namespace

cudaError_t IndexStore::apply(const StoreCalls &calls, cudaStream_t s) {
    StoreTimer tm(s);
    last_launches = 0;
    last_items = 0;
    last_repacked = last_rehashed = false;
    if (calls.M == 0) return cudaSuccess;
    ST_TRY(ensure_init(s));
    used_ = true;
    const uint32_t M = calls.M, n_chunks = (M + kCallChunk - 1) / kCallChunk;
    const uint64_t hist_n = (uint64_t)n_chunks * E_;
    ST_TRY(hist_.reserve(sizeof(uint32_t) * hist_n, &bytes_));
    ST_TRY(off_.reserve(sizeof(unsigned long long) * M, &bytes_));
    View v;
    fill_view(v);
    uint32_t *hist = hist_.as<uint32_t>();
    unsigned long long *off = off_.as<unsigned long long>();
    k_store_batch_clear<<<blocks_for(std::max<uint64_t>(hist_n, E_), 256), 256, 0, s>>>(v, hist, hist_n);
    k_store_hist<<<blocks_for(M, 256), 256, 0, s>>>(v, M, calls.ep, calls.n, hist);
    k_store_plan<<<blocks_for(E_, 128), 128, 0, s>>>(v, n_chunks, hist, calls.nb);
    tm.mark("plan");
    // log compaction (flat over 256-entry blocks): list the endpoints whose segment cannot take the batch; the read-back
    // below (needed anyway for the table sizes) tells whether there is anything to compact
    ST_TRY(list_e_.reserve(sizeof(uint32_t) * E_, &bytes_));
    ST_TRY(list_start_.reserve(sizeof(unsigned long long) * E_, &bytes_));
    ST_TRY(cudaMemsetAsync(&v.ctr[kCtrEvict], 0, sizeof(unsigned long long), s));
    k_compact_list<<<blocks_for(E_, 256), 256, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>());
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    last_launches += 4;
    if (ctr_host_[kCtrEvict] >> kEvictPackShift) {                 // endpoints listed (a brand-new one lists zero blocks)
        ST_TRY(blockcnt_.reserve(sizeof(uint32_t) * (log_cap_ / kEvictBlock + 1), &bytes_));
        ST_TRY(blockmask_.reserve(sizeof(uint32_t) * (log_cap_ / kEvictBlock + 1) * (kEvictBlock / 32), &bytes_));
        ST_TRY(log_hash_spare_.reserve(sizeof(unsigned long long) * std::max<uint64_t>(log_cap_, 64), &bytes_));
        ST_TRY(log_seq_spare_.reserve(sizeof(unsigned long long) * std::max<uint64_t>(log_cap_, 64), &bytes_));
        const unsigned cg = (unsigned)sm_count_ * 8;                // persistent: CTAs stride over the flat block space
        unsigned long long *nh = new_off_.as<unsigned long long>();          // scratch until repack_logs rewrites it
        k_compact_count<<<cg, kEvictBlock, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>(),
                                                   blockcnt_.as<uint32_t>(), blockmask_.as<uint32_t>());
        k_compact_scan<<<blocks_for((uint64_t)E_ * 32, 256), 256, 0, s>>>(v, blockcnt_.as<uint32_t>(), nh);
        k_compact_scatter<<<cg, kEvictBlock, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>(),
                                                     blockcnt_.as<uint32_t>(), blockmask_.as<uint32_t>(),
                                                     log_hash_spare_.as<unsigned long long>(), log_seq_spare_.as<unsigned long long>());
        k_compact_copyback<<<cg, kEvictBlock, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>(), nh,
                                                      log_hash_spare_.as<unsigned long long>(), log_seq_spare_.as<unsigned long long>());
        k_compact_finish<<<blocks_for(E_, 256), 256, 0, s>>>(v, nh);
        ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
        ST_TRY(cudaStreamSynchronize(s));
        last_launches += 5;
    }
    tm.mark("compact");
    const uint64_t total = ctr_host_[kCtrTotalItems];
    last_items = total;
    pt_used_ = ctr_host_[kCtrPtUsed];
    if ((pt_used_ + total) * 2 > pt_cap_) ST_TRY(grow_pair_table(total, s));
    if (ctr_host_[kCtrNeedRepack]) ST_TRY(repack_logs(s));
    ST_TRY(reserve_touch(2 * total, s));
    fill_view(v);
    tm.mark("grow");
    if (total) {
        k_store_offsets<<<n_chunks, kCallChunk, 0, s>>>(v, M, calls.ep, calls.n, hist, off);
        tm.mark("offsets");
        k_store_upsert<<<blocks_for((uint64_t)M * 32, 256), 256, 0, s>>>(v, M, calls.ep, calls.n,
                                                                         reinterpret_cast<const unsigned long long *>(calls.src), off,
                                                                         reinterpret_cast<const unsigned long long *>(calls.hashes));
        tm.mark("upsert");
        k_store_leak<<<std::min<uint32_t>(M, 592), 256, 0, s>>>(v, M, calls.ep, calls.n, off);
        ST_TRY(blockcnt_.reserve(sizeof(uint32_t) * (log_cap_ / kEvictBlock + 1), &bytes_));
        tm.mark("leak");
        ST_TRY(list_e_.reserve(sizeof(uint32_t) * E_, &bytes_));
        ST_TRY(list_start_.reserve(sizeof(unsigned long long) * E_, &bytes_));
        ST_TRY(cudaMemsetAsync(&v.ctr[kCtrEvict], 0, sizeof(unsigned long long), s));
        k_store_advance<<<blocks_for(E_, 256), 256, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>());
        const unsigned eg = (unsigned)sm_count_ * 8;     // persistent: CTAs stride over the flat block space
        k_evict_count<<<eg, kEvictBlock, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>(), blockcnt_.as<uint32_t>());
        tm.mark("ev_count");
        k_evict_cut<<<blocks_for((uint64_t)E_ * 32, 256), 256, 0, s>>>(v, blockcnt_.as<uint32_t>());
        tm.mark("ev_cut");
        k_evict_apply<<<eg, kEvictBlock, 0, s>>>(v, list_e_.as<uint32_t>(), list_start_.as<unsigned long long>());
        k_evict_finish<<<blocks_for(E_, 256), 256, 0, s>>>(v);
        tm.mark("ev_apply");
        last_launches += 8;
    }
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    in_map_ = ctr_host_[kCtrInMap];
    pt_used_ = ctr_host_[kCtrPtUsed];
    dirty_ = true;
    return cudaGetLastError();
}

// Room in the touch log for `more` entries (adds that enter the map + evictions that leave it).  Beyond kTouchMax the
// log is abandoned for this cycle and the next commit falls back to the bulk build.
cudaError_t IndexStore::reserve_touch(uint64_t more, cudaStream_t s) {
    constexpr uint64_t kTouchMax = 1ull << 27;            // 134 M entries = 1.6 GB
    if (touch_disabled_) return cudaSuccess;
    touch_upper_ += more;
    if (touch_upper_ > kTouchMax) {
        touch_disabled_ = true;
        return cudaSuccess;
    }
    if (touch_upper_ <= touch_cap_) return cudaSuccess;
    uint64_t want = std::max<uint64_t>(1 << 16, touch_cap_ * 2);
    while (want < touch_upper_) want *= 2;
    DevBuf nh, ne;
    size_t acc = 0;
    ST_TRY(nh.reserve(sizeof(unsigned long long) * want, &acc));
    ST_TRY(ne.reserve(sizeof(uint32_t) * want, &acc));
    if (touch_cap_) {
        ST_TRY(cudaMemcpyAsync(nh.p, touch_hash_.p, sizeof(unsigned long long) * touch_cap_, cudaMemcpyDeviceToDevice, s));
        ST_TRY(cudaMemcpyAsync(ne.p, touch_ep_.p, sizeof(uint32_t) * touch_cap_, cudaMemcpyDeviceToDevice, s));
        ST_TRY(cudaStreamSynchronize(s));
    }
    bytes_ -= touch_hash_.cap + touch_ep_.cap;
    std::swap(touch_hash_.p, nh.p);
    std::swap(touch_hash_.cap, nh.cap);
    std::swap(touch_ep_.p, ne.p);
    std::swap(touch_ep_.cap, ne.cap);
    bytes_ += touch_hash_.cap + touch_ep_.cap;
    touch_cap_ = want;
    return cudaSuccess;
}

// The read table now reflects the inverted map (bulk build or patch): start a new touch log.
cudaError_t IndexStore::touch_reset(cudaStream_t s) {
    touch_upper_ = 0;
    touch_disabled_ = false;
    if (!init_) return cudaSuccess;
    return cudaMemsetAsync(&ctr_.as<unsigned long long>()[kCtrTouch], 0, sizeof(unsigned long long) * 2, s);   // kCtrTouch, kCtrTouchLost
}

// Brings a bulk-built read table up to date from the touch log.  *patched = false: nothing was done (log unusable, the
// table or its interning table lacks room, the sentinel hash is involved, or the change set is too large to be worth
// it) -> bulk build.
cudaError_t IndexStore::patch_read_table(const ReadTableRef &rt, uint64_t table_pairs, cudaStream_t s, bool *patched,
                                         uint64_t *new_pairs, uint64_t *new_slots_used, uint64_t *new_post_used,
                                         uint64_t *new_intern_used) {
    *patched = false;
    if (!init_ || touch_disabled_) return cudaSuccess;
    View v;
    fill_view(v);
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    const uint64_t n_touch = ctr_host_[kCtrTouch];
    if (ctr_host_[kCtrTouchLost] || n_touch > touch_cap_) return cudaSuccess;
    if (n_touch == 0) {
        *patched = true;
        *new_pairs = table_pairs;
        *new_slots_used = rt.slots_used;
        *new_post_used = rt.post_used;
        *new_intern_used = rt.intern_used;
        return cudaSuccess;
    }
    // worth it only when the change set is small next to the table; and the table must keep its load factor
    if (n_touch > std::max<uint64_t>(1 << 16, table_pairs / 2)) return cudaSuccess;
    if ((rt.slots_used + n_touch) * 10 > rt.capacity * 6) return cudaSuccess;
    // so must the interning table, which only the bulk build empties: every spilled list a patch writes claims a key
    // (at most one per dirty slot, n_dirty <= n_touch) and the key of the list it replaces stays; its probes end only
    // at a free key
    if ((rt.intern_used + n_touch) * 10 > rt.capacity * 6) return cudaSuccess;
    if (n_touch >= 0xFFFFFFF0ull) return cudaSuccess;
    ST_TRY(patch_next_.reserve(sizeof(uint32_t) * n_touch, &bytes_));
    ST_TRY(patch_dirty_.reserve(sizeof(uint32_t) * n_touch, &bytes_));
    PatchView pv;
    pv.slots = rt.slots;
    pv.mask = rt.capacity - 1;
    pv.postings = rt.postings;
    pv.post_cap = rt.post_cap;
    pv.post_cursor = &v.ctr[kCtrPatchPost];
    pv.head = rt.head;
    pv.next = patch_next_.as<uint32_t>();
    pv.dirty = patch_dirty_.as<uint32_t>();
    pv.intern_keys = rt.intern_keys;
    pv.intern_vals = rt.intern_vals;
    pv.intern_claims = &v.ctr[kCtrPatchIntern];
    pv.presence = rt.presence;
    pv.presence_shift = rt.presence_shift;
    ST_TRY(cudaMemsetAsync(&v.ctr[kCtrPatchFlag], 0, sizeof(unsigned long long) * 6, s));     // flag .. intern
    ctr_host_[kCtrPatchPost] = rt.post_used;
    ST_TRY(cudaMemcpyAsync(&v.ctr[kCtrPatchPost], &ctr_host_[kCtrPatchPost], sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
    ST_TRY(cudaStreamSynchronize(s));
    k_patch_group<<<blocks_for(n_touch, 256), 256, 0, s>>>(v, pv, n_touch);
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    const uint64_t n_dirty = ctr_host_[kCtrPatchDirty];
    if (ctr_host_[kCtrPatchFlag]) return cudaSuccess;                    // sentinel hash touched: bulk build
    k_patch_apply<<<blocks_for(n_dirty, 128), 128, 0, s>>>(v, pv, n_dirty);
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    ST_TRY(cudaGetLastError());
    if (ctr_host_[kCtrPatchFlag]) return cudaSuccess;                    // out of posting space mid-way: bulk build
    k_patch_intern_claim<<<blocks_for(n_dirty, 128), 128, 0, s>>>(pv, n_dirty);
    k_patch_intern_apply<<<blocks_for(n_dirty, 128), 128, 0, s>>>(pv, n_dirty);
    ST_TRY(cudaMemcpyAsync(&ctr_host_[kCtrPatchIntern], &v.ctr[kCtrPatchIntern], sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    ST_TRY(cudaGetLastError());
    *new_pairs = table_pairs + ctr_host_[kCtrPatchAdd] - ctr_host_[kCtrPatchDel];
    *new_slots_used = rt.slots_used + ctr_host_[kCtrPatchClaims];
    *new_post_used = ctr_host_[kCtrPatchPost];
    *new_intern_used = rt.intern_used + ctr_host_[kCtrPatchIntern];
    last_patch_touches = n_touch;
    last_patch_dirty = n_dirty;
    *patched = true;
    return cudaSuccess;
}

cudaError_t IndexStore::apply_picks(const epp_decision *decisions, const uint64_t *hashes, const int32_t *nblocks,
                                    int64_t R, int32_t max_blocks, cudaStream_t s) {
    if (R <= 0) return cudaSuccess;
    const uint32_t M = (uint32_t)(2 * R);
    ST_TRY(call_ep_.reserve(sizeof(uint32_t) * M, &bytes_));
    ST_TRY(call_n_.reserve(sizeof(uint32_t) * M, &bytes_));
    ST_TRY(call_nb_.reserve(sizeof(int32_t) * M, &bytes_));
    ST_TRY(call_src_.reserve(sizeof(unsigned long long) * M, &bytes_));
    k_store_calls_from_picks<<<blocks_for((uint64_t)R, 256), 256, 0, s>>>(decisions, nblocks, R, max_blocks, E_, call_ep_.as<uint32_t>(),
                                                                          call_n_.as<uint32_t>(), call_nb_.as<int32_t>(),
                                                                          call_src_.as<unsigned long long>());
    StoreCalls c;
    c.M = M;
    c.ep = call_ep_.as<uint32_t>();
    c.n = call_n_.as<uint32_t>();
    c.nb = call_nb_.as<int32_t>();
    c.src = call_src_.as<uint64_t>();
    c.hashes = hashes;
    cudaError_t e = apply(c, s);
    last_launches += 1;
    return e;
}

cudaError_t IndexStore::remove_endpoint(uint32_t ep, cudaStream_t s) {
    if (ep >= E_ || !init_) return cudaSuccess;
    ST_TRY(reserve_touch(in_map_, s));            // at most every pair of the map leaves it
    View v;
    fill_view(v);
    k_store_remove_endpoint<<<1, 32, 0, s>>>(v, ep);
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    in_map_ = ctr_host_[kCtrInMap];
    dirty_ = true;
    return cudaGetLastError();
}

cudaError_t IndexStore::retain_endpoints(const uint8_t *active_dev, cudaStream_t s) {
    if (!init_) return cudaSuccess;
    ST_TRY(reserve_touch(in_map_, s));
    View v;
    fill_view(v);
    k_store_retain<<<blocks_for((uint64_t)E_ * 32, 256), 256, 0, s>>>(v, active_dev);
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    in_map_ = ctr_host_[kCtrInMap];
    dirty_ = true;
    return cudaGetLastError();
}

cudaError_t IndexStore::export_pairs(DevBuf &pair_hash, DevBuf &pair_ep, uint64_t *n_pairs, size_t *accounted,
                                     cudaStream_t s) {
    *n_pairs = 0;
    if (!init_) return cudaSuccess;
    View v;
    fill_view(v);
    ST_TRY(pair_hash.reserve(sizeof(uint64_t) * std::max<uint64_t>(in_map_, 1), accounted));
    ST_TRY(pair_ep.reserve(sizeof(uint32_t) * std::max<uint64_t>(in_map_, 1), accounted));
    ST_TRY(cudaMemsetAsync(&v.ctr[kCtrCursor], 0, sizeof(unsigned long long), s));
    k_store_export<<<blocks_for(pt_cap_ + E_, 256 * kExportPer), 256, 0, s>>>(v, pt_cap_, pair_hash.as<unsigned long long>(), pair_ep.as<uint32_t>());
    ST_TRY(cudaMemcpyAsync(ctr_host_, v.ctr, sizeof(unsigned long long) * kCtrN, cudaMemcpyDeviceToHost, s));
    ST_TRY(cudaStreamSynchronize(s));
    *n_pairs = ctr_host_[kCtrCursor];
    return cudaGetLastError();
}

}  // namespace epp
