// hash_fused.cu -- a1 (hashPrompt, approximateprefix/hashing.go:35-99) as one CTA-cooperative kernel with register-fed
// 128-bit global loads: the DEFAULT hash kernel of the throughput path (block sizes that are a multiple of 32
// bytes, 16-byte aligned prompts; everything else takes the generic kernels of hash_kernels.cu; DESIGN.md section 4.1).
//
// HBM traffic per request: every prompt byte is read at most once, the 8-byte pre-chain digests never leave the SM
// (shared-memory ring), the block hashes are written once (the PluginState stash PreRequest needs, plugin.go:150-157)
// -- or, with a presence bitmap (HashParams::presence), only up to the first block no endpoint can hold: the match
// kernel's global stop never lies beyond it.  With HashParams::skip as well, the prompt is also READ only that far
// (plus the ring's lookahead): a block hash depends on blocks 0..b alone, so no decision depends on the bytes past it.
//
// CTA = 9 warps, persistent, 32 request SLOTS refilled from a per-launch request counter (HashParams::req_next):
//   warps 0-7 (digest): thread (r = t/8, j = t%8) owns block j of the window the chain assigned to slot r for the
//       stage: 4 independent XXH64 accumulator chains over the block's 32-byte stripes, merge -> m, stored to the
//       stage's [r][j] cell.
//   warp 8 (chain): lane = slot.  Walks its request's window in block order (the only serial part of the digest:
//       m + len, one 8-byte round with h_{i-1}, avalanche), in place.  When a slot's request is done -- every full
//       window chained, or, with skip, a window start proven absent -- the lane finishes it (trailing partial block,
//       bound) and takes the next request from a CTA-local queue of 32 that one warp-wide ticket on req_next refills;
//       the new request's windows start kStages stages later, the stages already assigned still carry the old one.
//   Stages are handed over with named barriers (bar.arrive / bar.sync), 2-deep ring of stages of one window each: full
//   (digest -> chain), empty (chain -> digest).  With each empty hand-over the chain assigns the stage kStages ahead
//   (block 0 of a window and its number of full blocks per slot); once every request is taken and done it names the
//   last stage, and both sides leave the ring there.
//   A request closed at window c (block c*W proven absent) is known once window c has been chained; window c+1 is
//   assigned by then: it reads at most kStages - 1 windows past its closing window.
#include "hash_blocks.cuh"
#include "index.cuh"

namespace epp {

namespace {
constexpr int kWin = 8;
constexpr int kSlots = 32;
constexpr int kStages = 2;
constexpr int kBarFull = 1;               // named barrier ids 1..2
constexpr int kBarEmpty = 1 + kStages;    // 3..4
constexpr int kHashMinCtas = 4;

__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Lengths (hashing.go:58-66) of request r < R: writes in_len / nblocks / eff_len; -> offset, full blocks, tail bytes.
__device__ __forceinline__ void request_lengths(const HashParams &p, int64_t r, uint64_t &off, int32_t &nfull,
                                                int32_t &tail) {
    const int64_t bs = p.block_bytes;
    uint64_t len;
    if (p.offsets) { off = p.offsets[r]; len = p.lengths ? p.lengths[r] : p.offsets[r + 1] - off; }
    else { off = (uint64_t)r * p.uniform_len; len = p.uniform_len; }
    if (p.in_len) p.in_len[r] = (int64_t)len;
    int64_t eff = (int64_t)len;
    nfull = 0;
    tail = 0;
    if (eff < bs) {
        eff = 0;
    } else {
        const int64_t cap = bs * (int64_t)p.max_blocks;
        if (eff > cap) eff = cap;
        nfull = (int32_t)(eff / bs);
        tail = (int32_t)(eff - (int64_t)nfull * bs);
    }
    p.nblocks[r] = nfull + (tail ? 1 : 0);
    p.eff_len[r] = eff;
}

// Per-lane stop bound of the chain warp: the first window whose leading block reads as absent in the presence bitmap
// (one lookup per window of W blocks).  The word is loaded as soon as the window's leading hash is chained and examined
// once its other W - 1 hashes are, so the L2 latency hides behind them; a window proven absent is neither stored nor
// followed by more than the one window the ring has already assigned, and a row ends at its bound.
struct StopBound {
    int32_t bnd = INT32_MAX;        // a block proven absent (bound >= the global stop); INT32_MAX while none is
    int32_t pending = -1;           // block whose presence word is in flight, or -1
    uint32_t word = 0, bit = 0;

    __device__ __forceinline__ void issue(const HashParams &p, int32_t block, uint64_t h) {
        const uint32_t b = (uint32_t)(h >> p.presence_shift);
        word = __ldg(p.presence + (b >> 5));
        bit = h == kEmptyKey ? 32u : (b & 31);   // the all-ones hash lives in the side record: always present
        pending = block;
    }
    __device__ __forceinline__ void resolve() {
        if (bit < 32 && !((word >> bit) & 1u)) bnd = pending;
        pending = -1;
    }
};

// Chain warp, window k of the lane's request (row `row`): the serial part of the digest; the lane then writes the
// window's hashes straight from registers (64 bytes = two full sectors, 128-bit stores when the row pitch allows) -- no
// transpose through shared memory.  With p.presence, hashes at or past a proven-absent block are not stored (the match
// kernel never reads past it), nor computed once that block is known.
template <int W = kWin>
__device__ __forceinline__ uint64_t chain_window(const uint64_t *sm, const HashParams &p, uint64_t *row, int k,
                                                 int32_t nfull, uint64_t lenp8, uint64_t prev, StopBound &sb,
                                                 uint32_t &n_stored) {
    if (sb.bnd != INT32_MAX) return prev;
    const int32_t n_here = min(W, nfull - k * W);              // hashes of this window (>= 1)
    uint64_t hv[W];
#pragma unroll
    for (int j = 0; j < W; j++) {
        if (j < n_here) prev = xxh_chain_step32(sm[j], lenp8, prev);
        hv[j] = prev;
        if (j == 0 && p.presence) sb.issue(p, k * W, prev);    // the window's leading block: looked up at once
    }
    if (sb.pending >= 0) sb.resolve();                         // its word has had the window's other W - 1 steps
    const int32_t n_store = min(n_here, sb.bnd - k * W);
    if (n_store <= 0) return prev;
    n_stored += (uint32_t)n_store;
    uint64_t *dst = row + (int64_t)k * W;
    if (n_store == W && !(p.max_blocks & 1) && !(reinterpret_cast<uintptr_t>(p.hashes) & 15)) {   // the window starts 16-byte aligned
#pragma unroll
        for (int j = 0; j < W; j += 2)
            asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(dst + j), "l"(hv[j]), "l"(hv[j + 1]) : "memory");
    } else {
#pragma unroll
        for (int j = 0; j < W; j++)
            if (j < n_store) dst[j] = hv[j];
    }
    return prev;
}
}  // namespace

__global__ void __launch_bounds__(32 * kWin + 32, kHashMinCtas) k_hash_fused(HashParams p) {
    constexpr int W = kWin;
    constexpr int kDigestWarps = kSlots * W / 32;
    constexpr int kProducers = kSlots * W + 32;
    __shared__ uint64_t s_m[kStages][kSlots][(W + 1)];
    __shared__ const uint8_t *s_src[kStages][kSlots];     // block 0 of the window assigned to each slot for the stage
    __shared__ int32_t s_n[kStages][kSlots];              // its full blocks (0: nothing to load)
    __shared__ uint64_t s_q_off[kSlots], s_q_seed[kSlots];   // the chain's queue of requests not yet in a slot
    __shared__ int32_t s_q_nfull[kSlots], s_q_tail[kSlots];
    __shared__ int32_t s_end;                             // first stage nobody runs, INT32_MAX while unknown

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int t = threadIdx.x;
    const int64_t bs = p.block_bytes;
    const int n_stripes = (int)(bs >> 5);
    const uint64_t lenp8 = (uint64_t)bs + 8;
    const bool skip = p.presence && p.skip;
    uint64_t n_read = 0;                      // prompt bytes this thread loaded (p.read)

    if (warp < kDigestWarps) {
        __syncthreads();                      // the chain has assigned stages 0 .. kStages-1 and maybe s_end
        const int r = t / W, j = t % W;
        uint32_t n_loaded = 0;
        int k = 0;
        for (;; k++) {
            const int s = k % kStages;
            if (k >= kStages) bar_sync(kBarEmpty + s, kProducers);
            if (k >= *(volatile int32_t *)&s_end) break;
            if (j < s_n[s][r]) {
                s_m[s][r][j] = block_digest(s_src[s][r] + (uint64_t)j * (uint64_t)bs, n_stripes);
                n_loaded++;
            }
            bar_arrive(kBarFull + s, kProducers);     // bar.arrive orders the stores above for the threads of the barrier
        }
        for (int q = k + 1; q < k + kStages; q++)     // the chain's last empty hand-overs
            if (q >= kStages) bar_sync(kBarEmpty + q % kStages, kProducers);
        n_read = (uint64_t)n_loaded * (uint64_t)bs;
    } else {
        // lane state: the slot's request (rid < 0: none), its full blocks and the stage its window 0 is in (st0: stage
        // st0 + w holds window w); its offset and tail bytes are in s_off / s_tail
        __shared__ uint64_t s_off[kSlots];
        __shared__ int32_t s_tail[kSlots];
        int32_t rid = -1, nfull = 0, st0 = 0;
        uint64_t prev = 0;
        StopBound sb;
        uint32_t n_stored = 0;
        // the queue: request of entry 0, next entry, entries (-1: the request counter is exhausted); kept in shared
        // memory to spare the chain's registers
        __shared__ uint32_t s_q_base;
        __shared__ int32_t s_q_head, s_q_n;
        int end = INT32_MAX;

        // The slot's request is done: trailing partial block (hashing.go:90-96; when skipping, read only while the
        // request is open) and bound.
        auto finish = [&]() {
            if (sb.pending >= 0) sb.resolve();
            int32_t bnd = sb.bnd;
            const int32_t tail = s_tail[lane];
            if (tail && (!skip || bnd == INT32_MAX)) {
                n_read += (uint64_t)tail;
                const uint64_t h = hash_block_generic(p.data + s_off[lane] + (uint64_t)nfull * (uint64_t)bs, tail, prev);
                if (bnd == INT32_MAX && p.presence && !presence_maybe(p.presence, p.presence_shift, h)) bnd = nfull;
                if (nfull < bnd) {
                    p.hashes[(int64_t)rid * p.max_blocks + nfull] = h;
                    n_stored++;
                }
            }
            if (p.presence) p.bound[rid] = min(bnd, nfull + (tail ? 1 : 0));
            rid = -1;
        };
        // Every empty slot takes the next request; its window 0 goes to stage `first`.
        auto refill = [&](int first) {
            for (;;) {
                const unsigned need = __ballot_sync(0xffffffffu, rid < 0);
                const int q_head = s_q_head, q_n = s_q_n;
                if (!need || q_n < 0) return;
                __syncwarp();
                if (q_head == q_n) {          // one ticket of 32 requests for the queue
                    uint32_t base = 0;
                    if (lane == 0) base = atomicAdd(p.req_next, (uint32_t)kSlots);
                    base = __shfl_sync(0xffffffffu, base, 0);
                    if ((int64_t)base < p.R && lane == 0) {
                        s_q_base = base;
                        s_q_head = 0;
                        s_q_n = p.R - (int64_t)base < kSlots ? (int)(p.R - (int64_t)base) : kSlots;
                    }
                    if ((int64_t)base >= p.R && lane == 0) s_q_n = -1;
                    const int64_t r = (int64_t)base + lane;
                    if (r < p.R) {
                        uint64_t off;
                        int32_t nf, tl;
                        request_lengths(p, r, off, nf, tl);
                        s_q_off[lane] = off;
                        s_q_nfull[lane] = nf;
                        s_q_tail[lane] = tl;
                        s_q_seed[lane] = p.seeds[p.model_ids ? p.model_ids[r] : 0];
                    }
                    __syncwarp();
                    continue;
                }
                const int take = min(__popc(need), q_n - q_head);
                const int rank = __popc(need & ((1u << lane) - 1u));
                if (((need >> lane) & 1u) && rank < take) {
                    const int q = q_head + rank;
                    rid = (int32_t)(s_q_base + (uint32_t)q);
                    nfull = s_q_nfull[q];
                    s_off[lane] = s_q_off[q];
                    s_tail[lane] = s_q_tail[q];
                    prev = s_q_seed[q];
                    sb = StopBound();
                    st0 = first;
                    if (nfull == 0) finish();         // no full block: nothing for the ring
                }
                __syncwarp();                         // the queue entries are read before a ticket refills them
                if (lane == 0) s_q_head = q_head + take;
                __syncwarp();
            }
        };
        // Assigns the slot's next window (if any) to stage `stage`.
        auto assign = [&](int stage) {
            const int s = stage % kStages;
            const uint8_t *src = nullptr;
            int32_t n = 0;
            const int32_t w = stage - st0;
            if (rid >= 0 && w * W < nfull) {
                src = p.data + s_off[lane] + (uint64_t)w * W * (uint64_t)bs;
                n = min(W, nfull - w * W);
            }
            s_src[s][lane] = src;
            s_n[s][lane] = n;
        };
        // Once every request is taken and done, the last stage anybody runs is the last one already assigned.
        auto maybe_end = [&](int last) {
            if (end == INT32_MAX && s_q_n < 0 && !__any_sync(0xffffffffu, rid >= 0)) {
                end = last + 1;
                if (lane == 0) s_end = end;
            }
        };

        if (lane == 0) {
            s_q_head = s_q_n = 0;
            s_end = INT32_MAX;
        }
        __syncwarp();
        refill(0);
        for (int k = 0; k < kStages; k++) assign(k);
        maybe_end(-1);
        __syncthreads();
        for (int k = 0; k < end; k++) {
            const int s = k % kStages;
            bar_sync(kBarFull + s, kProducers);
            if (rid >= 0 && k >= st0) {       // window k - st0 of the slot's request is in the stage
                const int w = k - st0;
                prev = chain_window<W>(s_m[s][lane], p, p.hashes + (int64_t)rid * p.max_blocks, w, nfull, lenp8, prev,
                                       sb, n_stored);
                if ((w + 1) * W >= nfull || (skip && sb.bnd != INT32_MAX)) finish();
            }
            refill(k + kStages);
            assign(k + kStages);
            maybe_end(k + kStages - 1);
            bar_arrive(kBarEmpty + s, kProducers);
        }
        if (p.stored) {
            for (int o = 16; o; o >>= 1) n_stored += __shfl_xor_sync(0xffffffffu, n_stored, o);
            if (lane == 0 && n_stored) atomicAdd(p.stored, 8ull * n_stored);
        }
    }
    if (p.read) {                             // one atomic per warp and launch
        for (int o = 16; o; o >>= 1) n_read += __shfl_xor_sync(0xffffffffu, n_read, o);
        if (lane == 0 && n_read) atomicAdd(p.read, (unsigned long long)n_read);
    }
}

cudaError_t launch_hash_fused(const HashParams &p, int sm_count, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    if (!p.req_next) return cudaErrorInvalidValue;
    int dev = 0;
    cudaGetDevice(&dev);
    static int occ_dev[64] = {};                     // resident CTAs per SM, per device
    int &occ = occ_dev[dev & 63];
    if (!occ) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_hash_fused, 32 * kWin + 32, 0);
        if (occ < 1) occ = 1;
    }
    if (sm_count <= 0) sm_count = 132;
    const int64_t n_tiles = (p.R + kSlots - 1) / kSlots;
    const int grid = (int)(n_tiles < (int64_t)sm_count * occ ? n_tiles : (int64_t)sm_count * occ);
    cudaError_t e = cudaMemsetAsync(p.req_next, 0, sizeof(uint32_t), s);
    if (e != cudaSuccess) return e;
    k_hash_fused<<<grid, 32 * kWin + 32, 0, s>>>(p);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
