// hash_fused.cu -- a1 (hashPrompt, approximateprefix/hashing.go:35-99) as one CTA-cooperative kernel with register-fed
// 128-bit global loads: the DEFAULT hash kernel of the throughput path (block sizes that are a multiple of 32
// bytes, 16-byte aligned prompts; everything else takes the generic kernels of hash_kernels.cu).  hash_staged.cu is the
// cp.async-staged alternative behind EPP_HASH_STAGED=1 (DESIGN.md section 4.1).
//
// HBM traffic per request: every prompt byte is read exactly once, the 8-byte pre-chain digests never leave the SM
// (shared-memory ring), the block hashes are written once (the PluginState stash PreRequest needs, plugin.go:150-157)
// -- or, with a presence bitmap (HashParams::presence), only up to the first block no endpoint can hold: the match
// kernel's global stop never lies beyond it.
//
// CTA = 9 warps, tile = 32 requests:
//   warps 0-7 (digest): thread (r = t/8, j = t%8) owns block k*8+j of request r in window k: 4 independent XXH64
//       accumulator chains over the block's 32-byte stripes, merge -> m, stored to the stage's [r][j] cell.
//   warp 8 (chain): lane = request.  Walks the window's 8 blocks in order (the only serial part of the digest:
//       m + len, one 8-byte round with h_{i-1}, avalanche), in place.
//   Stages are handed over with named barriers (bar.arrive / bar.sync), 4-deep ring of stages of TWO windows each: full
//   (digest -> chain), empty (chain -> digest).
#include "hash_blocks.cuh"
#include "index.cuh"

namespace epp {

namespace {
constexpr int kWin = 8;
constexpr int kStages = 4;
constexpr int kSub = 2;                   // windows per ring stage (one barrier hand-over per kSub windows)
constexpr int kBarFull = 1;               // named barrier ids 1..4
constexpr int kBarEmpty = 1 + kStages;    // 5..8
constexpr int kHashMinCtas = 4;

__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Per-request lengths (hashing.go:58-66) for one tile; called by the first warp.
__device__ __forceinline__ void tile_lengths(const HashParams &p, int64_t r0, int t, uint64_t *s_off, int64_t *s_eff,
                                             int32_t *s_nfull, int32_t *s_maxfull) {
    const int64_t bs = p.block_bytes;
    const int64_t r = r0 + t;
    uint64_t off = 0;
    int64_t eff = 0;
    int32_t nfull = 0;
    if (r < p.R) {
        uint64_t len;
        if (p.offsets) { off = p.offsets[r]; len = p.lengths ? p.lengths[r] : p.offsets[r + 1] - off; }
        else { off = (uint64_t)r * p.uniform_len; len = p.uniform_len; }
        if (p.in_len) p.in_len[r] = (int64_t)len;
        eff = (int64_t)len;
        int32_t nb = 0;
        if (eff < bs) {
            eff = 0;
        } else {
            const int64_t cap = bs * (int64_t)p.max_blocks;
            if (eff > cap) eff = cap;
            nfull = (int32_t)(eff / bs);
            nb = nfull + ((eff % bs) ? 1 : 0);
        }
        p.nblocks[r] = nb;
        p.eff_len[r] = eff;
    }
    s_off[t] = off;
    s_eff[t] = eff;
    s_nfull[t] = nfull;
    int mx = nfull;
    for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (t == 0) *s_maxfull = mx;
}

// Per-lane stop bound of the chain warp: the first window whose leading block reads as absent in the presence bitmap
// (one lookup per window of W blocks).  The word is loaded right after the window is chained and examined only once the
// NEXT window has been chained, so the L2 latency hides behind that work instead of stalling the ring; a window is
// stored while no earlier one has been proven absent, so a row may run up to W - 1 hashes past its bound (never read).
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

// Chain warp, one window: the serial part of the digest for 32 requests at once (lane = request); every lane then
// writes its request's 8 hashes straight from registers (64 bytes = two full sectors per lane, 128-bit stores when the
// row pitch allows) -- no transpose through shared memory.  With p.presence, hashes at or past a proven-absent block
// are not stored (the match kernel never reads past it); every hash is still computed.
template <int TR, int W = kWin>
__device__ __forceinline__ uint64_t chain_window(uint64_t (*sm)[W + 1], const HashParams &p, int64_t r0, int k,
                                                 int lane, int32_t nfull, uint64_t lenp8, uint64_t prev,
                                                 StopBound &sb, uint32_t &n_stored) {
    const int32_t n_here = min(W, nfull - k * W);              // hashes of this window for my request (<= 0: none)
    if (lane >= TR || n_here <= 0) return prev;
    uint64_t hv[W];
#pragma unroll
    for (int j = 0; j < W; j++) {
        if (j < n_here) prev = xxh_chain_step32(sm[lane][j], lenp8, prev);
        hv[j] = prev;
    }
    if (sb.pending >= 0) sb.resolve();                         // the previous window's word has had this window's time
    const int32_t n_store = min(n_here, sb.bnd - k * W);
    if (n_store <= 0) return prev;
    n_stored += (uint32_t)n_store;
    uint64_t *dst = p.hashes + (r0 + lane) * (int64_t)p.max_blocks + (int64_t)k * W;
    if (n_store == W && !(p.max_blocks & 1) && !(reinterpret_cast<uintptr_t>(p.hashes) & 15)) {   // the window starts 16-byte aligned
#pragma unroll
        for (int j = 0; j < W; j += 2)
            asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(dst + j), "l"(hv[j]), "l"(hv[j + 1]) : "memory");
    } else {
#pragma unroll
        for (int j = 0; j < W; j++)
            if (j < n_store) dst[j] = hv[j];
    }
    if (p.presence && sb.bnd == INT32_MAX) sb.issue(p, k * W, hv[0]);        // closed requests issue no loads
    return prev;
}
}  // namespace

__global__ void __launch_bounds__(32 * kWin + 32, kHashMinCtas) k_hash_fused(HashParams p, int n_tiles) {
    constexpr int TR = 32, W = kWin;
    constexpr int kDigestWarps = TR * W / 32;
    constexpr int kProducers = TR * W + 32;
    __shared__ uint64_t s_m[kStages][kSub][TR][(W + 1)];
    __shared__ uint64_t s_off[TR];
    __shared__ int64_t s_eff[TR];
    __shared__ int32_t s_nfull[TR];
    __shared__ int32_t s_maxfull;

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int t = threadIdx.x;
    const int64_t bs = p.block_bytes;
    const int n_stripes = (int)(bs >> 5);
    const uint64_t lenp8 = (uint64_t)bs + 8;

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t r0 = (int64_t)tile * TR;
        if (t < 32) tile_lengths(p, r0, t, s_off, s_eff, s_nfull, &s_maxfull);
        __syncthreads();
        const int n_win = (s_maxfull + W - 1) / W;
        const int n_st = (n_win + kSub - 1) / kSub;                              // ring hand-overs of this tile

        if (warp < kDigestWarps) {
            const int r = t / W, j = t % W;
            const int32_t nfull = s_nfull[r];
            const uint8_t *src = p.data + s_off[r] + (uint64_t)j * (uint64_t)bs;     // block j of window 0; + W blocks per window
            const uint64_t win_bytes = (uint64_t)W * (uint64_t)bs;
            int32_t left = nfull - j;                                            // > 0: my block of this window is a full one
            for (int k = 0; k < n_st; k++) {
                const int s = k % kStages;
                if (k >= kStages) bar_sync(kBarEmpty + s, kProducers);
#pragma unroll
                for (int u = 0; u < kSub; u++, src += win_bytes, left -= W)
                    if (left > 0) s_m[s][u][r][j] = block_digest(src, n_stripes);
                bar_arrive(kBarFull + s, kProducers);     // bar.arrive orders the stores above for the threads of the barrier
            }
            const int first = n_st > kStages ? n_st - kStages : 0;
            for (int k = first; k < n_st; k++) bar_sync(kBarEmpty + (k % kStages), kProducers);
        } else {
            const int64_t r = r0 + lane;
            const int32_t nfull = s_nfull[lane];
            uint64_t prev = 0;
            StopBound sb;
            uint32_t n_stored = 0;
            if (r < p.R) prev = p.seeds[p.model_ids ? p.model_ids[r] : 0];
            for (int k = 0; k < n_st; k++) {
                const int s = k % kStages;
                bar_sync(kBarFull + s, kProducers);
#pragma unroll
                for (int u = 0; u < kSub; u++)
                    prev = chain_window<TR, W>(s_m[s][u], p, r0, k * kSub + u, lane, nfull, lenp8, prev, sb, n_stored);
                bar_arrive(kBarEmpty + s, kProducers);
            }
            if (sb.pending >= 0) sb.resolve();
            int32_t &bnd = sb.bnd;
            if (r < p.R) {                           // trailing partial block (hashing.go:90-96): generic tail, rare
                const int64_t eff = s_eff[lane];
                int32_t nb = nfull;
                if ((int64_t)nfull * bs < eff) {
                    nb++;
                    const uint64_t h = hash_block_generic(p.data + s_off[lane] + (uint64_t)nfull * (uint64_t)bs,
                                                          eff - (int64_t)nfull * bs, prev);
                    if (bnd == INT32_MAX && p.presence && !presence_maybe(p.presence, p.presence_shift, h)) bnd = nfull;
                    if (nfull < bnd) {
                        p.hashes[r * (int64_t)p.max_blocks + nfull] = h;
                        n_stored++;
                    }
                }
                if (p.presence) p.bound[r] = min(bnd, nb);
            }
            if (p.stored) {
                for (int o = 16; o; o >>= 1) n_stored += __shfl_xor_sync(0xffffffffu, n_stored, o);
                if (lane == 0) atomicAdd(p.stored, 8ull * n_stored);
            }
        }
        __syncthreads();
    }
}

cudaError_t launch_hash_fused(const HashParams &p, int sm_count, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    int dev = 0;
    cudaGetDevice(&dev);
    static int occ_dev[64] = {};                     // resident CTAs per SM, per device
    int &occ = occ_dev[dev & 63];
    if (!occ) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_hash_fused, 32 * kWin + 32, 0);
        if (occ < 1) occ = 1;
    }
    if (sm_count <= 0) sm_count = 132;
    const int n_tiles = (int)((p.R + 31) / 32);
    const int grid = n_tiles < sm_count * occ ? n_tiles : sm_count * occ;
    k_hash_fused<<<grid, 32 * kWin + 32, 0, s>>>(p, n_tiles);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
