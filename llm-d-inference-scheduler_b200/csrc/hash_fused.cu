// hash_fused.cu -- a1 (hashPrompt, approximateprefix/hashing.go:35-99) as one CTA-cooperative kernel with register-fed
// 128-bit global loads: the DEFAULT hash kernel of the throughput path (block sizes that are a multiple of 32
// bytes, 16-byte aligned prompts; everything else takes the generic kernels of hash_kernels.cu).  hash_staged.cu is the
// cp.async-staged alternative behind EPP_HASH_STAGED=1 (DESIGN.md section 4.1).
//
// HBM traffic per request: every prompt byte is read exactly once, the 8-byte pre-chain digests never leave the SM
// (shared-memory ring), the block hashes are written once (the PluginState stash PreRequest needs, plugin.go:150-157).
//
// CTA = 9 warps, tile = 32 requests:
//   warps 0-7 (digest): thread (r = t/8, j = t%8) owns block k*8+j of request r in window k: 4 independent XXH64
//       accumulator chains over the block's 32-byte stripes, merge -> m, stored to the stage's [r][j] cell.
//   warp 8 (chain): lane = request.  Walks the window's 8 blocks in order (the only serial part of the digest:
//       m + len, one 8-byte round with h_{i-1}, avalanche), in place.
//   Stages are handed over with named barriers (bar.arrive / bar.sync), 4-deep ring of stages of TWO windows each: full
//   (digest -> chain), empty (chain -> digest).
#include "hash_blocks.cuh"
#include "kernels.h"

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

// Chain warp, one window: the serial part of the digest for 32 requests at once (lane = request); every lane then
// writes its request's 8 hashes straight from registers (64 bytes = two full sectors per lane, 128-bit stores when the
// row pitch allows) -- no transpose through shared memory.
template <int TR, int W = kWin>
__device__ __forceinline__ uint64_t chain_window(uint64_t (*sm)[W + 1], const int32_t *s_nfull, const HashParams &p,
                                                 int64_t r0, int k, int lane, int32_t nfull, uint64_t lenp8,
                                                 uint64_t prev) {
    (void)s_nfull;
    const int32_t n_here = min(W, nfull - k * W);              // hashes of this window for my request (<= 0: none)
    if (lane >= TR || n_here <= 0) return prev;
    uint64_t hv[W];
#pragma unroll
    for (int j = 0; j < W; j++) {
        if (j < n_here) prev = xxh_chain_step32(sm[lane][j], lenp8, prev);
        hv[j] = prev;
    }
    uint64_t *dst = p.hashes + (r0 + lane) * (int64_t)p.max_blocks + (int64_t)k * W;
    if (n_here == W && !(p.max_blocks & 1) && !(reinterpret_cast<uintptr_t>(p.hashes) & 15)) {   // the window starts 16-byte aligned
#pragma unroll
        for (int j = 0; j < W; j += 2)
            asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(dst + j), "l"(hv[j]), "l"(hv[j + 1]) : "memory");
    } else {
#pragma unroll
        for (int j = 0; j < W; j++)
            if (j < n_here) dst[j] = hv[j];
    }
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
            if (r < p.R) prev = p.seeds[p.model_ids ? p.model_ids[r] : 0];
            for (int k = 0; k < n_st; k++) {
                const int s = k % kStages;
                bar_sync(kBarFull + s, kProducers);
#pragma unroll
                for (int u = 0; u < kSub; u++)
                    prev = chain_window<TR, W>(s_m[s][u], s_nfull, p, r0, k * kSub + u, lane, nfull, lenp8, prev);
                bar_arrive(kBarEmpty + s, kProducers);
            }
            if (r < p.R) {                           // trailing partial block (hashing.go:90-96): generic tail, rare
                const int64_t eff = s_eff[lane];
                if ((int64_t)nfull * bs < eff)
                    p.hashes[r * (int64_t)p.max_blocks + nfull] = hash_block_generic(
                        p.data + s_off[lane] + (uint64_t)nfull * (uint64_t)bs, eff - (int64_t)nfull * bs, prev);
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
