// hash_staged.cu -- a1 (hashPrompt, approximateprefix/hashing.go:35-99) with the prompt bytes staged through shared
// memory by cp.async and NO cross-warp synchronisation: one warp = one task of TR (16 or 32) requests.
//
//   digest phase, TR/4 sub-windows per window: sub-window g covers requests 4g..4g+3 x 8 blocks of 64 bytes (lane l:
//       request 4g + l/8, block l%8): four independent XXH64 accumulator chains over the block's two 32-byte stripes,
//       merge -> the 8-byte pre-chain digest m into the warp's own [TR][9] shared-memory tile.  The bytes come from the
//       warp's PRIVATE ring of DS sub-window slots (2 KiB each) filled by 16-byte cp.async (LDGSTS): one warp
//       instruction copies 512 contiguous bytes of one request; the 16-byte pieces are stored with an XOR swizzle so
//       that both the LDGSTS writes and the 128-bit shared loads are bank-conflict free.  Producer and consumer are
//       the same warp: the only synchronisation is cp.async.wait_group + __syncwarp, and DS-1 sub-windows stay in
//       flight per warp whatever the warp is doing.
//   chain phase: lane = request; the serial part of the digest (m + len, one 8-byte round with h_{i-1}, avalanche) for
//       TR requests per instruction, 8 steps per window; hashes written as 64-byte segments (the PluginState stash
//       PreRequest needs, plugin.go:150-157).
//
// Why this shape: in the CTA-cooperative kernels (hash_fused.cu
// and three staged variants of it) ONE chain warp per CTA carries the serial ~25-instruction dependency chain per
// block for 32 requests, and at 3-4 CTAs per SM those 3-4 latency-bound streams plus the named-barrier hand-over bound
// the kernel.  Here every warp chains its own requests and the chain phase of one warp overlaps the digest phases of
// its neighbours without any barrier.
// Fast path only: block_bytes == 64 and 16-byte aligned prompts (every BASELINE config); other shapes take
// hash_fused.cu / hash_kernels.cu.
#include "kernels.h"
#include "xxh64.cuh"

namespace epp {

namespace {
constexpr int kWin = 8;                    // blocks per window
constexpr int kBlock = 64;                 // bytes per block on this path
constexpr int kRowBytes = kWin * kBlock;   // 512: one request's bytes of one window
constexpr int kSlot = 4 * kRowBytes;       // one sub-window: 4 requests x 512 B
constexpr int kPitch = kWin + 1;           // u64 cells per request row (odd pitch: conflict-free lane = request reads)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void lds128(uint32_t addr, uint64_t &a, uint64_t &b) {
    asm volatile("ld.shared.v2.u64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "r"(addr) : "memory");
}

template <int TR>
struct TaskSmem {
    uint64_t m[TR][kPitch];
    uint64_t off[TR];
    int32_t nfull[TR];
};
}  // namespace

template <int TR, int DS, int WPC>
__global__ void __launch_bounds__(32 * WPC) k_hash_staged(HashParams p, int n_tasks) {
    extern __shared__ __align__(128) uint8_t s_dyn[];           // per warp: [DS] sub-window slots, then TaskSmem
    constexpr int kSub = TR / 4;                                 // sub-windows per window
    constexpr uint32_t kRing = DS * kSlot;
    constexpr uint32_t kPerWarp = kRing + (uint32_t)((sizeof(TaskSmem<TR>) + 127) & ~127u);
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int task = blockIdx.x * WPC + warp;
    if (task >= n_tasks) return;
    uint8_t *mine = s_dyn + (size_t)warp * kPerWarp;
    const uint32_t ring = smem_u32(mine);
    TaskSmem<TR> &ws = *reinterpret_cast<TaskSmem<TR> *>(mine + kRing);

    // ---- per-request lengths (hashing.go:58-66), lane = request
    const int64_t r0 = (int64_t)task * TR;
    const int64_t r = r0 + lane;
    const bool owner = lane < TR && r < p.R;
    uint64_t off = 0;
    int64_t eff = 0;
    int32_t nfull = 0;
    if (owner) {
        uint64_t len;
        if (p.offsets) { off = p.offsets[r]; len = p.lengths ? p.lengths[r] : p.offsets[r + 1] - off; }
        else { off = (uint64_t)r * p.uniform_len; len = p.uniform_len; }
        if (p.in_len) p.in_len[r] = (int64_t)len;
        eff = (int64_t)len;
        int32_t nb = 0;
        if (eff < kBlock) {
            eff = 0;
        } else {
            const int64_t cap = (int64_t)kBlock * (int64_t)p.max_blocks;
            if (eff > cap) eff = cap;
            nfull = (int32_t)(eff / kBlock);
            nb = nfull + ((eff % kBlock) ? 1 : 0);
        }
        p.nblocks[r] = nb;
        p.eff_len[r] = eff;
    }
    if (lane < TR) {
        ws.off[lane] = off;
        ws.nfull[lane] = nfull;
    }
    int mx = nfull, mn = lane < TR ? nfull : 0x7fffffff;
    for (int o = 16; o; o >>= 1) {
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    }
    __syncwarp();
    const int n_win = (mx + kWin - 1) / kWin;
    const int n_sub = n_win * kSub;                              // sub-window u = kSub * window + request group
    const int full_sub = (mn / kWin) * kSub;                     // sub-windows below this need no per-row length checks

    const uint64_t lenp8 = (uint64_t)kBlock + 8;
    const int q = lane >> 3, j = lane & 7;
    // this lane's copy target inside a row: 16-byte piece `lane` of the 512-byte row = piece lane%4 of block lane/4,
    // stored at piece position (lane%4) ^ ((lane/8) & 3)  [= piece ^ (block >> 1)]; its read position: block j of row q,
    // piece c at ((c ^ (j >> 1)) << 4)
    const uint32_t cp_dst = (uint32_t)((lane >> 2) * kBlock + (((lane & 3) ^ ((lane >> 3) & 3)) << 4));
    const uint32_t rd_row = (uint32_t)(q * kRowBytes + j * kBlock);
    const uint32_t sw = (uint32_t)((j >> 1) & 3);
    const uint8_t *lane_src = p.data + 16 * lane;

    auto issue = [&](int u) {                                    // one sub-window = 4 request rows x 512 B, one commit group
        if (u < n_sub) {
            const int k = u / kSub, g = u % kSub;
            const uint32_t dst = ring + (uint32_t)(u % DS) * (uint32_t)kSlot + cp_dst;
            const uint8_t *src = lane_src + (uint64_t)k * (uint64_t)kRowBytes;
            if (u < full_sub) {
#pragma unroll
                for (int qq = 0; qq < 4; qq++) cp_async16(dst + qq * kRowBytes, src + ws.off[4 * g + qq]);
            } else {
                const int blk = k * kWin + (lane >> 2);
#pragma unroll
                for (int qq = 0; qq < 4; qq++)
                    if (blk < ws.nfull[4 * g + qq]) cp_async16(dst + qq * kRowBytes, src + ws.off[4 * g + qq]);
            }
        }
        cp_async_commit();
    };

#pragma unroll
    for (int u = 0; u < DS - 1; u++) issue(u);
    uint64_t prev = 0;
    if (owner) prev = p.seeds[p.model_ids ? p.model_ids[r] : 0];
    for (int k = 0; k < n_win; k++) {
        // ---- digest phase
#pragma unroll 1
        for (int g = 0; g < kSub; g++) {
            const int u = k * kSub + g;
            cp_async_wait<DS - 2>();                             // sub-window u has landed (this lane's copies)
            __syncwarp();                                        // ... everybody's; sub-window u-1 is fully consumed
            issue(u + DS - 1);
            const int row = 4 * g + q;
            if (k * kWin + j < ws.nfull[row]) {
                const uint32_t a = ring + (uint32_t)(u % DS) * (uint32_t)kSlot + rd_row;
                uint64_t v[4], x[4];
                xxh_init(v);
                lds128(a + ((0u ^ sw) << 4), x[0], x[1]);
                lds128(a + ((1u ^ sw) << 4), x[2], x[3]);
#pragma unroll
                for (int c = 0; c < 4; c++) v[c] = xxh_round(v[c], x[c]);
                lds128(a + ((2u ^ sw) << 4), x[0], x[1]);
                lds128(a + ((3u ^ sw) << 4), x[2], x[3]);
#pragma unroll
                for (int c = 0; c < 4; c++) v[c] = xxh_round(v[c], x[c]);
                ws.m[row][j] = xxh_merge_all(v);
            }
        }
        __syncwarp();
        // ---- chain phase: lane = request
        if (lane < TR) {
#pragma unroll
            for (int jj = 0; jj < kWin; jj++) {
                if (k * kWin + jj < nfull) {
                    prev = xxh_chain_step32_lat(ws.m[lane][jj], lenp8, prev);
                    ws.m[lane][jj] = prev;
                }
            }
        }
        __syncwarp();
        // the 8 hashes of each request's window = one 64-byte segment; four request rows per instruction
#pragma unroll
        for (int it = 0; it < kSub; it++) {
            const int row = it * 4 + q;
            const int b = k * kWin + j;
            if (b < ws.nfull[row]) p.hashes[(r0 + row) * (int64_t)p.max_blocks + b] = ws.m[row][j];
        }
        __syncwarp();
    }
    cp_async_wait<0>();
    if (owner && (int64_t)nfull * kBlock < eff)                  // trailing partial block (hashing.go:90-96): rare
        p.hashes[r * (int64_t)p.max_blocks + nfull] =
            hash_block_generic(p.data + off + (uint64_t)nfull * (uint64_t)kBlock, eff - (int64_t)nfull * kBlock, prev);
}



namespace {
template <int TR, int DS, int WPC>
cudaError_t launch_shape(const HashParams &p, cudaStream_t s) {
    auto kernel = k_hash_staged<TR, DS, WPC>;
    constexpr size_t kPerWarp = (size_t)DS * kSlot + ((sizeof(TaskSmem<TR>) + 127) & ~(size_t)127);
    const size_t dyn = WPC * kPerWarp;
    static size_t dyn_set[64] = {};                              // per device (one static per instantiation)
    int dev = 0;
    cudaGetDevice(&dev);
    dev &= 63;
    if (dyn_set[dev] < dyn) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
        if (e != cudaSuccess) return e;
        dyn_set[dev] = dyn;
    }
    const int n_tasks = (int)((p.R + TR - 1) / TR);
    kernel<<<(n_tasks + WPC - 1) / WPC, 32 * WPC, dyn, s>>>(p, n_tasks);
    return cudaGetLastError();
}
}  // namespace

bool hash_staged_supported(const HashParams &p) {
    if (p.block_bytes != kBlock) return false;
    uint64_t bits = reinterpret_cast<uintptr_t>(p.data);
    bits |= p.offsets ? p.offsets_or_bits : p.uniform_len;
    return (bits & 15) == 0;
}

// shape: 1 = default (1644); else requests per task * 100 + ring slots * 10 + warps per CTA (A/B runs).
cudaError_t launch_hash_staged(const HashParams &p, int shape, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    cudaError_t e;
    switch (shape) {
        case 3244: e = launch_shape<32, 4, 4>(p, s); break;
        case 1634: e = launch_shape<16, 3, 4>(p, s); break;
        default: e = launch_shape<16, 4, 4>(p, s); break;      // 1644
    }
    if (launches) *launches += 1;
    return e;
}

}  // namespace epp
