// match_sparse.cu -- a2-a14 over the hash rows of a batch: the match / score / pick kernel of the throughput path (and of
// the endpoint-sharded mode): one warp per request, the per-request work is match_sparse.cuh.
#include "match_sparse.cuh"

namespace epp {

namespace {
constexpr int kWarps = 8;
}  // namespace

// MINCTA: resident CTAs per SM the register allocation is bounded for (8 -> 32 registers: 64 resident warps hide the
// probe latency; 6 -> 40 registers).  kTie / kStages: see match_sparse.cuh.
// Requests are taken dynamically: a warp's first request is its index in the grid, every further one comes off the
// launch's counter (p.req_next), so the warps that draw cheap (cold) prompts take more of them while the warps on long
// cached prefixes are busy, instead of the launch ending on the warps whose fixed share happened to be costliest.  The
// ticket is taken once the current request's probes are done, so the atomic's latency hides behind its scoring.
// kNoHit: the no-hit-lru builds (match_sparse.cuh match_request), launched as k_match_pick_sparse_nohit.
// kRand: the random-picker build (k_match_pick_sparse_rand).
template <bool kSharded, bool kTie, int kStages, bool kNoHit, bool kRand = false>
__device__ __forceinline__ void match_pick_sparse(const PickParams &p) {
    __shared__ sparse::Work s_work[kWarps];           // when counting
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t nwarps = gridDim.x * kWarps;
    const uint32_t R = (uint32_t)p.R;                  // < 2^31 (launch_match_pick_sparse)
    const bool counting = p.work_counters != nullptr;
    sparse::Work *wk = &s_work[warp];
    if (counting) {
        wk->postings[lane] = 0;
        if (lane == 0) wk->probes = 0;
    }
    uint32_t r = blockIdx.x * kWarps + warp;
    while (r < R) {
        int32_t ticket = 0;
        sparse::match_request<false, kSharded, kTie, kStages, sparse::NoFollow, kNoHit, kRand>(p, r, lane, counting, wk, p.req_next, ticket);
        r = nwarps + (uint32_t)__shfl_sync(0xffffffffu, ticket, 0);
    }
    if (counting) {
        unsigned long long postings = wk->postings[lane];
        for (int o = 16; o; o >>= 1) postings += __shfl_xor_sync(0xffffffffu, postings, o);
        if (lane == 0) {
            atomicAdd(&p.work_counters[0], wk->probes);
            atomicAdd(&p.work_counters[1], postings);
        }
    }
}

template <int MINCTA, bool kSharded, bool kTie, int kStages>
__global__ void __launch_bounds__(kWarps * 32, MINCTA) k_match_pick_sparse(PickParams p) {
    match_pick_sparse<kSharded, kTie, kStages, false>(p);
}
template <int MINCTA, bool kTie, int kStages>
__global__ void __launch_bounds__(kWarps * 32, MINCTA) k_match_pick_sparse_nohit(PickParams p) {
    match_pick_sparse<false, kTie, kStages, true>(p);
}
// Engines where some profile has a random picker: one build for every handler shape, tie rule and no-hit-lru setting
// (each is a run-time branch here: nohit_select reads a zero mask as "no scorer").
__global__ void __launch_bounds__(kWarps * 32, 6) k_match_pick_sparse_rand(PickParams p) {
    match_pick_sparse<false, true, 3, true, true>(p);
}

// The seeded sharded select (include/epp_engine.h "Seeded ties"): one warp per work item of k_shard_resolve, the items
// taken in grid stride (their count is on the device).
__global__ void __launch_bounds__(kWarps * 32, 6) k_match_pick_sparse_select(PickParams p, ShardSelView sv) {
    const int lane = threadIdx.x & 31;
    const int32_t nwarps = (int32_t)(gridDim.x * kWarps);
    const int32_t n = *sv.work_n;
    for (int32_t wi = (int32_t)(blockIdx.x * kWarps + (threadIdx.x >> 5)); wi < n; wi += nwarps) {
        int32_t ticket = 0;
        sparse::match_request<false, true, true, 1, sparse::NoFollow, false, false, true>(
            p, sv.work[wi].x / (uint32_t)sv.stages, lane, false, nullptr, nullptr, ticket, sparse::NoFollow(), &sv, wi);
    }
}

namespace {
template <void (*kernel)(PickParams)>
cudaError_t launch_kernel(const PickParams &p, int sm_count, cudaStream_t s) {
    int dev = 0;
    cudaGetDevice(&dev);
    static int occ_dev[64] = {};                       // per kernel and device: engines of one process may sit on different GPUs
    int &occ = occ_dev[dev & 63];
    if (!occ) {
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kWarps * 32, 0);
        if (occ < 1) occ = 1;
    }
    if (sm_count <= 0) sm_count = 132;
    const int64_t need = (p.R + kWarps - 1) / kWarps;
    const int grid = (int)(need < (int64_t)sm_count * occ ? need : (int64_t)sm_count * occ);
    kernel<<<grid, kWarps * 32, 0, s>>>(p);
    return cudaGetLastError();
}
template <int MINCTA, bool kSharded, bool kTie, int kStages>
cudaError_t launch_one(const PickParams &p, int sm_count, cudaStream_t s) {
    return launch_kernel<k_match_pick_sparse<MINCTA, kSharded, kTie, kStages>>(p, sm_count, s);
}
template <bool kTie, int kStages>
cudaError_t launch_nohit(const PickParams &p, int sm_count, cudaStream_t s) {
    return launch_kernel<k_match_pick_sparse_nohit<6, kTie, kStages>>(p, sm_count, s);
}
}  // namespace

cudaError_t launch_match_pick_sparse_select(const PickParams &p, const ShardSelView &sv, int sm_count, cudaStream_t s,
                                            int *launches) {
    const int64_t items = p.R * (int64_t)sv.stages;          // at most one item per request and stage
    if (items <= 0) return cudaSuccess;
    if (sm_count <= 0) sm_count = 132;
    const int64_t need = (items + kWarps - 1) / kWarps;
    const int grid = (int)(need < (int64_t)sm_count * 6 ? need : (int64_t)sm_count * 6);
    k_match_pick_sparse_select<<<grid, kWarps * 32, 0, s>>>(p, sv);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_match_pick_sparse(const PickParams &p, int sm_count, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    if (!p.req_next || p.R > INT32_MAX) return cudaErrorInvalidValue;
    const bool tie = p.tie_seed != 0;
    const int stages = handler_stages(p);
    cudaError_t e;
    // the hot configuration (one profile, lowest-slot ties) gets the 32-register build; the variants that carry more
    // code (stages, tie rule, sharding) keep 40 registers.  The sharded builds write one record per stage and always
    // take the lowest slot.
    if (p.global_masks) {
        if (stages == 1) e = launch_one<6, true, false, 1>(p, sm_count, s);
        else if (stages == 2) e = launch_one<6, true, false, 2>(p, sm_count, s);
        else e = launch_one<6, true, false, 3>(p, sm_count, s);
    }
    else if (any_random_picker(p)) e = launch_kernel<k_match_pick_sparse_rand>(p, sm_count, s);
    else if (p.nohit.mask) {
        if (stages == 1) e = tie ? launch_nohit<true, 1>(p, sm_count, s) : launch_nohit<false, 1>(p, sm_count, s);
        else if (stages == 2) e = tie ? launch_nohit<true, 2>(p, sm_count, s) : launch_nohit<false, 2>(p, sm_count, s);
        else e = tie ? launch_nohit<true, 3>(p, sm_count, s) : launch_nohit<false, 3>(p, sm_count, s);
    }
    else if (stages == 1 && !tie) e = launch_one<8, false, false, 1>(p, sm_count, s);
    else if (stages == 1) e = launch_one<6, false, true, 1>(p, sm_count, s);
    else if (stages == 2) e = tie ? launch_one<6, false, true, 2>(p, sm_count, s) : launch_one<6, false, false, 2>(p, sm_count, s);
    else e = tie ? launch_one<6, false, true, 3>(p, sm_count, s) : launch_one<6, false, false, 3>(p, sm_count, s);
    if (launches) *launches += 1;
    return e;
}

}  // namespace epp
