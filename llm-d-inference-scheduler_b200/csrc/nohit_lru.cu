// nohit_lru.cu -- the state of the no-hit-lru scorer (scorer/nohitlru/no_hit_lru.go) on the device.
//
// The reference keeps a golang-lru cache of endpoint names and Adds the targets of every cold request in PreRequest
// (:279-321).  After any sequence of Adds that cache holds the lruSize most recently Added distinct endpoints, ordered by
// their last Add, so the engine keeps one number per slot instead of a list: last_seq[e] = the sequence number of e's
// last Add (0 = not in the LRU).  A scheduling call with R requests owns the numbers seq0 + [0, 2R): request r's pick is
// Added as seq0 + 2r and its prefill pick as seq0 + 2r + 1, so atomicMax over the whole batch leaves exactly what the
// Adds in request order would.  Then the members are ranked by last_seq (k_pool_sort), all but the lruSize newest are
// dropped, and every profile with the scorer re-derives its cold column and its cold base / order / groups
// (launch_pool_order).  Every kernel after the touch returns at once when no request of the call was cold.
#include "kernels.h"

namespace epp {

namespace {
constexpr uint64_t kNoMember = 0xFFFFFFFFFFFFFFFFULL;

__global__ void k_nohit_touch(NoHitState st, const epp_decision *dec, const uint8_t *cold, int64_t R, uint64_t seq0) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || !cold[r]) return;
    const epp_decision d = dec[r];
    if (d.status != 0 || d.pick == EPP_NO_ENDPOINT) return;
    atomicMax(reinterpret_cast<unsigned long long *>(st.last_seq + d.pick), (unsigned long long)(seq0 + 2 * (uint64_t)r));
    if (d.prefill_pick != EPP_NO_ENDPOINT)
        atomicMax(reinterpret_cast<unsigned long long *>(st.last_seq + d.prefill_pick), (unsigned long long)(seq0 + 2 * (uint64_t)r + 1));
    *st.dirty = 1;
}

// Sort keys: members by last_seq ascending (oldest first), then every other slot.
__global__ void k_nohit_keys(NoHitState st, int32_t E, int32_t Epad, int32_t gated) {
    if (gated && !*st.dirty) return;
    const int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= Epad) return;
    const uint64_t s = k < E ? st.last_seq[k] : 0;
    st.sort_key[k] = s ? s : kNoMember;
    st.order[k] = (uint32_t)k;
}

// Capacity (golang-lru evicts the oldest beyond its size) and positions, oldest = 0.  One CTA.
__global__ void __launch_bounds__(1024) k_nohit_trim(NoHitState st, int32_t E, int32_t Epad, int32_t gated) {
    if (gated && !*st.dirty) return;
    __shared__ int32_t s_m;
    if (threadIdx.x == 0) s_m = 0;
    for (int32_t e = threadIdx.x; e < E; e += blockDim.x) st.pos[e] = -1;
    __syncthreads();
    for (int32_t k = threadIdx.x; k < Epad; k += blockDim.x)   // members form a prefix of the sorted keys
        if (st.sort_key[k] != kNoMember && (k + 1 == Epad || st.sort_key[k + 1] == kNoMember)) s_m = k + 1;
    __syncthreads();
    const int32_t m = s_m;
    const int32_t drop = m > st.lru_size ? m - st.lru_size : 0;
    for (int32_t k = threadIdx.x; k < m; k += blockDim.x) {
        const uint32_t e = st.order[k];
        if (k < drop) st.last_seq[e] = 0;
        else st.pos[e] = k - drop;
    }
    if (threadIdx.x == 0) *st.n_members = m - drop;
}

// scoreColdRequestByLRU (no_hit_lru.go:198-242) over the candidates in ascending slot order.  One CTA.
__global__ void __launch_bounds__(1024) k_nohit_column(NoHitState st, int32_t E, const uint8_t *cand, const int32_t *n_cand,
                                                       double *col, int32_t gated) {
    if (gated && !*st.dirty) return;
    __shared__ int32_t s_warp[32];
    __shared__ int32_t s_nu;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int32_t n = *n_cand;
    if (threadIdx.x == 0) s_nu = 0;
    __syncthreads();
    int32_t nu = 0;                                  // never-used candidates
    for (int32_t e = threadIdx.x; e < E; e += blockDim.x) nu += (cand[e] && st.pos[e] < 0) ? 1 : 0;
    atomicAdd(&s_nu, nu);
    __syncthreads();
    const int32_t nu_all = s_nu;
    const double denom = (double)(n - 1);
    int32_t carry = 0;                               // never-used candidates below the current chunk
    for (int32_t e0 = 0; e0 < E; e0 += blockDim.x) {
        const int32_t e = e0 + threadIdx.x;
        const bool c = e < E && cand[e];
        const bool never = c && st.pos[e] < 0;
        const uint32_t bal = __ballot_sync(0xffffffffu, never);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int32_t before = carry;
        for (int w = 0; w < warp; w++) before += s_warp[w];
        before += __popc(bal & ((1u << lane) - 1u));
        int32_t chunk = 0;
        for (int w = 0; w < nw; w++) chunk += s_warp[w];
        if (e < E) {
            double v = 0.0;
            if (c) {
                if (n <= 1) v = 1.0;                                                  // :239-242
                else if (never) v = __dsub_rn(1.0, __ddiv_rn((double)before, denom));  // :198-207
                else {                                                                // :211-229
                    v = __dsub_rn(1.0, __ddiv_rn((double)(nu_all + st.pos[e]), denom));
                    if (v < 0) v = 0;
                }
            }
            col[e] = v;
        }
        carry += chunk;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_nohit_cold_rows(int64_t R, int32_t E, const uint8_t *cand, const int32_t *match,
                                                         uint8_t *cold) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= R) return;
    const int32_t *row = match + r * (int64_t)E;
    bool hit = false;
    for (int32_t e = lane; e < E && !hit; e += 32) hit = cand[e] && row[e] > 0;
    const bool any = __any_sync(0xffffffffu, hit);
    if (lane == 0) cold[r] = any ? 0 : 1;
}
}  // namespace

cudaError_t launch_nohit_touch(const NoHitState &st, const epp_decision *dec, const uint8_t *cold, int64_t R, uint64_t seq0,
                               cudaStream_t s, int *launches) {
    if (R <= 0) return cudaSuccess;
    k_nohit_touch<<<(unsigned)((R + 255) / 256), 256, 0, s>>>(st, dec, cold, R, seq0);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_nohit_rank(const NoHitState &st, int32_t E, int32_t Epad, bool gated, cudaStream_t s, int *launches) {
    k_nohit_keys<<<(Epad + 255) / 256, 256, 0, s>>>(st, E, Epad, gated ? 1 : 0);
    cudaError_t e = launch_pool_sort(st.sort_key, st.order, Epad, gated ? st.dirty : nullptr, s);
    if (e != cudaSuccess) return e;
    k_nohit_trim<<<1, 1024, 0, s>>>(st, E, Epad, gated ? 1 : 0);
    if (launches) *launches += 3;
    return cudaGetLastError();
}

cudaError_t launch_nohit_column(const NoHitState &st, int32_t E, const uint8_t *cand, const int32_t *n_cand, double *col,
                                bool gated, cudaStream_t s, int *launches) {
    k_nohit_column<<<1, 1024, 0, s>>>(st, E, cand, n_cand, col, gated ? 1 : 0);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_nohit_clear(const NoHitState &st, cudaStream_t s, int *) {
    return cudaMemsetAsync(st.dirty, 0, sizeof(int32_t), s);
}

cudaError_t launch_nohit_cold_rows(int64_t R, int32_t E, const uint8_t *cand, const int32_t *match, uint8_t *cold,
                                   cudaStream_t s, int *launches) {
    if (R <= 0) return cudaSuccess;
    k_nohit_cold_rows<<<(unsigned)((R * 32 + 255) / 256), 256, 0, s>>>(R, E, cand, match, cold);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
