// inflight.cu -- the counters of the inflight-load producer (requestcontrol/dataproducer/inflightload/producer.go) on the
// device.
//
// The reference keeps two maps endpoint -> int64 (requests, estimated tokens): PreRequest (:110-129) adds 1 and the
// request's estimate to TargetEndpoints[0] of every profile result, ResponseBody (:131-168) takes them off again and an
// endpoint-delete event drops the entries (:86-97, 189-192).  The engine keeps one int64 pair per slot.  A scheduling
// call's adds are applied behind its last pick kernel by k_inflight_add; releases and resets are folded on the host and
// applied by k_inflight_apply at the start of the next call.  k_inflight_columns then writes the counters into the two
// f64 ext columns that the token-load and active-request scorers read (exact while |count| < 2^53).
#include "kernels.h"

namespace epp {

namespace {
// SimpleTokenEstimator.Estimate with RequestSizeBytes = L (token_estimator.go:55-56, 70-71): i = max(floor(L/4), 1),
// i + round(1.5 * i) with halves away from zero = 2i + ceil(i/2).
__device__ __forceinline__ int64_t inflight_est(int64_t L) {
    const int64_t i = L < 8 ? 1 : L / 4;
    return 2 * i + (i + 1) / 2;
}

// One thread per request, whole warps.  Stage k's endpoint of request r: its pick, prefill pick, encode pick.  Lanes with
// the same endpoint are merged by __match_any_sync and their leader adds the group's sums: a batch of cold requests
// under the lowest-slot tie rule puts every pick on one slot, and per-request atomics would serialise on it.
__global__ void __launch_bounds__(256) k_inflight_add(InflightState st, const epp_decision *dec, const epp_decision_detail *det,
                                                      const int64_t *in_len, int64_t R) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t ep[3] = {EPP_NO_ENDPOINT, EPP_NO_ENDPOINT, EPP_NO_ENDPOINT};
    int64_t tok = 0;
    if (r < R) {
        const epp_decision d = dec[r];
        if (d.status == 0) {                        // a Schedule error runs no PreRequest
            ep[0] = d.pick;
            ep[1] = d.prefill_pick;
            if (det) ep[2] = det[r].encode_pick;
            tok = inflight_est(in_len ? in_len[r] : 0);
        }
    }
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const uint32_t e = ep[k] < (uint32_t)st.E ? ep[k] : EPP_NO_ENDPOINT;
        const uint32_t peers = __match_any_sync(0xffffffffu, e);
        int64_t sum = 0;
        for (int j = 0; j < 32; j++) {
            const int64_t v = __shfl_sync(0xffffffffu, tok, j);
            if ((peers >> j) & 1u) sum += v;
        }
        if (e != EPP_NO_ENDPOINT && lane == __ffs(peers) - 1) {
            atomicAdd(reinterpret_cast<unsigned long long *>(st.req + e), (unsigned long long)__popc(peers));
            atomicAdd(reinterpret_cast<unsigned long long *>(st.tok + e), (unsigned long long)sum);
        }
    }
}

__global__ void k_inflight_apply(InflightState st, const InflightDelta *d, int32_t n) {
    const int32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const InflightDelta x = d[i];
    if (x.set) {
        st.req[x.slot] = x.req;
        st.tok[x.slot] = x.tok;
    } else {
        st.req[x.slot] += x.req;
        st.tok[x.slot] += x.tok;
    }
}

__global__ void k_inflight_columns(InflightState st) {
    const int32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= st.E) return;
    st.col_tok[e] = (double)st.tok[e];
    st.col_req[e] = (double)st.req[e];
}
}  // namespace

cudaError_t launch_inflight_add(const InflightState &st, const epp_decision *dec, const epp_decision_detail *det,
                                const int64_t *in_len, int64_t R, cudaStream_t s, int *launches) {
    if (R <= 0) return cudaSuccess;
    k_inflight_add<<<(unsigned)((R + 255) / 256), 256, 0, s>>>(st, dec, det, in_len, R);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_inflight_apply(const InflightState &st, const InflightDelta *d, int32_t n, cudaStream_t s, int *launches) {
    if (n <= 0) return cudaSuccess;
    k_inflight_apply<<<(n + 255) / 256, 256, 0, s>>>(st, d, n);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_inflight_columns(const InflightState &st, cudaStream_t s, int *launches) {
    k_inflight_columns<<<(st.E + 255) / 256, 256, 0, s>>>(st);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
