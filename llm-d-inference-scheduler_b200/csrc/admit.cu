// admit.cu -- the Admitter plugins of the request-control layer on the device: the latency-slo-admitter
// (requestcontrol/admitter/latencyslo/plugin.go:99-158) and the probabilistic-admitter
// (requestcontrol/admitter/probabilisticadmitter/plugin.go:125-162).
//
// The reference admits a request before Scheduler.Schedule; the engine picks first and then rewrites the rows an
// admitter rejects, before the call's after-pick updates read them.  Every admitted row is left exactly as the picks
// wrote it.  One warp per listed row (the host lists only the rows an admitter can reject).
#include <math.h>

#include "kernels.h"
#include "score.cuh"

namespace epp {

namespace {
constexpr uint64_t kAdmitDomain = 0x1D8E4E27C47D124FULL;

// Go's math.Max / math.Min: +-Inf first, then NaN, then the sign of zero.
__device__ __forceinline__ double go_max(double x, double y) {
    if (isinf(x) && x > 0) return x;
    if (isinf(y) && y > 0) return y;
    if (isnan(x) || isnan(y)) return __longlong_as_double(0x7FF8000000000001LL);
    if (x == 0 && x == y) return signbit(x) ? y : x;
    return x > y ? x : y;
}
__device__ __forceinline__ double go_min(double x, double y) {
    if (isinf(x) && x < 0) return x;
    if (isinf(y) && y < 0) return y;
    if (isnan(x) || isnan(y)) return __longlong_as_double(0x7FF8000000000001LL);
    if (x == 0 && x == y) return signbit(x) ? x : y;
    return x < y ? x : y;
}

__device__ __forceinline__ bool go_is_odd_int(double x) {
    if (fabs(x) >= 0x1.0p53) return false;
    double xi;
    const double xf = modf(x, &xi);
    return xf == 0 && ((long long)xi & 1) == 1;
}

// Go's math.Pow (math/pow.go): the special cases, then x**yf by Exp(yf * Log(x)) and x**yi by repeated squaring of
// Frexp's mantissa with the exponent kept apart, then Ldexp.  Exact for an integer y; Exp / Log are CUDA's.
__device__ double go_pow(double x, double y) {
    const double inf = __longlong_as_double(0x7FF0000000000000LL);
    const double nan = __longlong_as_double(0x7FF8000000000001LL);
    if (y == 0 || x == 1) return 1;
    if (y == 1) return x;
    if (isnan(x) || isnan(y)) return nan;
    if (x == 0) {
        if (y < 0) return signbit(x) && go_is_odd_int(y) ? -inf : inf;
        if (y > 0) return signbit(x) && go_is_odd_int(y) ? x : 0.0;
    }
    if (isinf(y)) {
        if (x == -1) return 1;
        if ((fabs(x) < 1) == (y > 0)) return 0;
        return inf;
    }
    if (isinf(x)) {
        if (x < 0) return go_pow(1 / x, -y);
        if (y < 0) return 0;
        if (y > 0) return inf;
    }
    if (y == 0.5) return sqrt(x);
    if (y == -0.5) return 1 / sqrt(x);
    double yi;
    double yf = modf(fabs(y), &yi);
    if (yf != 0 && x < 0) return nan;
    if (yi >= 0x1.0p63) {
        if (x == -1) return 1;
        if ((fabs(x) < 1) == (y > 0)) return 0;
        return inf;
    }
    double a1 = 1.0;
    long long ae = 0;
    if (yf != 0) {
        if (yf > 0.5) {
            yf--;
            yi++;
        }
        a1 = exp(yf * log(x));
    }
    int xe_i;
    double x1 = frexp(x, &xe_i);
    long long xe = xe_i;
    for (long long i = (long long)yi; i != 0; i >>= 1) {
        if (xe < -(1LL << 12) || (1LL << 12) < xe) {     // catastrophic overflow: Ldexp takes it
            ae += xe;
            break;
        }
        if (i & 1) {
            a1 *= x1;
            ae += xe;
        }
        x1 *= x1;
        xe <<= 1;
        if (x1 < .5) {
            x1 += x1;
            xe--;
        }
    }
    if (y < 0) {
        a1 = 1 / a1;
        ae = -ae;
    }
    // a1 is >= 2^-64 here, so any |ae| beyond 2^20 already gives 0 or Inf, as Go's Ldexp does for its int
    ae = ae < -(1LL << 20) ? -(1LL << 20) : (ae > (1LL << 20) ? (1LL << 20) : ae);
    return ldexp(a1, (int)ae);
}

// Is slot s a candidate of the row: in the pool and, for a subset row, in its ascending slot list.
__device__ __forceinline__ bool admit_candidate(const AdmitParams &p, const AdmitRow &row, uint32_t s) {
    if (s >= (uint32_t)p.E || p.role[s] == 0xFF) return false;
    if (row.sub_n == EPP_SUBSET_ALL) return true;
    const uint32_t *sl = p.sub_slots + row.sub_off;
    uint32_t lo = 0, hi = row.sub_n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (sl[mid] < s) lo = mid + 1;
        else hi = mid;
    }
    return lo < row.sub_n && sl[lo] == s;
}

__global__ void __launch_bounds__(256) k_admit(AdmitParams p) {
    const int64_t w = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= p.n_rows) return;
    const AdmitRow row = p.rows[w];
    // the candidate set: whole-pool aggregates from the snapshot, or folded here over the subset
    int32_t n = p.pool_n;
    bool idle = p.pool_idle != 0, cold = p.pool_cold != 0;
    double sum = p.pool_sat;
    if (row.sub_n != EPP_SUBSET_ALL) {
        n = 0;
        idle = cold = false;
        sum = 0.0;
        const uint32_t *sl = p.sub_slots + row.sub_off;
        for (uint32_t b = 0; b < row.sub_n; b += 32) {
            const uint32_t i = b + lane;
            bool in = false;
            double term = 0.0;
            if (i < row.sub_n) {
                const uint32_t s = sl[i];
                in = s < (uint32_t)p.E && p.role[s] != 0xFF;
                if (in) {
                    idle |= p.running[s] == 0;
                    cold |= p.kv[s] < 0.02;
                    term = go_max((double)p.waiting[s] / p.qdt, p.kv[s] / p.kvt);
                }
            }
            const uint32_t m = __ballot_sync(0xffffffffu, in);
            n += __popc(m);
            // the fold is a left fold in ascending slot order: one lane adds the terms one by one
            for (int j = 0; j < 32; j++) {
                const double t = __shfl_sync(0xffffffffu, term, j);
                if ((m >> j) & 1u) sum += t;
            }
        }
        idle = __any_sync(0xffffffffu, idle);
        cold = __any_sync(0xffffffffu, cold);
    }
    if (n == 0) return;                            // no candidate: the director's ServiceUnavailable (status -1) stands
    bool reject = false;
    if (row.flags & kAdmitProbabilistic) {
        const double sat = sum / (double)n;
        const double prob = go_min(go_pow(sat, p.power) * p.k, 1.0);
        const uint64_t key = 4ull * (p.ord_base + (uint64_t)row.row) + 3ull;
        const double u = (double)(mix64((p.tie_seed ^ kAdmitDomain) ^ mix64(key)) >> 11) * 0x1.0p-53;
        reject = u < prob;
    }
    if (!reject && (row.flags & kAdmitLatencySlo) && !idle && !cold) {
        bool has = false, valid = false;
        const uint32_t *ent = p.ent + row.pred_off;
        for (uint32_t b = 0; b < row.pred_n; b += 32) {
            const uint32_t i = b + lane;
            if (i < row.pred_n) {
                const uint32_t e = ent[i];
                if (admit_candidate(p, row, e & 0x7FFFFFFFu)) {
                    has = true;
                    valid |= (e >> 31) != 0;
                }
            }
        }
        has = __any_sync(0xffffffffu, has);
        valid = __any_sync(0xffffffffu, valid);
        reject = has && !valid;
    }
    if (!reject) return;
    const int64_t r = (int64_t)row.row;
    if (lane == 0) {
        epp_decision &d = p.dec[r];
        d.status = EPP_STATUS_REJECTED;
        d.pick = EPP_NO_ENDPOINT;
        d.score = 0.0;
        d.prefill_pick = EPP_NO_ENDPOINT;
        d.tie_count = 0;
        d.match_blocks = 0;
        if (p.det) {
            epp_decision_detail &x = p.det[r];
            x.prefill_score = 0.0;
            x.prefill_tie_count = 0;
            x.prefill_ran = 0;
            x.encode_score = 0.0;
            x.encode_pick = EPP_NO_ENDPOINT;
            x.encode_tie_count = 0;
            x.encode_ran = 0;
            x.reserved = 0;
        }
    }
    for (int j = lane; j < p.topk; j += 32) {
        const size_t o = (size_t)r * (size_t)p.topk + (size_t)j;
        for (int i = 0; i < kMaxProfiles; i++)
            if (p.topk_picks[i]) p.topk_picks[i][o] = EPP_NO_ENDPOINT;
        if (p.topk_scores) p.topk_scores[o] = 0.0;
    }
}
}  // namespace

cudaError_t launch_admit(const AdmitParams &p, cudaStream_t s, int *launches) {
    if (p.n_rows <= 0) return cudaSuccess;
    const int64_t threads = (int64_t)p.n_rows * 32;
    k_admit<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p);
    if (launches) ++*launches;
    return cudaGetLastError();
}

}  // namespace epp
