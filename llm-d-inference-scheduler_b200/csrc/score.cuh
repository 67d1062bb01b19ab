// score.cuh -- device-side scoring arithmetic shared by the pick kernels (a5-a10, a13).
//
// Arithmetic contract (SURVEY.md App. A.4/A.5): float64, IEEE round-to-nearest-even, NEVER fused -- every
// multiply/add/divide is an explicit __d*_rn intrinsic (the files are also compiled with -fmad=false).
// Scorer order = profile order; accumulation starts from +0.0 (scheduler_profile.go:155-168).
#pragma once
#include <math_constants.h>

#include "kernels.h"

namespace epp {

// ------------------------------------------------------------------------------------------------
// scorers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool filter_keeps(int filter, uint8_t role) {
    if (role == 0xFF) return false;                       // slot not in the pool
    switch (filter) {
        case EPP_FILTER_NONE: return true;
        case EPP_FILTER_DECODE:   // roles.go:46-48 (allowsNoLabel = true)
            return role == EPP_ROLE_NONE || role == EPP_ROLE_DECODE || role == EPP_ROLE_PREFILL_DECODE ||
                   role == EPP_ROLE_BOTH || role == EPP_ROLE_ENCODE_PREFILL_DECODE;
        case EPP_FILTER_PREFILL:  // roles.go:56-58
            return role == EPP_ROLE_PREFILL || role == EPP_ROLE_ENCODE_PREFILL || role == EPP_ROLE_PREFILL_DECODE ||
                   role == EPP_ROLE_BOTH || role == EPP_ROLE_ENCODE_PREFILL_DECODE;
        case EPP_FILTER_ENCODE:   // roles.go:68-70
            return role == EPP_ROLE_ENCODE || role == EPP_ROLE_ENCODE_PREFILL ||
                   role == EPP_ROLE_ENCODE_PREFILL_DECODE;
        default: return false;
    }
}

// Does the profile keep slot e: its role filter AND every label requirement (one bit test each).  The pool kernels are
// the only callers: every per-request kernel reads the cand[] they write.
__device__ __forceinline__ bool profile_keeps(int filter, const LabelFilterDev &lf, const PoolArrays &pool, int32_t e) {
    if (!filter_keeps(filter, pool.role[e])) return false;
    for (int i = 0; i < lf.n; i++)
        if (!((lf.mask[i] >> lf.lcode[(size_t)lf.key[i] * (size_t)pool.E + (size_t)e]) & 1ull)) return false;
    return true;
}

// enforceScoreRange, scheduler_profile.go:194-202 (NaN passes through, as in Go)
__device__ __forceinline__ double clamp01(double s) {
    if (s < 0.0) return 0.0;
    if (s > 1.0) return 1.0;
    return s;
}

// prefix-cache-scorer, scorer/prefix/plugin.go:100-111
__device__ __forceinline__ double prefix_score(int32_t match, int32_t total) {
    if (total == 0) return 0.0;
    return __ddiv_rn((double)match, (double)total);
}

// lora-affinity-scorer (scorer/loraaffinity/lora_affinity.go:76-100).  st: 0 = the request's adapter is neither active
// nor waiting on the endpoint, 1 = active, 2 = waiting.
__device__ __forceinline__ double lora_score(const LoraDev &L, uint32_t e, int st) {
    if (st == 1) return 1.0;
    const bool room = L.max_active && L.n_loaded[e] < L.max_active[e];
    if (room) return 0.8;
    return st == 2 ? 0.6 : 0.0;
}

// Residency state of adapter a on endpoint e (binary search in the adapter's endpoint list).
__device__ __forceinline__ int lora_lookup(const LoraDev &L, uint32_t a, uint32_t e) {
    if (!L.ptr || a >= (uint32_t)L.n_models) return 0;
    uint32_t lo = L.ptr[a];
    const uint32_t end = L.ptr[a + 1];
    uint32_t hi = end;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (L.ep[mid] < e) lo = mid + 1; else hi = mid;
    }
    return (lo < end && L.ep[lo] == e) ? (int)L.state[lo] : 0;
}

// Raw Scorer.Score value of one endpoint for the request-independent scorers.
// qminmax: [0..3] waiting / running min,max over the profile's candidates, [4 + s] max in-flight request count of
// active-request scorer s.
__device__ __forceinline__ double pool_score(const epp_scorer_cfg &sc, int s_index, const PoolArrays &pool,
                                             const int64_t *qminmax, int32_t e) {
    switch (sc.kind) {
        case EPP_SCORER_KV_UTIL:   // kvcache_utilization.go:79
            return __dsub_rn(1.0, pool.kv_usage[e]);
        case EPP_SCORER_QUEUE:     // queue.go:79-99
        case EPP_SCORER_RUNNING: { // runningrequest.go:79-99
            bool isq = sc.kind == EPP_SCORER_QUEUE;
            int64_t mn = qminmax[isq ? 0 : 2], mx = qminmax[isq ? 1 : 3];
            int64_t q = isq ? pool.waiting[e] : pool.running[e];
            if (mx == mn) return 1.0;
            return __ddiv_rn((double)(mx - q), (double)(mx - mn));
        }
        case EPP_SCORER_LOAD_AWARE: {  // load_aware.go:43-52, 87-97
            double thr = sc.param;
            if (!(thr > 0.0)) thr = 128.0;
            double w = (double)pool.waiting[e];
            if (w == 0.0) return 0.5;
            if (w > thr) w = thr;
            return __dmul_rn(0.5, __dsub_rn(1.0, __ddiv_rn(w, thr)));
        }
        case EPP_SCORER_EXTERNAL: {
            int col = (int)sc.param;
            if (col < 0 || col >= pool.n_ext_cols) return 0.0;
            return pool.ext[(size_t)col * (size_t)pool.E + (size_t)e];
        }
        case EPP_SCORER_TOKEN_LOAD: {   // token_load.go:84-112
            double thr = sc.param;
            if (!(thr > 0.0)) thr = 4194304.0;
            const int col = sc.column;
            double load = (col >= 0 && col < pool.n_ext_cols) ? pool.ext[(size_t)col * (size_t)pool.E + (size_t)e] : 0.0;
            if (load <= 0.0) return 1.0;
            if (load > thr) load = thr;
            return __dsub_rn(1.0, __ddiv_rn(load, thr));
        }
        case EPP_SCORER_ACTIVE_REQUEST: {   // active_request.go:140-173, NewActiveRequest :83-93
            const int col = sc.column;
            const int64_t idle = sc.param2 >= 0.0 ? (int64_t)sc.param2 : 0;
            const double max_busy = (sc.param >= 0.0 && sc.param <= 1.0) ? sc.param : 1.0;
            const int64_t c = (col >= 0 && col < pool.n_ext_cols) ? (int64_t)pool.ext[(size_t)col * (size_t)pool.E + (size_t)e] : 0;
            if (c <= idle) return 1.0;
            const int64_t mx = qminmax[4 + s_index];
            return __dmul_rn(__ddiv_rn((double)(mx - c), (double)mx), max_busy);
        }
        case EPP_SCORER_LORA_AFFINITY:      // request-independent part: the adapter is not resident on the endpoint
            return lora_score(pool.lora, (uint32_t)e, 0);
        case EPP_SCORER_NO_HIT_LRU:         // the warm score (no_hit_lru.go:159-165); the cold column is never read here
            return 0.5;
        default: return 0.0;
    }
}

// Ordered weighted sum of one endpoint (runScorerPlugins, scheduler_profile.go:151-174).
// lora_st: residency of the request's adapter on e (0 => the precomputed contribution already holds).
__device__ __forceinline__ double weighted_sum(const ProfileDev &pf, int32_t E, uint32_t e, int32_t match,
                                               int32_t total, const LoraDev &L = LoraDev{}, int lora_st = 0) {
    double acc = 0.0;
#pragma unroll 1
    for (int s = 0; s < pf.cfg.n_scorers; s++) {
        double term;
        if (pf.cfg.scorers[s].kind == EPP_SCORER_PREFIX)
            term = __dmul_rn(clamp01(prefix_score(match, total)), pf.cfg.scorers[s].weight);
        else if (lora_st && pf.cfg.scorers[s].kind == EPP_SCORER_LORA_AFFINITY)
            term = __dmul_rn(clamp01(lora_score(L, e, lora_st)), pf.cfg.scorers[s].weight);
        else
            term = pf.contrib[(size_t)s * (size_t)E + e];
        acc = __dadd_rn(acc, term);
    }
    return acc;
}

// ------------------------------------------------------------------------------------------------
// warp helpers
// ------------------------------------------------------------------------------------------------
struct Best {
    double val;
    uint32_t pick;
    uint32_t ties;
};
__device__ __forceinline__ void best_init(Best &b) { b.val = -CUDART_INF; b.pick = EPP_NO_ENDPOINT; b.ties = 0; }
__device__ __forceinline__ void best_add(Best &b, double v, uint32_t e, uint32_t n = 1) {
    if (v > b.val) { b.val = v; b.pick = e; b.ties = n; }
    else if (v == b.val) { b.ties += n; if (e < b.pick) b.pick = e; }
}
__device__ __forceinline__ Best best_warp_reduce(Best b) {
    double m = b.val;
    for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    uint32_t pk = (b.ties && b.val == m) ? b.pick : EPP_NO_ENDPOINT;
    uint32_t tc = (b.ties && b.val == m) ? b.ties : 0;
    for (int o = 16; o; o >>= 1) {
        pk = min(pk, __shfl_xor_sync(0xffffffffu, pk, o));
        tc += __shfl_xor_sync(0xffffffffu, tc, o);
    }
    Best r;
    r.val = m; r.pick = pk; r.ties = tc;
    return r;
}

// ------------------------------------------------------------------------------------------------
// tie rule (include/epp_engine.h, "Tie rule"): with tie_seed != 0 the pick is the member of rank
// tie_rank(seed, key, |arg-max set|) of the set in ascending slot order, key = 4 * request ordinal + profile index --
// a reproducible stand-in for the shuffle of maxscore/picker.go:91-102 (uniform over the set).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t mix64(uint64_t z) {           // SplitMix64 output function
    z += 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint32_t tie_rank(uint64_t seed, uint64_t key, uint32_t n) {
    const uint64_t m = mix64(seed ^ mix64(key));
    return (uint32_t)(((m >> 32) * (uint64_t)n) >> 32);
}
// The candidate of rank k (ascending slot id) among those whose score equals val: one warp scans all E slots.
// score_of(e) must reproduce the value the evaluation compared (bit for bit).
template <typename F>
__device__ inline uint32_t select_kth_scan(const ProfileDev &pf, int32_t E, double val, uint32_t k, int lane, F score_of) {
    for (uint32_t e0 = 0; e0 < (uint32_t)E; e0 += 32) {
        const uint32_t e = e0 + lane;
        const bool hit = e < (uint32_t)E && pf.cand[e] && score_of(e) == val;
        uint32_t bal = __ballot_sync(0xffffffffu, hit);
        const uint32_t c = __popc(bal);
        if (k < c) {
            for (uint32_t i = 0; i < k; i++) bal &= bal - 1;
            return e0 + (uint32_t)__ffs(bal) - 1u;
        }
        k -= c;
    }
    return EPP_NO_ENDPOINT;
}

// no-hit-lru isColdRequest (nohitlru/no_hit_lru.go:140-155) by a full scan: does no candidate of pf hold a block?
// cnt_of(slot) = the request's matchBlocks on the slot.  All lanes call it.
template <typename CntOf>
__device__ inline bool cold_scan(const ProfileDev &pf, int32_t E, int lane, CntOf cnt_of) {
    bool hit = false;
    for (uint32_t e = lane; e < (uint32_t)E && !hit; e += 32) hit = pf.cand[e] && cnt_of(e) > 0;
    return !__any_sync(0xffffffffu, hit);
}

// The profile set request-evaluation uses for profile pi: the cold set when the profile has a no-hit-lru scorer, has
// candidates and the request is cold for it (is_cold() is called only then, by all lanes); `cold` records the decision
// of the last such profile (no_hit_lru.go:264-266: every Score call overwrites the request's flag).
template <typename P, typename IsCold>
__device__ __forceinline__ const ProfileDev &nohit_select(const P &p, int pi, bool &cold, IsCold is_cold) {
    if (((p.nohit.mask >> pi) & 1) && *p.prof[pi].n_cand > 0) {
        cold = is_cold(p.prof[pi]);
        if (cold) return p.nohit.cold[pi];
    }
    return p.prof[pi];
}

// PrefixBasedPDDecider.disaggregate, prefix_based_pd_decider.go:99-149
__device__ __forceinline__ bool pd_decide(int64_t nct, int64_t in_len_bytes, int32_t match_blocks, int32_t bst) {
    if (nct == 0) return false;
    int64_t tokens = in_len_bytes / 4;                    // getUserInputLenInTokens, :152-167
    if (tokens < nct) return false;
    int64_t hit = (int64_t)match_blocks * (int64_t)bst;
    return (tokens - hit) >= nct;
}

// The stages of one decision after the matching (Scheduler.Schedule with the single / disagg profile handler):
// primary (decode) pick -> [encode stage for multimodal requests, disagg_profile_handler.go:284-295] -> [P/D decider ->
// prefill stage, :296-308].  eval(profile index, tie key) runs one SchedulerProfile for the request (all lanes call it
// together), match_of(slot) returns the request's matchBlocks on a slot.  P = PickParams or DensePickParams.
// kStages: how many stages are compiled in (1 = single profile, 2 = + P/D decider and prefill, 3 = + encode).
template <int kStages, typename P, typename Eval, typename MatchOf>
__device__ __forceinline__ void decide_stages(const P &p, int64_t r, int32_t total, int64_t in_len, Eval eval,
                                              MatchOf match_of, epp_decision &d, epp_decision_detail &dd) {
    const uint64_t key = 4 * (p.tie_base + (uint64_t)r);
    const Best b0 = eval(0, key);
    d.status = b0.ties ? 0 : -1;
    d.pick = b0.ties ? b0.pick : EPP_NO_ENDPOINT;
    d.score = b0.ties ? b0.val : 0.0;
    d.prefill_pick = EPP_NO_ENDPOINT;
    d.tie_count = b0.ties;
    d.total_blocks = total;
    d.match_blocks = b0.ties ? match_of(b0.pick) : 0;
    dd.prefill_score = 0.0; dd.prefill_tie_count = 0; dd.prefill_ran = 0;
    dd.encode_score = 0.0; dd.encode_pick = EPP_NO_ENDPOINT; dd.encode_tie_count = 0; dd.encode_ran = 0; dd.reserved = 0;
    if (!b0.ties) return;                                 // no decode endpoint: the cycle ends (ProcessResults :335-338)
    if (kStages >= 3 && p.encode_on && p.multimodal && p.multimodal[r]) {
        dd.encode_ran = 1;
        const Best b2 = eval(2, key + 2);
        if (b2.ties) { dd.encode_pick = b2.pick; dd.encode_score = b2.val; dd.encode_tie_count = b2.ties; }
    }
    if (kStages >= 2 && p.n_profiles >= 2) {
        const bool go = p.always_disagg || pd_decide(p.non_cached_tokens, in_len, d.match_blocks, p.block_size_tokens);
        if (go) {
            dd.prefill_ran = 1;
            const Best b1 = eval(1, key + 1);
            if (b1.ties) { d.prefill_pick = b1.pick; dd.prefill_score = b1.val; dd.prefill_tie_count = b1.ties; }
        }
    }
}

// Endpoint-sharded mode with the disagg handler (include/epp_engine.h, "Staged records"): this rank's best record of each
// of the n_stages stages of request r, out[0 .. n_stages).  Whether the prefill stage runs depends on the MERGED decode
// pick's match_blocks, which no rank knows yet, so a stage is evaluated whenever its decider can still come out true:
// prefill unless pd_decide is false for every match count (always_disagg, or 0 < non_cached_tokens <= tokens), encode for
// multimodal requests.  Every stage is evaluated even when this rank has no decode candidate (the decode pick may be
// another rank's).  A stage that is not evaluated gets status -1.  eval / match_of as in decide_stages; the records go to
// p.shard_out[r * n_stages ..].
template <typename P, typename Eval, typename MatchOf>
__device__ __forceinline__ void shard_stage_records(const P &p, int64_t r, int n_stages, int64_t in_len, Eval eval,
                                                    MatchOf match_of, int lane) {
    // decided up front: the request's length and flag need no registers while the stages are scored
    uint32_t runs = 1u;
    if (n_stages >= 2 && (p.always_disagg || (p.non_cached_tokens != 0 && in_len / 4 >= p.non_cached_tokens))) runs |= 2u;
    if (n_stages >= 3 && p.encode_on && p.multimodal && p.multimodal[r]) runs |= 4u;
#pragma unroll 1
    for (int st = 0; st < n_stages; st++) {
        epp_shard_best sb;
        sb.score = 0.0; sb.pick = EPP_NO_ENDPOINT; sb.tie_count = 0; sb.match_blocks = 0; sb.status = -1;
        if ((runs >> st) & 1u) {
            const Best b = eval(st, 4 * (p.tie_base + (uint64_t)r) + (uint64_t)st);
            const int32_t mb = b.ties ? match_of(b.pick) : 0;
            if (b.ties) { sb.score = b.val; sb.pick = b.pick; sb.tie_count = b.ties; sb.match_blocks = mb; sb.status = 0; }
        }
        if (lane == 0) p.shard_out[r * n_stages + st] = sb;
    }
}

}  // namespace epp
