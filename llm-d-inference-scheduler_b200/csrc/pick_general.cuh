// pick_general.cuh -- the GENERAL evaluation of one SchedulerProfile for one request (one warp):
//   * prefix-cache-affinity-filter between the role filter and the scorers (filter/prefixcacheaffinity/plugin.go:105-151):
//     the candidate set becomes request dependent, so the queue / running min-max and the active-request max the
//     scorers normalise with are recomputed over the narrowed set and the weighted sum is evaluated from the raw pool
//     arrays instead of the per-snapshot columns;
//   * the k best endpoints of the max-score picker (picker/maxscore/picker.go:87-115), group by group in descending
//     score order, every group of equal scores in the reproducible random order of include/epp_engine.h ("Top-k").
// Every step is a full scan over the E slots by the warp: the engine routes a batch here (dense-counter kernel /
// injected-match kernel) only when a profile configures the filter or pick_k > 1; the default configuration keeps the
// kernels of match_sparse.cuh / pick_kernels.cu, which never touch this code.
#pragma once
#include <cfloat>
#include <climits>

#include "pick_random.cuh"
#include "score.cuh"

namespace epp {
namespace gen {

constexpr uint32_t kFull = 0xffffffffu;
constexpr uint64_t kGolden = 0x9E3779B97F4A7C15ULL;
constexpr uint64_t kExploreDomain = 0xA0761D6478BD642FULL;

// matchBlocks / totalBlocks >= threshold (prefixCacheScore, plugin.go:160-171)
__device__ __forceinline__ bool is_sticky(int32_t c, int32_t total, double thr) {
    return total > 0 && __ddiv_rn((double)c, (double)total) >= thr;
}

struct Norm {                 // the request's candidate set of one profile
    bool sticky;              // narrowed to the sticky endpoints (else: every endpoint the role filter keeps)
    double thr;
    int64_t q[4 + EPP_MAX_SCORERS];   // scorer normalisation over the narrowed set (layout of ProfileDerived::qminmax)
};

__device__ __forceinline__ double explore_u(uint64_t seed, uint64_t key) {
    return (double)(mix64((seed ^ kExploreDomain) ^ mix64(key)) >> 11) * 0x1.0p-53;
}

// Plugin.Filter, plugin.go:105-151.  cnt_of(slot) = the request's matchBlocks on the slot.
template <typename CntOf>
__device__ inline void affinity_filter(const ProfileDev &pf, const GenView &g, int32_t E, int32_t total, int lane,
                                       uint64_t seed, uint64_t key, CntOf cnt_of, Norm &nm) {
    nm.sticky = false;
    const epp_profile_cfg &c = pf.cfg;
    nm.thr = c.affinity_threshold;
    if (!(c.affinity_threshold > 0.0) || *pf.n_cand <= 1) return;                        // :108
    if (seed && explore_u(seed, key) < c.exploration_probability) return;               // :113-117
    const bool have_ttft = c.ttft_column >= 0 && c.ttft_column < g.pool.n_ext_cols;
    const double *ttft = have_ttft ? g.pool.ext + (size_t)c.ttft_column * (size_t)E : nullptr;
    uint32_t ns = 0, nn = 0;
    long long mnw = LLONG_MAX, mxw = LLONG_MIN, mnr = LLONG_MAX, mxr = LLONG_MIN;
    double bs = DBL_MAX, bn = DBL_MAX;                                                   // bestTTFT, :173-184
    for (uint32_t e = lane; e < (uint32_t)E; e += 32) {
        if (!pf.cand[e]) continue;
        const double t = ttft ? ttft[e] : DBL_MAX;
        if (is_sticky(cnt_of(e), total, nm.thr)) {                                        // :120-127
            ns++;
            const long long w = g.pool.waiting[e], r = g.pool.running[e];
            mnw = min(mnw, w); mxw = max(mxw, w);
            mnr = min(mnr, r); mxr = max(mxr, r);
            if (t < bs) bs = t;
        } else {
            nn++;
            if (t < bn) bn = t;
        }
    }
    for (int o = 16; o; o >>= 1) {
        ns += __shfl_xor_sync(kFull, ns, o);
        nn += __shfl_xor_sync(kFull, nn, o);
        mnw = min(mnw, __shfl_xor_sync(kFull, mnw, o)); mxw = max(mxw, __shfl_xor_sync(kFull, mxw, o));
        mnr = min(mnr, __shfl_xor_sync(kFull, mnr, o)); mxr = max(mxr, __shfl_xor_sync(kFull, mxr, o));
        const double os = __shfl_xor_sync(kFull, bs, o), on = __shfl_xor_sync(kFull, bn, o);
        if (os < bs) bs = os;
        if (on < bn) bn = on;
    }
    if (ns == 0) return;                                                                 // :130-134
    if (c.max_ttft_penalty_ms > 0.0 && nn > 0 && __dsub_rn(bs, bn) > c.max_ttft_penalty_ms) return;   // :137-146
    nm.sticky = true;
    nm.q[0] = mnw; nm.q[1] = mxw; nm.q[2] = mnr; nm.q[3] = mxr;
    for (int s = 0; s < c.n_scorers; s++) {              // active-request scorers: max count over the narrowed set
        nm.q[4 + s] = 0;
        if (c.scorers[s].kind != EPP_SCORER_ACTIVE_REQUEST) continue;
        const int col = c.scorers[s].column;
        long long mx = 0;
        if (col >= 0 && col < g.pool.n_ext_cols)
            for (uint32_t e = lane; e < (uint32_t)E; e += 32)
                if (pf.cand[e] && is_sticky(cnt_of(e), total, nm.thr))
                    mx = max(mx, (long long)g.pool.ext[(size_t)col * (size_t)E + (size_t)e]);
        for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(kFull, mx, o));
        nm.q[4 + s] = mx;
    }
}

// runScorerPlugins over the narrowed set: the same ordered, clamped, unfused sum as weighted_sum(), with every scorer
// evaluated from the pool arrays and the set's own normalisation constants.  A narrowed set holds sticky endpoints only
// (matchBlocks > 0), so the request is warm for it and a no-hit-lru scorer adds its 0.5 (pool_score).
__device__ inline double weighted_sum_over(const ProfileDev &pf, const GenView &g, const Norm &nm, uint32_t e,
                                           int32_t match, int32_t total, const LoraDev &L, int lora_st) {
    double acc = 0.0;
#pragma unroll 1
    for (int s = 0; s < pf.cfg.n_scorers; s++) {
        const epp_scorer_cfg &sc = pf.cfg.scorers[s];
        double raw;
        if (sc.kind == EPP_SCORER_PREFIX) raw = prefix_score(match, total);
        else if (sc.kind == EPP_SCORER_LORA_AFFINITY) raw = lora_score(L, e, lora_st);
        else raw = pool_score(sc, s, g.pool, nm.q, (int32_t)e);
        acc = __dadd_rn(acc, __dmul_rn(clamp01(raw), sc.weight));
    }
    return acc;
}

// One profile for one request: filter chain, scores, and the first max(1, k) endpoints in picker order.  Returns the
// record of the arg-max set (value, pick 0, set size); picks_row / scores_row (k entries, or nullptr) receive the list.
// kRand: some profile of the engine has a random picker (the max-score builds carry none of that code).
template <bool kRand, typename CntOf>
__device__ inline Best eval(const ProfileDev &pf, const GenView &g, int32_t E, int32_t total, int lane,
                            const LoraDev &lora, uint32_t adapter, uint64_t seed, uint64_t key, CntOf cnt_of,
                            int32_t k, uint32_t *picks_row, double *scores_row) {
    Best first;
    best_init(first);
    if (k < 1) k = 1;
    if (picks_row) for (int j = lane; j < k; j += 32) picks_row[j] = EPP_NO_ENDPOINT;
    if (scores_row) for (int j = lane; j < k; j += 32) scores_row[j] = 0.0;
    __syncwarp();
    if (*pf.n_cand == 0) return first;
    Norm nm;
    affinity_filter(pf, g, E, total, lane, seed, key, cnt_of, nm);
    const bool use_lora = lora.enabled && lora.ptr;
    auto cand = [&](uint32_t e, int32_t c) { return pf.cand[e] && (!nm.sticky || is_sticky(c, total, nm.thr)); };
    auto score = [&](uint32_t e, int32_t c) {
        const int st = use_lora ? lora_lookup(lora, adapter, e) : 0;
        return nm.sticky ? weighted_sum_over(pf, g, nm, e, c, total, lora, st) : weighted_sum(pf, E, e, c, total, lora, st);
    };
    if (kRand && pf.cfg.picker) {     // random pickers: a narrowed set is all explicit, else the gaps of wcum
        uint32_t n = 0;
        for (uint32_t e0 = 0; e0 < (uint32_t)E; e0 += 32) {
            const uint32_t e = e0 + lane;
            n += __popc(__ballot_sync(kFull, e < (uint32_t)E && cand(e, cnt_of(e))));
        }
        // first k: successive draws without replacement, draw j with the seed tie_seed + j * kGolden; the endpoints
        // already emitted stay in the sequence with mass 0 (lane l holds emitted #l and #l + 32)
        uint32_t g0 = EPP_NO_ENDPOINT, g1 = EPP_NO_ENDPOINT;
        for (int32_t j = 0; j < k && (uint32_t)j < n; j++) {
            auto out_of = [&](uint32_t e) {
                bool o = false;
                for (int32_t t = 0; t < j; t++)
                    o |= e == __shfl_sync(kFull, t < 32 ? g0 : g1, t & 31);
                return o;
            };
            const Best b = rnd::draw_scan(pf, E, lane, !nm.sticky, n - (uint32_t)j, (uint32_t)j,
                                          seed + (uint64_t)j * kGolden, key,
                                          [&](uint32_t e) { return cand(e, cnt_of(e)); },
                                          [&](uint32_t e) { return cnt_of(e) > 0 || (use_lora && lora_lookup(lora, adapter, e) != 0); },
                                          [&](uint32_t e) { return score(e, cnt_of(e)); }, out_of);
            if (j == 0) first = b;
            if (lane == (j & 31)) { if (j < 32) g0 = b.pick; else g1 = b.pick; }
            if (lane == 0) {
                if (picks_row) picks_row[j] = b.pick;
                if (scores_row) scores_row[j] = b.val;
            }
        }
        return first;
    }
    double v = 0.0;                   // score of the current group
    bool have_v = false;              // a group is open: the next one lies strictly below v (the first may be +inf)
    uint32_t n_rem = 0;               // its members not emitted yet
    uint32_t g0 = EPP_NO_ENDPOINT, g1 = EPP_NO_ENDPOINT;   // emitted members of the current group: lane l holds #l and #l+32
    uint32_t n_taken = 0;
    for (int32_t j = 0; j < k; j++) {
        if (n_rem == 0) {             // next group: the best score strictly below the previous one
            Best b;
            best_init(b);
            for (uint32_t e = lane; e < (uint32_t)E; e += 32) {
                const int32_t c = cnt_of(e);
                if (!cand(e, c)) continue;
                const double sc = score(e, c);
                if (!have_v || sc < v) best_add(b, sc, e);
            }
            b = best_warp_reduce(b);
            if (!b.ties) break;       // fewer candidates than k
            v = b.val;
            have_v = true;
            n_rem = b.ties;
            n_taken = 0;
            g0 = g1 = EPP_NO_ENDPOINT;
            if (j == 0) first = b;
        }
        // the member of rank `rank` (ascending slot) among the group's members not emitted yet
        uint32_t rank = seed ? tie_rank(seed + (uint64_t)j * kGolden, key, n_rem) : 0u;
        uint32_t pick = EPP_NO_ENDPOINT;
        for (uint32_t e0 = 0; e0 < (uint32_t)E && pick == EPP_NO_ENDPOINT; e0 += 32) {
            const uint32_t e = e0 + lane;
            bool hit = false;
            if (e < (uint32_t)E) {
                const int32_t c = cnt_of(e);
                hit = cand(e, c) && score(e, c) == v;
            }
            if (n_taken && __any_sync(kFull, hit))
                for (uint32_t t = 0; t < n_taken; t++) {
                    const uint32_t te = __shfl_sync(kFull, t < 32 ? g0 : g1, (int)(t & 31));
                    if (te == e) hit = false;
                }
            uint32_t bal = __ballot_sync(kFull, hit);
            const uint32_t cnt = __popc(bal);
            if (rank < cnt) {
                for (uint32_t i = 0; i < rank; i++) bal &= bal - 1;
                pick = e0 + (uint32_t)__ffs(bal) - 1u;
            } else {
                rank -= cnt;
            }
        }
        if (pick == EPP_NO_ENDPOINT) break;                 // cannot happen: n_rem members remain
        if (lane == (int)(n_taken & 31)) { if (n_taken < 32) g0 = pick; else g1 = pick; }
        n_taken++;
        n_rem--;
        if (j == 0) first.pick = pick;
        if (lane == 0) {
            if (picks_row) picks_row[j] = pick;
            if (scores_row) scores_row[j] = v;
        }
    }
    return first;
}

}  // namespace gen
}  // namespace epp
