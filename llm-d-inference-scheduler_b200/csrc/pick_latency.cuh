// pick_latency.cuh -- the general evaluation of one chain SchedulerProfile (a latency piece, the context-length-aware
// plugin or both) for one request (one warp), as defined in include/epp_engine.h ("Latency predictions", "Context length"):
//   [role + label + context-length filters] -> [affinity A1] -> [slo-headroom-tier-filter T] -> [affinity A2] -> scorers
//   -> picker,
// with the latency-scorer (scorer/latency/plugin.go:144-395) and the context-length scorer among the scorers.  The request-level state (the A1 / T / A2
// decisions, the scored bucket, its per-dimension min / max, alpha and beta) is computed once per stage by warp
// reductions; after that a slot's membership and score are per-slot predicates over its entry, which each lane finds by
// binary search in the request's ascending entry list.
// The chain walks an index domain (PoolDom: every slot of the pool; ListDom: a restricted request's listed slots), so
// the _lat builds of the dense-counter and injected-match kernels and the subset kernel share one evaluation.
#pragma once
#include <cfloat>
#include <climits>

#include "pick_general.cuh"

namespace epp {
namespace lat {

constexpr uint64_t kA1Domain = 0x8EBC6AF09C88C6E3ULL;
constexpr uint64_t kTierDomain = 0x589965CC75374CC3ULL;
constexpr double kEps = 1e-9;        // scorer/latency/plugin.go:41

__device__ __forceinline__ double draw_u(uint64_t seed, uint64_t dom, uint64_t key) {
    return (double)(mix64((seed ^ dom) ^ mix64(key)) >> 11) * 0x1.0p-53;
}

// int(x) of Go on amd64 (CVTTSD2SQ): truncation toward zero, 0x8000000000000000 for NaN and out-of-range values
__device__ __forceinline__ long long go_int(double x) {
    if (!(x > -0x1.0p63 && x < 0x1.0p63)) return LLONG_MIN;
    return (long long)x;
}

__device__ __forceinline__ uint32_t warp_sum(uint32_t v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(gen::kFull, v, o);
    return v;
}

// The context-length-aware plugin of one profile for one request (context_length_aware.go): the first-stage filter
// predicate and the score of slot e, from e's range (kernels.h LatView::rng) and the request's ctx.
struct CtxLen {
    const longlong2 *rng;          // nullptr: the profile does not list the plugin
    long long ctx;
    bool filter;
    __device__ __forceinline__ bool keep(uint32_t e) const {
        if (!filter) return true;
        const longlong2 r = rng[e];
        if (r.x < 0) return r.x == kRangeAbsent;                                      // no label keeps, invalid drops
        return ctx >= r.x && ctx <= r.y;
    }
    // calculateRangeScore; differences wrap like Go's int arithmetic
    __device__ __forceinline__ double score(uint32_t e) const {
        const longlong2 r = rng[e];
        if (r.x == kRangeAbsent) return 0.5;
        if (r.x < 0) return 0.0;
        if (ctx >= r.x && ctx <= r.y) {
            const long long w = r.y - r.x;
            if (w == 0) return 1.0;
            const double ws = __ddiv_rn(1.0, __dadd_rn(1.0, __ddiv_rn((double)w, 10000.0)));
            const double pos = __ddiv_rn((double)(r.y - ctx), (double)w);
            const double raw = __dadd_rn(__dmul_rn(0.7, ws), __dmul_rn(0.3, pos));
            return __dadd_rn(0.3, __dmul_rn(raw, 0.7));
        }
        const long long d = (long long)(ctx > r.y ? (unsigned long long)ctx - (unsigned long long)r.y
                                                  : (unsigned long long)r.x - (unsigned long long)ctx);
        return __ddiv_rn(0.3, __dadd_rn(1.0, __ddiv_rn((double)d, 1000.0)));
    }
};

// Profile pi's plugin for absolute row `row` of the call, whose true prompt length is L: ctx is the caller's count, or
// int(float64(L) * 0.25).
__device__ __forceinline__ CtxLen ctx_len(const LatView &lv, int pi, int64_t row, int64_t L) {
    CtxLen c;
    c.rng = lv.rng[pi];
    c.filter = c.rng && ((lv.cl_filter >> pi) & 1);
    const long long t = (c.rng && lv.ctx) ? lv.ctx[row] : -1;
    c.ctx = t >= 0 ? t : go_int(__dmul_rn((double)L, 0.25));
    return c;
}

// The request's entries, ascending slot.
struct Req {
    const epp_prediction *ent;
    uint32_t n;
    __device__ __forceinline__ const epp_prediction *find(uint32_t e) const {
        uint32_t lo = 0, hi = n;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (ent[mid].slot < e) lo = mid + 1; else hi = mid;
        }
        return (lo < n && ent[lo].slot == e) ? ent + lo : nullptr;
    }
};

// The index domain of an evaluation: members i of [0, n), member i is slot at(i) with matchBlocks cnt(i);
// n_cand(pf, lane, cl) is the number of members that pass the first stage of profile pf (role, label and context-length
// filters); with the context-length filter on it depends on the request.
template <typename CntOf>
struct PoolDom {                   // i -> i over the whole pool
    uint32_t n;
    CntOf cnt_of;
    __device__ __forceinline__ uint32_t at(uint32_t i) const { return i; }
    __device__ __forceinline__ int32_t cnt(uint32_t i) const { return cnt_of(i); }
    __device__ __forceinline__ uint32_t n_cand(const ProfileDev &pf, int lane, const CtxLen &cl) const {
        if (!cl.filter) return (uint32_t)*pf.n_cand;
        uint32_t c = 0;
        for (uint32_t i = lane; i < n; i += 32) c += pf.cand[i] && cl.keep(i);
        return warp_sum(c);
    }
};
template <typename CntOf>
__device__ __forceinline__ PoolDom<CntOf> pool_dom(int32_t E, CntOf cnt_of) { return PoolDom<CntOf>{(uint32_t)E, cnt_of}; }

struct ListDom {                   // i -> sl[i] over a restricted request's ascending slot list (endpoint subsets)
    const uint32_t *sl;
    const int32_t *hit;            // whole-pool matchBlocks per listed slot
    uint32_t n;
    __device__ __forceinline__ uint32_t at(uint32_t i) const { return sl[i]; }
    __device__ __forceinline__ int32_t cnt(uint32_t i) const { return hit[i]; }
    __device__ __forceinline__ uint32_t n_cand(const ProfileDev &pf, int lane, const CtxLen &cl) const {
        uint32_t c = 0;
        for (uint32_t i0 = 0; i0 < n; i0 += 32)
            c += __popc(__ballot_sync(gen::kFull, i0 + lane < n && pf.cand[sl[i0 + lane]] && cl.keep(sl[i0 + lane])));
        return c;
    }
};

// both headrooms >= 0 (sloheadroomtier/plugin.go:102)
__device__ __forceinline__ bool meets(const epp_prediction *p) { return p->ttft_headroom >= 0.0 && p->tpot_headroom >= 0.0; }

enum { kTierAll = 0, kTierPos = 1, kTierNeg = 2 };
enum { kBucketPos = 0, kBucketIdle = 1, kBucketTpot = 2, kBucketTtft = 3, kBucketBoth = 4, kComposite = 5 };

// The scored bucket of Score (plugin.go:172-235); p == nullptr: no entry (positive, headrooms 0).
__device__ __forceinline__ bool in_bucket(int bucket, const epp_prediction *p) {
    if (!p) return bucket == kBucketPos;
    const bool tn = p->ttft_headroom < 0.0, pn = p->tpot_headroom < 0.0;
    switch (bucket) {
        case kBucketPos: return !tn && !pn;
        case kBucketIdle: return (tn || pn) && p->dispatched == 0;
        case kBucketTpot: return !tn && pn;
        case kBucketTtft: return tn && !pn;
        case kBucketBoth: return tn && pn;
        default: return false;
    }
}

struct State {
    bool a1, a2;
    int tier;
    gen::Norm nm;                   // normalisation over the final set (nm.sticky / nm.thr unused)
    bool scorer;                    // the profile lists the latency scorer
    int bucket;
    bool most;
    double alpha, beta, mn_t, rng_t, mn_p, rng_p;
    long long max_q;
    double wkv, wq, wpref;
};

// prefix-cache-affinity-filter (plugin.go:105-151) over the n members of in_set, TTFT from the entries (bestTTFT,
// :173-184, skips members without one).  True: the set narrows to the sticky members.
template <typename InSet, typename Dom>
__device__ inline bool affinity(double thr, double explore, double penalty, uint64_t dom, uint32_t n, const Req &q,
                                int32_t total, int lane, uint64_t seed, uint64_t key, InSet in_set, const Dom &ix) {
    if (!(thr > 0.0) || n <= 1) return false;                                           // :108
    if (seed && draw_u(seed, dom, key) < explore) return false;                         // :113-117
    uint32_t ns = 0, nn = 0;
    double bs = DBL_MAX, bn = DBL_MAX;
    for (uint32_t i = lane; i < ix.n; i += 32) {
        if (!in_set(i)) continue;
        const epp_prediction *p = q.find(ix.at(i));
        const double t = p ? p->ttft : DBL_MAX;
        if (gen::is_sticky(ix.cnt(i), total, thr)) { ns++; if (t < bs) bs = t; }
        else { nn++; if (t < bn) bn = t; }
    }
    for (int o = 16; o; o >>= 1) {
        ns += __shfl_xor_sync(gen::kFull, ns, o);
        nn += __shfl_xor_sync(gen::kFull, nn, o);
        const double os = __shfl_xor_sync(gen::kFull, bs, o), on = __shfl_xor_sync(gen::kFull, bn, o);
        if (os < bs) bs = os;
        if (on < bn) bn = on;
    }
    if (ns == 0) return false;                                                           // :130-134
    if (penalty > 0.0 && nn > 0 && __dsub_rn(bs, bn) > penalty) return false;            // :137-146
    return true;
}

// The latency scorer's raw score of final-set member e (p = its entry or nullptr).
__device__ __forceinline__ double score_raw(const State &st, const PoolArrays &pool, uint32_t e, const epp_prediction *p,
                                            int32_t match, int32_t total) {
    if (st.bucket == kComposite) {                                                       // compositeScores, :323-367
        const long long q = pool.waiting[e];
        const double rel = st.max_q > 0 ? __ddiv_rn((double)(st.max_q - q), (double)st.max_q) : 1.0;
        const double kv_free = __dsub_rn(1.0, pool.kv_usage[e]);
        const double c = __dadd_rn(__dadd_rn(__dmul_rn(st.wkv, kv_free), __dmul_rn(st.wq, rel)),
                                   __dmul_rn(st.wpref, prefix_score(match, total)));
        return __ddiv_rn((double)go_int(round(__dadd_rn(0.0, __dmul_rn(100.0, c)))), 100.0);
    }
    if (!in_bucket(st.bucket, p)) return 0.0;
    const double ht = p ? fabs(p->ttft_headroom) : 0.0, hp = p ? fabs(p->tpot_headroom) : 0.0;   // scoreBucket, :246-318
    const double nt = st.rng_t > kEps ? __ddiv_rn(__dsub_rn(ht, st.mn_t), st.rng_t) : 0.5;
    const double np = st.rng_p > kEps ? __ddiv_rn(__dsub_rn(hp, st.mn_p), st.rng_p) : 0.5;
    const double comb = __dadd_rn(__dmul_rn(st.alpha, nt), __dmul_rn(st.beta, np));
    const double x = st.most ? comb : __dsub_rn(1.0, comb);
    return __ddiv_rn((double)(go_int(__dmul_rn(x, 100.0)) + 1), 100.0);
}

// runScorerPlugins over the final set (weighted_sum_over with the latency and context-length scorers).
__device__ inline double weighted_sum(const ProfileDev &pf, const GenView &g, const State &st, const CtxLen &cl, uint32_t e,
                                      const epp_prediction *p, int32_t match, int32_t total, const LoraDev &L, int lora_st) {
    double acc = 0.0;
#pragma unroll 1
    for (int s = 0; s < pf.cfg.n_scorers; s++) {
        const epp_scorer_cfg &sc = pf.cfg.scorers[s];
        double raw;
        if (sc.kind == EPP_SCORER_PREFIX) raw = prefix_score(match, total);
        else if (sc.kind == EPP_SCORER_LORA_AFFINITY) raw = lora_score(L, e, lora_st);
        else if (sc.kind == EPP_SCORER_LATENCY) raw = score_raw(st, g.pool, e, p, match, total);
        else if (sc.kind == EPP_SCORER_CONTEXT_LENGTH) raw = cl.score(e);
        else raw = pool_score(sc, s, g.pool, st.nm.q, (int32_t)e);
        acc = __dadd_rn(acc, __dmul_rn(clamp01(raw), sc.weight));
    }
    return acc;
}

// The request-level state of the chain and the scorer over the members of ix (E: the pool's, the stride of its
// columns).  Returns the final set's size.
template <typename Dom>
__device__ inline uint32_t prepare(const ProfileDev &pf, const epp_latency_cfg &lc, const CtxLen &cl, const GenView &g,
                                   const Req &q, int32_t E, int32_t total, int lane, uint64_t seed, uint64_t key, const Dom &ix,
                                   State &st) {
    const epp_profile_cfg &c = pf.cfg;
    st.a1 = st.a2 = false;
    st.tier = kTierAll;
    auto in1 = [&](uint32_t i) { return pf.cand[ix.at(i)] && cl.keep(ix.at(i)) && (!st.a1 || gen::is_sticky(ix.cnt(i), total, lc.a1_affinity_threshold)); };
    auto in2 = [&](uint32_t i) {
        if (!in1(i)) return false;
        if (st.tier == kTierAll) return true;
        const epp_prediction *p = q.find(ix.at(i));
        return (st.tier == kTierPos) == (p && meets(p));
    };
    auto in = [&](uint32_t i) { return in2(i) && (!st.a2 || gen::is_sticky(ix.cnt(i), total, c.affinity_threshold)); };
    // A1 over the filtered candidates
    if (lc.tier_filter)
        st.a1 = affinity(lc.a1_affinity_threshold, lc.a1_exploration_probability, lc.a1_max_ttft_penalty_ms, kA1Domain,
                         ix.n_cand(pf, lane, cl), q, total, lane, seed, key, in1, ix);
    // T over A1's set (sloheadroomtier/plugin.go:84-138)
    uint32_t n1 = 0, npos = 0, nneg = 0;
    for (uint32_t i = lane; i < ix.n; i += 32) {
        if (!in1(i)) continue;
        n1++;
        const epp_prediction *p = q.find(ix.at(i));
        if (p) { if (meets(p)) npos++; else nneg++; }
    }
    n1 = warp_sum(n1); npos = warp_sum(npos); nneg = warp_sum(nneg);
    uint32_t n2 = n1;
    if (lc.tier_filter && n1 > 1 && (npos || nneg)) {
        nneg = n1 - npos;                                                               // + the no-prediction endpoints
        if (npos && nneg) st.tier = (seed && draw_u(seed, kTierDomain, key) < lc.epsilon_explore_neg) ? kTierNeg : kTierPos;
        else st.tier = npos ? kTierPos : kTierNeg;
        n2 = st.tier == kTierPos ? npos : nneg;
    }
    // A2: the profile's own affinity filter, today's draw
    st.a2 = affinity(c.affinity_threshold, c.exploration_probability, c.max_ttft_penalty_ms, gen::kExploreDomain, n2, q,
                     total, lane, seed, key, in2, ix);
    // normalisation over the final set; the latency scorer's bucket
    uint32_t n = 0, has = 0, pos = 0, idle = 0, tpot = 0, ttft = 0;
    long long mnw = LLONG_MAX, mxw = LLONG_MIN, mnr = LLONG_MAX, mxr = LLONG_MIN, mxq = 0;
    for (uint32_t i = lane; i < ix.n; i += 32) {
        if (!in(i)) continue;
        const uint32_t e = ix.at(i);
        n++;
        const long long w = g.pool.waiting[e], r = g.pool.running[e];
        mnw = min(mnw, w); mxw = max(mxw, w);
        mnr = min(mnr, r); mxr = max(mxr, r);
        mxq = max(mxq, w);
        const epp_prediction *p = q.find(e);
        if (!p) { pos++; continue; }
        has++;
        pos += in_bucket(kBucketPos, p);
        idle += in_bucket(kBucketIdle, p);
        tpot += in_bucket(kBucketTpot, p);
        ttft += in_bucket(kBucketTtft, p);
    }
    for (int o = 16; o; o >>= 1) {
        mnw = min(mnw, __shfl_xor_sync(gen::kFull, mnw, o)); mxw = max(mxw, __shfl_xor_sync(gen::kFull, mxw, o));
        mnr = min(mnr, __shfl_xor_sync(gen::kFull, mnr, o)); mxr = max(mxr, __shfl_xor_sync(gen::kFull, mxr, o));
        mxq = max(mxq, __shfl_xor_sync(gen::kFull, mxq, o));
    }
    n = warp_sum(n); has = warp_sum(has); pos = warp_sum(pos); idle = warp_sum(idle); tpot = warp_sum(tpot); ttft = warp_sum(ttft);
    st.nm.sticky = false;
    st.nm.thr = 0.0;
    st.nm.q[0] = mnw; st.nm.q[1] = mxw; st.nm.q[2] = mnr; st.nm.q[3] = mxr;
    st.scorer = false;
    for (int s = 0; s < c.n_scorers; s++) {
        st.nm.q[4 + s] = 0;
        if (c.scorers[s].kind == EPP_SCORER_LATENCY) st.scorer = true;
        if (c.scorers[s].kind != EPP_SCORER_ACTIVE_REQUEST) continue;
        const int col = c.scorers[s].column;
        long long mx = 0;
        if (col >= 0 && col < g.pool.n_ext_cols)
            for (uint32_t i = lane; i < ix.n; i += 32)
                if (in(i)) mx = max(mx, (long long)g.pool.ext[(size_t)col * (size_t)E + (size_t)ix.at(i)]);
        for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(gen::kFull, mx, o));
        st.nm.q[4 + s] = mx;
    }
    st.max_q = mxq;
    st.most = false;
    if (!st.scorer) { st.bucket = kComposite; return n; }
    if (!has) {                                                                          // compositeScores weights, :326-334
        st.bucket = kComposite;
        double wkv = lc.composite_kv_weight, wq = lc.composite_queue_weight, wp = lc.composite_prefix_weight;
        double sw = __dadd_rn(__dadd_rn(wkv, wq), wp);
        if (sw <= 0.0) { wkv = 1.0; wq = 0.0; wp = 0.0; sw = 1.0; }
        st.wkv = __ddiv_rn(wkv, sw); st.wq = __ddiv_rn(wq, sw); st.wpref = __ddiv_rn(wp, sw);
        return n;
    }
    if (pos) { st.bucket = kBucketPos; st.most = lc.strategy == EPP_HEADROOM_MOST; }
    else if (idle) st.bucket = kBucketIdle;
    else if (tpot) st.bucket = kBucketTpot;
    else if (ttft) st.bucket = kBucketTtft;
    else st.bucket = kBucketBoth;
    double mnt = DBL_MAX, mxt = -DBL_MAX, mnp = DBL_MAX, mxp = -DBL_MAX;
    for (uint32_t i = lane; i < ix.n; i += 32) {
        if (!in(i)) continue;
        const epp_prediction *p = q.find(ix.at(i));
        if (!in_bucket(st.bucket, p)) continue;
        const double ht = p ? fabs(p->ttft_headroom) : 0.0, hp = p ? fabs(p->tpot_headroom) : 0.0;
        if (ht < mnt) mnt = ht;
        if (ht > mxt) mxt = ht;
        if (hp < mnp) mnp = hp;
        if (hp > mxp) mxp = hp;
    }
    for (int o = 16; o; o >>= 1) {
        mnt = fmin(mnt, __shfl_xor_sync(gen::kFull, mnt, o)); mxt = fmax(mxt, __shfl_xor_sync(gen::kFull, mxt, o));
        mnp = fmin(mnp, __shfl_xor_sync(gen::kFull, mnp, o)); mxp = fmax(mxp, __shfl_xor_sync(gen::kFull, mxp, o));
    }
    st.mn_t = mnt; st.mn_p = mnp;
    st.rng_t = __dsub_rn(mxt, mnt);
    st.rng_p = __dsub_rn(mxp, mnp);
    const double sab = __dadd_rn(lc.ttft_weight, lc.tpot_weight);                        // normalizedWeights, :376-382
    if (sab <= 0.0) { st.alpha = 1.0; st.beta = 0.0; }
    else { st.alpha = __ddiv_rn(lc.ttft_weight, sab); st.beta = __ddiv_rn(lc.tpot_weight, sab); }
    if (st.rng_t <= kEps && st.rng_p > kEps) { st.alpha = 0.0; st.beta = 1.0; }        // :277-281
    else if (st.rng_p <= kEps && st.rng_t > kEps) { st.alpha = 1.0; st.beta = 0.0; }
    return n;
}

// One latency profile for one request: the chain, scores, and the first max(1, k) endpoints in picker order (the
// contract of gen::eval, over the final set), all over the members of ix: the candidates are its members that pass
// pf's filters, and every set size, range and draw population is taken over them.  Picks are slots.
template <bool kRand, typename Dom>
__device__ inline Best eval(const ProfileDev &pf, const epp_latency_cfg &lc, const CtxLen &cl, const GenView &g, const Req &q,
                            int32_t E, int32_t total, int lane, const LoraDev &lora, uint32_t adapter, uint64_t seed,
                            uint64_t key, const Dom &ix, int32_t k, uint32_t *picks_row, double *scores_row) {
    Best first;
    best_init(first);
    if (k < 1) k = 1;
    if (picks_row) for (int j = lane; j < k; j += 32) picks_row[j] = EPP_NO_ENDPOINT;
    if (scores_row) for (int j = lane; j < k; j += 32) scores_row[j] = 0.0;
    __syncwarp();
    if (ix.n_cand(pf, lane, cl) == 0) return first;
    State st;
    const uint32_t n = prepare(pf, lc, cl, g, q, E, total, lane, seed, key, ix, st);
    const bool use_lora = lora.enabled && lora.ptr;
    auto cand = [&](uint32_t i) {
        const uint32_t e = ix.at(i);
        if (!pf.cand[e] || !cl.keep(e)) return false;
        if (st.a1 && !gen::is_sticky(ix.cnt(i), total, lc.a1_affinity_threshold)) return false;
        if (st.tier != kTierAll) {
            const epp_prediction *p = q.find(e);
            if ((st.tier == kTierPos) != (p && meets(p))) return false;
        }
        return !st.a2 || gen::is_sticky(ix.cnt(i), total, pf.cfg.affinity_threshold);
    };
    auto score = [&](uint32_t i) {
        const uint32_t e = ix.at(i);
        const int ls = use_lora ? lora_lookup(lora, adapter, e) : 0;
        return weighted_sum(pf, g, st, cl, e, q.find(e), ix.cnt(i), total, lora, ls);
    };
    if (kRand && pf.cfg.picker) {     // random pickers: every member is an explicit item
        uint32_t g0 = EPP_NO_ENDPOINT, g1 = EPP_NO_ENDPOINT;
        for (int32_t j = 0; j < k && (uint32_t)j < n; j++) {
            auto out_of = [&](uint32_t e) {
                bool o = false;
                for (int32_t t = 0; t < j; t++)
                    o |= e == __shfl_sync(gen::kFull, t < 32 ? g0 : g1, t & 31);
                return o;
            };
            Best b = rnd::draw_scan(pf, (int32_t)ix.n, lane, false, n - (uint32_t)j, (uint32_t)j, seed + (uint64_t)j * gen::kGolden,
                                    key, cand, [](uint32_t) { return true; }, score, out_of);
            if (lane == (j & 31)) { if (j < 32) g0 = b.pick; else g1 = b.pick; }     // members, as out_of compares them
            b.pick = ix.at(b.pick);
            if (j == 0) first = b;
            if (lane == 0) {
                if (picks_row) picks_row[j] = b.pick;
                if (scores_row) scores_row[j] = b.val;
            }
        }
        return first;
    }
    double v = 0.0;
    bool have_v = false;
    uint32_t n_rem = 0;
    uint32_t g0 = EPP_NO_ENDPOINT, g1 = EPP_NO_ENDPOINT;
    uint32_t n_taken = 0;
    for (int32_t j = 0; j < k; j++) {
        if (n_rem == 0) {
            Best b;
            best_init(b);
            for (uint32_t i = lane; i < ix.n; i += 32) {
                if (!cand(i)) continue;
                const double sc = score(i);
                if (!have_v || sc < v) best_add(b, sc, i);
            }
            b = best_warp_reduce(b);
            if (!b.ties) break;
            v = b.val;
            have_v = true;
            n_rem = b.ties;
            n_taken = 0;
            g0 = g1 = EPP_NO_ENDPOINT;
            if (j == 0) first = b;
        }
        uint32_t rank = seed ? tie_rank(seed + (uint64_t)j * gen::kGolden, key, n_rem) : 0u;
        uint32_t pick = EPP_NO_ENDPOINT;
        for (uint32_t i0 = 0; i0 < ix.n && pick == EPP_NO_ENDPOINT; i0 += 32) {
            const uint32_t i = i0 + lane;
            bool hit = i < ix.n && cand(i) && score(i) == v;
            if (n_taken && __any_sync(gen::kFull, hit))
                for (uint32_t t = 0; t < n_taken; t++) {
                    const uint32_t te = __shfl_sync(gen::kFull, t < 32 ? g0 : g1, (int)(t & 31));
                    if (te == i) hit = false;
                }
            uint32_t bal = __ballot_sync(gen::kFull, hit);
            const uint32_t cnt = __popc(bal);
            if (rank < cnt) {
                for (uint32_t i = 0; i < rank; i++) bal &= bal - 1;
                pick = i0 + (uint32_t)__ffs(bal) - 1u;
            } else {
                rank -= cnt;
            }
        }
        if (pick == EPP_NO_ENDPOINT) break;
        if (lane == (int)(n_taken & 31)) { if (n_taken < 32) g0 = pick; else g1 = pick; }
        n_taken++;
        n_rem--;
        if (j == 0) first.pick = pick;
        if (lane == 0) {
            if (picks_row) picks_row[j] = ix.at(pick);
            if (scores_row) scores_row[j] = v;
        }
    }
    if (first.ties) first.pick = ix.at(first.pick);
    return first;
}

}  // namespace lat
}  // namespace epp
