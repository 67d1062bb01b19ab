// pick_kernels.cu -- a3-a14: prefix match (global-stop rule), load scorers, ordered weighted sum, arg-max pick,
// and the decode -> decider -> prefill two-stage pick.
//
// Arithmetic contract (SURVEY.md App. A.4/A.5): float64, IEEE round-to-nearest-even, NEVER fused -- every
// multiply/add/divide below is an explicit __d*_rn intrinsic (the file is also compiled with -fmad=false).
// Scorer order = profile order; accumulation starts from +0.0 (scheduler_profile.go:155-168).
//
// Work decomposition: all request-independent terms are derived once per pool snapshot (k_pool_*): per profile the
// candidate mask (role filter), queue min/max over the candidates, each scorer's clamp(score)*weight column and
// the ordered base sum every endpoint has when its prefix match is 0, plus the candidates sorted by
// (base desc, slot asc).  Per request only the few endpoints that actually hold a prefix need arithmetic; the
// best of all the others is the first unmatched entry of the sorted order.  This is exact, not an approximation:
// an unmatched endpoint's weighted sum is bit-identical to its base.
#include <math_constants.h>

#include <climits>

#include "index.cuh"
#include "pick_general.cuh"
#include "pick_latency.cuh"
#include "pick_random.cuh"
#include "score.cuh"

namespace epp {

// ------------------------------------------------------------------------------------------------
// pool snapshot -> derived per-profile arrays
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_pool_candidates(PoolArrays pool, int filter, LabelFilterDev labels,
                                                          uint32_t shard_begin, uint32_t shard_end, uint8_t *cand,
                                                          int32_t *n_cand, int64_t *qminmax) {
    __shared__ long long s_mn[2][32], s_mx[2][32];
    __shared__ int s_cnt[32];
    long long mnw = LLONG_MAX, mxw = LLONG_MIN, mnr = LLONG_MAX, mxr = LLONG_MIN;
    int cnt = 0;
    for (int e = threadIdx.x; e < pool.E; e += blockDim.x) {
        bool k = profile_keeps(filter, labels, pool, e);
        bool local = k && (uint32_t)e >= shard_begin && (uint32_t)e < shard_end;
        cand[e] = local ? 1 : 0;
        if (k) {      // queue min/max span every candidate of the pool, not only this shard's (queue.go:79-91)
            long long w = pool.waiting[e], r = pool.running[e];
            mnw = min(mnw, w); mxw = max(mxw, w);
            mnr = min(mnr, r); mxr = max(mxr, r);
        }
        if (local) cnt++;
    }
    for (int o = 16; o; o >>= 1) {
        mnw = min(mnw, __shfl_xor_sync(0xffffffffu, mnw, o));
        mxw = max(mxw, __shfl_xor_sync(0xffffffffu, mxw, o));
        mnr = min(mnr, __shfl_xor_sync(0xffffffffu, mnr, o));
        mxr = max(mxr, __shfl_xor_sync(0xffffffffu, mxr, o));
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { s_mn[0][w] = mnw; s_mx[0][w] = mxw; s_mn[1][w] = mnr; s_mx[1][w] = mxr; s_cnt[w] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int nw = blockDim.x >> 5;
        for (int i = 1; i < nw; i++) {
            s_mn[0][0] = min(s_mn[0][0], s_mn[0][i]); s_mx[0][0] = max(s_mx[0][0], s_mx[0][i]);
            s_mn[1][0] = min(s_mn[1][0], s_mn[1][i]); s_mx[1][0] = max(s_mx[1][0], s_mx[1][i]);
            s_cnt[0] += s_cnt[i];
        }
        qminmax[0] = s_mn[0][0]; qminmax[1] = s_mx[0][0];
        qminmax[2] = s_mn[1][0]; qminmax[3] = s_mx[1][0];
        *n_cand = s_cnt[0];
    }
}

// active-request scorers: max in-flight request count over the profile's candidates (whole pool, like the queue
// min/max), starting from 0 (active_request.go:144-155) -> qminmax[4 + s].
__global__ void __launch_bounds__(1024) k_pool_aux(PoolArrays pool, epp_profile_cfg cfg, int filter, LabelFilterDev labels,
                                                   int64_t *qminmax) {
    __shared__ long long s_mx[32];
    for (int s = 0; s < cfg.n_scorers; s++) {
        if (cfg.scorers[s].kind != EPP_SCORER_ACTIVE_REQUEST) continue;
        const int col = cfg.scorers[s].column;
        long long mx = 0;
        if (col >= 0 && col < pool.n_ext_cols)
            for (int e = threadIdx.x; e < pool.E; e += blockDim.x)
                if (profile_keeps(filter, labels, pool, e)) mx = max(mx, (long long)pool.ext[(size_t)col * (size_t)pool.E + (size_t)e]);
        for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if ((threadIdx.x & 31) == 0) s_mx[threadIdx.x >> 5] = mx;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int i = 1; i < (int)(blockDim.x >> 5); i++) s_mx[0] = max(s_mx[0], s_mx[i]);
            qminmax[4 + s] = s_mx[0];
        }
        __syncthreads();
    }
}

__device__ __forceinline__ uint64_t desc_key(double x) {
    // order-preserving map double -> u64 (ascending), then inverted so that an ASCENDING sort of the key
    // yields DESCENDING scores.
    uint64_t b = (uint64_t)__double_as_longlong(x);
    uint64_t asc = (b & 0x8000000000000000ULL) ? ~b : (b | 0x8000000000000000ULL);
    return ~asc;
}

// nohit_col: raw cold no-hit-lru score per slot, nullptr = the warm 0.5 (no_hit_lru.go:159-165).
__global__ void k_pool_terms(PoolArrays pool, epp_profile_cfg cfg, const uint8_t *cand, const int64_t *qminmax,
                             double *contrib, double *base, uint64_t *sort_key, uint32_t *order, int32_t Epad,
                             const double *nohit_col, const int32_t *gate) {
    if (gate && !*gate) return;
    int32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= Epad) return;
    if (e >= pool.E || !cand[e]) {
        if (e < pool.E) {
            base[e] = 0.0;
            for (int s = 0; s < cfg.n_scorers; s++) contrib[(size_t)s * (size_t)pool.E + e] = 0.0;
        }
        sort_key[e] = 0xFFFFFFFFFFFFFFFFULL;
        order[e] = (uint32_t)e;
        return;
    }
    double acc = 0.0;
    for (int s = 0; s < cfg.n_scorers; s++) {
        double raw;
        if (cfg.scorers[s].kind == EPP_SCORER_PREFIX) raw = 0.0;
        else if (cfg.scorers[s].kind == EPP_SCORER_NO_HIT_LRU) raw = nohit_col ? nohit_col[e] : 0.5;
        else raw = pool_score(cfg.scorers[s], s, pool, qminmax, e);
        double term = __dmul_rn(clamp01(raw), cfg.scorers[s].weight);
        contrib[(size_t)s * (size_t)pool.E + e] = term;
        acc = __dadd_rn(acc, term);
    }
    base[e] = acc;
    sort_key[e] = desc_key(acc);
    order[e] = (uint32_t)e;
}

// Single-CTA bitonic sort of (sort_key asc, slot asc) over Epad (power of two) entries in global memory.
__global__ void __launch_bounds__(1024) k_pool_sort(uint64_t *key, uint32_t *order, int32_t Epad, const int32_t *gate) {
    if (gate && !*gate) return;
    for (int32_t k = 2; k <= Epad; k <<= 1) {
        for (int32_t j = k >> 1; j > 0; j >>= 1) {
            for (int32_t i = threadIdx.x; i < Epad; i += blockDim.x) {
                int32_t ixj = i ^ j;
                if (ixj > i) {
                    uint64_t ka = key[i], kb = key[ixj];
                    uint32_t oa = order[i], ob = order[ixj];
                    bool a_gt_b = ka > kb || (ka == kb && oa > ob);
                    bool up = (i & k) == 0;
                    if (up ? a_gt_b : !a_gt_b) {
                        key[i] = kb; key[ixj] = ka;
                        order[i] = ob; order[ixj] = oa;
                    }
                }
            }
            __syncthreads();
        }
    }
}

__global__ void k_pool_groups(const double *base, const uint32_t *order, const int32_t *n_cand, uint32_t *grp_size,
                              const int32_t *gate) {
    if (gate && !*gate) return;
    int32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    int32_t n = *n_cand;
    if (k >= n) return;
    double b = base[order[k]];
    if (k > 0 && base[order[k - 1]] == b) return;        // not a group leader
    int32_t end = k + 1;
    while (end < n && base[order[end]] == b) end++;
    for (int32_t i = k; i < end; i++) grp_size[i] = (uint32_t)(end - k);
}

// Random pickers (pick_random.cuh): the candidates in ascending slot order, and over them wcum[i] = the left fold (+0.0
// first) of the weighted-random masses of the bases of cands[0 .. i), icum[i] = how many of those bases are +inf.  One
// CTA: each chunk of 1024 slots is compacted by the block, then one thread folds it in order (the fold is sequential by
// definition: round-to-nearest addition is not associative).
__global__ void __launch_bounds__(1024) k_pool_cum(const uint8_t *cand, const double *base, int32_t E, epp_profile_cfg cfg,
                                                   uint32_t *cands, double *wcum, uint32_t *icum, const int32_t *gate) {
    if (gate && !*gate) return;
    __shared__ double s_m[1024];
    __shared__ uint8_t s_inf[1024];
    __shared__ uint32_t s_wc[32];
    const double sigma = rnd::mass_scale(cfg);
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    uint32_t q = 0;                                   // candidates before the chunk (every thread keeps the same count)
    double acc = 0.0;                                 // thread 0: wcum[q]
    uint32_t ic = 0;                                  // thread 0: icum[q]
    if (t == 0) { wcum[0] = 0.0; icum[0] = 0; }
    for (int32_t e0 = 0; e0 < E; e0 += 1024) {
        const int32_t e = e0 + t;
        const bool c = e < E && cand[e];
        const uint32_t bal = __ballot_sync(0xffffffffu, c);
        if (lane == 0) s_wc[w] = __popc(bal);
        __syncthreads();
        uint32_t before = 0, nc = 0;
        for (int i = 0; i < 32; i++) { if (i < w) before += s_wc[i]; nc += s_wc[i]; }
        if (c) {
            const uint32_t pos = before + __popc(bal & ((1u << lane) - 1u));
            const double b = base[e];
            s_m[pos] = rnd::mass_of(b, sigma);
            s_inf[pos] = rnd::is_pinf(b) ? 1 : 0;
            cands[q + pos] = (uint32_t)e;
        }
        __syncthreads();
        if (t == 0)
            for (uint32_t i = 0; i < nc; i++) {
                acc = __dadd_rn(acc, s_m[i]);
                ic += s_inf[i];
                wcum[q + i + 1] = acc;
                icum[q + i + 1] = ic;
            }
        q += nc;
        __syncthreads();
    }
}

cudaError_t launch_pool_sort(uint64_t *key, uint32_t *order, int32_t Epad, const int32_t *gate, cudaStream_t s) {
    k_pool_sort<<<1, 1024, 0, s>>>(key, order, Epad, gate);
    return cudaGetLastError();
}

cudaError_t launch_pool_order(const PoolArrays &pool, const epp_profile_cfg &prof, const ProfileDerived &d, int32_t Epad,
                              const double *nohit_col, const int32_t *gate, cudaStream_t s, int *launches) {
    k_pool_terms<<<(Epad + 255) / 256, 256, 0, s>>>(pool, prof, d.cand, d.qminmax, d.contrib, d.base, d.sort_key,
                                                    d.order, Epad, nohit_col, gate);
    k_pool_sort<<<1, 1024, 0, s>>>(d.sort_key, d.order, Epad, gate);
    k_pool_groups<<<(pool.E + 255) / 256, 256, 0, s>>>(d.base, d.order, d.n_cand, d.grp_size, gate);
    if (launches) *launches += 3;
    if (d.wcum) {
        k_pool_cum<<<1, 1024, 0, s>>>(d.cand, d.base, pool.E, prof, d.cands, d.wcum, d.icum, gate);
        if (launches) *launches += 1;
    }
    return cudaGetLastError();
}

cudaError_t launch_pool_prepare(const PoolArrays &pool, const epp_profile_cfg &prof, const LabelFilterDev &labels,
                                const ProfileDerived &d, int32_t Epad, uint32_t shard_begin, uint32_t shard_end,
                                cudaStream_t s, int *launches) {
    k_pool_candidates<<<1, 1024, 0, s>>>(pool, prof.filter, labels, shard_begin, shard_end, d.cand, d.n_cand, d.qminmax);
    for (int i = 0; i < prof.n_scorers; i++)
        if (prof.scorers[i].kind == EPP_SCORER_ACTIVE_REQUEST) {
            k_pool_aux<<<1, 1024, 0, s>>>(pool, prof, prof.filter, labels, d.qminmax);
            if (launches) *launches += 1;
            break;
        }
    if (launches) *launches += 1;
    return launch_pool_order(pool, prof, d, Epad, nullptr, nullptr, s, launches);
}

// ------------------------------------------------------------------------------------------------
// fused lookup + match + score + pick: one warp per request
// ------------------------------------------------------------------------------------------------
constexpr int kListCap = 128;   // matched-endpoint list per request; beyond it the warp falls back to a dense scan
constexpr int kPickWarps = 8;

__device__ __forceinline__ uint32_t cnt_get(const uint32_t *cnt32, uint32_t e) {
    return (cnt32[e >> 1] >> ((e & 1u) * 16u)) & 0xFFFFu;
}

// Evaluate one profile for the current request.  cnt32 holds the per-endpoint match counts; list/nl the
// distinct matched endpoints (nl > kListCap => overflow => dense scan).
__device__ inline Best eval_profile_inner(const ProfileDev &pf, int32_t E, const uint32_t *cnt32, const uint32_t *list,
                                          uint32_t nl, int32_t total, int lane, const LoraDev &lora, uint32_t adapter);

// + the tie rule (score.cuh): the member of rank k of the arg-max set, found by one more scan over the slots.
// kForce: the member of rank force_rank instead (the seeded sharded select, include/epp_engine.h "Seeded ties").
template <bool kRand, bool kForce = false>
__device__ inline Best eval_profile(const ProfileDev &pf, int32_t E, const uint32_t *cnt32, const uint32_t *list,
                                    uint32_t nl, int32_t total, int lane, const LoraDev &lora, uint32_t adapter,
                                    uint64_t tie_seed, uint64_t tie_key, uint32_t force_rank = 0) {
    if (kRand && pf.cfg.picker) {                     // random pickers: explicit = matched or lora-resident candidates
        const bool use_lora = lora.enabled && lora.ptr;
        return rnd::draw_scan(pf, E, lane, true, (uint32_t)*pf.n_cand, 0u, tie_seed, tie_key,
                              [&](uint32_t e) { return pf.cand[e] != 0; },
                              [&](uint32_t e) { return cnt_get(cnt32, e) > 0 || (use_lora && lora_lookup(lora, adapter, e) != 0); },
                              [&](uint32_t e) {
                                  const uint32_t c = cnt_get(cnt32, e);
                                  if (use_lora) return weighted_sum(pf, E, e, (int32_t)c, total, lora, lora_lookup(lora, adapter, e));
                                  return c ? weighted_sum(pf, E, e, (int32_t)c, total) : pf.base[e];
                              },
                              [](uint32_t) { return false; });
    }
    Best b = eval_profile_inner(pf, E, cnt32, list, nl, total, lane, lora, adapter);
    if (kForce || (tie_seed && b.ties > 1)) {
        const bool use_lora = lora.enabled && lora.ptr;
        b.pick = select_kth_scan(pf, E, b.val, kForce ? force_rank : tie_rank(tie_seed, tie_key, b.ties), lane, [&](uint32_t e) {
            const uint32_t c = cnt_get(cnt32, e);
            if (use_lora) return weighted_sum(pf, E, e, (int32_t)c, total, lora, lora_lookup(lora, adapter, e));
            return c ? weighted_sum(pf, E, e, (int32_t)c, total) : pf.base[e];
        });
    }
    return b;
}

__device__ inline Best eval_profile_inner(const ProfileDev &pf, int32_t E, const uint32_t *cnt32, const uint32_t *list,
                                          uint32_t nl, int32_t total, int lane, const LoraDev &lora, uint32_t adapter) {
    Best b;
    best_init(b);
    int32_t ncand = *pf.n_cand;
    if (ncand == 0) return b;
    if (lora.enabled && lora.ptr) {
        // lora-affinity makes the score of some unmatched endpoints request-dependent: plain scan of every candidate
        for (uint32_t e = lane; e < (uint32_t)E; e += 32) {
            if (!pf.cand[e]) continue;
            best_add(b, weighted_sum(pf, E, e, (int32_t)cnt_get(cnt32, e), total, lora, lora_lookup(lora, adapter, e)), e);
        }
        return best_warp_reduce(b);
    }
    if (nl <= (uint32_t)kListCap) {
        for (uint32_t j = lane; j < nl; j += 32) {       // endpoints holding part of the prefix
            uint32_t e = list[j];
            if (pf.cand[e]) best_add(b, weighted_sum(pf, E, e, (int32_t)cnt_get(cnt32, e), total), e);
        }
        b = best_warp_reduce(b);
        // best of everyone else = first unmatched entry of the (base desc, slot asc) order
        for (int32_t k0 = 0; k0 < ncand; k0 += 32) {
            int32_t k = k0 + lane;
            uint32_t e = k < ncand ? pf.order[k] : EPP_NO_ENDPOINT;
            bool un = k < ncand && cnt_get(cnt32, e) == 0;
            uint32_t bal = __ballot_sync(0xffffffffu, un);
            if (bal) {
                int first = __ffs(bal) - 1;
                uint32_t ue = __shfl_sync(0xffffffffu, e, first);
                double ubase = pf.base[ue];
                uint32_t gsz = pf.grp_size[k0 + first];
                uint32_t same = 0;                        // matched candidates sharing that base value
                for (uint32_t j = lane; j < nl; j += 32) {
                    uint32_t me = list[j];
                    if (pf.cand[me] && pf.base[me] == ubase) same++;
                }
                for (int o = 16; o; o >>= 1) same += __shfl_xor_sync(0xffffffffu, same, o);
                best_add(b, ubase, ue, gsz - same);
                break;
            }
        }
    } else {
        for (uint32_t e = lane; e < (uint32_t)E; e += 32) {
            if (!pf.cand[e]) continue;
            uint32_t c = cnt_get(cnt32, e);
            best_add(b, c ? weighted_sum(pf, E, e, (int32_t)c, total) : pf.base[e], e);
        }
        b = best_warp_reduce(b);
    }
    return b;
}

// gen::eval for profile pi of request r, with the request's top-k rows (all rows are reset first: a stage that does
// not run leaves EPP_NO_ENDPOINT).
template <bool kRand, typename P, typename CntOf>
__device__ inline Best gen_eval_profile(const P &p, const ProfileDev &pf, int pi, int64_t r, int32_t total, int lane,
                                        uint32_t adapter, uint64_t key, CntOf cnt_of) {
    const int32_t k = p.gen.topk > 1 ? p.gen.topk : 1;
    if (pi == 0 && k > 1) {
        for (int q = 0; q < kMaxProfiles; q++)
            if (p.gen.topk_picks[q]) for (int j = lane; j < k; j += 32) p.gen.topk_picks[q][r * k + j] = EPP_NO_ENDPOINT;
        __syncwarp();
    }
    return gen::eval<kRand>(pf, p.gen, p.E, total, lane, p.lora, adapter, p.tie_seed, key, cnt_of, k,
                     (k > 1 && p.gen.topk_picks[pi]) ? p.gen.topk_picks[pi] + r * k : nullptr,
                     (k > 1 && pi == 0 && p.gen.topk_scores) ? p.gen.topk_scores + r * k : nullptr);
}

// lat::eval for chain profile pi of request r (the row handling of gen_eval_profile).
template <bool kRand, typename P, typename CntOf>
__device__ inline Best lat_eval_profile(const P &p, const LatView &lv, int pi, int64_t r, int32_t total, int lane,
                                        uint32_t adapter, uint64_t key, CntOf cnt_of) {
    const int32_t k = p.gen.topk > 1 ? p.gen.topk : 1;
    if (pi == 0 && k > 1) {
        for (int q = 0; q < kMaxProfiles; q++)
            if (p.gen.topk_picks[q]) for (int j = lane; j < k; j += 32) p.gen.topk_picks[q][r * k + j] = EPP_NO_ENDPOINT;
        __syncwarp();
    }
    lat::Req q;
    q.n = lv.cnt ? lv.cnt[lv.r0 + r] : 0u;
    q.ent = q.n ? lv.ent + lv.off[lv.r0 + r] : nullptr;
    const lat::CtxLen cl = lat::ctx_len(lv, pi, lv.r0 + r, p.in_len ? p.in_len[r] : 0);
    return lat::eval<kRand>(p.prof[pi], lv.cfg[pi], cl, p.gen, q, p.E, total, lane, p.lora, adapter, p.tie_seed, key,
                            lat::pool_dom(p.E, cnt_of), k,
                            (k > 1 && p.gen.topk_picks[pi]) ? p.gen.topk_picks[pi] + r * k : nullptr,
                            (k > 1 && pi == 0 && p.gen.topk_scores) ? p.gen.topk_scores + r * k : nullptr);
}

// kRand: the engine has a random picker (k_match_pick_rand); the max-score build carries none of its code.
// kLat: the engine has latency profiles (k_match_pick_lat*): those evaluate through lat::eval with the request's entries.
// kSel: the seeded sharded select (k_match_pick_select): the items of sv->dense_list, each one profile with the rank of
// its member forced, written to sv->sel.
template <bool kRand, bool kLat = false, bool kSel = false>
__device__ __forceinline__ void match_pick_dense(const PickParams &p, int32_t cnt_words, uint32_t *gscratch,
                                                 const LatView *lv = nullptr, const ShardSelView *sv = nullptr) {
    extern __shared__ uint32_t smem[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int64_t gwarp = (int64_t)blockIdx.x * kPickWarps + warp;
    const int64_t nwarps = (int64_t)gridDim.x * kPickWarps;
    // the overflow pass runs over a full grid and its list is almost always empty: a warp without a request leaves
    // before it clears its counters (no block-wide barrier below)
    const int64_t n_work = kSel ? (int64_t)*sv->dense_n : (p.req_list ? (int64_t)*p.req_list_n : p.R);
    if (gwarp >= n_work) return;
    uint32_t *cnt32;
    uint32_t *list;
    if (gscratch) {
        cnt32 = gscratch + (size_t)gwarp * (size_t)cnt_words;   // kept all-zero between requests
        list = smem + warp * (kListCap + 4);
    } else {
        uint32_t *mine = smem + (size_t)warp * (size_t)(cnt_words + kListCap + 4);
        cnt32 = mine;
        list = mine + cnt_words;
        for (int i = lane; i < cnt_words; i += 32) cnt32[i] = 0;
    }
    uint32_t *list_n = list + kListCap;
    unsigned long long w_probes = 0, w_postings = 0;    // algorithmic work of this warp's requests
    __syncwarp();

    for (int64_t wi = gwarp; wi < n_work; wi += nwarps) {
        const int64_t r = kSel ? (int64_t)(sv->work[sv->dense_list[wi]].x / (uint32_t)sv->stages)
                               : (p.req_list ? (int64_t)p.req_list[wi] : wi);
        const int32_t total = p.nblocks[r];
        const int32_t stored = p.bound ? p.bound[r] : total;      // block `stored` < total: a proven miss
        if (lane == 0) *list_n = 0;
        __syncwarp();
        // ---- a2/a3: probe in block order, global stop at the first block nobody holds (plugin.go:214-230)
        const uint64_t *row = p.hashes + r * (int64_t)p.max_blocks;
        for (int32_t c0 = 0; c0 < total; c0 += 32) {
            int32_t i = c0 + lane;
            bool active = i < total;
            Hit hit;
            hit.cnt = 0;
            bool found = false;
            if (i < stored) found = probe(p.index, row[i], hit);
            if (!found) hit.cnt = 0;
            const uint32_t cnt = hit.cnt;
            uint32_t miss;
            if (p.global_masks) {   // sharded: a block is missing only if NO rank holds it
                uint32_t word = p.global_masks[r * (int64_t)p.mask_words + (c0 >> 5)];
                uint32_t valid = (total - c0) >= 32 ? 0xffffffffu : ((1u << (total - c0)) - 1u);
                miss = ~word & valid;
            } else {
                miss = __ballot_sync(0xffffffffu, active && !found);
            }
            int32_t limit = miss ? c0 + (__ffs(miss) - 1) : total;
            if (active && i < limit) {
                w_postings += cnt;
                for (uint32_t k = 0; k < cnt; k++) {
                    uint32_t e = posting(p.index, hit, k);
                    if (e >= p.index.ep_begin && e < p.index.ep_end && e < (uint32_t)p.E) {
                        uint32_t sh = (e & 1u) * 16u;
                        uint32_t old = atomicAdd(&cnt32[e >> 1], 1u << sh);
                        if (((old >> sh) & 0xFFFFu) == 0) {
                            uint32_t pos = atomicAdd(list_n, 1u);
                            if (pos < (uint32_t)kListCap) list[pos] = e;
                        }
                    }
                }
            }
            if (lane == 0) w_probes += (unsigned long long)((miss ? limit + 1 : min(total, c0 + 32)) - c0);
            if (miss) break;
        }
        __syncwarp();
        const uint32_t nl = *list_n;

        // ---- a5-a14: the profiles of the handler
        const uint32_t adapter = p.model_ids ? p.model_ids[r] : 0u;
        epp_decision d;
        epp_decision_detail dd;
        auto cnt_of = [&](uint32_t e) { return (int32_t)cnt_get(cnt32, e); };
        bool cold = false;
        auto is_cold = [&](const ProfileDev &pf) { return cold_scan(pf, p.E, lane, cnt_of); };
        bool staged = false;
        if constexpr (kSel) {
            const uint2 it = sv->work[sv->dense_list[wi]];
            const Best b = eval_profile<false, true>(p.prof[it.x % (uint32_t)sv->stages], p.E, cnt32, list, nl, total, lane,
                                                     p.lora, adapter, 0, 0, it.y);
            if (lane == 0) {
                epp_shard_sel s;
                s.pick = b.pick;
                s.match_blocks = (int32_t)cnt_get(cnt32, b.pick);
                sv->sel[it.x] = s;
            }
            staged = true;                               // nothing else is written
        } else if constexpr (kLat) {
            decide_stages<3>(p, r, total, p.n_profiles >= 2 ? p.in_len[r] : 0,
                          [&](int pi, uint64_t key) {
                              if ((lv->mask >> pi) & 1) return lat_eval_profile<kRand>(p, *lv, pi, r, total, lane, adapter, key, cnt_of);
                              return gen_eval_profile<kRand>(p, nohit_select(p, pi, cold, is_cold), pi, r, total, lane, adapter, key, cnt_of);
                          },
                          cnt_of, d, dd);
        } else if (p.gen.on) {       // affinity filter / top-k: full-scan evaluation (pick_general.cuh)
            decide_stages<3>(p, r, total, p.n_profiles >= 2 ? p.in_len[r] : 0,
                          [&](int pi, uint64_t key) { return gen_eval_profile<kRand>(p, nohit_select(p, pi, cold, is_cold), pi, r, total, lane, adapter, key, cnt_of); },
                          cnt_of, d, dd);
        } else {
            // endpoint-sharded mode under the disagg handler (never with a random picker or no-hit-lru): one record per stage
            if constexpr (!kRand) {
                if (p.shard_out && handler_stages(p) > 1) {
                    staged = true;
                    shard_stage_records(p, r, handler_stages(p), p.in_len[r],
                                        [&](int pi, uint64_t key) { return eval_profile<false>(p.prof[pi], p.E, cnt32, list, nl, total, lane, p.lora, adapter, p.tie_seed, key); },
                                        cnt_of, lane);
                }
            }
            if (!staged)
                decide_stages<3>(p, r, total, p.n_profiles >= 2 ? p.in_len[r] : 0,
                              [&](int pi, uint64_t key) { return eval_profile<kRand>(nohit_select(p, pi, cold, is_cold), p.E, cnt32, list, nl, total, lane, p.lora, adapter, p.tie_seed, key); },
                              cnt_of, d, dd);
        }
        if (lane == 0 && p.nohit.cold_out) p.nohit.cold_out[r] = cold ? 1 : 0;
        if constexpr (!kSel) {
            if (lane == 0 && !staged) {
                if (p.shard_out) {
                    epp_shard_best sb;
                    sb.score = d.score; sb.pick = d.pick; sb.tie_count = d.tie_count;
                    sb.match_blocks = d.match_blocks; sb.status = d.status;
                    p.shard_out[r] = sb;
                } else {
                    p.out[r] = d;
                    if (p.detail) p.detail[r] = dd;
                }
            }
        }
        // ---- a4: dense match row (Produce parity mode only)
        if (p.out_match) {
            int32_t *mrow = p.out_match + r * (int64_t)p.E;
            if (nl <= (uint32_t)kListCap) {
                for (int32_t e = lane; e < p.E; e += 32) mrow[e] = 0;
                __syncwarp();
                for (uint32_t j = lane; j < nl; j += 32) mrow[list[j]] = (int32_t)cnt_get(cnt32, list[j]);
            } else {
                for (int32_t e = lane; e < p.E; e += 32) mrow[e] = (int32_t)cnt_get(cnt32, (uint32_t)e);
            }
        }
        __syncwarp();
        // ---- reset the counters this request touched
        if (nl <= (uint32_t)kListCap) {
            for (uint32_t j = lane; j < nl; j += 32) cnt32[list[j] >> 1] = 0;
        } else {
            for (int i = lane; i < cnt_words; i += 32) cnt32[i] = 0;
        }
        __syncwarp();
    }
    if (p.work_counters) {
        for (int o = 16; o; o >>= 1) w_postings += __shfl_xor_sync(0xffffffffu, w_postings, o);
        if (lane == 0) {
            atomicAdd(&p.work_counters[0], w_probes);
            atomicAdd(&p.work_counters[1], w_postings);
        }
    }
}

__global__ void __launch_bounds__(kPickWarps * 32) k_match_pick(PickParams p, int32_t cnt_words, uint32_t *gscratch) {
    match_pick_dense<false>(p, cnt_words, gscratch);
}
__global__ void __launch_bounds__(kPickWarps * 32) k_match_pick_rand(PickParams p, int32_t cnt_words, uint32_t *gscratch) {
    match_pick_dense<true>(p, cnt_words, gscratch);
}

__global__ void __launch_bounds__(kPickWarps * 32) k_match_pick_select(PickParams p, int32_t cnt_words, uint32_t *gscratch, ShardSelView sv) {
    match_pick_dense<false, false, true>(p, cnt_words, gscratch, nullptr, &sv);
}

__global__ void __launch_bounds__(kPickWarps * 32) k_match_pick_lat(PickParams p, int32_t cnt_words, uint32_t *gscratch, LatView lv) {
    match_pick_dense<false, true>(p, cnt_words, gscratch, &lv);
}
__global__ void __launch_bounds__(kPickWarps * 32) k_match_pick_lat_rand(PickParams p, int32_t cnt_words, uint32_t *gscratch, LatView lv) {
    match_pick_dense<true, true>(p, cnt_words, gscratch, &lv);
}

// The engine allocates gscratch when E does not fit in shared memory; see engine.cu.
size_t match_pick_smem_bytes(int32_t E, bool global_counts) {
    int32_t cnt_words = (E + 1) / 2;
    size_t per_warp = (size_t)(global_counts ? 0 : cnt_words) + kListCap + 4;
    return per_warp * sizeof(uint32_t) * kPickWarps;
}
int match_pick_warps_per_cta() { return kPickWarps; }

cudaError_t launch_match_pick(const PickParams &p, uint32_t *gscratch, int grid, size_t smem, cudaStream_t s,
                                  int *launches) {
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_set[64] = {};                 // function attributes are per device: engines of one process may sit on several GPUs
    if (!attr_set[dev & 63]) {
        cudaError_t e = cudaFuncSetAttribute(k_match_pick, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_match_pick_rand, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 63] = true;
    }
    int32_t cnt_words = (p.E + 1) / 2;
    if (any_random_picker(p)) k_match_pick_rand<<<grid, kPickWarps * 32, smem, s>>>(p, cnt_words, gscratch);
    else k_match_pick<<<grid, kPickWarps * 32, smem, s>>>(p, cnt_words, gscratch);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_match_pick_select(const PickParams &p, const ShardSelView &sv, uint32_t *gscratch, int grid, size_t smem,
                                     cudaStream_t s, int *launches) {
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_set[64] = {};
    if (!attr_set[dev & 63]) {
        const cudaError_t e = cudaFuncSetAttribute(k_match_pick_select, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 63] = true;
    }
    k_match_pick_select<<<grid, kPickWarps * 32, smem, s>>>(p, (p.E + 1) / 2, gscratch, sv);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_match_pick_lat(const PickParams &p, const LatView &lv, uint32_t *gscratch, int grid, size_t smem,
                                  cudaStream_t s, int *launches) {
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_set[64] = {};
    if (!attr_set[dev & 63]) {
        cudaError_t e = cudaFuncSetAttribute(k_match_pick_lat, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_match_pick_lat_rand, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 63] = true;
    }
    int32_t cnt_words = (p.E + 1) / 2;
    if (any_random_picker(p)) k_match_pick_lat_rand<<<grid, kPickWarps * 32, smem, s>>>(p, cnt_words, gscratch, lv);
    else k_match_pick_lat<<<grid, kPickWarps * 32, smem, s>>>(p, cnt_words, gscratch, lv);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// decision logic on injected dense match info (KAT / plugin-parity mode)
// ------------------------------------------------------------------------------------------------
template <bool kRand>
__device__ inline Best eval_profile_dense(const ProfileDev &pf, int32_t E, const int32_t *mrow, int32_t total,
                                          int lane, const LoraDev &lora, uint32_t adapter, uint64_t tie_seed,
                                          uint64_t tie_key) {
    Best b;
    best_init(b);
    const bool use_lora = lora.enabled && lora.ptr;
    auto score_of = [&](uint32_t e) {
        return weighted_sum(pf, E, e, mrow[e], total, lora, use_lora ? lora_lookup(lora, adapter, e) : 0);
    };
    if (kRand && pf.cfg.picker)
        return rnd::draw_scan(pf, E, lane, true, (uint32_t)*pf.n_cand, 0u, tie_seed, tie_key,
                              [&](uint32_t e) { return pf.cand[e] != 0; },
                              [&](uint32_t e) { return mrow[e] > 0 || (use_lora && lora_lookup(lora, adapter, e) != 0); }, score_of,
                              [](uint32_t) { return false; });
    for (uint32_t e = lane; e < (uint32_t)E; e += 32) {
        if (!pf.cand[e]) continue;
        best_add(b, score_of(e), e);
    }
    b = best_warp_reduce(b);
    if (tie_seed && b.ties > 1) b.pick = select_kth_scan(pf, E, b.val, tie_rank(tie_seed, tie_key, b.ties), lane, score_of);
    return b;
}

template <bool kRand, bool kLat = false>
__device__ __forceinline__ void dense_pick(const DensePickParams &p, const LatView *lv = nullptr) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= p.R) return;
    const int32_t *mrow = p.match + r * (int64_t)p.E;
    int32_t total = p.total[r];
    const uint32_t adapter = p.model_ids ? p.model_ids[r] : 0u;
    epp_decision d;
    epp_decision_detail dd;
    auto cnt_of = [&](uint32_t e) { return mrow[e]; };
    bool cold = false;
    auto is_cold = [&](const ProfileDev &pf) { return cold_scan(pf, p.E, lane, cnt_of); };
    if constexpr (kLat) {
        decide_stages<3>(p, r, total, p.in_len ? p.in_len[r] : 0,
                      [&](int pi, uint64_t key) {
                          if ((lv->mask >> pi) & 1) return lat_eval_profile<kRand>(p, *lv, pi, r, total, lane, adapter, key, cnt_of);
                          return gen_eval_profile<kRand>(p, nohit_select(p, pi, cold, is_cold), pi, r, total, lane, adapter, key, cnt_of);
                      },
                      cnt_of, d, dd);
    } else if (p.gen.on) {
        decide_stages<3>(p, r, total, p.in_len ? p.in_len[r] : 0,
                      [&](int pi, uint64_t key) { return gen_eval_profile<kRand>(p, nohit_select(p, pi, cold, is_cold), pi, r, total, lane, adapter, key, cnt_of); },
                      cnt_of, d, dd);
    } else {
        decide_stages<3>(p, r, total, p.in_len ? p.in_len[r] : 0,
                      [&](int pi, uint64_t key) { return eval_profile_dense<kRand>(nohit_select(p, pi, cold, is_cold), p.E, mrow, total, lane, p.lora, adapter, p.tie_seed, key); },
                      cnt_of, d, dd);
    }
    if (lane == 0 && p.nohit.cold_out) p.nohit.cold_out[r] = cold ? 1 : 0;
    if (lane == 0) {
        p.out[r] = d;
        if (p.detail) p.detail[r] = dd;
    }
}

__global__ void __launch_bounds__(256) k_dense_pick(DensePickParams p) { dense_pick<false>(p); }
__global__ void __launch_bounds__(256) k_dense_pick_rand(DensePickParams p) { dense_pick<true>(p); }

cudaError_t launch_dense_pick(const DensePickParams &p, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    int64_t threads = p.R * 32;
    if (any_random_picker(p)) k_dense_pick_rand<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p);
    else k_dense_pick<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) k_dense_pick_lat(DensePickParams p, LatView lv) { dense_pick<false, true>(p, &lv); }
__global__ void __launch_bounds__(256) k_dense_pick_lat_rand(DensePickParams p, LatView lv) { dense_pick<true, true>(p, &lv); }

cudaError_t launch_dense_pick_lat(const DensePickParams &p, const LatView &lv, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    int64_t threads = p.R * 32;
    if (any_random_picker(p)) k_dense_pick_lat_rand<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p, lv);
    else k_dense_pick_lat<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(p, lv);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

// Scorer.Score parity (dense [R][E] output).
__global__ void k_score_dense(int64_t R, int32_t E, ProfileDev pw, ProfileDev pcold, const uint8_t *cold,
                              const double *nohit_col, PoolArrays pool,
                              const int64_t *qminmax, const int32_t *match, const int32_t *total, const uint32_t *model_ids,
                              int32_t scorer_index, double *out) {
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= R * (int64_t)E) return;
    int64_t r = idx / E;
    int32_t e = (int32_t)(idx % E);
    const ProfileDev &pf = (cold && cold[r]) ? pcold : pw;
    bool c = pf.cand[e] != 0;
    const int lora_st = (pool.lora.enabled && pool.lora.ptr) ? lora_lookup(pool.lora, model_ids ? model_ids[r] : 0u, (uint32_t)e) : 0;
    double v;
    if (scorer_index < 0) {
        v = c ? weighted_sum(pf, E, (uint32_t)e, match[idx], total[r], pool.lora, lora_st) : -1.0;
    } else if (!c) {
        v = 0.0;
    } else {
        const epp_scorer_cfg &sc = pf.cfg.scorers[scorer_index];
        if (sc.kind == EPP_SCORER_NO_HIT_LRU)        // no_hit_lru.go:259-275
            v = (cold && cold[r]) ? nohit_col[e] : 0.5;
        else
            v = sc.kind == EPP_SCORER_PREFIX ? prefix_score(match[idx], total[r])
                : (sc.kind == EPP_SCORER_LORA_AFFINITY ? lora_score(pool.lora, (uint32_t)e, lora_st)
                                                       : pool_score(sc, scorer_index, pool, qminmax, e));
    }
    out[idx] = v;
}

cudaError_t launch_score_dense(int64_t R, int32_t E, const ProfileDev &prof, const ProfileDev &prof_cold,
                               const uint8_t *cold, const double *nohit_col, const PoolArrays &pool,
                               const int64_t *qminmax, const int32_t *match, const int32_t *total,
                               const uint32_t *model_ids, int32_t scorer_index, double *out, cudaStream_t s,
                               int *launches) {
    int64_t n = R * (int64_t)E;
    if (n <= 0) return cudaSuccess;
    k_score_dense<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(R, E, prof, prof_cold, cold, nohit_col, pool, qminmax, match, total,
                                                             model_ids, scorer_index, out);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// endpoint-sharded mode (SURVEY.md 8(e)): presence masks + merge of the per-shard best records
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_shard_probe(int64_t R, int32_t max_blocks, const uint64_t *hashes,
                                                     const int32_t *nblocks, IndexView index, uint32_t *out_masks,
                                                     int32_t mask_words) {
    const int lane = threadIdx.x & 31;
    const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= R) return;
    const int32_t total = nblocks[r];
    const uint64_t *row = hashes + r * (int64_t)max_blocks;
    for (int32_t w = 0; w < mask_words; w++) {
        int32_t i = w * 32 + lane;
        bool hit = false;
        if (i < total) {
            Hit h;
            hit = probe(index, row[i], h);
        }
        uint32_t word = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) out_masks[r * (int64_t)mask_words + w] = word;
    }
}

cudaError_t launch_shard_probe(int64_t R, int32_t max_blocks, const uint64_t *hashes, const int32_t *nblocks,
                               const IndexView &index, uint32_t *out_masks, int32_t mask_words, cudaStream_t s,
                               int *launches) {
    if (R <= 0) return cudaSuccess;
    int64_t threads = R * 32;
    k_shard_probe<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(R, max_blocks, hashes, nblocks, index, out_masks,
                                                                   mask_words);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

// Stage st of request r over every rank's record: the max score, lowest slot id among equals, ties summed; mb = the
// match_blocks of the winning record.
__device__ __forceinline__ Best merge_stage(const ShardMergeParams &p, int64_t r, int st, int32_t &mb) {
    Best b;
    best_init(b);
    mb = 0;
    for (int32_t k = 0; k < p.n_ranks; k++) {
        epp_shard_best sb = p.all_best[((int64_t)k * p.R + r) * p.stages + st];
        if (sb.status != 0) continue;
        uint32_t before = b.pick;
        best_add(b, sb.score, sb.pick, sb.tie_count);
        if (b.pick != before) mb = sb.match_blocks;
    }
    return b;
}

// The decision of request r from the reduced stages (stage(st, mb) -> the stage's Best, mb = its pick's match count), as
// decide_stages makes it from one pool.
template <typename Stage>
__device__ __forceinline__ void shard_decide(const ShardMergeParams &p, int64_t r, Stage stage) {
    int32_t mb;
    const Best b = stage(0, mb);
    epp_decision d;
    d.status = b.ties ? 0 : -1;
    d.pick = b.ties ? b.pick : EPP_NO_ENDPOINT;
    d.score = b.ties ? b.val : 0.0;
    d.prefill_pick = EPP_NO_ENDPOINT;
    d.tie_count = b.ties;
    d.total_blocks = p.nblocks[r];
    d.match_blocks = b.ties ? mb : 0;
    epp_decision_detail dd;
    dd.prefill_score = 0.0; dd.prefill_tie_count = 0; dd.prefill_ran = 0;
    dd.encode_score = 0.0; dd.encode_pick = EPP_NO_ENDPOINT; dd.encode_tie_count = 0; dd.encode_ran = 0; dd.reserved = 0;
    if (b.ties && p.stages >= 3 && p.multimodal && p.multimodal[r]) {   // no decode pick: no other stage runs
        dd.encode_ran = 1;
        const Best b2 = stage(2, mb);
        if (b2.ties) { dd.encode_pick = b2.pick; dd.encode_score = b2.val; dd.encode_tie_count = b2.ties; }
    }
    if (b.ties && p.stages >= 2 &&
        (p.always_disagg || pd_decide(p.non_cached_tokens, p.in_len[r], d.match_blocks, p.block_size_tokens))) {
        dd.prefill_ran = 1;
        const Best b1 = stage(1, mb);
        if (b1.ties) { d.prefill_pick = b1.pick; dd.prefill_score = b1.val; dd.prefill_tie_count = b1.ties; }
    }
    p.out[r] = d;
    if (p.detail) p.detail[r] = dd;
}

__global__ void k_shard_merge(ShardMergeParams p) {
    int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    shard_decide(p, r, [&](int st, int32_t &mb) { return merge_stage(p, r, st, mb); });
}

cudaError_t launch_shard_merge(const ShardMergeParams &p, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    k_shard_merge<<<(unsigned)((p.R + 255) / 256), 256, 0, s>>>(p);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

// Seeded ties (include/epp_engine.h, "Seeded ties").  The arg-max set of stage st over every rank is the union of the
// local sets of the records at the max (b, from merge_stage); the shard ranges are disjoint, so in ascending slot order
// it is those local sets taken in the order of their lowest members, the records' picks.  -> the rank (index in
// all_best) that owns member tie_rank(seed, 4 * (tie_base + r) + st, b.ties) and its rank in that rank's local set;
// rank -1 when no rank has a candidate.  At most n_ranks passes over n_ranks records.
struct ShardOwner {
    int32_t rank;
    uint32_t local;
};
__device__ __forceinline__ ShardOwner shard_owner(const ShardMergeParams &p, const ShardSeedParams &sp, int64_t r, int st,
                                                  const Best &b) {
    ShardOwner o{-1, 0u};
    if (!b.ties) return o;
    uint32_t rho = b.ties > 1 ? tie_rank(sp.tie_seed, 4 * (sp.tie_base + (uint64_t)r) + (uint64_t)st, b.ties) : 0u;
    int64_t after = -1;                                  // the pick of the last local set passed
    for (int32_t n = 0; n < p.n_ranks; n++) {
        int32_t next = -1;
        uint32_t lo = EPP_NO_ENDPOINT;
        for (int32_t k = 0; k < p.n_ranks; k++) {
            const epp_shard_best sb = p.all_best[((int64_t)k * p.R + r) * p.stages + st];
            if (sb.status == 0 && sb.score == b.val && (int64_t)sb.pick > after && (next < 0 || sb.pick < lo)) {
                next = k;
                lo = sb.pick;
            }
        }
        if (next < 0) break;
        const uint32_t c = p.all_best[((int64_t)next * p.R + r) * p.stages + st].tie_count;
        if (rho < c) { o.rank = next; o.local = rho; break; }
        rho -= c;
        after = lo;
    }
    return o;
}

// One thread per (request, stage): this rank's entry -- the owner's record pick when this rank owns it (the member of
// local rank 0 is that pick), EPP_NO_ENDPOINT otherwise -- and a work item for each owned member of local rank >= 1.
__global__ void k_shard_resolve(ShardMergeParams p, ShardSeedParams sp) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.R * p.stages) return;
    const int64_t r = i / p.stages;
    const int st = (int)(i % p.stages);
    int32_t mb;
    const Best b = merge_stage(p, r, st, mb);
    const ShardOwner o = shard_owner(p, sp, r, st, b);
    epp_shard_sel s;
    s.pick = EPP_NO_ENDPOINT;
    s.match_blocks = 0;
    if (o.rank >= 0) {
        const epp_shard_best own = p.all_best[((int64_t)o.rank * p.R + r) * p.stages + st];
        if (own.pick >= sp.ep_begin && own.pick < sp.ep_end) {
            s.pick = own.pick;
            s.match_blocks = own.match_blocks;
            if (o.local) sp.work[atomicAdd(sp.work_n, 1)] = make_uint2((uint32_t)i, o.local);
        }
    }
    sp.sel[i] = s;
}

cudaError_t launch_shard_resolve(const ShardMergeParams &p, const ShardSeedParams &sp, cudaStream_t s, int *launches) {
    const int64_t n = p.R * p.stages;
    if (n <= 0) return cudaSuccess;
    k_shard_resolve<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, sp);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

// The decisions as k_shard_merge builds them, each stage's pick and match count taken from its owner's entry.
__global__ void k_shard_finish(ShardMergeParams p, ShardSeedParams sp) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= p.R) return;
    shard_decide(p, r, [&](int st, int32_t &mb) {
        Best b = merge_stage(p, r, st, mb);
        const ShardOwner o = shard_owner(p, sp, r, st, b);
        if (o.rank >= 0) {
            const epp_shard_sel s = sp.all_sel[((int64_t)o.rank * p.R + r) * p.stages + st];
            b.pick = s.pick;
            mb = s.match_blocks;
        }
        return b;
    });
}

cudaError_t launch_shard_finish(const ShardMergeParams &p, const ShardSeedParams &sp, cudaStream_t s, int *launches) {
    if (p.R <= 0) return cudaSuccess;
    k_shard_finish<<<(unsigned)((p.R + 255) / 256), 256, 0, s>>>(p, sp);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
