// subset_pick.cu -- per-request endpoint subsets (include/epp_engine.h, "Endpoint subsets"): the gateway's
// x-gateway-destination-endpoint-subset hint hands Scheduler.Schedule only the endpoints of the subset
// (requestcontrol/candidates.go:98-167, director.go:222-243).  One warp re-decides one restricted request after the
// batch's ordinary match kernels have decided it over the whole pool:
//   * match: the request's stored hash row is walked through the read table up to the GLOBAL stop (the first block no
//     endpoint holds, approximateprefix/plugin.go:214-230 -- the index is not narrowed) and only holders in the request's
//     slot list are counted, one int32 counter per list entry (posting lists are duplicate-free and the warp handles one
//     block at a time, so no two lanes bump the same counter);
//   * decide: every profile's candidates are the listed slots that pass its role filter; the affinity filter, the
//     queue / running min-max, the active-request max, the no-hit-lru cold test and ranks, tie counts and ranks, the
//     first-k lists and the random pickers' populations are all taken over those candidates (never over the per-snapshot
//     arrays, which describe the whole pool).
// Every step scans the request's list (ascending slot order), so a request costs O(blocks * holders * log S + S) for S
// listed slots.  The kernels of match_sparse.cuh / pick_kernels.cu are not touched: this one only runs for batches that
// carry a restricted request.  On an engine with latency profiles, k_subset_pick_lat evaluates those profiles with the
// chain of pick_latency.cuh over the request's list (lat::ListDom) and the request's predictions; its other profiles,
// the match walk and the rest of the row's handling are k_subset_pick's.
#include <cfloat>
#include <climits>

#include "index.cuh"
#include "pick_general.cuh"
#include "pick_latency.cuh"

namespace epp {
namespace {

constexpr int kSubsetWarps = 4;            // warps per CTA (one restricted request each)
constexpr uint32_t kFull = 0xffffffffu;

// Position of slot e in the ascending list sl[0 .. n), or n when it is not listed.
__device__ __forceinline__ uint32_t list_find(const uint32_t *sl, uint32_t n, uint32_t e) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (sl[mid] < e) lo = mid + 1; else hi = mid;
    }
    return (lo < n && sl[lo] == e) ? lo : n;
}

// The scorers' normalisation over the selected entries of the list (layout of ProfileDerived::qminmax): waiting and
// running min / max, the active-request scorers' max in-flight count starting from 0 (active_request.go:144-155).
template <typename Sel>
__device__ inline uint32_t norm_over(const epp_profile_cfg &c, const PoolArrays &pool, const uint32_t *sl, uint32_t n,
                                     int lane, Sel sel, int64_t *q) {
    uint32_t cnt = 0;
    long long mnw = LLONG_MAX, mxw = LLONG_MIN, mnr = LLONG_MAX, mxr = LLONG_MIN;
    for (uint32_t i = lane; i < n; i += 32) {
        if (!sel(i)) continue;
        const uint32_t e = sl[i];
        const long long w = pool.waiting[e], r = pool.running[e];
        cnt++;
        mnw = min(mnw, w); mxw = max(mxw, w);
        mnr = min(mnr, r); mxr = max(mxr, r);
    }
    for (int o = 16; o; o >>= 1) {
        cnt += __shfl_xor_sync(kFull, cnt, o);
        mnw = min(mnw, __shfl_xor_sync(kFull, mnw, o)); mxw = max(mxw, __shfl_xor_sync(kFull, mxw, o));
        mnr = min(mnr, __shfl_xor_sync(kFull, mnr, o)); mxr = max(mxr, __shfl_xor_sync(kFull, mxr, o));
    }
    q[0] = mnw; q[1] = mxw; q[2] = mnr; q[3] = mxr;
    for (int s = 0; s < c.n_scorers; s++) {
        q[4 + s] = 0;
        if (c.scorers[s].kind != EPP_SCORER_ACTIVE_REQUEST) continue;
        const int col = c.scorers[s].column;
        long long mx = 0;
        if (col >= 0 && col < pool.n_ext_cols)
            for (uint32_t i = lane; i < n; i += 32)
                if (sel(i)) mx = max(mx, (long long)pool.ext[(size_t)col * (size_t)pool.E + (size_t)sl[i]]);
        for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(kFull, mx, o));
        q[4 + s] = mx;
    }
    return cnt;
}

struct SubsetReq {                 // one restricted request, as the warp sees it
    const uint32_t *sl;            // its slots, ascending
    const int32_t *hit;            // matchBlocks per listed slot
    int32_t *num;                  // scratch per listed slot: the no-hit-lru cold rank's numerator
    uint32_t n;
    int32_t total;
    uint32_t adapter;
};

// One SchedulerProfile over the request's listed slots: role filter -> [affinity filter] -> scorers -> picker.  Returns
// the record of the pick (value, slot, size of the arg-max set / the random population); picks_row / scores_row
// (k entries, or nullptr) receive the first-k list.  has_nohit: the profile lists the no-hit-lru scorer; *cold is set to
// the request's cold bit for it when the profile has candidates.
__device__ Best eval_subset(const ProfileDev &pf, const PickParams &p, const SubsetView &sv, const SubsetReq &q, int lane,
                            uint64_t key, bool has_nohit, bool *cold, int32_t k, uint32_t *picks_row, double *scores_row) {
    Best first;
    best_init(first);
    if (k < 1) k = 1;
    if (picks_row) for (int j = lane; j < k; j += 32) picks_row[j] = EPP_NO_ENDPOINT;
    if (scores_row) for (int j = lane; j < k; j += 32) scores_row[j] = 0.0;
    __syncwarp();
    const epp_profile_cfg &c = pf.cfg;
    const PoolArrays &pool = p.gen.pool;
    const uint32_t *sl = q.sl;
    const uint32_t n = q.n;
    const int32_t total = q.total;
    gen::Norm nm;
    nm.sticky = false;
    nm.thr = c.affinity_threshold;
    auto in_role = [&](uint32_t i) { return pf.cand[sl[i]] != 0; };
    const uint32_t n_role = norm_over(c, pool, sl, n, lane, in_role, nm.q);
    if (n_role == 0) return first;

    // no-hit-lru isColdRequest (no_hit_lru.go:140-155) over the candidates, and the cold ranks (:198-250): never-used
    // candidates by their index in slot order, LRU members by neverUsedCount + their position in the (global) LRU
    bool is_cold = false;
    if (has_nohit) {
        bool h = false;
        for (uint32_t i = lane; i < n && !h; i += 32) h = in_role(i) && q.hit[i] > 0;
        is_cold = !__any_sync(kFull, h);
        *cold = is_cold;
        if (is_cold) {
            uint32_t nu_all = 0;
            for (uint32_t i = lane; i < n; i += 32) nu_all += (in_role(i) && sv.nohit_pos[sl[i]] < 0) ? 1u : 0u;
            for (int o = 16; o; o >>= 1) nu_all += __shfl_xor_sync(kFull, nu_all, o);
            uint32_t carry = 0;
            for (uint32_t i0 = 0; i0 < n; i0 += 32) {
                const uint32_t i = i0 + lane;
                const bool cd = i < n && in_role(i);
                const int32_t pos = cd ? sv.nohit_pos[sl[i]] : 0;
                const uint32_t never = __ballot_sync(kFull, cd && pos < 0);
                if (cd) q.num[i] = pos < 0 ? (int32_t)(carry + __popc(never & ((1u << lane) - 1u))) : (int32_t)nu_all + pos;
                carry += __popc(never);
            }
            __syncwarp();
        }
    }
    const double denom = (double)((int32_t)n_role - 1);

    // prefix-cache-affinity-filter (filter/prefixcacheaffinity/plugin.go:105-151) over the candidates
    if (c.affinity_threshold > 0.0 && n_role > 1 && !(p.tie_seed && gen::explore_u(p.tie_seed, key) < c.exploration_probability)) {
        const bool have_ttft = c.ttft_column >= 0 && c.ttft_column < pool.n_ext_cols;
        const double *ttft = have_ttft ? pool.ext + (size_t)c.ttft_column * (size_t)pool.E : nullptr;
        uint32_t ns = 0, nn = 0;
        double bs = DBL_MAX, bn = DBL_MAX;
        for (uint32_t i = lane; i < n; i += 32) {
            if (!in_role(i)) continue;
            const double t = ttft ? ttft[sl[i]] : DBL_MAX;
            if (gen::is_sticky(q.hit[i], total, nm.thr)) { ns++; if (t < bs) bs = t; }
            else { nn++; if (t < bn) bn = t; }
        }
        for (int o = 16; o; o >>= 1) {
            ns += __shfl_xor_sync(kFull, ns, o);
            nn += __shfl_xor_sync(kFull, nn, o);
            const double os = __shfl_xor_sync(kFull, bs, o), on = __shfl_xor_sync(kFull, bn, o);
            if (os < bs) bs = os;
            if (on < bn) bn = on;
        }
        if (ns > 0 && !(c.max_ttft_penalty_ms > 0.0 && nn > 0 && __dsub_rn(bs, bn) > c.max_ttft_penalty_ms)) {
            nm.sticky = true;
            norm_over(c, pool, sl, n, lane, [&](uint32_t i) { return in_role(i) && gen::is_sticky(q.hit[i], total, nm.thr); }, nm.q);
        }
    }
    auto cand = [&](uint32_t i) { return in_role(i) && (!nm.sticky || gen::is_sticky(q.hit[i], total, nm.thr)); };
    const bool use_lora = p.lora.enabled && p.lora.ptr;
    // runScorerPlugins over the candidates: ordered, clamped, unfused (scheduler_profile.go:151-174)
    auto score = [&](uint32_t i) {
        const uint32_t e = sl[i];
        double acc = 0.0;
#pragma unroll 1
        for (int s = 0; s < c.n_scorers; s++) {
            const epp_scorer_cfg &sc = c.scorers[s];
            double raw;
            if (sc.kind == EPP_SCORER_PREFIX) raw = prefix_score(q.hit[i], total);
            else if (sc.kind == EPP_SCORER_LORA_AFFINITY) raw = lora_score(p.lora, e, use_lora ? lora_lookup(p.lora, q.adapter, e) : 0);
            else if (sc.kind == EPP_SCORER_NO_HIT_LRU) {
                if (!is_cold) raw = 0.5;                                                        // :159-165
                else if (n_role <= 1) raw = 1.0;                                                // :239-242
                else {
                    raw = __dsub_rn(1.0, __ddiv_rn((double)q.num[i], denom));
                    if (raw < 0) raw = 0;
                }
            } else raw = pool_score(sc, s, pool, nm.q, (int32_t)e);
            acc = __dadd_rn(acc, __dmul_rn(clamp01(raw), sc.weight));
        }
        return acc;
    };

    if (c.picker != EPP_PICKER_MAX_SCORE) {
        // random pickers: every candidate is an explicit item (no gaps); emitted entries stay in the sequence with mass 0
        uint32_t nc = 0;
        for (uint32_t i0 = 0; i0 < n; i0 += 32) nc += __popc(__ballot_sync(kFull, i0 + lane < n && cand(i0 + lane)));
        uint32_t g0 = rnd::kNone, g1 = rnd::kNone;            // emitted list positions: lane l holds #l and #l + 32
        const double sigma = rnd::mass_scale(c);
        for (int32_t j = 0; j < k && (uint32_t)j < nc; j++) {
            auto out_of = [&](uint32_t i) {
                bool o = false;
                for (int32_t t = 0; t < j; t++) o |= i == __shfl_sync(kFull, t < 32 ? g0 : g1, t & 31);
                return o;
            };
            const uint32_t pop = nc - (uint32_t)j;
            const double u = rnd::pick_u(p.tie_seed + (uint64_t)j * gen::kGolden, key);
            auto nth = [&](uint32_t r) -> uint32_t {
                for (uint32_t i0 = 0; i0 < n; i0 += 32) {
                    const uint32_t i = i0 + lane;
                    const bool o = out_of(i);
                    uint32_t bal = __ballot_sync(kFull, i < n && !o && cand(i));
                    const uint32_t cnt = __popc(bal);
                    if (r < cnt) {
                        for (uint32_t t = 0; t < r; t++) bal &= bal - 1;
                        return i0 + (uint32_t)__ffs(bal) - 1u;
                    }
                    r -= cnt;
                }
                return rnd::kNone;
            };
            uint32_t pi;
            if (c.picker == EPP_PICKER_RANDOM) {
                pi = nth(rnd::pick_rank(u, pop));
            } else {
                auto feed = [&](rnd::Walker &w) {
                    for (uint32_t i0 = 0; i0 < n && w.pick == rnd::kNone; i0 += 32) {
                        const uint32_t i = i0 + lane;
                        const bool o = out_of(i);
                        const bool x = i < n && cand(i);
                        double m = 0.0;
                        bool inf = false;
                        if (x && !o) {
                            const double s = score(i);
                            m = rnd::mass_of(s, sigma);
                            inf = rnd::is_pinf(s);
                        }
                        uint32_t xm = __ballot_sync(kFull, x);
                        while (xm) {
                            const int l = __ffs(xm) - 1;
                            xm &= xm - 1;
                            const double ml = __shfl_sync(kFull, m, l);
                            const bool il = __shfl_sync(kFull, (int)inf, l) != 0;
                            w.item(0, ml, il, i0 + (uint32_t)l);
                        }
                    }
                    w.finish(0);
                };
                pi = rnd::weighted_pick(pf, false, u, pop, feed, nth);
            }
            Best b;
            b.pick = sl[pi];
            b.val = score(pi);
            b.ties = pop;
            if (j == 0) first = b;
            if (lane == (j & 31)) { if (j < 32) g0 = pi; else g1 = pi; }
            if (lane == 0) {
                if (picks_row) picks_row[j] = b.pick;
                if (scores_row) scores_row[j] = b.val;
            }
        }
        return first;
    }

    // max-score picker: group by group in descending score order, each group in the tie rule's order
    double v = 0.0;
    bool have_v = false;
    uint32_t n_rem = 0, n_taken = 0;
    uint32_t g0 = EPP_NO_ENDPOINT, g1 = EPP_NO_ENDPOINT;       // emitted list positions of the current group
    for (int32_t j = 0; j < k; j++) {
        if (n_rem == 0) {
            Best b;
            best_init(b);
            for (uint32_t i = lane; i < n; i += 32) {
                if (!cand(i)) continue;
                const double sc = score(i);
                if (!have_v || sc < v) best_add(b, sc, i);      // pick = list position (ascending slot order)
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
        uint32_t rank = p.tie_seed ? tie_rank(p.tie_seed + (uint64_t)j * gen::kGolden, key, n_rem) : 0u;
        uint32_t pick = EPP_NO_ENDPOINT;
        for (uint32_t i0 = 0; i0 < n && pick == EPP_NO_ENDPOINT; i0 += 32) {
            const uint32_t i = i0 + lane;
            bool hit = i < n && cand(i) && score(i) == v;
            if (n_taken && __any_sync(kFull, hit))
                for (uint32_t t = 0; t < n_taken; t++)
                    if (__shfl_sync(kFull, t < 32 ? g0 : g1, (int)(t & 31)) == i) hit = false;
            uint32_t bal = __ballot_sync(kFull, hit);
            const uint32_t cnt = __popc(bal);
            if (rank < cnt) {
                for (uint32_t t = 0; t < rank; t++) bal &= bal - 1;
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
            if (picks_row) picks_row[j] = sl[pick];
            if (scores_row) scores_row[j] = v;
        }
    }
    if (first.ties) first.pick = sl[first.pick];
    return first;
}

// One restricted request per warp.  kLat: the engine has latency profiles (lv): those evaluate through lat::eval over
// the listed slots with the request's predictions (LatView rows are the call's absolute rows, as SubsetRow::row is).
template <bool kLat>
__device__ __forceinline__ void subset_pick(const PickParams &p, const SubsetView &sv, const LatView *lv = nullptr) {
    const int lane = threadIdx.x & 31;
    const int32_t j = (int32_t)blockIdx.x * kSubsetWarps + (int32_t)(threadIdx.x >> 5);
    if (j >= sv.n_rows) return;
    const SubsetRow row = sv.rows[j];
    const int64_t r = (int64_t)row.row - sv.r0;
    SubsetReq q;
    q.sl = sv.slots + row.off;
    q.hit = sv.hits + row.off;
    q.num = sv.scratch + row.off;
    q.n = row.n;
    q.total = p.nblocks[r];
    q.adapter = p.model_ids ? p.model_ids[r] : 0u;
    int32_t *hit = sv.hits + row.off;
    for (uint32_t i = lane; i < q.n; i += 32) hit[i] = 0;
    __syncwarp();

    // ---- match: probe in block order up to the global stop, count the listed holders (plugin.go:214-230)
    const int32_t total = q.total;
    const int32_t stored = p.bound ? p.bound[r] : total;          // block `stored` < total: a proven miss
    const uint64_t *hrow = p.hashes + r * (int64_t)p.max_blocks;
    for (int32_t c0 = 0; c0 < total; c0 += 32) {
        const int32_t i = c0 + lane;
        Hit h;
        h.cnt = 0;
        bool found = false;
        if (i < stored && i < total) found = probe(p.index, hrow[i], h);
        if (!found) h.cnt = 0;
        const uint32_t miss = __ballot_sync(kFull, i < total && !found);
        const int32_t limit = miss ? c0 + (__ffs(miss) - 1) : min(total, c0 + 32);
        if (q.n)
            for (int32_t b = 0; b < limit - c0; b++) {       // one block at a time: its holders are distinct
                Hit hb;
                hb.cnt = __shfl_sync(kFull, h.cnt, b);
#pragma unroll
                for (int w = 0; w < kInlineIds; w++) hb.w[w] = __shfl_sync(kFull, h.w[w], b);
                for (uint32_t t = lane; t < hb.cnt; t += 32) {
                    const uint32_t at = list_find(q.sl, q.n, posting(p.index, hb, t));
                    if (at < q.n) hit[at]++;
                }
                __syncwarp();
            }
        if (miss) break;
    }
    __syncwarp();

    // ---- the stages of the handler over the listed slots
    const int32_t k = p.gen.topk > 1 ? p.gen.topk : 1;
    if (k > 1) {
        for (int pq = 1; pq < kMaxProfiles; pq++)
            if (p.gen.topk_picks[pq]) for (int t = lane; t < k; t += 32) p.gen.topk_picks[pq][r * k + t] = EPP_NO_ENDPOINT;
        __syncwarp();
    }
    bool cold = false;
    auto eval = [&](int pi, uint64_t key) {
        if constexpr (kLat) {
            if ((lv->mask >> pi) & 1) {
                lat::Req lq;
                lq.n = lv->cnt ? lv->cnt[row.row] : 0u;
                lq.ent = lq.n ? lv->ent + lv->off[row.row] : nullptr;
                const lat::CtxLen cl = lat::ctx_len(*lv, pi, row.row, p.in_len[r]);
                return lat::eval<true>(p.prof[pi], lv->cfg[pi], cl, p.gen, lq, p.E, total, lane, p.lora, q.adapter, p.tie_seed, key,
                                       lat::ListDom{q.sl, q.hit, q.n}, k,
                                       (k > 1 && p.gen.topk_picks[pi]) ? p.gen.topk_picks[pi] + r * k : nullptr,
                                       (k > 1 && pi == 0 && p.gen.topk_scores) ? p.gen.topk_scores + r * k : nullptr);
            }
        }
        return eval_subset(p.prof[pi], p, sv, q, lane, key, (p.nohit.mask >> pi) & 1, &cold, k,
                           (k > 1 && p.gen.topk_picks[pi]) ? p.gen.topk_picks[pi] + r * k : nullptr,
                           (k > 1 && pi == 0 && p.gen.topk_scores) ? p.gen.topk_scores + r * k : nullptr);
    };
    auto match_of = [&](uint32_t e) {
        const uint32_t at = list_find(q.sl, q.n, e);
        return at < q.n ? q.hit[at] : 0;
    };
    epp_decision d;
    epp_decision_detail dd;
    decide_stages<3>(p, r, total, p.n_profiles >= 2 ? p.in_len[r] : 0, eval, match_of, d, dd);
    if (lane == 0) {
        if (p.nohit.cold_out) p.nohit.cold_out[r] = cold ? 1 : 0;
        p.out[r] = d;
        if (p.detail) p.detail[r] = dd;
    }
}

__global__ void __launch_bounds__(kSubsetWarps * 32) k_subset_pick(PickParams p, SubsetView sv) { subset_pick<false>(p, sv); }
__global__ void __launch_bounds__(kSubsetWarps * 32) k_subset_pick_lat(PickParams p, SubsetView sv, LatView lv) {
    subset_pick<true>(p, sv, &lv);
}

}  // namespace

cudaError_t launch_subset_pick(const PickParams &p, const SubsetView &sv, const LatView *lv, cudaStream_t s, int *launches) {
    if (sv.n_rows <= 0) return cudaSuccess;
    const unsigned grid = (unsigned)((sv.n_rows + kSubsetWarps - 1) / kSubsetWarps);
    if (lv) k_subset_pick_lat<<<grid, kSubsetWarps * 32, 0, s>>>(p, sv, *lv);
    else k_subset_pick<<<grid, kSubsetWarps * 32, 0, s>>>(p, sv);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace epp
