// match_sparse.cuh -- a2-a14 for ONE request by ONE warp over hashes resident in HBM / L2: index lookup with the
// global-stop rule (approximateprefix/plugin.go:214-230), per-endpoint match counts, ordered weighted sum
// (scheduler_profile.go:151-174), arg-max pick (maxscore/picker.go:87-115) and the decode -> decider -> prefill second
// stage (disagg_profile_handler.go:264-308).  No shared memory (except the optional work tally), one atomic per request
// (the throughput kernel's request counter).
//
// Shared by the throughput kernel (match_sparse.cu: one warp per request over the hash rows of a whole batch, incl. the
// endpoint-sharded variant) and by the latency kernel (cycle_small.cu: one warp of the request's CTA follows the hash
// chain as it is produced).
//
//   * 32 blocks are probed per step, two 128-bit loads per 32-byte slot.  Probe chains are followed only as far as the
//     stop rule needs them: once a lane has proven its block absent, the lanes behind it (which cannot change the walk)
//     stop probing -- a cold prompt costs the probe chain of block 0, not the longest chain of 32 unrelated blocks;
//   * matched endpoints live in a LANE-DISTRIBUTED register map: lane j holds (endpoint E_j, count C_j), j <
//     n_distinct <= 32; membership tests are ballots;
//   * counting is run-length based: posting lists are sorted, duplicate-free and (when spilled) interned, and unused
//     id words of a slot are zero by construction of the table (index_kernels.cu: finalize_slot, index_store.cu:
//     k_patch_apply), so "same endpoint set" is equality of the six words (cnt, ids[0..4]); the blocks of one cached
//     prefix form a few runs of identical sets and a run adds its length to each of its endpoints.
//
// Exactness: a request whose matched-endpoint set exceeds the map's capacity is appended to
// PickParams::overflow_list and handled by the dense-counter kernel (pick_kernels.cu), never approximated.
#pragma once
#include "index.cuh"
#include "pick_random.cuh"
#include "score.cuh"

namespace epp {
namespace sparse {

constexpr uint32_t kNoKey = 0xFFFFFFFFu;
constexpr uint32_t kFull = 0xffffffffu;

struct LaneMap {                   // one entry per lane
    uint32_t e;                    // endpoint held by this lane (kNoKey = none)
    uint32_t c;                    // its match count
    uint32_t n;                    // distinct endpoints so far (warp-uniform); 33 = overflowed (one register, no flag)
    __device__ __forceinline__ bool overflow() const { return n > 32; }
};

// count[e] += c for a warp-uniform (e, c).
__device__ __forceinline__ void map_add(LaneMap &m, uint32_t e, uint32_t c, int lane) {
    const uint32_t holder = __ballot_sync(kFull, m.e == e);
    if (holder) {
        if (lane == __ffs(holder) - 1) m.c += c;
    } else if (m.n < 32) {
        if (lane == (int)m.n) { m.e = e; m.c = c; }
        m.n++;
    } else {
        m.n = 33;
    }
}

__device__ __forceinline__ uint32_t map_get(const LaneMap &m, uint32_t e) {   // warp-uniform e
    const uint32_t holder = __ballot_sync(kFull, m.e == e);
    const uint32_t c = __shfl_sync(kFull, m.c, holder ? __ffs(holder) - 1 : 0);
    return holder ? c : 0;
}

// Lane-parallel membership: is MY candidate e (different per lane) one of the matched endpoints?
__device__ __forceinline__ bool map_contains_any(const LaneMap &m, uint32_t e) {
    bool hit = false;
    for (uint32_t j = 0; j < m.n; j++) hit |= (e == __shfl_sync(kFull, m.e, (int)j));
    return hit;
}

// The member of rank k (ascending slot order) of the arg-max set S = A u U (see eval_profile_lanes): one lower bound
// per A lane in parallel and, failing that, one warp-uniform binary search over the equal-base group G.  Rare path
// (ties only): kept out of line so that it costs the common path no registers.
static __device__ __noinline__ uint32_t select_tied(const ProfileDev &pf, const LaneMap &m, int lane, bool in_a, bool in_x_all,
                                             bool have_u, uint32_t gpos, uint32_t ue, uint32_t k) {
    const bool in_x = in_x_all && have_u;
    const uint32_t mask_a = __ballot_sync(kFull, in_a), mask_x = __ballot_sync(kFull, in_x);
    // G = order[gs .. gs + gsz): the X members with a smaller slot than ue precede it inside the group
    const uint32_t gs = have_u ? gpos - __popc(__ballot_sync(kFull, in_x && m.e < ue)) : 0u;
    const uint32_t gsz = have_u ? pf.grp_size[gpos] : 0u;
    uint32_t ca = 0, cx = 0;
    for (uint32_t j = 0; j < m.n; j++) {
        const uint32_t ej = __shfl_sync(kFull, m.e, (int)j);
        ca += ((mask_a >> j) & 1u) && ej < m.e;
        cx += ((mask_x >> j) & 1u) && ej < m.e;
    }
    uint32_t pos = 0;
    if (in_a && have_u) {                          // lower bound of my slot in G
        uint32_t lo = 0, hi = gsz;
        while (lo < hi) {
            const uint32_t mid = (lo + hi) >> 1;
            if (pf.order[gs + mid] < m.e) lo = mid + 1; else hi = mid;
        }
        pos = lo;
    }
    const uint32_t found = __ballot_sync(kFull, in_a && ca + pos - (have_u ? cx : 0u) == k);
    if (found) return __shfl_sync(kFull, m.e, __ffs(found) - 1);
    // the member is an unmatched entry of G: the largest position of rank <= k
    uint32_t lo = 0, hi = gsz - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        const uint32_t x = pf.order[gs + mid];
        const uint32_t f = mid - __popc(__ballot_sync(kFull, in_x && m.e < x)) + __popc(__ballot_sync(kFull, in_a && m.e < x));
        if (f <= k) lo = mid; else hi = mid - 1;
    }
    return pf.order[gs + lo];
}

// One profile for the current request (SchedulerProfile.Run): matched candidates from the lane map, everyone else
// from the precomputed (base desc, slot asc) order -- an unmatched endpoint's ordered weighted sum is bit-identical to
// its precomputed base, so only the first unmatched entry of the order (and the size of its equal-base group) matters.
// tie_seed != 0: the pick is the member of rank tie_rank(...) of the arg-max set in ascending slot order (score.cuh).
// The set is S = A u U: A = matched candidates whose score is the maximum, U = the unmatched members of the equal-base
// group G of the order (only when that base IS the maximum); X = matched candidates sitting inside G.  G is sorted by
// slot, |A|, |X| <= 32: the rank of a slot x in S is #{a in A: a < x} + lower_bound_G(x) - #{x' in X: x' < x}, so the
// member is found with one lower bound per A lane (in parallel) and, failing that, one warp-uniform binary search over G.
// kForce: the member of rank force_rank (>= 1) instead (the seeded sharded select, include/epp_engine.h "Seeded ties").
template <bool kTie, bool kForce = false>
__device__ __forceinline__ Best eval_profile_lanes(const ProfileDev &pf, int32_t E, const LaneMap &m, int32_t total,
                                                   int lane, const LoraDev &lora, int lora_st, uint64_t tie_seed,
                                                   uint64_t tie_key, uint32_t force_rank = 0) {
    Best b;
    best_init(b);
    const int32_t ncand = *pf.n_cand;
    if (ncand == 0) return b;
    if (m.n == 0) {                                   // nobody holds a block of this prompt: the head of the order wins
        const uint32_t ue = pf.order[0];
        best_add(b, pf.base[ue], ue, pf.grp_size[0]);
        if (kForce) b.pick = pf.order[force_rank];
        else if (kTie && tie_seed && b.ties > 1) b.pick = pf.order[tie_rank(tie_seed, tie_key, b.ties)];
        return b;
    }
    const bool mine = (uint32_t)lane < m.n && pf.cand[m.e];
    double myv = 0.0;
    if (mine) {
        myv = weighted_sum(pf, E, m.e, (int32_t)m.c, total, lora, lora_st);
        best_add(b, myv, m.e);
    }
    b = best_warp_reduce(b);
    bool have_u = false;
    bool in_x = false;
    uint32_t gpos = 0, ue = kNoKey;
    double ubase = 0.0;
    for (int32_t k0 = 0; k0 < ncand; k0 += 32) {
        const int32_t k = k0 + lane;
        const uint32_t e = k < ncand ? pf.order[k] : kNoKey;
        const bool matched = map_contains_any(m, e);   // shuffles inside: EVERY lane must call it (no short-circuit)
        const bool un = k < ncand && !matched;
        const uint32_t bal = __ballot_sync(kFull, un);
        if (bal) {
            const int first = __ffs(bal) - 1;
            ue = __shfl_sync(kFull, e, first);
            ubase = pf.base[ue];
            gpos = (uint32_t)(k0 + first);
            const uint32_t gsz = pf.grp_size[gpos];
            in_x = mine && pf.base[m.e] == ubase;
            const uint32_t same = __popc(__ballot_sync(kFull, in_x));
            best_add(b, ubase, ue, gsz - same);
            have_u = true;
            break;
        }
    }
    if (kForce || (kTie && tie_seed && b.ties > 1))
        b.pick = select_tied(pf, m, lane, mine && myv == b.val, in_x, have_u && ubase == b.val, gpos, ue,
                             kForce ? force_rank : tie_rank(tie_seed, tie_key, b.ties));
    return b;
}

// One profile with a random picker (include/epp_engine.h "Random pickers"): the explicit candidates are the map's (matched
// endpoints and lora-affinity entries), at most 32.  Each lane finds its entry's rank in slot order and its position among
// the candidates (one binary search per lane, in parallel); the fold then walks the items and the gaps between them in
// warp-uniform steps, and a pick inside a gap costs one binary search over wcum.  Kept out of line: the builds that carry
// it are launched only for engines with a random picker.
static __device__ __noinline__ Best eval_random_lanes(const ProfileDev &pf, int32_t E, const LaneMap &m, int32_t total,
                                                      int lane, const LoraDev &lora, int lora_st, uint64_t seed,
                                                      uint64_t key) {
    Best b;
    best_init(b);
    const uint32_t n = (uint32_t)*pf.n_cand;
    if (n == 0) return b;
    const double u = rnd::pick_u(seed, key);
    const bool x = (uint32_t)lane < m.n && pf.cand[m.e];
    const double s = x ? weighted_sum(pf, E, m.e, (int32_t)m.c, total, lora, lora_st) : 0.0;
    uint32_t pick;
    if (pf.cfg.picker == EPP_PICKER_RANDOM) {
        pick = pf.cands[rnd::pick_rank(u, n)];
    } else {
        const double mass = x ? rnd::mass_of(s, rnd::mass_scale(pf.cfg)) : 0.0;
        const bool inf = x && rnd::is_pinf(s);
        const uint32_t xmask = __ballot_sync(kFull, x);
        uint32_t rk = 0;                               // rank of my entry among the explicit ones, ascending slot
        for (uint32_t j = 0; j < m.n; j++) {
            const uint32_t ej = __shfl_sync(kFull, m.e, (int)j);
            rk += ((xmask >> j) & 1u) && ej < m.e;
        }
        uint32_t pos = 0;                              // its position among the candidates
        if (x) {
            uint32_t lo = 0, hi = n;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (pf.cands[mid] < m.e) lo = mid + 1; else hi = mid;
            }
            pos = lo;
        }
        const uint32_t nx = __popc(xmask);
        auto feed = [&](rnd::Walker &w) {
            for (uint32_t q = 0; q < nx && w.pick == rnd::kNone; q++) {
                const int l = __ffs(__ballot_sync(kFull, x && rk == q)) - 1;
                const uint32_t pl = __shfl_sync(kFull, pos, l);
                const double ml = __shfl_sync(kFull, mass, l);
                const bool il = __shfl_sync(kFull, (int)inf, l) != 0;
                w.item(pl, ml, il, __shfl_sync(kFull, m.e, l));
            }
            w.finish(n);
        };
        pick = rnd::weighted_pick(pf, true, u, n, feed, [&](uint32_t r) { return pf.cands[r]; });
    }
    // the pick's score: its own weighted sum when it is an explicit entry, else its base
    const uint32_t holder = __ballot_sync(kFull, x && m.e == pick);
    const double hs = __shfl_sync(kFull, s, holder ? __ffs(holder) - 1 : 0);
    b.val = holder ? hs : pf.base[pick];
    b.pick = pick;
    b.ties = n;
    return b;
}

// Adds one chunk's postings to the lane map.  (cnt, w0..w4) = this lane's slot words, all zero when the block is
// beyond the stop or absent.  Runs of lanes with identical words are added at once.
__device__ __forceinline__ void count_chunk(LaneMap &m, const IndexView &ix, uint32_t cnt, uint32_t w0, uint32_t w1,
                                            uint32_t w2, uint32_t w3, uint32_t w4, uint32_t shard_lo, uint32_t shard_hi,
                                            int lane) {
    // run boundaries: a lane starts a run when its words differ from the previous lane's
    uint32_t d = cnt ^ __shfl_up_sync(kFull, cnt, 1);
    d |= w0 ^ __shfl_up_sync(kFull, w0, 1);
    d |= w1 ^ __shfl_up_sync(kFull, w1, 1);
    d |= w2 ^ __shfl_up_sync(kFull, w2, 1);
    d |= w3 ^ __shfl_up_sync(kFull, w3, 1);
    d |= w4 ^ __shfl_up_sync(kFull, w4, 1);
    const uint32_t bounds = __ballot_sync(kFull, d != 0 || lane == 0);
    uint32_t heads = bounds & __ballot_sync(kFull, cnt != 0);                    // heads of the non-empty runs
    while (heads) {
        const int s = __ffs(heads) - 1;
        heads &= heads - 1;
        const uint32_t after = bounds & ~((2u << s) - 1u);              // next run boundary behind s
        const int end = after ? __ffs(after) - 1 : 32;
        const uint32_t len = (uint32_t)(end - s);
        const uint32_t rc = __shfl_sync(kFull, cnt, s);
        const uint32_t r0 = __shfl_sync(kFull, w0, s);
        if (rc <= (uint32_t)kInlineIds) {
            if (r0 >= shard_lo && r0 < shard_hi) map_add(m, r0, len, lane);
            if (rc > 1) { const uint32_t e = __shfl_sync(kFull, w1, s); if (e >= shard_lo && e < shard_hi) map_add(m, e, len, lane); }
            if (rc > 2) { const uint32_t e = __shfl_sync(kFull, w2, s); if (e >= shard_lo && e < shard_hi) map_add(m, e, len, lane); }
            if (rc > 3) { const uint32_t e = __shfl_sync(kFull, w3, s); if (e >= shard_lo && e < shard_hi) map_add(m, e, len, lane); }
            if (rc > 4) { const uint32_t e = __shfl_sync(kFull, w4, s); if (e >= shard_lo && e < shard_hi) map_add(m, e, len, lane); }
        } else {
            // spilled (interned) list: r0 is the offset into the postings array
            for (uint32_t k0 = 0; k0 < rc && !m.overflow(); k0 += 32) {
                const uint32_t mine = (k0 + lane < rc) ? ix.postings[r0 + k0 + lane] : kNoKey;
                const uint32_t nk = min(32u, rc - k0);
                for (uint32_t k = 0; k < nk && !m.overflow(); k++) {
                    const uint32_t e = __shfl_sync(kFull, mine, (int)k);
                    if (e >= shard_lo && e < shard_hi) map_add(m, e, len, lane);
                }
            }
        }
    }
}

template <bool kCg, typename T>
__device__ __forceinline__ T ld_row(const T *p) {
    if (kCg) return __ldcg(p);        // written earlier by THIS kernel (fused cycle): read at L2, never a stale L1 line
    return *p;
}

// Work a warp did for its requests (SURVEY 8(d) P and M), tallied in the calling kernel's shared memory so that the
// probe loop carries no totals in registers: blocks probed (added by lane 0) and postings counted (one total per lane).
struct Work {
    unsigned long long probes;
    unsigned long long postings[32];
};

// The whole decision for request r (all 32 lanes of one warp call it together).  kCg: the per-request inputs
// (hashes, nblocks, in_len) were produced earlier in the same kernel launch.
// kSharded: endpoint-sharded mode (the stop rule comes from p.global_masks).
// kTie: the reproducible random tie rule is compiled in (epp_config.tie_seed != 0); the deterministic lowest-slot
// build carries none of its code or registers.
// kStages: stages of the handler compiled in (score.cuh: decide_stages).
// Follow: the request's hashes are still being produced by another warp of the CTA (cycle_small.cu): wait(n) returns
// once hashes [0, n) can be read with hash(i) (shared memory).  NoFollow: they are all in the row p.hashes.
struct NoFollow {
    static constexpr bool kOn = false;
    __device__ __forceinline__ void wait(int32_t) const {}
    __device__ __forceinline__ uint64_t hash(int32_t) const { return 0; }
};
// Returns false when the request was handed to the dense-counter kernel (p.overflow_list) instead of being decided.
// req_next != nullptr: once the probes are done, lane 0 takes a ticket off *req_next into `ticket` (k_match_pick_sparse:
// the warp's next request, fetched while this one is scored).
// kNoHit: a profile has a no-hit-lru scorer (PickParams::nohit): the lane map decides, with one ballot, whether the request
// is cold for the profile, which selects the profile's warm or cold set (same candidates, different base / order / groups).
// kRand: some profile has a random picker (epp_profile_cfg.picker): those profiles are decided by eval_random_lanes.
// kSel: the seeded sharded select (k_match_pick_sparse_select): request r is work item sv->work[wi], whose one profile
// is evaluated with the rank of its member forced; the member and its match count go to sv->sel, an overflow appends wi
// to sv->dense_list.
template <bool kCg, bool kSharded, bool kTie, int kStages, typename Follow = NoFollow, bool kNoHit = false, bool kRand = false,
          bool kSel = false>
__device__ __forceinline__ bool match_request(const PickParams &p, const uint32_t r, const int lane, const bool counting,
                                              Work *wk, int32_t *req_next, int32_t &ticket, const Follow fw = Follow(),
                                              const ShardSelView *sv = nullptr, int32_t wi = 0) {
    const uint32_t shard_lo = p.index.ep_begin, shard_hi = min(p.index.ep_end, (uint32_t)p.E);
    const IndexSlot *slots = p.index.slots;
    const uint32_t mask32 = (uint32_t)p.index.mask;
    const int32_t total = ld_row<kCg>(p.nblocks + r);
    // hashes [0, stored) are in the row; block `stored` < total is a proven miss (PickParams::bound)
    const int32_t stored = (!Follow::kOn && p.bound) ? ld_row<kCg>(p.bound + r) : total;
    const uint64_t *row = p.hashes + r * (int64_t)p.max_blocks;
    LaneMap m;
    m.e = kNoKey; m.c = 0; m.n = 0;
    // ---- a2/a3: probe in block order, 32 blocks per step; global stop at the first block nobody holds
    int32_t limit = total;                                        // < total once the walk has stopped at block `limit`
    uint64_t hnext = (!Follow::kOn && lane < stored) ? ld_row<kCg>(row + lane) : 0;
    for (int32_t cq = 0; cq < total && limit == total; cq += 32) {
        const int32_t i = cq + lane;
        uint64_t hcur;
        if (Follow::kOn) {
            fw.wait(min(total, cq + 32));
            hcur = i < total ? fw.hash(i) : 0;
        } else {
            hcur = hnext;
            if (i + 32 < stored) hnext = ld_row<kCg>(row + i + 32);   // next chunk's hashes in flight during this one
        }
        const bool valid = i < total;
        // endpoint-sharded mode: a block is missing only if NO rank holds it, and that is known up front
        uint32_t gmiss = 0;
        if (kSharded) {
            const uint32_t word = p.global_masks[r * (int64_t)p.mask_words + (cq >> 5)];
            const uint32_t vmask = (total - cq) >= 32 ? kFull : ((1u << (total - cq)) - 1u);
            gmiss = ~word & vmask;
        }
        const uint32_t relevant = (kSharded && gmiss) ? ((1u << (__ffs(gmiss) - 1)) - 1u) : kFull;
        uint32_t cnt = 0, w0 = 0, w1 = 0, w2 = 0, w3 = 0, w4 = 0;
        bool pending = i < stored && ((relevant >> lane) & 1u);     // lanes in [stored, total): absent, never probed
        if (pending && (hcur == kEmptyKey || !slots)) {           // the sentinel hash lives in a side record
            Hit hs;
            if (probe(p.index, hcur, hs)) { cnt = hs.cnt; w0 = hs.w[0]; w1 = hs.w[1]; w2 = hs.w[2]; w3 = hs.w[3]; w4 = hs.w[4]; }
            if (cnt > (uint32_t)kInlineIds) { w1 = w2 = w3 = w4 = 0; }
            pending = false;
        }
        uint32_t idx = (uint32_t)hcur & mask32;
        for (;;) {
            const uint32_t pend0 = __ballot_sync(kFull, pending);
            if (!pend0) break;
            if (!kSharded) {
                const uint32_t missm0 = __ballot_sync(kFull, valid && !pending && cnt == 0);
                const uint32_t below0 = missm0 ? ((1u << (__ffs(missm0) - 1)) - 1u) : kFull;
                if (!(pend0 & below0)) break;
                if (!((below0 >> lane) & 1u)) pending = false;
            }
            if (pending) {
                // straight into (cnt, w0..w4), which a pending lane holds as zeros: no second set of slot registers
                uint64_t key;
                Hit hs;
                load_slot(slots + idx, key, hs);
                cnt = hs.cnt; w0 = hs.w[0]; w1 = hs.w[1]; w2 = hs.w[2]; w3 = hs.w[3]; w4 = hs.w[4];
                if (key == hcur) {                                // cnt == 0: every holder was evicted (tombstone)
                    pending = false;
                } else {
                    cnt = 0; w0 = 0; w1 = 0; w2 = 0; w3 = 0; w4 = 0;
                    if (key == kEmptyKey) pending = false;        // a never-used slot ends the probe chain: absent
                    else idx = (idx + 1) & mask32;
                }
            }
        }
        // lanes that stopped early (pending) hold cnt == 0 and sit behind the stop
        const uint32_t miss = kSharded ? gmiss : __ballot_sync(kFull, valid && cnt == 0);
        limit = miss ? cq + (__ffs(miss) - 1) : total;
        if (i >= limit) { cnt = 0; w0 = 0; w1 = 0; w2 = 0; w3 = 0; w4 = 0; }
        if (counting) wk->postings[lane] += cnt;
        if (limit > cq) count_chunk(m, p.index, cnt, w0, w1, w2, w3, w4, shard_lo, shard_hi, lane);
    }
    if (counting && lane == 0) wk->probes += (unsigned long long)min(limit + 1, total);   // up to and including the stop
    if (req_next && lane == 0) ticket = atomicAdd(req_next, 1);
    // ---- lora-affinity: the endpoints where the request's adapter is active or waiting get a request-dependent
    //      score, so they join the map (count 0) and are evaluated one by one like the prefix holders
    int lora_st = 0;
    if (p.lora.enabled && p.lora.ptr && !m.overflow()) {
        const uint32_t a = p.model_ids ? p.model_ids[r] : 0u;
        if (a < (uint32_t)p.lora.n_models) {
            const uint32_t lo = p.lora.ptr[a], hi = p.lora.ptr[a + 1];
            for (uint32_t k0 = lo; k0 < hi && !m.overflow(); k0 += 32) {
                const uint32_t mine_e = (k0 + lane < hi) ? p.lora.ep[k0 + lane] : kNoKey;
                const uint32_t nk = min(32u, hi - k0);
                for (uint32_t k = 0; k < nk && !m.overflow(); k++) {
                    const uint32_t e = __shfl_sync(kFull, mine_e, (int)k);
                    if (e >= shard_lo && e < shard_hi) map_add(m, e, 0, lane);
                }
            }
            if ((uint32_t)lane < m.n) lora_st = lora_lookup(p.lora, a, m.e);
        }
    }
    if (m.overflow()) {
        // hand the request to the dense-counter kernel
        if constexpr (kSel) {
            if (lane == 0) sv->dense_list[atomicAdd(sv->dense_n, 1)] = wi;
        } else {
            if (lane == 0 && p.overflow_list) p.overflow_list[atomicAdd(p.overflow_n, 1)] = (int32_t)r;
        }
        return false;
    }
    if constexpr (kSel) {
        const uint2 it = sv->work[wi];
        const Best b = eval_profile_lanes<true, true>(p.prof[it.x % (uint32_t)sv->stages], p.E, m, total, lane, p.lora,
                                                      lora_st, 0, 0, it.y);
        const uint32_t mb = m.n ? map_get(m, b.pick) : 0u;
        if (lane == 0) {
            epp_shard_sel s;
            s.pick = b.pick;
            s.match_blocks = (int32_t)mb;
            sv->sel[it.x] = s;
        }
        return true;
    }
    // ---- a5-a14: the profiles of the handler
    if constexpr (kSharded && kStages > 1) {
        // endpoint-sharded disagg handler: one record per stage, each a scoring pass over the same lane map
        shard_stage_records(p, r, kStages, p.in_len[r],
                            [&](int pi, uint64_t key) {
                                return eval_profile_lanes<kTie>(p.prof[pi], p.E, m, total, lane, p.lora, lora_st, p.tie_seed, key);
                            },
                            [&](uint32_t e) { return m.n ? (int32_t)map_get(m, e) : 0; }, lane);
        return true;
    }
    epp_decision d;
    epp_decision_detail dd;
    bool cold = false;
    decide_stages<kStages>(p, r, total, (kStages >= 2 && p.n_profiles >= 2) ? ld_row<kCg>(p.in_len + r) : 0,
                  [&](int pi, uint64_t key) {
                      if (!kNoHit) {
                          if (kRand && p.prof[pi].cfg.picker)
                              return eval_random_lanes(p.prof[pi], p.E, m, total, lane, p.lora, lora_st, p.tie_seed, key);
                          return eval_profile_lanes<kTie>(p.prof[pi], p.E, m, total, lane, p.lora, lora_st, p.tie_seed, key);
                      }
                      // a hit = a matched candidate with count > 0 (lora-affinity entries join the map with count 0)
                      const ProfileDev &pf = nohit_select(p, pi, cold, [&](const ProfileDev &w) {
                          return !__ballot_sync(kFull, (uint32_t)lane < m.n && m.c > 0 && w.cand[m.e]);
                      });
                      if (kRand && pf.cfg.picker) return eval_random_lanes(pf, p.E, m, total, lane, p.lora, lora_st, p.tie_seed, key);
                      return eval_profile_lanes<kTie>(pf, p.E, m, total, lane, p.lora, lora_st, p.tie_seed, key);
                  },
                  [&](uint32_t e) { return m.n ? (int32_t)map_get(m, e) : 0; }, d, dd);
    if (kNoHit && lane == 0 && p.nohit.cold_out) p.nohit.cold_out[r] = cold ? 1 : 0;
    if (lane == 0) {
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
    return true;
}

}  // namespace sparse
}  // namespace epp
