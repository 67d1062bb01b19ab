// pick_random.cuh -- the random-picker (picker/random/picker.go:86-104) and the weighted-random-picker
// (picker/weightedrandom/picker.go:111-155) for one request by one warp, as defined in include/epp_engine.h ("Random
// pickers").
//
// The weighted draw folds the request's explicit candidates (the few whose score depends on the request) and the gaps
// between them; a gap's mass is the difference of two entries of the profile set's prefix array wcum (k_pool_cum), so a
// request costs O(explicit + log n) however many candidates the profile has.  Every lane runs the same fold on warp-uniform
// values: the result is one double sequence, bit-identical to the restatement in tools/picker_model.py.
#pragma once
#include "score.cuh"

namespace epp {
namespace rnd {

constexpr uint64_t kPickDomain = 0xE7037ED1A0B428DBULL;
constexpr uint32_t kNone = 0xFFFFFFFFu;

__device__ __forceinline__ double pick_u(uint64_t seed, uint64_t key) {
    return (double)(mix64((seed ^ kPickDomain) ^ mix64(key)) >> 11) * 0x1.0p-53;
}
// min(floor(u * n), n - 1)
__device__ __forceinline__ uint32_t pick_rank(double u, uint32_t n) {
    const uint32_t k = (uint32_t)__dmul_rn(u, (double)n);
    return k < n ? k : n - 1;
}
// 2^-128 when the profile's sum of |weight| exceeds 2^960, else 1: every sum of masses stays finite
__device__ __forceinline__ double mass_scale(const epp_profile_cfg &c) {
    double s = 0.0;
    for (int i = 0; i < c.n_scorers; i++) s = __dadd_rn(s, fabs(c.scorers[i].weight));
    return s > 0x1.0p960 ? 0x1.0p-128 : 1.0;
}
__device__ __forceinline__ bool is_pinf(double s) { return s == CUDART_INF; }
__device__ __forceinline__ double mass_of(double s, double sigma) {
    return (s > 0.0 && !is_pinf(s)) ? __dmul_rn(s, sigma) : 0.0;
}

// The fold over the item sequence: gap [a, pos), explicit candidate at position pos, ..., final gap [a, n).
// mode 0 sums W and counts the +inf candidates; mode 1 finds the first item whose running sum exceeds t; mode 2 finds the
// +inf candidate of rank k.  gaps == false: every candidate is explicit (the positions are ignored).
struct Walker {
    const ProfileDev *pf;
    bool gaps;
    int mode;
    double t;
    uint32_t k;
    double S;
    uint32_t ninf;
    uint32_t a;
    uint32_t pick;
    __device__ __forceinline__ Walker(const ProfileDev &p, bool g, int md, double tt, uint32_t kk)
        : pf(&p), gaps(g), mode(md), t(tt), k(kk), S(0.0), ninf(0), a(0), pick(kNone) {}
    __device__ __forceinline__ void gap(uint32_t b) {
        if (!gaps || pick != kNone || b <= a) return;
        if (mode == 2) {
            const uint32_t c = pf->icum[b] - pf->icum[a];
            if (k < c) {                                   // first i with icum[i+1] - icum[a] > k
                uint32_t lo = a, hi = b - 1;
                while (lo < hi) {
                    const uint32_t mid = (lo + hi) >> 1;
                    if (pf->icum[mid + 1] - pf->icum[a] > k) hi = mid; else lo = mid + 1;
                }
                pick = pf->cands[lo];
            } else {
                k -= c;
            }
            return;
        }
        const double wa = pf->wcum[a];
        const double ns = __dadd_rn(S, __dsub_rn(pf->wcum[b], wa));
        if (mode == 1 && ns > t) {                         // first i with S + (wcum[i+1] - wcum[a]) > t
            uint32_t lo = a, hi = b - 1;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (__dadd_rn(S, __dsub_rn(pf->wcum[mid + 1], wa)) > t) hi = mid; else lo = mid + 1;
            }
            pick = pf->cands[lo];
            return;
        }
        S = ns;
        if (mode == 0) ninf += pf->icum[b] - pf->icum[a];
    }
    __device__ __forceinline__ void item(uint32_t pos, double m, bool inf, uint32_t e) {
        gap(pos);
        if (pick != kNone) return;
        a = pos + 1;
        if (mode == 2) {
            if (inf) { if (k == 0) pick = e; else k--; }
            return;
        }
        const double ns = __dadd_rn(S, m);
        if (mode == 1 && ns > t) { pick = e; return; }
        S = ns;
        if (mode == 0) ninf += inf ? 1u : 0u;
    }
    __device__ __forceinline__ void finish(uint32_t n) { gap(n); }
};

// The weighted-random pick: feed(w) presents the item sequence to Walker w (all lanes, warp-uniform); n = population size,
// nth(r) = the population member of rank r (ascending slot), for the W == 0 fallback.
template <typename Feed, typename Nth>
__device__ __forceinline__ uint32_t weighted_pick(const ProfileDev &pf, bool gaps, double u, uint32_t n, Feed feed, Nth nth) {
    Walker w0(pf, gaps, 0, 0.0, 0);
    feed(w0);
    if (w0.ninf) {
        Walker w2(pf, gaps, 2, 0.0, pick_rank(u, w0.ninf));
        feed(w2);
        return w2.pick;
    }
    const double W = w0.S;
    if (!(W > 0.0)) return nth(pick_rank(u, n));
    double t = __dmul_rn(u, W);
    if (t >= W) t = __longlong_as_double(__double_as_longlong(W) - 1);
    Walker w1(pf, gaps, 1, t, 0);
    feed(w1);
    return w1.pick;
}

// Full-scan form (dense-counter, injected-match and general evaluation kernels).  cand_of(e): e is a candidate (with
// gaps: one of pf's, whose positions index pf.cands / wcum / icum); expl_of(e): e is explicit (asked for candidates only,
// only when gaps); score_of(e): e's weighted score.  out_of(e): e was already emitted into the request's first-k list --
// it stays in the sequence as an explicit item of mass 0 and leaves the population; out_of is called by every lane
// (e may be >= E) since it may shuffle.  n = the population (candidates not out), n_out = how many are out.
template <typename CandOf, typename ExplOf, typename ScoreOf, typename OutOf>
__device__ inline Best draw_scan(const ProfileDev &pf, int32_t E, int lane, bool gaps, uint32_t n, uint32_t n_out,
                                 uint64_t seed, uint64_t key, CandOf cand_of, ExplOf expl_of, ScoreOf score_of,
                                 OutOf out_of) {
    Best b;
    best_init(b);
    if (n == 0) return b;
    const double u = pick_u(seed, key);
    auto nth = [&](uint32_t r) -> uint32_t {
        if (gaps && !n_out) return pf.cands[r];
        for (uint32_t e0 = 0; e0 < (uint32_t)E; e0 += 32) {
            const uint32_t e = e0 + lane;
            const bool o = out_of(e);
            uint32_t bal = __ballot_sync(0xffffffffu, e < (uint32_t)E && !o && cand_of(e));
            const uint32_t c = __popc(bal);
            if (r < c) {
                for (uint32_t i = 0; i < r; i++) bal &= bal - 1;
                return e0 + (uint32_t)__ffs(bal) - 1u;
            }
            r -= c;
        }
        return kNone;
    };
    uint32_t pick;
    if (pf.cfg.picker == EPP_PICKER_RANDOM) {
        pick = nth(pick_rank(u, n));
    } else {
        const double sigma = mass_scale(pf.cfg);
        auto feed = [&](Walker &w) {
            uint32_t q = 0;                                // population members before this chunk
            for (uint32_t e0 = 0; e0 < (uint32_t)E && w.pick == kNone; e0 += 32) {
                const uint32_t e = e0 + lane;
                const bool o = out_of(e);
                const bool c = e < (uint32_t)E && cand_of(e);
                const bool x = c && (!gaps || o || expl_of(e));
                double m = 0.0;
                bool inf = false;
                if (x && !o) {
                    const double s = score_of(e);
                    m = mass_of(s, sigma);
                    inf = is_pinf(s);
                }
                const uint32_t cm = __ballot_sync(0xffffffffu, c);
                uint32_t xm = __ballot_sync(0xffffffffu, x);
                while (xm) {
                    const int l = __ffs(xm) - 1;
                    xm &= xm - 1;
                    const double ml = __shfl_sync(0xffffffffu, m, l);
                    const bool il = __shfl_sync(0xffffffffu, (int)inf, l) != 0;
                    w.item(q + __popc(cm & ((1u << l) - 1u)), ml, il, e0 + (uint32_t)l);
                }
                q += __popc(cm);
            }
            w.finish(n + n_out);                          // every candidate, the emitted ones included
        };
        pick = weighted_pick(pf, gaps, u, n, feed, nth);
    }
    b.pick = pick;
    b.val = score_of(pick);
    b.ties = n;
    return b;
}

}  // namespace rnd
}  // namespace epp
