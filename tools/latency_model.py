"""CPU restatement of the latency pieces (include/epp_engine.h "Latency predictions"): the slo-headroom-tier-filter
(filter/sloheadroomtier/plugin.go:84-138), the latency-scorer (scorer/latency/plugin.go:144-395: Score, scoreBucket,
compositeScores), the prefix-cache-affinity-filter reading TTFT from the request's predictions, the two-gate chain with
its draws, and a scheduling model built on the C oracle.

The three Go functions are restated line by line on Python floats (IEEE doubles, no fused multiply-add: Go's amd64
arithmetic).  The oracle itself knows neither the predictions nor the latency scorer, so a profile is decided as the label
model does it: the chain runs here, the pool handed to the oracle holds only the final set (every other slot absent), and
the latency scorer becomes an external column holding this module's scores.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import picker_model as pm  # noqa: E402

M64 = (1 << 64) - 1
A1_DOMAIN = 0x8EBC6AF09C88C6E3
TIER_DOMAIN = 0x589965CC75374CC3
EXPLORE_DOMAIN = 0xA0761D6478BD642F
EPS = 1e-9
W_MAX, MIN_WEIGHT = 100, 0
SCORER_EXTERNAL, SCORER_LATENCY = 4, 10
INT64_MIN = -(1 << 63)


class Info:
    """LatencyPredictionInfo as the plugins read it."""

    def __init__(self, ttft, ttft_headroom, tpot_headroom, dispatched):
        self.ttft, self.ttft_headroom, self.tpot_headroom, self.dispatched = ttft, ttft_headroom, tpot_headroom, dispatched


def draw_u(seed: int, domain: int, key: int) -> float:
    return (pm.mix64(((seed ^ domain) ^ pm.mix64(key)) & M64) >> 11) * 2.0 ** -53


def go_int(x: float) -> int:
    """int(x) of Go on amd64: truncation toward zero; NaN and out-of-range give math.MinInt64."""
    if not (-2.0 ** 63 < x < 2.0 ** 63):
        return INT64_MIN
    return int(x)


def go_round(x: float) -> float:
    """math.Round: the nearest integer, halves away from zero."""
    if math.isnan(x) or math.isinf(x):
        return x
    t = float(math.trunc(x))
    if abs(x - t) >= 0.5:
        t += math.copysign(1.0, x)
    return t


# ---- filter/sloheadroomtier/plugin.go:84-138 -------------------------------------------------------------------------
def tier_filter(endpoints, info, eps_neg, rand):
    """endpoints: ordered list; info: endpoint -> Info (absent = no attribute); rand(): the draw."""
    if len(endpoints) <= 1:
        return endpoints
    positive, negative, no_prediction = [], [], []
    for ep in endpoints:
        i = info.get(ep)
        if i is None:
            no_prediction.append(ep)
            continue
        if i.ttft_headroom >= 0 and i.tpot_headroom >= 0:
            positive.append(ep)
        else:
            negative.append(ep)
    if len(positive) == 0 and len(negative) == 0:
        return endpoints
    negative = negative + no_prediction
    if len(positive) > 0 and len(negative) > 0:
        if rand() < eps_neg:
            return negative
        return positive
    if len(positive) > 0:
        return positive
    return negative


# ---- scorer/latency/plugin.go:144-395 --------------------------------------------------------------------------------
def normalized_weights(a, b):
    s = a + b
    if s <= 0:
        return 1.0, 0.0
    return a / s, b / s


def score_bucket(cfg, data, scores, force_least):
    alpha, beta = normalized_weights(cfg["ttft_weight"], cfg["tpot_weight"])
    min_t, max_t = sys.float_info.max, -sys.float_info.max
    min_p, max_p = sys.float_info.max, -sys.float_info.max
    for _, th, tp, _i in data:
        h = abs(th)
        if h < min_t:
            min_t = h
        if h > max_t:
            max_t = h
        h = abs(tp)
        if h < min_p:
            min_p = h
        if h > max_p:
            max_p = h
    rt = max_t - min_t
    rp = max_p - min_p
    if rt <= EPS and rp > EPS:
        alpha, beta = 0.0, 1.0
    elif rp <= EPS and rt > EPS:
        alpha, beta = 1.0, 0.0
    for ep, th, tp, _i in data:
        nt = (abs(th) - min_t) / rt if rt > EPS else 0.5
        np_ = (abs(tp) - min_p) / rp if rp > EPS else 0.5
        combined = alpha * nt + beta * np_
        strategy = "least" if force_least else cfg["strategy"]
        if strategy == "most":
            w = float(go_int(combined * float(W_MAX - MIN_WEIGHT)) + MIN_WEIGHT + 1)
        else:
            w = float(go_int((1.0 - combined) * float(W_MAX - MIN_WEIGHT)) + MIN_WEIGHT + 1)
        scores[ep] = w / float(W_MAX)


def composite_scores(cfg, endpoints, waiting, kv, prefix):
    scores = {}
    wkv, wq, wpref = cfg["composite_kv_weight"], cfg["composite_queue_weight"], cfg["composite_prefix_weight"]
    sumw = wkv + wq + wpref
    if sumw <= 0:
        wkv, wq, wpref = 1.0, 0.0, 0.0
        sumw = 1.0
    wkv /= sumw
    wq /= sumw
    wpref /= sumw
    max_q = 0
    for ep in endpoints:
        if waiting[ep] > max_q:
            max_q = waiting[ep]
    q_range = float(max_q)
    for ep in endpoints:
        q = waiting[ep]
        rel = 1.0
        if q_range > 0:
            rel = float(max_q - q) / q_range
        kv_free = 1.0 - kv[ep]
        composite = wkv * kv_free + wq * rel + wpref * prefix[ep]
        w = go_int(go_round(float(MIN_WEIGHT) + float(W_MAX - MIN_WEIGHT) * composite))
        scores[ep] = float(w) / float(W_MAX)
    return scores


def latency_score(cfg, endpoints, info, waiting, kv, prefix):
    """Score: endpoint -> score over the ordered endpoints."""
    scores = {ep: 0.0 for ep in endpoints}
    data, has = [], False
    for ep in endpoints:
        i = info.get(ep)
        if i is not None:
            data.append((ep, i.ttft_headroom, i.tpot_headroom, i))
            has = True
        else:
            data.append((ep, 0.0, 0.0, None))
    if not has:
        return composite_scores(cfg, endpoints, waiting, kv, prefix)
    positive, negative = [], []
    for d in data:
        if d[3] is not None and (d[1] < 0 or d[2] < 0):
            negative.append(d)
        else:
            positive.append(d)
    if positive:
        score_bucket(cfg, positive, scores, False)
        return scores
    idle = [d for d in negative if d[3] is not None and d[3].dispatched == 0]
    if idle:
        score_bucket(cfg, idle, scores, True)
        return scores
    neg_tpot, neg_ttft, both = [], [], []
    for d in negative:
        if d[3] is None:
            both.append(d)
            continue
        tn, pn = d[1] < 0, d[2] < 0
        if tn and pn:
            both.append(d)
        elif tn:
            neg_ttft.append(d)
        elif pn:
            neg_tpot.append(d)
        else:
            both.append(d)
    for bucket in (neg_tpot, neg_ttft, both):
        if bucket:
            score_bucket(cfg, bucket, scores, True)
            return scores
    score_bucket(cfg, negative, scores, True)
    return scores


# ---- filter/prefixcacheaffinity/plugin.go:105-151 with TTFT from the request's predictions ---------------------------
def affinity_filter(endpoints, match, total, thr, explore, penalty, info, rand):
    if len(endpoints) <= 1 or thr <= 0:
        return endpoints
    if rand() < explore:
        return endpoints
    pcs = lambda ep: (match[ep] / total) if total > 0 else 0.0  # noqa: E731
    sticky = [ep for ep in endpoints if pcs(ep) >= thr]
    non = [ep for ep in endpoints if pcs(ep) < thr]
    if not sticky:
        return endpoints

    def best(eps):
        b = sys.float_info.max
        for ep in eps:
            i = info.get(ep)
            if i is not None and i.ttft < b:
                b = i.ttft
        return b
    if penalty > 0 and non:
        if best(sticky) - best(non) > penalty:
            return endpoints
    return sticky


# ---- the chain and a profile decision --------------------------------------------------------------------------------
DEFAULT_CFG = dict(tier_filter=0, epsilon_explore_neg=0.01, a1_affinity_threshold=0.0, a1_exploration_probability=0.01,
                   a1_max_ttft_penalty_ms=5000.0, ttft_weight=0.8, tpot_weight=0.2, strategy="least",
                   composite_kv_weight=1.0, composite_queue_weight=1.0, composite_prefix_weight=1.0)


def chain(cands, match, total, info, lcfg, a2, seed, key):
    """The final set of [A1] -> [T] -> [A2] over the ordered candidates.  a2 = (threshold, exploration, penalty) or None.
    With seed == 0 no stage explores."""
    never = lambda: 1.0  # noqa: E731
    s = list(cands)
    if lcfg["tier_filter"]:
        if lcfg["a1_affinity_threshold"] > 0:
            s = affinity_filter(s, match, total, lcfg["a1_affinity_threshold"], lcfg["a1_exploration_probability"],
                                lcfg["a1_max_ttft_penalty_ms"], info,
                                (lambda: draw_u(seed, A1_DOMAIN, key)) if seed else never)
        s = tier_filter(s, info, lcfg["epsilon_explore_neg"], (lambda: draw_u(seed, TIER_DOMAIN, key)) if seed else never)
    if a2 is not None:
        s = affinity_filter(s, match, total, a2[0], a2[1], a2[2], info,
                            (lambda: draw_u(seed, EXPLORE_DOMAIN, key)) if seed else never)
    return s


def profile_decide(orc, filter_kind, scorers, picker, role, kv, waiting, running, match, total, info, lcfg=None, a2=None,
                   seed=0, key=0, k=1, keep=None, lora=None):
    """One latency profile for one request -> dict(ties, picks, scores, final).  scorers: oracle tuples (kind, weight,
    param[, column[, param2]]) with kind SCORER_LATENCY for the latency scorer; picker: 0 max-score, 1 random,
    2 weighted-random; keep: bool [E] of the label filters or None; lora: (state, max_active, loaded) for the request's
    adapter or None."""
    lcfg = dict(DEFAULT_CFG, **(lcfg or {}))
    E = len(role)
    cands = [e for e in range(E) if role[e] != 0xFF and orc.lib().orc_role_filter_keeps(filter_kind, int(role[e]))
             and (keep is None or keep[e])]
    final = chain(cands, match, total, info, lcfg, a2, seed, key)
    prefix = [(match[e] / total) if total > 0 else 0.0 for e in range(E)]
    lat = latency_score(lcfg, final, info, waiting, kv, prefix)
    col = np.zeros(E, dtype=np.float64)
    for e, v in lat.items():
        col[e] = v
    r = np.full(E, 0xFF, dtype=np.uint8)
    for e in final:
        r[e] = role[e]
    pool = orc.PoolState(r, kv, waiting, running, col)
    if lora is not None:
        pool.set_lora(*lora)
    sc = [(SCORER_EXTERNAL, s[1], 0.0) if s[0] == SCORER_LATENCY else s for s in scorers]
    prof = orc.make_profile(filter_kind, sc)
    picks, pscores, ties, allsc = orc.profile_run_topk(prof, pool, np.asarray(match, dtype=np.int32), total, k, seed, key)
    if picker and final:
        weights = [s[1] for s in scorers]
        score = {e: float(allsc[e]) for e in final}
        # the draws rank the candidates in ascending slot order; the tier filter's negative side lists the endpoints
        # without a prediction last, so the chain's order is not that order
        drawn = pm.draw_k(picker, sorted(final), None, score, set(final), seed, key, weights, k, gaps=False)
        picks = [p for p, _ in drawn]
        pscores = [s for _, s in drawn]
        ties = len(final)
    return dict(ties=ties, picks=picks, scores=pscores, final=final)
