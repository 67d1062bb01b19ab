"""Landscapes for endpoint subsets on a latency engine (include/epp_engine.h "Latency predictions"), checked on the CPU
with tools/latency_model.py alone: each one puts a restricted request on an edge of the chain that the subset moves
(profile_decide with keep = the subset, whole-pool match counts).  tests/test_subset_latency_gpu.py runs the same
landscapes on the device."""
from __future__ import annotations

import numpy as np

from tools import latency_model as lm

E = 48
TOTAL = 10
LAT, QUEUE, KV, PREFIX = 10, 2, 1, 0
ABSENT = (44, 45, 46, 47)

CHART = dict(scorers=[(LAT, 1.0, 0.0)], picker=0, a2=(0.80, 0.0, 5000.0),
             lcfg=dict(tier_filter=1, epsilon_explore_neg=0.0, a1_affinity_threshold=0.99,
                       a1_exploration_probability=0.0, a1_max_ttft_penalty_ms=5000.0))


def pool():
    rng = np.random.default_rng(21)
    role = np.zeros(E, np.uint8)
    role[list(ABSENT)] = 0xFF
    kv = rng.choice([0.0, 0.25, 0.5, 0.75], E)
    waiting = rng.integers(0, 6, E)
    running = rng.integers(0, 6, E)
    return role, kv, waiting, running


def case(name):
    """-> dict(match [E], info {slot: Info}, subset [...], waiting override or None)."""
    match = np.zeros(E, np.int32)
    match[::5] = 3
    waiting = None
    if name == "tier_flip":               # the pool keeps its positive tier; the subset holds no positive endpoint
        info = {e: lm.Info(50.0, 20.0 if e < 20 else -10.0, 5.0, 1) for e in range(E)}
        subset = list(range(20, 40))
    elif name == "a1_gate":               # A1 narrows the pool to slot 5; the subset has one candidate (and an absent slot)
        match[5] = 10
        info = {e: lm.Info(50.0, float(e), 5.0, 1) for e in range(E)}
        subset = [7, 45]
    elif name == "sticky_excluded":       # the pool's only sticky endpoints (3, 4) are outside the subset
        match[3] = match[4] = 10
        info = {e: lm.Info(50.0, float(e % 7), 1.0 + e % 3, 1) for e in range(E)}
        subset = list(range(8, 30))
    elif name == "composite":             # the subset's members have no entry, the others do
        info = {e: lm.Info(50.0, float(e), 2.0, 0) for e in range(E) if not 10 <= e < 26}
        subset = list(range(10, 26))
    elif name == "range_extreme":         # the pool's largest |TTFT headroom| and queue are outside the subset
        info = {e: lm.Info(50.0, 1000.0 if e == 2 else float(e % 11), float(e % 5), 1) for e in range(E)}
        waiting = np.arange(E) % 6
        waiting[2] = 40
        subset = list(range(3, 33))
    else:
        raise ValueError(name)
    return dict(match=match, info=info, subset=subset, waiting=waiting)


CASES = ["tier_flip", "a1_gate", "sticky_excluded", "composite", "range_extreme"]


def keep_of(subset):
    k = np.zeros(E, bool)
    k[list(subset)] = True
    return k


def _cands(role, keep=None):
    return [e for e in range(E) if role[e] != 0xFF and (keep is None or keep[e])]


def test_subset_flips_the_tier():
    role, _, _, _ = pool()
    c = case("tier_flip")
    never = lambda: 1.0  # noqa: E731
    whole = lm.tier_filter(_cands(role), c["info"], 0.0, never)
    sub = lm.tier_filter(_cands(role, keep_of(c["subset"])), c["info"], 0.0, never)
    assert all(c["info"][e].ttft_headroom >= 0 for e in whole)
    assert sub and all(c["info"][e].ttft_headroom < 0 for e in sub)


def test_a1_gate_fires_only_in_the_subset():
    role, _, _, _ = pool()
    c = case("a1_gate")
    never = lambda: 1.0  # noqa: E731
    cw = _cands(role)
    cs = _cands(role, keep_of(c["subset"]))
    assert lm.affinity_filter(cw, c["match"], TOTAL, 0.99, 0.0, 5000.0, c["info"], never) == [5]
    assert cs == [7]                                             # slot 45 is not in the pool
    assert lm.affinity_filter(cs, c["match"], TOTAL, 0.99, 0.0, 5000.0, c["info"], never) == [7]


def test_subset_excludes_the_only_sticky_endpoints():
    role, _, _, _ = pool()
    c = case("sticky_excluded")
    never = lambda: 1.0  # noqa: E731
    cw = _cands(role)
    cs = _cands(role, keep_of(c["subset"]))
    assert lm.affinity_filter(cw, c["match"], TOTAL, 0.80, 0.0, 5000.0, c["info"], never) == [3, 4]
    assert lm.affinity_filter(cs, c["match"], TOTAL, 0.80, 0.0, 5000.0, c["info"], never) == cs


def test_subset_without_entries_takes_the_composite_fallback():
    role, kv, waiting, running = pool()
    c = case("composite")
    prefix = [c["match"][e] / TOTAL for e in range(E)]
    cfg = dict(lm.DEFAULT_CFG)
    cs = _cands(role, keep_of(c["subset"]))
    assert not any(e in c["info"] for e in cs)
    assert lm.latency_score(cfg, cs, c["info"], waiting, kv, prefix) == lm.composite_scores(cfg, cs, waiting, kv, prefix)
    whole = lm.latency_score(cfg, _cands(role), c["info"], waiting, kv, prefix)
    assert whole != lm.composite_scores(cfg, _cands(role), waiting, kv, prefix)


def test_dropping_the_extreme_changes_range_and_max_q():
    role, kv, _, running = pool()
    c = case("range_extreme")
    waiting = c["waiting"]
    prefix = [c["match"][e] / TOTAL for e in range(E)]
    cfg = dict(lm.DEFAULT_CFG)
    cw, cs = _cands(role), _cands(role, keep_of(c["subset"]))
    sw = lm.latency_score(cfg, cw, c["info"], waiting, kv, prefix)
    ss = lm.latency_score(cfg, cs, c["info"], waiting, kv, prefix)
    assert any(sw[e] != ss[e] for e in cs)                       # |headroom| range without slot 2's 1000
    qw = lm.composite_scores(cfg, cw, waiting, kv, prefix)
    qs = lm.composite_scores(cfg, cs, waiting, kv, prefix)
    assert any(qw[e] != qs[e] for e in cs)                       # maxQ without slot 2's 40


def test_profile_decide_narrows_to_the_subset(orc):
    """The whole chain on each landscape: the subset's decision differs from the pool's, and stays inside the subset."""
    role, kv, waiting, running = pool()
    for name in CASES:
        c = case(name)
        w = waiting if c["waiting"] is None else c["waiting"]
        args = (orc, 0, CHART["scorers"], CHART["picker"], role, kv, w, running, c["match"], TOTAL, c["info"],
                CHART["lcfg"], CHART["a2"], 0, 0, 4)
        whole = lm.profile_decide(*args)
        sub = lm.profile_decide(*args, keep=keep_of(c["subset"]))
        assert sub["picks"] and set(sub["picks"]) <= set(c["subset"]), name
        assert (sub["picks"], sub["scores"]) != (whole["picks"], whole["scores"]), name
