"""The latency pieces without a GPU: tools/latency_model.py on cases restated from the reference's plugin code, the
ctypes layout of the new ABI records, and pack_predictions."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tools import latency_model as lm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def info(th, tp, disp=1, ttft=10.0):
    return lm.Info(ttft, th, tp, disp)


CFG = dict(lm.DEFAULT_CFG)


def score(endpoints, inf, waiting=None, kv=None, prefix=None, **cfg):
    n = max(endpoints) + 1
    return lm.latency_score(dict(CFG, **cfg), endpoints, inf, waiting or [0] * n, kv or [0.0] * n, prefix or [0.0] * n)


# ---- tier filter (sloheadroomtier/plugin.go:84-138) ------------------------------------------------------------------
def test_tier_single_endpoint_kept():
    assert lm.tier_filter([3], {3: info(-1, -1)}, 0.0, lambda: 0.5) == [3]


def test_tier_no_predictions_keeps_all():
    assert lm.tier_filter([0, 1, 2], {}, 0.0, lambda: 0.5) == [0, 1, 2]


def test_tier_positive_kept_no_prediction_joins_negative():
    inf = {0: info(1, 1), 1: info(-1, 1)}
    assert lm.tier_filter([0, 1, 2], inf, 0.01, lambda: 0.5) == [0]
    assert lm.tier_filter([0, 1, 2], inf, 0.9, lambda: 0.5) == [1, 2]


def test_tier_only_negative_or_no_prediction():
    assert lm.tier_filter([0, 1], {0: info(-1, 1)}, 0.0, lambda: 0.0) == [0, 1]


def test_tier_zero_headroom_is_positive():
    assert lm.tier_filter([0, 1], {0: info(0.0, 0.0), 1: info(-0.5, 0)}, 0.0, lambda: 0.5) == [0]


# ---- latency scorer (scorer/latency/plugin.go:144-395) ---------------------------------------------------------------
def test_score_no_entry_is_positive_headroom_zero():
    s = score([0, 1, 2], {0: info(10, 2), 1: info(-5, 1)})
    assert s[1] == 0.0                       # negative: outside the positive bucket
    assert s[0] == 0.01 and s[2] == 1.01     # least: the most headroom scores lowest; the entry-less one counts as 0


def test_score_most_strategy():
    s = score([0, 1], {0: info(10, 2), 1: info(20, 4)}, strategy="most")
    assert s == {0: 0.01, 1: 1.01}


def test_score_idle_preferred_among_negative():
    s = score([0, 1, 2], {0: info(-10, -1, 0), 1: info(-1, -1, 3), 2: info(-30, -2, 0)})
    assert s[1] == 0.0 and s[0] > 0 and s[2] > 0


def test_score_bucket_order():
    inf = {0: info(-1, -1), 1: info(-1, 2), 2: info(3, -1)}
    s = score([0, 1, 2], inf)
    assert s[2] > 0 and s[0] == 0 and s[1] == 0          # TPOT-only negative first
    s = score([0, 1], {0: info(-1, -1), 1: info(-1, 2)})
    assert s[1] > 0 and s[0] == 0                        # then TTFT-only


def test_score_zero_range_renormalisation():
    # TTFT range 0, TPOT range > eps: all weight to TPOT
    s = score([0, 1], {0: info(5, 1), 1: info(5, 3)})
    assert s == {0: 1.01, 1: 0.01}
    # both ranges 0: n = 0.5 on both dimensions, least -> int(50) + 1
    s = score([0, 1], {0: info(5, 1), 1: info(5, 1)})
    assert s == {0: 0.51, 1: 0.51}


def test_score_truncation_not_rounding():
    # combined = 0.8 * 1/3 + 0.2 * 0.5 -> least: int((1 - combined) * 100) truncates
    s = score([0, 1, 2], {0: info(0, 0), 1: info(1, 1), 2: info(3, 2)})
    a, b = 0.8, 0.2
    comb = a * (1 / 3) + b * 0.5
    assert s[1] == float(int((1.0 - comb) * 100) + 1) / 100


def test_composite_fallback():
    s = score([0, 1], {}, waiting=[4, 0], kv=[0.5, 0.0], prefix=[1.0, 0.0])
    # (1/3 * 0.5 + 1/3 * 0 + 1/3 * 1) -> round(50) / 100; (1/3 + 1/3 + 0) -> round(66.67) / 100
    assert s == {0: 0.5, 1: 0.67}
    s = score([0, 1], {}, waiting=[0, 0], kv=[0.0, 0.0], composite_kv_weight=0, composite_queue_weight=0,
              composite_prefix_weight=0)
    assert s == {0: 1.0, 1: 1.0}


def test_go_round_and_int():
    assert lm.go_round(0.5) == 1.0 and lm.go_round(-0.5) == -1.0 and lm.go_round(2.5) == 3.0
    assert lm.go_round(0.49999999999999994) == 0.0
    assert lm.go_int(-0.7) == 0 and lm.go_int(float("nan")) == lm.INT64_MIN and lm.go_int(1e300) == lm.INT64_MIN


# ---- chain -----------------------------------------------------------------------------------------------------------
def test_chain_two_gates():
    match = [10, 10, 9, 0, 0]
    inf = {0: info(-1, 1), 1: info(5, 5), 2: info(5, 5), 3: info(5, 5)}
    cfg = dict(CFG, tier_filter=1, a1_affinity_threshold=0.99)
    # A1 keeps {0, 1}; T keeps the positive {1}; A2 sees a set of one
    assert lm.chain(range(5), match, 10, inf, cfg, (0.8, 0.0, 5000.0), 0, 0) == [1]
    # without A1: T keeps {1, 2, 3}; A2 keeps the sticky {1, 2}
    cfg["a1_affinity_threshold"] = 0.0
    assert lm.chain(range(5), match, 10, inf, cfg, (0.8, 0.0, 5000.0), 0, 0) == [1, 2]


def test_ttft_gate_reads_predictions():
    match = [10, 0, 0]
    inf = {0: info(1, 1, ttft=9000.0), 1: info(1, 1, ttft=10.0)}
    assert lm.affinity_filter([0, 1, 2], match, 10, 0.8, 0.0, 5000.0, inf, lambda: 1.0) == [0, 1, 2]
    inf[0] = info(1, 1, ttft=100.0)
    assert lm.affinity_filter([0, 1, 2], match, 10, 0.8, 0.0, 5000.0, inf, lambda: 1.0) == [0]
    # without entries bestTTFT is MaxFloat64 on both sides: the gate never breaks
    assert lm.affinity_filter([0, 1, 2], match, 10, 0.8, 0.0, 1.0, {}, lambda: 1.0) == [0]


def test_draws_are_distinct():
    u = [lm.draw_u(7, d, 12) for d in (lm.A1_DOMAIN, lm.TIER_DOMAIN, lm.EXPLORE_DOMAIN)]
    assert len(set(u)) == 3 and all(0.0 <= x < 1.0 for x in u)


# ---- ABI -------------------------------------------------------------------------------------------------------------
PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "epp_engine.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu\n", sizeof(epp_prediction), offsetof(epp_prediction, ttft),
           offsetof(epp_prediction, tpot_headroom), sizeof(epp_predictions), offsetof(epp_predictions, entries));
    printf("%zu %zu %zu %zu\n", sizeof(epp_latency_cfg), offsetof(epp_latency_cfg, strategy),
           offsetof(epp_latency_cfg, composite_kv_weight), offsetof(epp_latency_cfg, composite_prefix_weight));
    printf("%d\n", (int)EPP_SCORER_LATENCY);
    return 0;
}
"""


def test_ctypes_layout(tmp_path):
    from oracle import pyoracle  # noqa: F401  (the package imports below need the repository on sys.path)
    import importlib
    capi = importlib.import_module("llm-d-inference-scheduler_b200._capi")
    src = tmp_path / "probe.c"
    src.write_text(PROBE)
    exe = tmp_path / "probe"
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    P, Ps, L = capi.Prediction, capi.Predictions, capi.LatencyCfg
    assert list(map(int, out[0].split())) == [C.sizeof(P), P.ttft.offset, P.tpot_headroom.offset, C.sizeof(Ps),
                                              Ps.entries.offset]
    assert list(map(int, out[1].split())) == [C.sizeof(L), L.strategy.offset, L.composite_kv_weight.offset,
                                              L.composite_prefix_weight.offset]
    assert int(out[2]) == capi.SCORER_LATENCY == 10
    assert C.sizeof(P) == 32


def test_pack_predictions():
    import importlib
    eng = importlib.import_module("llm-d-inference-scheduler_b200.engine")
    counts, offs, ent = eng.pack_predictions([None, [(5, 1.0, 2.0, -1.0, 0), (2, 3.0, 1.0, 1.0, 4)], []])
    assert list(counts) == [0, 2, 0] and list(offs) == [0, 0, 2]
    assert list(ent["slot"]) == [2, 5] and list(ent["dispatched"]) == [4, 0]
    assert ent.dtype.itemsize == 32
    with pytest.raises(ValueError):
        eng.pack_predictions([[(1, 1.0, 1.0, 1.0, 0), (1, 2.0, 1.0, 1.0, 0)]])
    with pytest.raises(ValueError):
        eng.pack_predictions([[(-1, 1.0, 1.0, 1.0, 0)]])


# ---- the GPU landscapes reach their edges ----------------------------------------------------------------------------
def test_gpu_landscapes_reach_their_edges():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_latency_profile_gpu as g
    buckets = {}
    for name in g.LANDSCAPES:
        _, _, preds = g.landscape(name, 24, 1)
        d = preds[0] or {}
        vals = list(d.values())
        buckets[name] = (len(vals), sum(v.ttft_headroom >= 0 and v.tpot_headroom >= 0 for v in vals))
    assert buckets["all_positive"][0] == buckets["all_positive"][1] == g.E
    assert buckets["all_negative_busy"][1] == 0 and buckets["both_bucket"][1] == 0
    assert buckets["none"][0] == 0 and 0 < buckets["partial"][0] < g.E
    _, total, _ = g.landscape("none_idle", 4, 1)
    assert (total == 0).all()
    _, _, preds = g.landscape("zero_range_both", 2, 1)
    assert len({(v.ttft_headroom, v.tpot_headroom) for v in preds[0].values()}) == 1


# ---- the reference's own cases (sloheadroomtier/plugin_test.go, scorer/latency/plugin_test.go), through the model ----
def _tier_ep(th, tp, has=True):
    return lm.Info(100.0, th, tp, 0) if has else None


def _tier(eps, specs, explore):
    inf = {name: i for name, i in zip(eps, specs) if i is not None}
    return lm.tier_filter(list(eps), inf, explore, lambda: 0.5)


def test_ref_filter_single_endpoint():
    assert len(_tier(["a"], [_tier_ep(-1, -1)], 0.01)) == 1


def test_ref_filter_no_predictions():
    assert len(_tier(["a", "b"], [None, None], 0.01)) == 2


def test_ref_filter_all_positive():
    assert len(_tier(["a", "b"], [_tier_ep(100, 50), _tier_ep(200, 80)], 0.0)) == 2


def test_ref_filter_all_negative():
    assert len(_tier(["a", "b"], [_tier_ep(-100, -50), _tier_ep(-200, -80)], 0.0)) == 2


def test_ref_filter_both_tiers_select_positive():
    r = _tier(["pos1", "pos2", "neg1"], [_tier_ep(100, 50), _tier_ep(200, 80), _tier_ep(-100, -50)], 0.0)
    assert r == ["pos1", "pos2"]


def test_ref_filter_both_tiers_epsilon_explore_neg():
    assert _tier(["pos1", "neg1"], [_tier_ep(100, 50), _tier_ep(-100, -50)], 1.0) == ["neg1"]


def test_ref_filter_no_prediction_goes_to_negative():
    assert _tier(["pos1", "nopred"], [_tier_ep(100, 50), None], 1.0) == ["nopred"]


def _plugins():
    import importlib
    return importlib.import_module("llm-d-inference-scheduler_b200.plugins")


def test_ref_factory_valid_config():
    pl = _plugins()
    assert pl.SLOHeadroomTierFilterFactory("test", b'{"epsilonExploreNeg": 0.05}').epsilonExploreNeg == 0.05


def test_ref_factory_invalid_epsilon():
    pl = _plugins()
    with pytest.raises(ValueError, match=r"epsilonExploreNeg must be in \[0, 1\], got 1.500000"):
        pl.SLOHeadroomTierFilterFactory("test", b'{"epsilonExploreNeg": 1.5}')


def _lat_case(eps):
    """eps: [(kv, queue, running, (ttft_headroom, tpot_headroom, ttft, dispatched) or None)] -> model scores."""
    n = len(eps)
    inf = {i: lm.Info(p[2], p[0], p[1], p[3]) for i, (_, _, _, p) in enumerate(eps) if p is not None}
    s = lm.latency_score(dict(CFG), list(range(n)), inf, [e[1] for e in eps], [e[0] for e in eps], [0.0] * n)
    return [s[i] for i in range(n)]


def test_ref_score_positive_headroom():
    s1, s2 = _lat_case([(0.3, 0, 5, (100, 20, 50, 0)), (0.5, 0, 8, (30, 5, 120, 0))])
    assert s1 != 0 and s2 != 0


def test_ref_score_negative_only():
    s1, s2 = _lat_case([(0.5, 0, 5, (-10, -5, 110, 0)), (0.6, 0, 8, (-100, -30, 200, 0))])
    assert s1 != 0 and s2 != 0 and s1 > s2


def test_ref_score_tier_split():
    s1, s2 = _lat_case([(0.3, 0, 5, (10, 2, 90, 0)), (0.5, 0, 8, (50, 10, 50, 0))])
    assert s1 != 0 and s2 != 0 and s1 > s2


def test_ref_score_idle_pod_preference():
    busy, idle = _lat_case([(0.5, 0, 5, (-50, -10, 150, 5)), (0.5, 0, 0, (-50, -10, 150, 0))])
    assert idle != 0 and busy == 0


def test_ref_score_hierarchical_buckets():
    s = _lat_case([(0.5, 0, 5, (-50, -10, 150, 0)), (0.4, 0, 3, (-30, 5, 130, 0)), (0.6, 0, 4, (10, -8, 90, 0))])
    assert all(x != 0 for x in s)


def test_ref_score_composite_fallback():
    s1, s2 = _lat_case([(0.2, 0, 3, None), (0.8, 5, 10, None)])
    assert s1 > s2


# ---- prefixcacheaffinity cases placed in the two-gate chain --------------------------------------------------------
def test_ref_affinity_in_chain():
    cfg = dict(CFG, tier_filter=1, epsilon_explore_neg=0.0, a1_affinity_threshold=0.99, a1_exploration_probability=0.0)
    pos = {i: info(5, 5, ttft=100.0) for i in range(4)}
    # below threshold: A1 keeps all, T keeps all (every one positive), A2 narrows to the 0.8-sticky ones
    assert lm.chain(range(4), [8, 9, 2, 0], 10, pos, cfg, (0.8, 0.0, 5000.0), 0, 0) == [0, 1]
    # no sticky endpoint anywhere: everything survives
    assert lm.chain(range(4), [1, 2, 3, 0], 10, pos, cfg, (0.8, 0.0, 5000.0), 0, 0) == [0, 1, 2, 3]
    # A1's TTFT gate broken by the sticky endpoint's predicted TTFT: A1 keeps all, A2 (no penalty) sticks
    slow = dict(pos)
    slow[0] = info(5, 5, ttft=9000.0)
    assert lm.chain(range(4), [10, 9, 0, 0], 10, slow, cfg, (0.8, 0.0, 0.0), 0, 0) == [0, 1]
    # total blocks 0: the prefix score is 0 for everyone, nobody is sticky
    assert lm.chain(range(3), [0, 0, 0], 0, pos, cfg, (0.8, 0.0, 5000.0), 0, 0) == [0, 1, 2]


# ---- factories and the chain of SchedulerProfile -------------------------------------------------------------------
def test_latency_scorer_factory():
    pl = _plugins()
    s = pl.LatencyScorerFactory("ls", b'{"TTFTWEIGHT": 0.5, "unknown": 3}')      # Go: case-insensitive keys
    assert s.config.ttftWeight == 0.5 and s.config.tpotWeight == 0.2 and s.config.compositeKVWeight == 1.0
    assert pl.LatencyScorerFactory("ls", b"null").config == pl.LatencyScorerConfig()
    assert pl.LatencyScorerFactory("ls", b"").config == pl.LatencyScorerConfig()
    odd = pl.LatencyScorerFactory("ls", {"headroomSelectionStrategy": "sideways"})
    assert pl._latency_fields(None, None, odd)["strategy"] == 0                  # the switch's default: least
    most = pl.LatencyScorerFactory("ls", '{"headroomSelectionStrategy": "most"}')
    assert pl._latency_fields(None, None, most)["strategy"] == 1
    for bad in (b"{", b'{"ttftWeight": "x"}', b"[1]", b'{"headroomSelectionStrategy": 3}'):
        with pytest.raises(ValueError, match="failed to unmarshal config"):
            pl.LatencyScorerFactory("ls", bad)
    with pytest.raises(ValueError, match="failed to unmarshal config"):
        pl.SLOHeadroomTierFilterFactory("t", b'{"epsilonExploreNeg": true}')
    assert pl.SLOHeadroomTierFilterFactory("t", None).epsilonExploreNeg == 0.01


def test_latency_prediction_info():
    pl = _plugins()
    i = pl.NewLatencyPredictionInfo(True, False, 1.5, -2.0, 30.0, 4.0, 7)
    assert (i.TTFTValid(), i.TPOTValid(), i.IsValid(), i.TTFTHeadroom(), i.TPOTHeadroom(), i.TTFT(), i.TPOT(),
            i.DispatchedRequestCount()) == (True, False, False, 1.5, -2.0, 30.0, 4.0, 7)
    assert i.entry(3) == (3, 30.0, 1.5, -2.0, 7)


def test_chain_accept_reject():
    pl = _plugins()
    A = lambda t=0.8: pl.PrefixCacheAffinityFilter(t)  # noqa: E731
    T = pl.SLOHeadroomTierFilter
    role = pl.NewDecodeRole()
    lab = pl.NewByLabel("l", "k", True)
    ok = [[A(0.99), T(), A()], [role, lab, A(0.99), T(), A()], [T()], [T(), A()], [A(), T()], [lab, T(), A()], [A()]]
    for chain in ok:
        pl.SchedulerProfile().WithFilters(*chain)
    bad = [[A(), A()], [lab, A(), lab], [A(), lab, T()], [T(), A(), A()], [T(), lab], [A(), A(), T()], [T(), T()],
           [T(), A(), lab]]
    for chain in bad:
        with pytest.raises(AssertionError):
            pl.SchedulerProfile().WithFilters(*chain)


def test_chart_profile_spec():
    pl = _plugins()
    p = pl.SchedulerProfile().WithFilters(pl.PrefixCacheAffinityFilter(0.99), pl.SLOHeadroomTierFilterFactory("t", None),
                                          pl.PrefixCacheAffinityFilter(0.80)) \
        .WithScorers(pl.NewWeightedScorer(pl.LatencyScorerFactory("ls", None), 1.0)) \
        .WithPicker(pl.NewWeightedRandomPicker())
    spec = p.spec()
    assert spec.affinity.affinity_threshold == 0.80 and spec.picker == 2
    assert spec.latency == dict(tier_filter=1, epsilon_explore_neg=0.01, a1_affinity_threshold=0.99,
                                a1_exploration_probability=0.01, a1_max_ttft_penalty_ms=5000.0, ttft_weight=0.8,
                                tpot_weight=0.2, strategy=0, composite_kv_weight=1.0, composite_queue_weight=1.0,
                                composite_prefix_weight=1.0)
    assert [s.kind for s in spec.scorers] == [10]
    plain = pl.SchedulerProfile().WithFilters(pl.PrefixCacheAffinityFilter()).spec()
    assert plain.latency is None and plain.affinity.affinity_threshold == 0.80
