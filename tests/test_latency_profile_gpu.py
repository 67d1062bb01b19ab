"""Latency profiles on the GPU (include/epp_engine.h "Latency predictions") against tools/latency_model.py, bit for bit:
status, pick, score bits, tie count, match_blocks, total_blocks, the prefill fields and the first-k lists with their
scores.  pick_k = 64 on pools of 48 reads every member's score."""
from __future__ import annotations

import numpy as np
import pytest

from tools import latency_model as lm

pytestmark = pytest.mark.gpu

E = 48
NO = 0xFFFFFFFF
LAT, QUEUE, KV, PREFIX, RUNNING = 10, 2, 1, 0, 5


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def pool(seed):
    rng = np.random.default_rng(seed)
    role = np.zeros(E, np.uint8)
    role[rng.choice(E, 4, replace=False)] = 0xFF
    kv = rng.choice([0.0, 0.25, 0.5, 0.75], E)
    waiting = rng.integers(0, 6, E)
    running = rng.integers(0, 6, E)
    return role, kv, waiting, running


def set_pool(eng, role, kv, waiting, running):
    ids = np.flatnonzero(role != 0xFF).astype(np.uint32)
    eng.pool_set(ids, role[ids], kv[ids], waiting[ids], running[ids])


def landscape(name, R, seed):
    """-> (match [R][E], total [R], predictions: list of R dicts slot -> Info or None)."""
    rng = np.random.default_rng(seed)
    match = np.zeros((R, E), np.int32)
    total = np.full(R, 10, np.int32)
    preds = []
    for r in range(R):
        sticky = rng.choice(E, 6, replace=False)
        match[r, sticky[:3]] = 10
        match[r, sticky[3:]] = 9
        match[r, rng.choice(E, 6)] = rng.integers(1, 8, 6)
        d = {}
        for e in range(E):
            ttft = float(rng.integers(1, 400))
            disp = int(rng.integers(0, 3))
            if name == "all_positive":
                th, tp = float(rng.integers(0, 200)), float(rng.integers(0, 50))
            elif name == "mixed":
                th, tp = float(rng.integers(-100, 100)), float(rng.integers(-20, 20))
            elif name == "all_negative_idle":
                th, tp = -float(rng.integers(1, 100)), float(rng.integers(-20, 20))
            elif name == "all_negative_busy":
                th, tp, disp = -float(rng.integers(1, 100)), float(rng.integers(-20, 20)), int(rng.integers(1, 4))
            elif name == "ttft_only_bucket":
                th, tp, disp = -float(rng.integers(1, 100)), float(rng.integers(0, 20)), 1
            elif name == "both_bucket":
                th, tp, disp = -float(rng.integers(1, 100)), -float(rng.integers(1, 20)), 1
            elif name == "zero_range_ttft":
                th, tp = 50.0, float(rng.integers(0, 40))
            elif name == "zero_range_tpot":
                th, tp = float(rng.integers(0, 400)), 7.0
            elif name == "zero_range_both":
                th, tp = 3.0, 3.0
            elif name == "truncation":
                th, tp = float(rng.integers(0, 101)), 0.0       # alpha = 1: x * 100 lands on every truncation edge
            elif name in ("partial", "ttft_gate"):
                if rng.random() < 0.5:
                    continue
                th, tp = float(rng.integers(-50, 150)), float(rng.integers(-5, 20))
                if name == "ttft_gate":
                    ttft = 6000.0 if match[r, e] >= 9 else ttft
            elif name in ("none", "none_idle"):
                continue
            else:
                raise ValueError(name)
            d[e] = lm.Info(ttft, th, tp, disp)
        if name == "none_idle":
            total[r] = 0
            match[r] = 0
        preds.append(d if d or name not in ("none", "none_idle") else None)
    return match, total, preds


LANDSCAPES = ["all_positive", "mixed", "all_negative_idle", "all_negative_busy", "ttft_only_bucket", "both_bucket",
              "zero_range_ttft", "zero_range_tpot", "zero_range_both", "truncation", "partial", "ttft_gate", "none",
              "none_idle"]

CHART = dict(scorers=[(LAT, 1.0, 0.0)], picker=2, a2=(0.80, 0.3, 5000.0),
             lcfg=dict(tier_filter=1, epsilon_explore_neg=0.3, a1_affinity_threshold=0.99,
                       a1_exploration_probability=0.3, a1_max_ttft_penalty_ms=5000.0))
PROFILES = {
    "chart": CHART,
    "mixed_scorers": dict(scorers=[(QUEUE, 2.0, 0.0), (KV, 2.0, 0.0), (PREFIX, 3.0, 0.0), (LAT, 1.5, 0.0),
                                   (RUNNING, 1.0, 0.0)], picker=0, a2=(0.80, 0.2, 100.0),
                          lcfg=dict(tier_filter=1, epsilon_explore_neg=0.5, strategy="most")),
    "tier_only": dict(scorers=[(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0)], picker=0, a2=None,
                      lcfg=dict(tier_filter=1, epsilon_explore_neg=0.5)),
    "scorer_only_random": dict(scorers=[(LAT, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=1, a2=None,
                               lcfg=dict(ttft_weight=0.0, tpot_weight=0.0, composite_kv_weight=2.0,
                                         composite_queue_weight=0.0, composite_prefix_weight=1.0)),
}


def _spec(epp, p):
    aff = None if p["a2"] is None else epp.AffinityFilterSpec(*p["a2"])
    return epp.ProfileSpec(0, [epp.ScorerSpec(k, w, pa) for k, w, pa in p["scorers"]], aff, p["picker"])


def _lat_kwargs(epp, lcfg):
    kw = dict(lcfg)
    if "strategy" in kw:
        kw["strategy"] = epp.capi.HEADROOM_MOST if kw["strategy"] == "most" else epp.capi.HEADROOM_LEAST
    return kw


def _pred_lists(preds):
    return [None if d is None else [(e, i.ttft, i.ttft_headroom, i.tpot_headroom, i.dispatched) for e, i in d.items()]
            for d in preds]


def _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, lists, seed, k, base=0, pre=None, nct=0,
           in_len=None):
    for r in range(match.shape[0]):
        key = 4 * (base + r)
        info = preds[r] or {}
        m = lm.profile_decide(orc, 0, p["scorers"], p["picker"], role, kv, waiting, running, match[r], int(total[r]),
                              info, p["lcfg"], p["a2"], seed, key, k)
        ok = bool(m["picks"])
        assert dec[r]["status"] == (0 if ok else -1), r
        assert dec[r]["tie_count"] == (m["ties"] if ok else 0), r
        assert int(dec[r]["total_blocks"]) == int(total[r])
        if not ok:
            continue
        assert dec[r]["pick"] == m["picks"][0], (r, m["final"])
        assert np.float64(dec[r]["score"]).tobytes() == np.float64(m["scores"][0]).tobytes(), r
        assert dec[r]["match_blocks"] == match[r, m["picks"][0]]
        if lists is not None:
            n = len(m["picks"])
            assert list(lists["primary"][r, :n]) == m["picks"], r
            assert lists["primary_scores"][r, :n].tobytes() == np.asarray(m["scores"], np.float64).tobytes(), r
            assert all(x == NO for x in lists["primary"][r, n:])
        if pre is not None:
            go = nct and lm_pd(nct, int(in_len[r]), int(match[r, m["picks"][0]]))
            assert det[r]["prefill_ran"] == int(bool(go)), r
            if go:
                q = lm.profile_decide(orc, 0, pre["scorers"], pre["picker"], role, kv, waiting, running, match[r],
                                      int(total[r]), info, pre["lcfg"], pre["a2"], seed, key + 1, 1) \
                    if pre.get("latency", True) else None
                assert dec[r]["prefill_pick"] == q["picks"][0], r
                assert np.float64(det[r]["prefill_score"]).tobytes() == np.float64(q["scores"][0]).tobytes(), r
                assert det[r]["prefill_tie_count"] == q["ties"], r


def lm_pd(nct, in_len, mb, bst=16):
    tokens = in_len // 4
    return tokens >= nct and tokens - mb * bst >= nct


def _engine(epp, p, seed, k, prefill=None, nct=0):
    kw = dict(tie_seed=seed, pick_k=k)
    if prefill is not None:
        kw.update(prefill=_spec(epp, prefill), non_cached_tokens=nct)
    eng = epp.Engine(E, _spec(epp, p), **kw)
    eng.latency_profile_set(0, **_lat_kwargs(epp, p["lcfg"]))
    if prefill is not None:
        eng.latency_profile_set(1, **_lat_kwargs(epp, prefill["lcfg"]))
    return eng


@pytest.mark.parametrize("prof", list(PROFILES))
@pytest.mark.parametrize("seed", [0, 0x5EED])
@pytest.mark.parametrize("k", [1, 4, 64])
def test_with_match_landscapes(epp, orc, prof, seed, k):
    p = PROFILES[prof]
    role, kv, waiting, running = pool(7)
    with _engine(epp, p, seed, k) as eng:
        set_pool(eng, role, kv, waiting, running)
        base = 0
        for li, name in enumerate(LANDSCAPES):
            match, total, preds = landscape(name, 24, 100 + li)
            out = eng.schedule_with_match(match, total, topk=k > 1, predictions=_pred_lists(preds))
            dec, det = out[0], out[1]
            lists = out[2] if k > 1 else None
            _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, lists, seed, k, base)
            base += 24


def test_composite_max_q_zero(epp, orc):
    p = PROFILES["scorer_only_random"]
    role, kv, _, running = pool(8)
    waiting = np.zeros(E, np.int64)
    with _engine(epp, p, 0x77, 64) as eng:
        set_pool(eng, role, kv, waiting, running)
        match, total, preds = landscape("none_idle", 8, 5)
        dec, det, lists = eng.schedule_with_match(match, total, topk=True)          # no predictions at all
        _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, lists, 0x77, 64)


def test_set_of_one_after_a1(epp, orc):
    p = CHART
    role, kv, waiting, running = pool(9)
    match = np.zeros((4, E), np.int32)
    total = np.full(4, 10, np.int32)
    match[:, 5] = 10                                            # the one sticky endpoint for 0.99
    match[:, 6:12] = 9
    preds = [{e: lm.Info(10.0, -5.0 if e == 5 else 5.0, 1.0, 1) for e in range(E)} for _ in range(4)]
    with _engine(epp, p, 0, 64) as eng:
        set_pool(eng, role, kv, waiting, running)
        dec, det, lists = eng.schedule_with_match(match, total, topk=True, predictions=_pred_lists(preds))
        _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, lists, 0, 64)
        assert all(d["pick"] == 5 and d["tie_count"] == 1 for d in dec)


def test_pd_latency_decode_default_prefill(epp, orc):
    p = PROFILES["mixed_scorers"]
    pre = dict(scorers=[(QUEUE, 2.0, 0.0), (KV, 2.0, 0.0), (PREFIX, 3.0, 0.0)], picker=0, a2=None, lcfg={})
    pre_lat = dict(PROFILES["tier_only"])
    role, kv, waiting, running = pool(10)
    for prefill in (pre, pre_lat):
        with _engine(epp, p, 0x99, 1, prefill=prefill, nct=8) as eng:
            set_pool(eng, role, kv, waiting, running)
            match, total, preds = landscape("mixed", 32, 11)
            in_len = np.random.default_rng(3).integers(0, 2000, 32).astype(np.int64)
            dec, det = eng.schedule_with_match(match, total, input_len_bytes=in_len, predictions=_pred_lists(preds))
            _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, None, 0x99, 1, pre=prefill, nct=8,
                   in_len=in_len)


@pytest.mark.parametrize("device", [False, True])
def test_schedule_paths(epp, orc, device):
    """The hash + dense-counter path (k_match_pick_lat): an empty index, so every match is 0 and total = the blocks."""
    import torch
    p = PROFILES["chart"]
    role, kv, waiting, running = pool(12)
    R = 40
    rng = np.random.default_rng(4)
    lens = rng.integers(0, 700, R)
    offs = np.zeros(R + 1, np.uint64)
    offs[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(offs[-1]) or 1).astype(np.uint8)
    _, _, preds = landscape("mixed", R, 13)
    with _engine(epp, p, 0x1234, 64) as eng:
        eng.register_model(b"m")
        set_pool(eng, role, kv, waiting, running)
        if device:
            dec, det, lists = eng.schedule(torch.from_numpy(data).cuda(), offsets=torch.from_numpy(offs.astype(np.int64)).cuda(),
                                           topk=True, predictions=_pred_lists(preds))
            torch.cuda.synchronize()
            dec = np.frombuffer(dec.cpu().numpy().tobytes(), dtype=epp.DECISION_DTYPE)[:R]
            det = np.frombuffer(det.cpu().numpy().tobytes(), dtype=epp.DETAIL_DTYPE)[:R]
            lists = {k2: v.cpu().numpy().view(np.uint32 if k2 != "primary_scores" else np.float64) for k2, v in lists.items()}
        else:
            dec, det, lists = eng.schedule(data, offsets=offs, topk=True, predictions=_pred_lists(preds))
        total = dec["total_blocks"].astype(np.int32)
        match = np.zeros((R, E), np.int32)
        _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, lists, 0x1234, 64)


def test_plain_schedule_is_no_predictions(epp, orc):
    p = CHART
    role, kv, waiting, running = pool(14)
    match, total, preds = landscape("mixed", 16, 15)
    with _engine(epp, p, 0x42, 1) as eng:
        set_pool(eng, role, kv, waiting, running)
        dec, det = eng.schedule_with_match(match, total)
        _check(orc, p, role, kv, waiting, running, match, total, [None] * 16, dec, det, None, 0x42, 1)


def test_rejections_change_nothing(epp, orc):
    p = CHART
    role, kv, waiting, running = pool(16)
    match, total, preds = landscape("mixed", 8, 17)
    good = _pred_lists(preds)
    with _engine(epp, p, 0x42, 1) as eng:
        set_pool(eng, role, kv, waiting, running)
        bad_slot = [list(x) for x in good]
        bad_slot[3] = bad_slot[3] + [(E, 1.0, 1.0, 1.0, 0)]
        bad_nan = [list(x) for x in good]
        bad_nan[2] = [(0, float("nan"), 1.0, 1.0, 0)]
        bad_inf = [list(x) for x in good]
        bad_inf[1] = [(0, 1.0, float("inf"), 1.0, 0)]
        for bad in (bad_slot, bad_nan, bad_inf):
            with pytest.raises(epp.EngineError):
                eng.schedule_with_match(match, total, predictions=bad)
        # not ascending / wrong struct_size through the raw ABI
        import ctypes as C
        counts, offs, ent = epp.pack_predictions(good)
        ent2 = ent.copy()
        o = int(offs[0])
        ent2[o], ent2[o + 1] = ent[o + 1], ent[o]
        for arr, size in ((ent2, C.sizeof(epp.capi.Predictions)), (ent, 8)):
            pr = epp.capi.Predictions()
            pr.struct_size = size
            pr.counts, pr.offsets, pr.entries = counts.ctypes.data, offs.ctypes.data, arr.ctypes.data
            d = np.zeros(8, epp.DECISION_DTYPE)
            rc = eng._lib.epp_schedule_with_match_predicted(eng._h, 8, match.ctypes.data, total.ctypes.data, None, None, 0,
                                                            d.ctypes.data, None, 0, None, C.byref(pr))
            assert rc == epp.capi.EPP_ERR_INVALID
        with pytest.raises(epp.EngineError):           # subsets on a latency engine
            eng.schedule(np.zeros(64, np.uint8), uniform_len=8, subsets=[None] * 7 + [[1, 2]])
        for si in (-1, 0):                             # epp_score of a latency profile / the latency scorer
            out = np.zeros((8, E), np.float64)
            rc = eng._lib.epp_score(eng._h, 8, match.ctypes.data, total.ctypes.data, None, 0, si, out.ctypes.data, 0)
            assert rc == epp.capi.EPP_ERR_INVALID
        assert eng.stats()["n_decisions"] == 0
        dec, det = eng.schedule_with_match(match, total, predictions=good)      # ordinals start at 0: nothing advanced
        _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, None, 0x42, 1)
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0)])) as eng:
        set_pool(eng, role, kv, waiting, running)
        with pytest.raises(epp.EngineError):
            eng.schedule_with_match(match, total, predictions=good)


def test_config_rejections(epp):
    with pytest.raises(epp.EngineError):           # no-hit-lru on a latency profile
        epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(LAT, 1.0), epp.ScorerSpec(9, 1.0)]))
    with pytest.raises(epp.EngineError):           # ttft_column >= 0 on a latency profile
        epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(LAT, 1.0)], epp.AffinityFilterSpec(0.8, 0.0, 1.0, 0)), n_ext_cols=1)
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0)])) as eng:
        for bad in (dict(a1_affinity_threshold=0.9), dict(tier_filter=1, epsilon_explore_neg=1.5),
                    dict(tier_filter=1, strategy=7), dict(tier_filter=2)):
            with pytest.raises(epp.EngineError):
                eng.latency_profile_set(0, **bad)
        eng.latency_profile_set(0, tier_filter=1)
        set_pool(eng, np.zeros(E, np.uint8), np.zeros(E), np.zeros(E), np.zeros(E))
        with pytest.raises(epp.EngineError):           # fixed once the pool is set
            eng.latency_profile_set(0, tier_filter=0)


# ---- role and label filters ahead of the chain, and a LoRA scorer mixed with the latency scorer ---------------------
def test_labels_role_and_lora(epp, orc):
    LORA = 8
    p = dict(scorers=[(LAT, 1.0, 0.0), (LORA, 1.0, 0.0), (QUEUE, 1.0, 0.0)], picker=0, a2=(0.8, 0.2, 5000.0),
             lcfg=dict(tier_filter=1, epsilon_explore_neg=0.4, a1_affinity_threshold=0.99, a1_exploration_probability=0.2))
    role, kv, waiting, running = pool(20)
    rng = np.random.default_rng(21)
    role = np.where(role == 0xFF, role, rng.choice([0, 1, 2, 3], E)).astype(np.uint8)    # decode filter drops prefill
    zone = rng.choice(["a", "b"], E)
    keep = zone == "a"
    max_active = np.full(E, 2, np.int32)
    loaded = rng.integers(0, 3, E).astype(np.int32)
    state = rng.choice([0, 1, 2], E, p=[0.6, 0.2, 0.2]).astype(np.uint8)
    spec = _spec(epp, p)
    spec.filter = epp.capi.FILTER_DECODE
    spec.labels = [("zone", epp.capi.LABEL_IN, ["a"])]
    eng = epp.Engine(E, spec, tie_seed=0x51, pick_k=64)
    eng.latency_profile_set(0, **_lat_kwargs(epp, p["lcfg"]))
    with eng:
        eng.register_model(b"base")
        eng.register_model(b"adapter")
        set_pool(eng, role, kv, waiting, running)
        ids = np.flatnonzero(role != 0xFF).astype(np.uint32)
        eng.pool_set_labels(ids, [{"zone": str(zone[i])} for i in ids])
        eng.pool_set_lora(ids, max_active[ids], loaded[ids], [(int(e), 1, int(state[e])) for e in ids if state[e]])
        match, total, preds = landscape("mixed", 24, 22)
        mids = np.ones(24, np.uint32)
        dec, det, lists = eng.schedule_with_match(match, total, topk=True, model_ids=mids, predictions=_pred_lists(preds))
    for r in range(24):
        m = lm.profile_decide(orc, epp.capi.FILTER_DECODE, p["scorers"], 0, role, kv, waiting, running, match[r],
                              int(total[r]), preds[r], p["lcfg"], p["a2"], 0x51, 4 * r, 64, keep=keep,
                              lora=(state, max_active, loaded))
        assert dec[r]["pick"] == m["picks"][0] and dec[r]["tie_count"] == m["ties"], r
        n = len(m["picks"])
        assert list(lists["primary"][r, :n]) == m["picks"], r
        assert lists["primary_scores"][r, :n].tobytes() == np.asarray(m["scores"], np.float64).tobytes(), r


# ---- the reference's plugin cases through the engine ----------------------------------------------------------------
REF_SCORER_CASES = {       # scorer/latency/plugin_test.go: (kv, queue, running, (ttft_headroom, tpot_headroom, ttft, dispatched))
    "positive_headroom": [(0.3, 0, 5, (100, 20, 50, 0)), (0.5, 0, 8, (30, 5, 120, 0))],
    "negative_only": [(0.5, 0, 5, (-10, -5, 110, 0)), (0.6, 0, 8, (-100, -30, 200, 0))],
    "tier_split": [(0.3, 0, 5, (10, 2, 90, 0)), (0.5, 0, 8, (50, 10, 50, 0))],
    "idle_pod_preference": [(0.5, 0, 5, (-50, -10, 150, 5)), (0.5, 0, 0, (-50, -10, 150, 0))],
    "hierarchical_buckets": [(0.5, 0, 5, (-50, -10, 150, 0)), (0.4, 0, 3, (-30, 5, 130, 0)), (0.6, 0, 4, (10, -8, 90, 0))],
    "composite_fallback": [(0.2, 0, 3, None), (0.8, 5, 10, None)],
}


@pytest.mark.parametrize("case", list(REF_SCORER_CASES))
def test_reference_scorer_cases(epp, orc, case):
    eps = REF_SCORER_CASES[case]
    n = len(eps)
    p = dict(scorers=[(LAT, 1.0, 0.0)], picker=0, a2=None, lcfg={})
    role = np.full(E, 0xFF, np.uint8)
    role[:n] = 0
    kv = np.zeros(E)
    waiting = np.zeros(E, np.int64)
    running = np.zeros(E, np.int64)
    for i, (k, q, rr, _) in enumerate(eps):
        kv[i], waiting[i], running[i] = k, q, rr
    preds = [{i: lm.Info(e[3][2], e[3][0], e[3][1], e[3][3]) for i, e in enumerate(eps) if e[3] is not None} or None]
    match = np.zeros((1, E), np.int32)
    total = np.zeros(1, np.int32)
    with _engine(epp, p, 0, 64) as eng:
        set_pool(eng, role, kv, waiting, running)
        dec, det, lists = eng.schedule_with_match(match, total, topk=True, predictions=_pred_lists(preds))
    _check(orc, p, role, kv, waiting, running, match, total, preds, dec, det, lists, 0, 64)


# ---- rows past the first chunk: chunked host batches and pipelined device batches (LatView.r0 != 0) ---------------
def test_chunked_host_batch(epp, orc):
    p = PROFILES["mixed_scorers"]
    role, kv, waiting, running = pool(30)
    R, L = 4, 20 << 20                        # 20 MiB prompts: one request per 48 MiB chunk
    data = np.zeros(R * L, np.uint8)
    for r in range(R):
        data[r * L:r * L + 64 * (r + 1)] = r + 1
    _, _, preds = landscape("mixed", R, 31)
    with _engine(epp, p, 0x31, 64) as eng:
        eng.register_model(b"m")
        set_pool(eng, role, kv, waiting, running)
        dec, det, lists = eng.schedule(data, uniform_len=L, topk=True, predictions=_pred_lists(preds))
    match = np.zeros((R, E), np.int32)
    _check(orc, p, role, kv, waiting, running, match, dec["total_blocks"].astype(np.int32), preds, dec, det, lists, 0x31, 64)


def test_pipelined_device_batch(epp, orc):
    import torch
    p = PROFILES["mixed_scorers"]
    role, kv, waiting, running = pool(32)
    R, L = 8192, 64
    rng = np.random.default_rng(33)
    data = rng.integers(0, 256, R * L).astype(np.uint8)
    _, _, preds = landscape("mixed", R, 34)
    with _engine(epp, p, 0x33, 1) as eng:
        eng.register_model(b"m")
        set_pool(eng, role, kv, waiting, running)
        out, _ = eng.schedule(torch.from_numpy(data).cuda(), uniform_len=L, asynchronous=True, detail=False,
                              predictions=_pred_lists(preds))
        eng.synchronize()
        dec = np.frombuffer(out.cpu().numpy().tobytes(), dtype=epp.DECISION_DTYPE)[:R]
    match = np.zeros((R, E), np.int32)
    total = dec["total_blocks"].astype(np.int32)
    for r in range(0, R, 97):                 # rows of both chunks
        m = lm.profile_decide(orc, 0, p["scorers"], 0, role, kv, waiting, running, match[r], int(total[r]), preds[r],
                              p["lcfg"], p["a2"], 0x33, 4 * r, 1)
        assert dec[r]["pick"] == m["picks"][0], r
        assert np.float64(dec[r]["score"]).tobytes() == np.float64(m["scores"][0]).tobytes(), r
        assert dec[r]["tie_count"] == m["ties"], r


# ---- the batcher from many threads, different predictions per request -----------------------------------------------
def test_batcher_threads(epp, orc):
    import threading
    p = CHART
    role, kv, waiting, running = pool(40)
    R = 256
    _, _, preds = landscape("mixed", R, 41)
    prompts = [bytes([r % 251]) * (16 + r) for r in range(R)]
    out = [None] * R
    with _engine(epp, p, 0, 1) as eng:
        eng.register_model(b"m")
        set_pool(eng, role, kv, waiting, running)
        b = epp.Batcher(eng, max_batch=64, max_delay_us=300)
        try:
            def worker(t):
                for r in range(t, R, 16):
                    tk = b.submit(prompts[r], predictions=_pred_lists([preds[r]])[0])
                    out[r] = b.wait(tk)[0]
            th = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            # no state change from refused submits; a subset on a latency engine is refused at submit time
            with pytest.raises(epp.EngineError):
                b.submit(prompts[0], subset=[1, 2])
            with pytest.raises(epp.EngineError):
                b.submit(prompts[0], predictions=[(1, 1.0, 1.0, 1.0, 0), (1, 2.0, 1.0, 1.0, 0)])
            with pytest.raises(epp.EngineError):
                b.submit(prompts[0], predictions=[(E, 1.0, 1.0, 1.0, 0)])
            with pytest.raises(epp.EngineError):
                b.submit(prompts[0], predictions=[(0, float("nan"), 1.0, 1.0, 0)])
            with pytest.raises(epp.EngineError):
                b.submit(prompts[0], predictions=[(i, 1.0, 1.0, 1.0, 0) for i in range(1025)])
            plain = b.wait(b.submit(prompts[0]))[0]     # a plain request next to the refused ones is decided
            assert plain["status"] in (0, -1)
        finally:
            b.close()
    # the model needs each request's ordinal, which the batcher assigns in flush order: compare every request against
    # the model at the flush-independent parts (a seed-0 engine draws nothing in the chain; the picker draws depend on
    # the ordinal, so the pick must be a member of the model's final set and its score the model's score there)
    for r in range(R):
        m = lm.profile_decide(orc, 0, p["scorers"], 0, role, kv, waiting, running, np.zeros(E, np.int32),
                              int(out[r]["total_blocks"]), preds[r], p["lcfg"], p["a2"], 0, 0, E)
        assert out[r]["status"] == 0 and out[r]["tie_count"] == len(m["final"]), r
        assert int(out[r]["pick"]) in m["final"], r
        sc = dict(zip(m["picks"], m["scores"]))
        assert np.float64(out[r]["score"]).tobytes() == np.float64(sc[int(out[r]["pick"])]).tobytes(), r


def test_batcher_refuses_predictions_without_latency_profile(epp):
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0)])) as eng:
        eng.register_model(b"m")
        b = epp.Batcher(eng, max_batch=8, max_delay_us=100)
        try:
            with pytest.raises(epp.EngineError):
                b.submit(b"abc", predictions=[(0, 1.0, 1.0, 1.0, 0)])
        finally:
            b.close()


# ---- the Python plugin layer: the chart profile built from the factories ---------------------------------------------
def test_scheduler_chart_profile(epp, orc):
    pl = epp.plugins
    prof = pl.SchedulerProfile().WithFilters(
        pl.PrefixCacheAffinityFilter(0.99, 0.3), pl.SLOHeadroomTierFilterFactory("t", b'{"epsilonExploreNeg": 0.3}'),
        pl.PrefixCacheAffinityFilter(0.80, 0.3)) \
        .WithScorers(pl.NewWeightedScorer(pl.LatencyScorerFactory("ls", None), 1.0)) \
        .WithPicker(pl.NewWeightedRandomPicker())
    sched = pl.Scheduler(pl.SingleProfileHandler(), {"p": prof}, max_endpoints=E, tie_seed=0x77)
    try:
        rng = np.random.default_rng(50)
        eps = [pl.NewEndpoint(pl.EndpointMetadata(f"e{i}"), pl.Metrics(WaitingQueueSize=int(rng.integers(0, 5)),
                                                                        KVCacheUsagePercent=0.25)) for i in range(12)]
        preds = []
        for _ in range(6):
            preds.append({i: pl.NewLatencyPredictionInfo(True, True, float(rng.integers(-50, 50)),
                                                         float(rng.integers(-5, 5)), float(rng.integers(1, 300)), 5.0,
                                                         int(rng.integers(0, 2))) for i in range(12) if rng.random() < 0.8})
        res = sched.Schedule([pl.InferenceRequest(Prompt=b"x" * 64) for _ in range(6)], eps, predictions=preds)
        role = np.full(E, 0xFF, np.uint8)
        role[:12] = 0
        kv = np.zeros(E)
        kv[:12] = 0.25
        waiting = np.zeros(E, np.int64)
        waiting[:12] = [e.metrics.WaitingQueueSize for e in eps]
        lcfg = dict(tier_filter=1, epsilon_explore_neg=0.3, a1_affinity_threshold=0.99, a1_exploration_probability=0.01,
                    a1_max_ttft_penalty_ms=5000.0)
        lcfg["a1_exploration_probability"] = 0.3
        for r in range(6):
            info = {i: lm.Info(v.TTFT(), v.TTFTHeadroom(), v.TPOTHeadroom(), v.DispatchedRequestCount())
                    for i, v in preds[r].items()}
            m = lm.profile_decide(orc, 0, [(LAT, 1.0, 0.0)], 2, role, kv, waiting, np.zeros(E, np.int64),
                                  np.zeros(E, np.int32), 0, info, lcfg, (0.8, 0.3, 5000.0), 0x77, 4 * r, 1)
            assert res[r].ProfileResults["p"].TargetSlots == m["picks"], r
        # the attribute path: LatencyPredictionInfoKey on the endpoints, the same for every request
        for i, e in enumerate(eps):
            if i in preds[0]:
                e.Put(pl.LatencyPredictionInfoKey, preds[0][i])
        one = sched.Schedule(pl.InferenceRequest(Prompt=b"x" * 64), eps)
        info = {i: lm.Info(v.TTFT(), v.TTFTHeadroom(), v.TPOTHeadroom(), v.DispatchedRequestCount())
                for i, v in preds[0].items()}
        m = lm.profile_decide(orc, 0, [(LAT, 1.0, 0.0)], 2, role, kv, waiting, np.zeros(E, np.int64),
                              np.zeros(E, np.int32), 0, info, lcfg, (0.8, 0.3, 5000.0), 0x77, 4 * 6, 1)
        assert one.ProfileResults["p"].TargetSlots == m["picks"]
    finally:
        sched.engine.close()
