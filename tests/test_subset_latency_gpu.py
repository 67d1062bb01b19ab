"""Endpoint subsets on a latency engine (epp_schedule_subset_predicted, epp_submit_subset_predicted; k_subset_pick_lat)
against tools/latency_model.py, bit for bit: status, pick, score bits, tie count, match_blocks, the prefill and encode
fields and the first-k lists.  A restricted request's expectation is profile_decide with keep = its subset and the
whole pool's match counts.  The index is built so that prompt r's first match[r][e] blocks are held by slot e (prompts of
10 blocks, no two sharing a block), so every landscape's match counts are real prefix matches walked by the kernel."""
from __future__ import annotations

import threading

import numpy as np
import pytest

import test_subset_latency_cpu as cases
from test_latency_profile_gpu import LANDSCAPES, PROFILES, _lat_kwargs, _pred_lists, _spec, landscape, lm_pd
from tools import latency_model as lm

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
PB = 640                       # prompt bytes: 10 blocks of 16 tokens
QUEUE, KV, PREFIX, LAT = 2, 1, 0, 10


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def make_pool(E, seed, absent=4):
    rng = np.random.default_rng(seed)
    role = np.zeros(E, np.uint8)
    role[rng.choice(E, absent, replace=False)] = 0xFF
    return role, rng.choice([0.0, 0.25, 0.5, 0.75], E), rng.integers(0, 6, E), rng.integers(0, 6, E)


def engine(epp, E, p, seed, k, prefill=None, nct=0, encode=None, **kw):
    kw.update(tie_seed=seed, pick_k=k, block_size_tokens=16, max_prefix_blocks=16)
    if prefill is not None:
        kw.update(prefill=_spec(epp, prefill), non_cached_tokens=nct)
    if encode is not None:
        kw.update(encode=_spec(epp, encode))
    eng = epp.Engine(E, _spec(epp, p), **kw)
    for pi, q in ((0, p), (1, prefill), (2, encode)):
        if q is not None and q.get("latency", True):
            eng.latency_profile_set(pi, **_lat_kwargs(epp, q["lcfg"]))
    eng.register_model(b"m")
    return eng


def set_pool(eng, role, kv, waiting, running):
    ids = np.flatnonzero(role != 0xFF).astype(np.uint32)
    eng.pool_set(ids, role[ids], kv[ids], waiting[ids], running[ids])


def load(eng, match, seed):
    """Prompts [R][PB] whose whole-pool match counts are `match`, with the index that gives them."""
    R, E = match.shape
    prompts = np.random.default_rng(seed).integers(0, 256, (R, PB)).astype(np.uint8)
    h, nb = eng.hash_prompts(prompts, uniform_len=PB)
    assert (nb == 10).all()
    rs, es = np.nonzero(match)
    hs = np.concatenate([h[r, :match[r, e]] for r, e in zip(rs, es)]) if rs.size else np.zeros(0, np.uint64)
    eps = np.concatenate([np.full(match[r, e], e, np.uint32) for r, e in zip(rs, es)]) if rs.size else np.zeros(0, np.uint32)
    eng.index_load_snapshot(hs, eps)
    got, total = eng.prefix_match(prompts, uniform_len=PB)
    assert (got == match).all() and (total == 10).all()
    return prompts


def keep_of(E, subset):
    k = np.zeros(E, bool)
    k[[e for e in subset if e < E]] = True
    return k


def check(orc, p, pool, match, preds, subsets, dec, det, lists, seed, k, base=0, rows=None, pre=None, nct=0, enc=None,
          mm=None):
    role, kv, waiting, running = pool
    E = match.shape[1]
    for r in (range(match.shape[0]) if rows is None else rows):
        key = 4 * (base + r)
        info = preds[r] or {}
        keep = None if subsets is None or subsets[r] is None else keep_of(E, subsets[r])
        m = lm.profile_decide(orc, 0, p["scorers"], p["picker"], role, kv, waiting, running, match[r], 10, info,
                              p["lcfg"], p["a2"], seed, key, k, keep=keep)
        ok = bool(m["picks"])
        where = (r, None if keep is None else len(subsets[r]))
        assert dec[r]["status"] == (0 if ok else -1), where
        assert dec[r]["tie_count"] == (m["ties"] if ok else 0), where
        assert int(dec[r]["total_blocks"]) == 10
        if lists is not None:
            n = len(m["picks"])
            assert list(lists["primary"][r, :n]) == m["picks"], where
            assert lists["primary_scores"][r, :n].tobytes() == np.asarray(m["scores"], np.float64).tobytes(), where
            assert all(x == NO for x in lists["primary"][r, n:]), where
        if not ok:
            continue
        assert dec[r]["pick"] == m["picks"][0], where
        assert keep is None or keep[m["picks"][0]]
        assert np.float64(dec[r]["score"]).tobytes() == np.float64(m["scores"][0]).tobytes(), where
        assert dec[r]["match_blocks"] == match[r, m["picks"][0]], where
        for q, pi, ran, pick, score, ties in ((enc, 2, "encode_ran", "encode_pick", "encode_score", "encode_tie_count"),
                                              (pre, 1, "prefill_ran", "prefill_pick", "prefill_score", "prefill_tie_count")):
            if q is None:
                continue
            go = (mm is not None and mm[r]) if pi == 2 else lm_pd(nct, PB, int(match[r, m["picks"][0]]))
            assert det[r][ran] == int(bool(go)), (where, ran)
            if not go:
                continue
            qm = lm.profile_decide(orc, 0, q["scorers"], q["picker"], role, kv, waiting, running, match[r], 10, info,
                                   q["lcfg"], q["a2"], seed, key + pi, 1, keep=keep)
            got = dec[r]["prefill_pick"] if pi == 1 else det[r]["encode_pick"]
            assert got == (qm["picks"][0] if qm["picks"] else NO), (where, ran)
            if qm["picks"]:
                assert np.float64(det[r][score]).tobytes() == np.float64(qm["scores"][0]).tobytes(), (where, ran)
                assert det[r][ties] == qm["ties"], (where, ran)


def shaped_subsets(rng, E, R, role):
    """Row shapes in turn: the whole pool (no subset), empty, 1, 31, 32, 33 slots, every slot, a random half."""
    out = []
    for r in range(R):
        c = r % 8
        if c == 0:
            out.append(None)
        elif c == 1:
            out.append([])
        elif c in (2, 3, 4, 5):
            n = (1, 31, 32, 33)[c - 2]
            out.append(sorted(rng.choice(E, min(n, E), replace=False).tolist()))
        elif c == 6:
            out.append(list(range(E)))
        else:
            out.append(sorted(rng.choice(E, E // 2, replace=False).tolist()))
    return out


def reshape_entries(rng, preds, subsets):
    """Every third restricted row keeps only the entries inside its list, every third only those outside it (disjoint);
    the others keep all (a superset of the list)."""
    out = []
    for r, (d, s) in enumerate(zip(preds, subsets)):
        if d is None or s is None or r % 3 == 0:
            out.append(d)
            continue
        inside = set(s)
        out.append({e: i for e, i in d.items() if (e in inside) == (r % 3 == 1)} or None)
    return out


def cpu_rows(E):
    """The landscapes of test_subset_latency_cpu.py as rows: (match [E], info, subset)."""
    assert E == cases.E
    return [(c["match"], c["info"], c["subset"]) for c in map(cases.case, cases.CASES) if c["waiting"] is None]


@pytest.mark.parametrize("prof", list(PROFILES))
@pytest.mark.parametrize("seed", [0, 0x5EED])
@pytest.mark.parametrize("k", [1, 4, 64])
def test_landscapes(epp, orc, prof, seed, k):
    p = PROFILES[prof]
    E = cases.E
    pool = cases.pool()
    rng = np.random.default_rng(k * 31 + seed)
    matches, preds, subsets = [], [], []
    for li, name in enumerate(LANDSCAPES):
        m, _, pr = landscape(name, 16, 100 + li)
        s = shaped_subsets(rng, E, 16, pool[0])
        matches.append(m)
        preds += reshape_entries(rng, pr, s)
        subsets += s
    for m, info, s in cpu_rows(E):
        matches.append(m[None])
        preds.append(info)
        subsets.append(s)
    match = np.concatenate(matches)
    with engine(epp, E, p, seed, k) as eng:
        set_pool(eng, *pool)
        prompts = load(eng, match, 3)
        out = eng.schedule(prompts, uniform_len=PB, topk=k > 1, subsets=subsets, predictions=_pred_lists(preds))
        check(orc, p, pool, match, preds, subsets, out[0], out[1], out[2] if k > 1 else None, seed, k)


def test_range_extreme_landscape(epp, orc):
    """test_subset_latency_cpu's range_extreme: the pool's queue extreme lies outside the subset."""
    c = cases.case("range_extreme")
    role, kv, _, running = cases.pool()
    pool = (role, kv, c["waiting"], running)
    p = dict(PROFILES["mixed_scorers"])
    with engine(epp, cases.E, p, 0x5EED, 4) as eng:
        set_pool(eng, *pool)
        match = np.repeat(c["match"][None], 4, 0)
        prompts = load(eng, match, 4)
        subsets = [None, c["subset"], c["subset"], None]
        preds = [c["info"], c["info"], None, None]
        dec, det, lists = eng.schedule(prompts, uniform_len=PB, topk=True, subsets=subsets, predictions=_pred_lists(preds))
        check(orc, p, pool, match, preds, subsets, dec, det, lists, 0x5EED, 4)


def random_rows(rng, E, R, sizes):
    match = np.zeros((R, E), np.int32)
    preds, subsets = [], []
    for r in range(R):
        sticky = rng.choice(E, 8, replace=False)
        match[r, sticky[:4]] = 10
        match[r, sticky[4:]] = rng.integers(5, 10, 4)
        n = sizes[r % len(sizes)]
        s = sorted(rng.choice(E, n, replace=False).tolist())
        if r % 2:
            s = sorted(set(s) | set(sticky[:2].tolist()))[:n] if n > 2 else s
        subsets.append(s)
        mode = r % 3                                   # entries: everywhere, inside the list only, outside it only
        inside = set(s)
        d = {}
        for e in range(E):
            if (mode == 1 and e not in inside) or (mode == 2 and e in inside) or rng.random() < 0.2:
                continue
            d[e] = lm.Info(float(rng.integers(1, 400)), float(rng.integers(-60, 120)), float(rng.integers(-10, 30)),
                           int(rng.integers(0, 3)))
        preds.append(d or None)
    return match, preds, subsets


@pytest.mark.parametrize("prof", ["chart", "mixed_scorers", "scorer_only_random"])
def test_long_lists(epp, orc, prof):
    """Lists of 1, 64, 65 and 1024 slots on a pool of 1100."""
    p = PROFILES[prof]
    E = 1100
    pool = make_pool(E, 8, absent=20)
    match, preds, subsets = random_rows(np.random.default_rng(9), E, 16, [1, 64, 65, 1024])
    with engine(epp, E, p, 0x5EED, 4) as eng:
        set_pool(eng, *pool)
        prompts = load(eng, match, 5)
        dec, det, lists = eng.schedule(prompts, uniform_len=PB, topk=True, subsets=subsets, predictions=_pred_lists(preds))
        check(orc, p, pool, match, preds, subsets, dec, det, lists, 0x5EED, 4)


@pytest.mark.parametrize("kind", ["device", "async", "pipelined"])
def test_batch_kinds(epp, orc, kind):
    import torch
    p = PROFILES["chart"]
    E = 48
    pool = make_pool(E, 11)
    R = 8192 + 96 if kind == "pipelined" else 200
    rng = np.random.default_rng(12)
    restricted = list(range(3, R, 37))
    match = np.zeros((R, E), np.int32)
    m, _, pr = landscape("mixed", len(restricted), 13)
    match[restricted] = m
    preds = [None] * R
    subsets = [None] * R
    for i, r in enumerate(restricted):
        preds[r] = pr[i]
        subsets[r] = sorted(rng.choice(E, (1, 31, 32, 33, 40)[i % 5], replace=False).tolist())
    for r in range(1, R, 53):                         # unrestricted rows with predictions
        if subsets[r] is None:
            preds[r] = pr[r % len(pr)]
    with engine(epp, E, p, 0x5EED, 4) as eng:
        set_pool(eng, *pool)
        prompts = load(eng, match, 14)
        data = torch.from_numpy(prompts.reshape(-1)).cuda()
        dec, det, lists = eng.schedule(data, uniform_len=PB, topk=True, subsets=subsets, predictions=_pred_lists(preds),
                                       asynchronous=kind != "device")
        eng.synchronize()
        torch.cuda.synchronize()
        dec = np.frombuffer(dec.cpu().numpy().tobytes(), dtype=epp.DECISION_DTYPE)[:R]
        det = np.frombuffer(det.cpu().numpy().tobytes(), dtype=epp.DETAIL_DTYPE)[:R]
        lists = {k2: v.cpu().numpy().view(np.uint32 if k2 != "primary_scores" else np.float64) for k2, v in lists.items()}
        assert eng.stats()["last_kernel_ms"][6] > 0
        rows = restricted + list(range(1, R, 53)) + list(range(0, R, 401))
        check(orc, p, pool, match, preds, subsets, dec, det, lists, 0x5EED, 4, rows=rows)


def test_pd_and_encode(epp, orc):
    """Decode latency profile, a latency or default prefill profile (the P/D decider at match 9 | 10 of 10 blocks with
    non_cached_tokens 8), and a latency encode profile for the multimodal rows."""
    p = PROFILES["mixed_scorers"]
    enc = dict(scorers=[(LAT, 1.0, 0.0), (KV, 1.0, 0.0)], picker=0, a2=None, lcfg=dict(tier_filter=1, epsilon_explore_neg=0.5))
    pre_default = dict(scorers=[(QUEUE, 2.0, 0.0), (KV, 2.0, 0.0), (PREFIX, 3.0, 0.0)], picker=0, a2=None, lcfg={},
                       latency=False)
    E = 48
    pool = make_pool(E, 15)
    rng = np.random.default_rng(16)
    for pre in (PROFILES["tier_only"], pre_default):
        match, _, preds = landscape("mixed", 64, 17)
        subsets = shaped_subsets(rng, E, 64, pool[0])
        mm = (np.arange(64) % 3 == 1).astype(np.uint8)
        with engine(epp, E, p, 0x99, 1, prefill=pre, nct=8, encode=enc) as eng:
            set_pool(eng, *pool)
            prompts = load(eng, match, 18)
            dec, det = eng.schedule(prompts, uniform_len=PB, multimodal=mm, subsets=subsets, predictions=_pred_lists(preds))
            check(orc, p, pool, match, preds, subsets, dec, det, None, 0x99, 1, pre=pre, nct=8, enc=enc, mm=mm)
            assert det["prefill_ran"].any() and not det["prefill_ran"].all()


def test_inflight_counts_subset_picks(epp, orc):
    p = PROFILES["chart"]
    E = 48
    pool = make_pool(E, 19)
    match, _, preds = landscape("mixed", 64, 20)
    subsets = shaped_subsets(np.random.default_rng(21), E, 64, pool[0])
    with engine(epp, E, p, 0x5EED, 1, inflight_load=True) as eng:
        set_pool(eng, *pool)
        prompts = load(eng, match, 22)
        dec, det = eng.schedule(prompts, uniform_len=PB, subsets=subsets, predictions=_pred_lists(preds))
        check(orc, p, pool, match, preds, subsets, dec, det, None, 0x5EED, 1)
        req, _ = eng.inflight_get()
        picks = dec["pick"][dec["status"] == 0].astype(np.int64)
        assert (req == np.bincount(picks, minlength=E)).all()


@pytest.mark.parametrize("prof", ["chart", "mixed_scorers", "scorer_only_random"])
def test_whole_pool_subset_is_no_subset(epp, orc, prof):
    """Every picker: a subset listing every slot decides bit for bit as no subset, first-k lists included."""
    p = PROFILES[prof]
    E = 48
    pool = make_pool(E, 23)
    match, _, preds = landscape("partial", 48, 24)
    outs = []
    for subsets in ([list(range(E))] * 48, None):
        with engine(epp, E, p, 0x5EED, 64) as eng:
            set_pool(eng, *pool)
            prompts = load(eng, match, 25)
            outs.append(eng.schedule(prompts, uniform_len=PB, topk=True, subsets=subsets, predictions=_pred_lists(preds)))
    (d1, t1, l1), (d2, t2, l2) = outs
    assert d1.tobytes() == d2.tobytes() and t1.tobytes() == t2.tobytes()
    for name in l1:
        assert np.asarray(l1[name]).tobytes() == np.asarray(l2[name]).tobytes(), name
    check(orc, p, pool, match, preds, None, d2, t2, l2, 0x5EED, 64)


def test_rejections_change_nothing(epp, orc):
    p = PROFILES["chart"]
    E = 48
    pool = make_pool(E, 26)
    match, _, preds = landscape("mixed", 8, 27)
    good = _pred_lists(preds)
    subsets = [None, [1, 2, 3], [], list(range(0, E, 2)), None, [5], [7, 9], None]
    with engine(epp, E, p, 0x42, 1) as eng:
        set_pool(eng, *pool)
        prompts = load(eng, match, 28)
        bad_pred = [list(x) for x in good]
        bad_pred[3] = bad_pred[3] + [(E, 1.0, 1.0, 1.0, 0)]
        bad_nan = [list(x) for x in good]
        bad_nan[6] = [(0, float("nan"), 1.0, 1.0, 0)]
        for s, pr in ((subsets, bad_pred), (subsets, bad_nan), (subsets[:5] + [[E]] + subsets[6:], good)):
            with pytest.raises(epp.EngineError):
                eng.schedule(prompts, uniform_len=PB, subsets=s, predictions=pr)
        with pytest.raises(epp.EngineError):           # the subset-only call still refuses a latency engine
            eng.schedule(prompts, uniform_len=PB, subsets=subsets)
        assert eng.stats()["n_decisions"] == 0
        dec, det = eng.schedule(prompts, uniform_len=PB, subsets=subsets, predictions=good)   # ordinals start at 0
        check(orc, p, pool, match, preds, subsets, dec, det, None, 0x42, 1)


def test_batcher(epp, orc):
    """16 threads mixing plain, predicted and subset-predicted submits, with refused submits beside them.  tie_seed 0
    and a max-score picker: a decision does not depend on the request's ordinal."""
    p = PROFILES["mixed_scorers"]
    E = 48
    pool = make_pool(E, 29)
    R = 256
    match, _, preds = landscape("mixed", R, 30)
    subsets = shaped_subsets(np.random.default_rng(31), E, R, pool[0])
    kinds = [r % 3 for r in range(R)]                   # 0 plain, 1 predicted, 2 subset + predicted
    eff_preds = [None if kinds[r] == 0 else preds[r] for r in range(R)]
    eff_sub = [subsets[r] if kinds[r] == 2 else None for r in range(R)]
    with engine(epp, E, p, 0, 1) as eng:
        set_pool(eng, *pool)
        prompts = load(eng, match, 32)
        plist = _pred_lists(eff_preds)
        out = [None] * R
        errs = []
        with epp.Batcher(eng, max_batch=32, max_delay_us=200) as b:
            def worker(t):
                try:
                    for r in range(t, R, 16):
                        if kinds[r] == 0:
                            tk = b.submit(prompts[r])
                        elif kinds[r] == 1:
                            tk = b.submit(prompts[r], predictions=plist[r] or [])
                        else:
                            tk = b.submit(prompts[r], subset=eff_sub[r], predictions=plist[r] or [])
                        out[r] = b.wait(tk)
                        for bad in ({"subset": [E]}, {"predictions": [(E, 1.0, 1.0, 1.0, 0)]}):
                            try:
                                b.submit(prompts[r], **dict(dict(subset=[1], predictions=[]), **bad))
                                errs.append(r)
                            except epp.EngineError:
                                pass
                except Exception as e:                  # surfaced below
                    errs.append(e)
            th = [threading.Thread(target=worker, args=(t,)) for t in range(16)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            with pytest.raises(epp.EngineError):        # the subset-only submit still refuses a latency engine
                b.submit(prompts[0], subset=[1, 2])
        assert not errs, errs[:3]
        dec = np.array([o[0] for o in out], dtype=epp.DECISION_DTYPE)
        det = np.array([o[1] for o in out], dtype=epp.DETAIL_DTYPE)
        check(orc, p, pool, match, eff_preds, eff_sub, dec, det, None, 0, 1)
