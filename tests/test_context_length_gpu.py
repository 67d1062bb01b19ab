"""The context-length-aware scorer and filter on the GPU (include/epp_engine.h "Context length") against
tools/context_length_model.py, bit for bit: status, pick, score bits, tie count, match_blocks, the prefill / encode fields
and the first-k lists with their scores, on the injected-match, host, device, async, subset and batcher paths."""
from __future__ import annotations

import threading

import numpy as np
import pytest

from tools import context_length_model as cm
from tools import latency_model as lm

pytestmark = pytest.mark.gpu

E = 48
NO = 0xFFFFFFFF
PB = 640                       # prompt bytes: 10 blocks of 16 tokens; default ctx = 160
CL, LAT, QUEUE, KV, PREFIX, RUNNING, NOHIT = 11, 10, 2, 1, 0, 5, 9
KEY = cm.DEFAULT_LABEL
VALUES = ["0-100", "100-200", "150-150", "160-160", "0-2048", " 0 - 2048 ", "+0-+10", "007-9", "161-5000", "0-159",
          "0-9223372036854775807", "0-9223372036854775808", "1-2-3", "", "10-5", "abc", "200-100000", "5000-9000"]


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def make_pool(seed, absent=4):
    rng = np.random.default_rng(seed)
    role = np.zeros(E, np.uint8)
    role[rng.choice(E, absent, replace=False)] = 0xFF
    return role, rng.choice([0.0, 0.25, 0.5, 0.75], E), rng.integers(0, 6, E), rng.integers(0, 6, E)


def make_labels(seed, key=KEY):
    """Per slot: None (no labels), {} (other labels only) or {key: value}."""
    rng = np.random.default_rng(seed)
    out = []
    for e in range(E):
        c = rng.integers(0, 10)
        out.append(None if c == 0 else {"other": "x"} if c == 1 else {key: VALUES[rng.integers(0, len(VALUES))], "z": "1"})
    return out


def ranges_of(labels, key=KEY):
    return [cm.endpoint_state(lb, key) for lb in labels]


def set_pool(eng, pool, labels=None):
    role, kv, waiting, running = pool
    ids = np.flatnonzero(role != 0xFF).astype(np.uint32)
    eng.pool_set(ids, role[ids], kv[ids], waiting[ids], running[ids])
    if labels is not None:
        all_ids = np.arange(E, dtype=np.uint32)
        eng.pool_set_labels(all_ids, labels)


def ctx_values(rng, R):
    """Row ctx in turn: the default (-1), the edges of the label ranges, random."""
    edges = [0, 1, 9, 10, 11, 99, 100, 101, 149, 150, 151, 159, 160, 161, 199, 200, 201, 2047, 2048, 2049, 4999, 5000, 5001,
             9000, 9001, 100000, 100001, (1 << 62)]
    return np.array([-1 if r % 5 == 0 else edges[r % len(edges)] if r % 3 else int(rng.integers(0, 12000))
                     for r in range(R)], np.int64)


def landscape(R, seed):
    rng = np.random.default_rng(seed)
    match = np.zeros((R, E), np.int32)
    for r in range(R):
        sticky = rng.choice(E, 6, replace=False)
        match[r, sticky[:3]] = 10
        match[r, sticky[3:]] = 9
        match[r, rng.choice(E, 6)] = rng.integers(1, 8, 6)
    return match


PROFILES = {
    "score_only": dict(scorers=[(QUEUE, 2.0, 0.0), (KV, 2.0, 0.0), (PREFIX, 3.0, 0.0), (CL, 1.5, 0.0)], picker=0, a2=None,
                       filt=False, lcfg=None),
    "filter_affinity": dict(scorers=[(CL, 1.0, 0.0), (QUEUE, 1.0, 0.0), (RUNNING, 1.0, 0.0)], picker=0,
                            a2=(0.80, 0.3, 5000.0), filt=True, lcfg=None),
    "filter_random": dict(scorers=[(CL, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=1, a2=None, filt=True, lcfg=None),
    "filter_weighted": dict(scorers=[(QUEUE, 1.0, 0.0), (CL, 2.0, 0.0)], picker=2, a2=None, filt=True, lcfg=None),
    "with_latency": dict(scorers=[(CL, 1.0, 0.0), (LAT, 1.0, 0.0), (KV, 0.5, 0.0)], picker=0, a2=(0.80, 0.2, 100.0),
                         filt=True, lcfg=dict(tier_filter=1, epsilon_explore_neg=0.5)),
}


def _spec(epp, p, label=None):
    aff = None if p["a2"] is None else epp.AffinityFilterSpec(*p["a2"])
    cl = dict(label=label, enable_filtering=p["filt"])
    return epp.ProfileSpec(0, [epp.ScorerSpec(k, w, pa) for k, w, pa in p["scorers"]], aff, p["picker"], latency=p["lcfg"],
                           context_length=cl)


def engine(epp, p, seed, k, prefill=None, encode=None, nct=0, labels=(None, None, None), **kw):
    kw.update(tie_seed=seed, pick_k=k, block_size_tokens=16, max_prefix_blocks=16)
    if prefill is not None:
        kw.update(prefill=_spec(epp, prefill, labels[1]), non_cached_tokens=nct)
    if encode is not None:
        kw.update(encode=_spec(epp, encode, labels[2]))
    eng = epp.Engine(E, _spec(epp, p, labels[0]), **kw)
    eng.register_model(b"m")
    return eng


def decide(orc, p, pool, match_r, total, ranges, ctx, seed, key, k, info=None, keep=None):
    role, kv, waiting, running = pool
    return cm.profile_decide(orc, 0, p["scorers"], p["picker"], role, kv, waiting, running, match_r, total, ranges, ctx,
                             p["filt"], info, p["lcfg"], p["a2"], seed, key, k, keep=keep)


def check(orc, p, pool, match, total, ranges, ctx, dec, det, lists, seed, k, base=0, keeps=None, preds=None, pre=None,
          enc=None, mm=None, nct=0, in_len=PB):
    for r in range(match.shape[0]):
        key = 4 * (base + r)
        keep = None if keeps is None else keeps[r]
        info = None if preds is None else preds[r]
        m = decide(orc, p, pool, match[r], int(total[r]), ranges[0], int(ctx[r]), seed, key, k, info, keep)
        ok = bool(m["picks"])
        assert dec[r]["status"] == (0 if ok else -1), r
        assert dec[r]["tie_count"] == (m["ties"] if ok else 0), r
        if lists is not None:
            n = len(m["picks"])
            assert list(lists["primary"][r, :n]) == m["picks"], r
            assert lists["primary_scores"][r, :n].tobytes() == np.asarray(m["scores"], np.float64).tobytes(), r
            assert all(x == NO for x in lists["primary"][r, n:]), r
        if not ok:
            continue
        assert dec[r]["pick"] == m["picks"][0], (r, m["final"])
        assert np.float64(dec[r]["score"]).tobytes() == np.float64(m["scores"][0]).tobytes(), r
        assert dec[r]["match_blocks"] == match[r, m["picks"][0]], r
        for q, pi, ran, pick, score, ties in ((enc, 2, "encode_ran", "encode_pick", "encode_score", "encode_tie_count"),
                                              (pre, 1, "prefill_ran", "prefill_pick", "prefill_score", "prefill_tie_count")):
            if q is None:
                continue
            go = bool(mm[r]) if pi == 2 else (in_len // 4 >= nct and in_len // 4 - int(match[r, m["picks"][0]]) * 16 >= nct)
            assert det[r][ran] == int(go), (r, ran)
            if not go:
                continue
            qm = decide(orc, q, pool, match[r], int(total[r]), ranges[pi], int(ctx[r]), seed, key + pi, 1, info, keep)
            got = dec[r]["prefill_pick"] if pi == 1 else det[r]["encode_pick"]
            assert got == (qm["picks"][0] if qm["picks"] else NO), (r, ran)
            if qm["picks"]:
                assert np.float64(det[r][score]).tobytes() == np.float64(qm["scores"][0]).tobytes(), (r, ran)
                assert det[r][ties] == qm["ties"], (r, ran)


def resolved(ctx, in_len=PB):
    return np.array([c if c >= 0 else cm.default_ctx(in_len) for c in ctx], np.int64)


def load(eng, match, seed):
    """Prompts [R][PB] whose whole-pool match counts are `match`, with the index that gives them."""
    R = match.shape[0]
    prompts = np.random.default_rng(seed).integers(0, 256, (R, PB)).astype(np.uint8)
    h, nb = eng.hash_prompts(prompts, uniform_len=PB)
    rs, es = np.nonzero(match)
    hs = np.concatenate([h[r, :match[r, e]] for r, e in zip(rs, es)]) if rs.size else np.zeros(0, np.uint64)
    eps = np.concatenate([np.full(match[r, e], e, np.uint32) for r, e in zip(rs, es)]) if rs.size else np.zeros(0, np.uint32)
    eng.index_load_snapshot(hs, eps)
    got, total = eng.prefix_match(prompts, uniform_len=PB)
    assert (got == match).all() and (total == 10).all()
    return prompts


@pytest.mark.parametrize("prof", list(PROFILES))
@pytest.mark.parametrize("seed", [0, 0x5EED])
@pytest.mark.parametrize("k", [1, 4])
def test_with_match(epp, orc, prof, seed, k):
    p = PROFILES[prof]
    pool = make_pool(7)
    labels = make_labels(11)
    rng = np.random.default_rng(seed + k)
    R = 96
    match = landscape(R, 5)
    total = np.full(R, 10, np.int32)
    ctx = ctx_values(rng, R)
    in_len = np.full(R, PB, np.int64)
    with engine(epp, p, seed, k) as eng:
        set_pool(eng, pool, labels)
        out = eng.schedule_with_match(match, total, input_len_bytes=in_len, topk=k > 1, context_tokens=ctx)
        check(orc, p, pool, match, total, [ranges_of(labels)], resolved(ctx), out[0], out[1], out[2] if k > 1 else None,
              seed, k)


@pytest.mark.parametrize("kind", ["host", "device", "async"])
@pytest.mark.parametrize("prof", ["filter_affinity", "filter_weighted", "with_latency"])
def test_batch_kinds_and_subsets(epp, orc, kind, prof):
    import torch
    p = PROFILES[prof]
    pool = make_pool(3)
    labels = make_labels(23)
    rng = np.random.default_rng(9)
    R = 64
    match = landscape(R, 8)
    ctx = ctx_values(rng, R)
    subsets = [None if r % 4 else sorted(rng.choice(E, 20, replace=False).tolist()) for r in range(R)]
    keeps = [None if s is None else np.isin(np.arange(E), s) for s in subsets]
    preds = None
    if p["lcfg"]:
        preds = [{e: lm.Info(float(rng.integers(1, 400)), float(rng.integers(-50, 150)), float(rng.integers(-5, 20)), 0)
                  for e in range(E) if rng.random() < 0.5} for _ in range(R)]
    plist = None if preds is None else [[(e, i.ttft, i.ttft_headroom, i.tpot_headroom, i.dispatched) for e, i in d.items()]
                                        for d in preds]
    with engine(epp, p, 0x5EED, 4) as eng:
        set_pool(eng, pool, labels)
        prompts = load(eng, match, 4)
        data = prompts if kind == "host" else torch.from_numpy(prompts).cuda()
        dec, det, lists = eng.schedule(data, uniform_len=PB, topk=True, subsets=subsets, predictions=plist,
                                       context_tokens=ctx, asynchronous=kind == "async")
        if kind != "host":
            eng.synchronize()
            dec = epp.decisions_from_torch(dec)
            det = det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
            lists = {n: v.cpu().numpy().view(np.uint32 if n != "primary_scores" else np.float64) for n, v in lists.items()}
        check(orc, p, pool, match, np.full(R, 10), [ranges_of(labels)], resolved(ctx), dec, det, lists, 0x5EED, 4,
              keeps=keeps, preds=preds)


def test_default_ctx_is_quarter_length(epp, orc):
    """No token counts: ctx = int(float64(L) * 0.25) of input_len_bytes, the same decisions as explicit L // 4."""
    p = PROFILES["filter_affinity"]
    pool = make_pool(5)
    labels = make_labels(31)
    R = 64
    match = landscape(R, 12)
    total = np.full(R, 10, np.int32)
    in_len = np.random.default_rng(2).integers(0, 40000, R).astype(np.int64)
    in_len[:4] = [0, 3, 4, 642]
    with engine(epp, p, 0x5EED, 1) as a, engine(epp, p, 0x5EED, 1) as b:
        set_pool(a, pool, labels)
        set_pool(b, pool, labels)
        d1, _ = a.schedule_with_match(match, total, input_len_bytes=in_len)
        d2, _ = b.schedule_with_match(match, total, input_len_bytes=in_len, context_tokens=in_len // 4)
        assert d1.tobytes() == d2.tobytes()
        check(orc, p, pool, match, total, [ranges_of(labels)], in_len // 4, d1, None, None, 0x5EED, 1)


def test_filtered_extremes_and_empty_decode_set(epp, orc):
    """The endpoints the filter drops hold the pool's queue and running extremes; a request whose range matches no
    endpoint gets status -1 while its neighbours are decided."""
    p = dict(PROFILES["filter_affinity"], a2=None)
    role, kv, waiting, running = make_pool(1, absent=0)
    labels = [{KEY: "0-100"} if e % 2 else {KEY: "101-200"} for e in range(E)]
    waiting = np.where(np.arange(E) % 2 == 1, 1000 + np.arange(E), waiting)
    running = np.where(np.arange(E) % 2 == 1, 0, running + 50)
    pool = (role, kv, waiting, running)
    R = 6
    match = landscape(R, 3)
    total = np.full(R, 10, np.int32)
    ctx = np.array([50, 150, 300, 100, 101, 5000], np.int64)
    with engine(epp, p, 0, 1) as eng:
        set_pool(eng, pool, labels)
        dec, det = eng.schedule_with_match(match, total, input_len_bytes=np.full(R, PB, np.int64), context_tokens=ctx)
        assert list(dec["status"]) == [0, 0, -1, 0, 0, -1]
        check(orc, p, pool, match, total, [ranges_of(labels)], ctx, dec, det, None, 0, 1)


def test_pd_and_encode_with_different_labels(epp, orc):
    dec_p = PROFILES["filter_affinity"]
    pre_p = dict(PROFILES["score_only"])
    enc_p = dict(PROFILES["filter_random"])
    pool = make_pool(13)
    lab = make_labels(41)
    for e in range(E):                                     # a second range key read by the prefill and encode profiles
        lab[e] = dict(lab[e] or {}, **{"pd-range": VALUES[(e * 7) % len(VALUES)]})
    R = 64
    match = landscape(R, 14)
    rng = np.random.default_rng(4)
    ctx = ctx_values(rng, R)
    mm = (np.arange(R) % 3 == 0).astype(np.uint8)
    with engine(epp, dec_p, 0x5EED, 1, prefill=pre_p, encode=enc_p, nct=8,
                labels=(None, "pd-range", "pd-range")) as eng:
        set_pool(eng, pool, lab)
        prompts = load(eng, match, 6)
        dec, det = eng.schedule(prompts, uniform_len=PB, multimodal=mm, context_tokens=ctx)
        rg = ranges_of(lab, "pd-range")
        check(orc, dec_p, pool, match, np.full(R, 10), [ranges_of(lab), rg, rg], resolved(ctx), dec, det, None, 0x5EED, 1,
              pre=pre_p, enc=enc_p, mm=mm, nct=8)


def test_label_snapshots_between_async_batches(epp, orc):
    import torch
    p = PROFILES["filter_weighted"]
    pool = make_pool(17)
    la, lb = make_labels(51), make_labels(52)
    R = 48
    match = landscape(R, 19)
    ctx = ctx_values(np.random.default_rng(5), R)
    with engine(epp, p, 0x5EED, 1) as eng:
        set_pool(eng, pool, la)
        prompts = torch.from_numpy(load(eng, match, 7)).cuda()
        d1, _ = eng.schedule(prompts, uniform_len=PB, context_tokens=ctx, asynchronous=True)
        eng.pool_set_labels(np.arange(E, dtype=np.uint32), lb)
        d2, _ = eng.schedule(prompts, uniform_len=PB, context_tokens=ctx, asynchronous=True)
        eng.synchronize()
        for i, (d, lab) in enumerate(((d1, la), (d2, lb))):
            check(orc, p, pool, match, np.full(R, 10), [ranges_of(lab)], resolved(ctx), epp.decisions_from_torch(d), None,
                  None, 0x5EED, 1, base=i * R)


def test_batcher_submit_ctx(epp, orc):
    p = PROFILES["filter_affinity"]
    pool = make_pool(21)
    labels = make_labels(61)
    R = 64
    match = landscape(R, 22)
    ctx = ctx_values(np.random.default_rng(8), R)
    with engine(epp, p, 0, 1) as eng:
        set_pool(eng, pool, labels)
        prompts = load(eng, match, 9)
        got = {}
        with epp.Batcher(eng, max_batch=16, max_delay_us=100) as b:
            def worker(rows):
                for r in rows:
                    t = b.submit(prompts[r], subset=None if r % 7 else list(range(0, E, 2)), context_tokens=int(ctx[r]))
                    got[r] = b.wait(t)[0]
            ts = [threading.Thread(target=worker, args=(range(i, R, 8),)) for i in range(8)]
            for t in ts:
                t.start()
            for t in ts:
                t.join()
        rg = ranges_of(labels)
        rc = resolved(ctx)
        for r in range(R):
            keep = None if r % 7 else np.arange(E) % 2 == 0
            m = decide(orc, p, pool, match[r], 10, rg, int(rc[r]), 0, 0, 1, None, keep)
            d = got[r]
            assert d["status"] == (0 if m["picks"] else -1), r
            if m["picks"]:
                assert d["pick"] == m["picks"][0], r
                assert np.float64(d["score"]).tobytes() == np.float64(m["scores"][0]).tobytes(), r
                assert d["tie_count"] == m["ties"], r


def test_rejections(epp, orc):
    p = PROFILES["filter_affinity"]
    pool = make_pool(2)
    with pytest.raises(epp.EngineError):                   # two instances in one profile
        epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(CL, 1.0, 0.0), epp.ScorerSpec(CL, 1.0, 0.0)]))
    with pytest.raises(epp.EngineError):                   # no-hit-lru on the same profile
        epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(CL, 1.0, 0.0), epp.ScorerSpec(NOHIT, 1.0, 0.0)]))
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0, 0.0)])) as plain:
        with pytest.raises(epp.EngineError):               # the profile does not list the scorer
            plain.context_length_set(0, None, True)
    with engine(epp, p, 0, 1) as eng:
        with pytest.raises(epp.EngineError):
            eng.context_length_set(0, "", False)
        with pytest.raises(epp.EngineError):
            eng.shard_set(0, E // 2)
        set_pool(eng, pool, make_labels(3))
        with pytest.raises(epp.EngineError) as ei:         # fixed once the pool is set
            eng.context_length_set(0, None, False)
        assert ei.value.code == -5
        R = 8
        match = landscape(R, 1)
        total = np.full(R, 10, np.int32)
        for bad in (np.full(R, -2, np.int64), np.full(R - 1, 5, np.int64)):
            with pytest.raises((epp.EngineError, ValueError)):
                eng.schedule_with_match(match, total, context_tokens=bad)
        with pytest.raises(epp.EngineError):
            eng.score(match, total, 0, 0)                  # the scorer's index
        with pytest.raises(epp.EngineError):
            eng.score(match, total, 0, -1)                 # the weighted sum of its profile
        assert eng.stats()["n_decisions"] == 0             # nothing above changed an ordinal
        with epp.Batcher(eng, max_batch=4, max_delay_us=0) as b:
            with pytest.raises(epp.EngineError):
                b.submit(b"x" * 64, context_tokens=-2)
