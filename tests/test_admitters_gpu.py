"""The latency-slo-admitter and probabilistic-admitter on the GPU (include/epp_engine.h "Admission") against
tools/admission_model.py, byte for byte.  Every call is made twice, on two engines with the same configuration and the
same history: one without admitters, one with them and the call's admission inputs.  The second must return the first's
rows with exactly the model's rejected rows rewritten, and its after-pick state (in-flight counters, no-hit-lru LRU,
indexed picks) must be what the admitted rows alone produce."""
from __future__ import annotations

import threading

import numpy as np
import pytest

from tools import admission_model as am

pytestmark = pytest.mark.gpu

E = 64
PB = 256
QUEUE, KV, PREFIX, NOHIT, LAT = 2, 1, 0, 9, 10


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def make_pool(seed, idle=False, cold=False, absent=6, neg_waiting=False):
    """Slot-indexed pool arrays.  Without idle / cold every present slot is busy (running > 0) and warm (kv >= 0.02)."""
    rng = np.random.default_rng(seed)
    present = np.ones(E, bool)
    present[rng.choice(E, absent, replace=False)] = False
    kv = rng.choice([0.05, 0.1, 0.2, 0.3, 0.5, 0.75], E)
    waiting = rng.integers(-2 if neg_waiting else 0, 8, E).astype(np.int32)
    running = rng.integers(1, 6, E).astype(np.int32)
    live = np.flatnonzero(present)
    if idle:
        running[live[3]] = 0
    if cold:
        kv[live[5]] = 0.01
    return dict(present=present, kv=kv, waiting=waiting, running=running)


def set_pool(eng, pool):
    eng.register_model(b"m")
    ids = np.flatnonzero(pool["present"]).astype(np.uint32)
    eng.pool_set(ids, np.zeros(ids.size, np.uint8), pool["kv"][ids], pool["waiting"][ids], pool["running"][ids])


def inputs(R, seed, pool, subsets=False, with_pred=True):
    """Per-request admission inputs over every landscape of the contract: priorities, SLOs (0, NaN, +Inf, > 0),
    predictions all valid / all invalid / single bits / absent / only on non-candidates, subsets (empty, outside the
    pool, small)."""
    rng = np.random.default_rng(seed)
    prio = rng.choice([-3, -1, -1, -1, 0, 2], R).astype(np.int32)
    slo_vals = [0.0, np.nan, np.inf, 50.0, 100.0, -1.0]
    ttft = np.array([slo_vals[i] for i in rng.integers(0, len(slo_vals), R)])
    tpot = np.array([slo_vals[i] for i in rng.integers(0, len(slo_vals), R)])
    absent = np.flatnonzero(~pool["present"])
    subs, preds, valid = [], [], []
    for r in range(R):
        sub = None
        if subsets:
            c = r % 6
            sub = None if c == 0 else [] if c == 1 else list(absent[:2]) if c == 2 else \
                sorted(rng.choice(E, int(rng.integers(1, 12)), replace=False).tolist())
        subs.append(sub)
        if not with_pred:
            continue
        kind = r % 5
        if kind == 0:
            preds.append(None)
            valid.append(None)
            continue
        slots = rng.choice(absent, min(2, absent.size), replace=False) if kind == 1 else \
            rng.choice(E, int(rng.integers(1, 10)), replace=False)
        v = {2: 3, 3: 0}.get(kind, None)
        bits = [v if v is not None else int(rng.integers(0, 4)) for _ in slots]
        preds.append([(int(s), 10.0, 1.0 - b, 1.0 - (b >> 1), 0) for s, b in zip(slots, bits)])
        valid.append(bits)
    return prio, ttft, tpot, (subs if subsets else None), (preds if with_pred else None), (valid if with_pred else None)


def pred_slots(preds):
    return None if preds is None else [None if p is None else [e[0] for e in p] for p in preds]


def engines(epp, acfg, lat=False, **kw):
    """(base, adm): the same engine configuration, the second with the admitters."""
    scorers = [epp.ScorerSpec(QUEUE, 2.0), epp.ScorerSpec(KV, 2.0), epp.ScorerSpec(PREFIX, 3.0)]
    if lat:
        scorers.append(epp.ScorerSpec(LAT, 1.0))
    prof = lambda: epp.ProfileSpec(0, list(scorers), latency=dict(tier_filter=1) if lat else None)   # noqa: E731
    out = []
    for with_adm in (False, True):
        eng = epp.Engine(E, prof(), **kw)
        if with_adm:
            eng.admission_set(**acfg)
        out.append(eng)
    return out


def acfg_of(latency_slo=True, probabilistic=True, **p):
    c = dict(latency_slo=latency_slo, probabilistic=probabilistic)
    c.update(p)
    return c


def model_cfg(acfg):
    c = dict(am.DEFAULTS)
    c.update({k: v for k, v in acfg.items() if k in am.DEFAULTS})
    c.update(latency_slo=acfg["latency_slo"], probabilistic=acfg["probabilistic"])
    return c


def check_band(acfg, pool, prio, subs, tie_seed, ord_base):
    """With a fractional power Exp / Log are not pinned: count the rows whose draw lies within 2^-40 of p."""
    if float(acfg.get("power", 5.0)).is_integer() or not acfg["probabilistic"]:
        return 0
    cfg = model_cfg(acfg)
    n = 0
    for r in range(len(prio)):
        if prio[r] >= 0:
            continue
        slots = np.flatnonzero(pool["present"]) if subs is None or subs[r] is None else \
            [s for s in sorted(set(subs[r])) if pool["present"][s]]
        if len(slots) == 0:
            continue
        eps = [am.Endpoint(int(pool["waiting"][s]), float(pool["kv"][s]), int(pool["running"][s])) for s in slots]
        p, u = am.probabilistic_p(eps, cfg), am.draw(tie_seed, ord_base + r)
        n += abs(u - p) <= 2.0 ** -40 * p
    return n


def assert_rows(got, want, what):
    for a, b, name in zip(got, want, ("decisions", "details", "first-k")):
        if b is None:
            continue
        if isinstance(b, dict):
            for k in b:
                assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), f"{what}: {k}"
        else:
            assert a.tobytes() == b.tobytes(), f"{what}: {name} differ"


POOLS = [dict(), dict(idle=True), dict(cold=True), dict(neg_waiting=True)]
THRESH = [dict(), dict(queue_depth_threshold=40, kv_cache_util_threshold=4.0, k=3.0),
          dict(queue_depth_threshold=1000, kv_cache_util_threshold=100.0), dict(power=2.5, k=1.0, queue_depth_threshold=20)]


@pytest.mark.parametrize("pi", range(len(POOLS)))
@pytest.mark.parametrize("ti", range(len(THRESH)))
@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
def test_injected_match_landscapes(epp, pi, ti, tie_seed):
    R = 400
    pool = make_pool(11 + pi, **POOLS[pi])
    acfg = acfg_of(**THRESH[ti])
    base, adm = engines(epp, acfg, lat=True, tie_seed=tie_seed)
    with base, adm:
        for e in (base, adm):
            set_pool(e, pool)
        rng = np.random.default_rng(pi * 7 + ti)
        for call in range(2):
            prio, ttft, tpot, _, preds, valid = inputs(R, 100 * ti + call, pool)
            match = rng.integers(0, 4, (R, E)).astype(np.int32)
            total = np.full(R, 8, np.int32)
            ord_base = base.stats()["n_decisions"]
            want = base.schedule_with_match(match, total, predictions=preds)
            got = adm.schedule_with_match(match, total, predictions=preds,
                                          admission=dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot, pred_valid=valid))
            rej = am.rejects(model_cfg(acfg), pool, prio, ttft, tpot, pred_slots(preds), valid, None, tie_seed, ord_base)
            assert check_band(acfg, pool, prio, None, tie_seed, ord_base) == 0
            assert_rows(got, am.apply(want[0], want[1], rej), f"pool {pi} thresholds {ti} call {call}")
            if ti == 0 and pi == 0:
                assert rej.any()


def batch_prompts(R, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 1 << 31, (R, PB // 4), dtype=np.int64).astype(np.uint32)


@pytest.mark.parametrize("path", ["host", "device", "async"])
@pytest.mark.parametrize("subsets", [False, True])
def test_schedule_paths(epp, path, subsets):
    import torch
    R = 8192 + 512 if path == "async" else 700
    pool = make_pool(5, neg_waiting=True)
    acfg = acfg_of(queue_depth_threshold=30, kv_cache_util_threshold=2.0, k=2.0)
    base, adm = engines(epp, acfg, inflight_load=True, tie_seed=3)
    with base, adm:
        for e in (base, adm):
            set_pool(e, pool)
        prio, ttft, tpot, subs, preds, valid = inputs(R, 9, pool, subsets=subsets)
        prompts = batch_prompts(R, 1)
        ad = dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot, pred_valid=valid)
        ord_base = base.stats()["n_decisions"]

        def run(eng, admission):
            kw = dict(uniform_len=PB, subsets=subs, predictions=preds if admission else None, admission=admission)
            if path == "host":
                return eng.schedule(prompts, **kw)
            data = torch.from_numpy(prompts.view(np.int32)).cuda()
            dec, det = eng.schedule(data, asynchronous=path == "async", **kw)
            eng.synchronize()
            torch.cuda.synchronize()
            return epp.decisions_from_torch(dec), det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)

        want = run(base, None)
        got = run(adm, ad)
        rej = am.rejects(model_cfg(acfg), pool, prio, ttft, tpot, pred_slots(preds), valid, subs, 3, ord_base)
        assert rej.any() and (~rej).any()
        assert_rows(got, am.apply(want[0], want[1], rej), f"{path} subsets={subsets}")
        st = adm.stats()
        if path != "host":
            assert st["last_kernel_ms"][7] > 0
        # in-flight counters: the admitted rows' adds only
        req, tok = adm.inflight_get()
        exp = np.zeros(E, np.int64)
        for r in np.flatnonzero(got[0]["status"] == 0):
            exp[got[0]["pick"][r]] += 1
        assert np.array_equal(np.asarray(req)[:E], exp)


def test_topk_nohit_and_index(epp):
    R = 500
    pool = make_pool(21, idle=False)
    acfg = acfg_of(latency_slo=False, queue_depth_threshold=30, kv_cache_util_threshold=2.0, k=2.0)
    base, adm = [epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0), epp.ScorerSpec(NOHIT, 1.0, 64.0)]),
                            pick_k=4, tie_seed=9) for _ in range(2)]
    adm.admission_set(**acfg)
    with base, adm:
        for e in (base, adm):
            set_pool(e, pool)
        prio, ttft, tpot, _, _, _ = inputs(R, 4, pool, with_pred=False)
        prompts = batch_prompts(R, 2)
        ord_base = base.stats()["n_decisions"]
        want = base.schedule(prompts, uniform_len=PB, topk=True, keep_hashes=True)
        got = adm.schedule(prompts, uniform_len=PB, topk=True, keep_hashes=True,
                           admission=dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot))
        rej = am.rejects(model_cfg(acfg), pool, prio, ttft, tpot, None, None, None, 9, ord_base)
        assert rej.any()
        assert_rows(got, am.apply(want[0], want[1], rej, want[2]), "top-k")
        # no-hit-lru: cold admitted picks only, in request order
        lru = adm.nohit_lru_get()
        order = []
        for r in np.flatnonzero(got[0]["status"] == 0):
            p = int(got[0]["pick"][r])
            if p in order:
                order.remove(p)
            order.append(p)
        assert list(lru) == order[-64:]
        # epp_index_add_picked indexes the admitted rows only
        adm.index_add_picked()
        hashes = adm.hash_prompts(prompts, uniform_len=PB)[0]
        for r in range(0, R, 37):
            got_eps = adm.index_get(int(hashes[r, 0]))
            assert got_eps == ({int(got[0]["pick"][r])} if got[0]["status"][r] == 0 else set())


def test_latency_slo_only_plain_engine_and_small_path(epp):
    R = 64
    pool = make_pool(31)
    acfg = acfg_of(probabilistic=False)
    base, adm = engines(epp, acfg)
    with base, adm:
        for e in (base, adm):
            set_pool(e, pool)
        prompts = batch_prompts(R, 3)
        # no sheddable row: the same single-launch small-batch path as without admission inputs
        base.schedule(prompts, uniform_len=PB)
        adm.schedule(prompts, uniform_len=PB, admission=dict(priority=np.zeros(R, np.int32)))
        assert adm.stats()["last_kernel_launches"] == base.stats()["last_kernel_launches"]
        prio, ttft, tpot, _, preds, valid = inputs(R, 8, pool)
        ord_base = base.stats()["n_decisions"]
        want = base.schedule(prompts, uniform_len=PB)
        got = adm.schedule(prompts, uniform_len=PB, predictions=preds,
                           admission=dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot, pred_valid=valid))
        rej = am.rejects(model_cfg(acfg), pool, prio, ttft, tpot, pred_slots(preds), valid, None, 0, ord_base)
        assert rej.any()
        assert_rows(got, am.apply(want[0], want[1], rej), "latency-slo only")
        # refusals: no pred_valid with predictions, a wrong struct (via an admitter-less engine); nothing moves
        n0 = adm.stats()["n_decisions"]
        with pytest.raises(epp.EngineError):
            adm.schedule(prompts, uniform_len=PB, predictions=preds, admission=dict(priority=prio))
        with pytest.raises(epp.EngineError):
            base.schedule(prompts, uniform_len=PB, admission=dict(priority=prio))
        with pytest.raises(epp.EngineError):
            adm.admission_set(probabilistic=True)                     # after the pool
        assert adm.stats()["n_decisions"] == n0
        want = base.schedule(prompts, uniform_len=PB)
        got = adm.schedule(prompts, uniform_len=PB, predictions=preds,
                           admission=dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot, pred_valid=valid))
        rej = am.rejects(model_cfg(acfg), pool, prio, ttft, tpot, pred_slots(preds), valid, None, 0, n0)
        assert_rows(got, am.apply(want[0], want[1], rej), "after refusals")


def test_config_refusals(epp):
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0)])) as eng:
        for bad in (dict(queue_depth_threshold=0), dict(kv_cache_util_threshold=0.0), dict(power=-1.0), dict(k=0.0),
                    dict(power=float("inf")), dict(k=float("nan"))):
            with pytest.raises(epp.EngineError):
                eng.admission_set(probabilistic=True, **bad)


def test_pd_encode(epp):
    R = 300
    pool = make_pool(41)
    acfg = acfg_of(queue_depth_threshold=30, kv_cache_util_threshold=2.0, k=2.0)
    mk = lambda: epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0)]),   # noqa: E731
                            epp.ProfileSpec(0, [epp.ScorerSpec(KV, 1.0)]), always_disagg=True,
                            encode=epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0)]), inflight_load=True)
    base, adm = mk(), mk()
    adm.admission_set(**acfg)
    with base, adm:
        for e in (base, adm):
            set_pool(e, pool)
        prio, ttft, tpot, _, preds, valid = inputs(R, 12, pool)
        prompts = batch_prompts(R, 4)
        mm = (np.arange(R) % 3 == 0).astype(np.uint8)
        ord_base = base.stats()["n_decisions"]
        want = base.schedule(prompts, uniform_len=PB, multimodal=mm)
        got = adm.schedule(prompts, uniform_len=PB, multimodal=mm, predictions=preds,
                           admission=dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot, pred_valid=valid))
        rej = am.rejects(model_cfg(acfg), pool, prio, ttft, tpot, pred_slots(preds), valid, None, 0, ord_base)
        assert rej.any()
        assert_rows(got, am.apply(want[0], want[1], rej), "P/D + encode")
        req, _ = adm.inflight_get()
        exp = np.zeros(E, np.int64)
        for r in np.flatnonzero(got[0]["status"] == 0):
            for p in (got[0]["pick"][r], got[0]["prefill_pick"][r], got[1]["encode_pick"][r]):
                if p != am.EPP_NO_ENDPOINT:
                    exp[p] += 1
        assert np.array_equal(np.asarray(req)[:E], exp)


def test_batcher_mixed_submits(epp):
    R = 96
    pool = make_pool(51)
    acfg = acfg_of(queue_depth_threshold=30, kv_cache_util_threshold=2.0, k=2.0)
    _, adm = engines(epp, acfg)
    with adm:
        set_pool(adm, pool)
        prio, ttft, tpot, _, preds, valid = inputs(R, 13, pool)
        prompts = batch_prompts(R, 5)
        b = epp.Batcher(adm, max_batch=R, max_delay_us=1000000)
        tickets = [None] * R

        def submit(r):
            if r % 4 == 0:
                tickets[r] = b.submit(prompts[r])
            else:
                tickets[r] = b.submit(prompts[r], predictions=preds[r], admission=dict(
                    priority=int(prio[r]), ttft_slo=float(ttft[r]), tpot_slo=float(tpot[r]), pred_valid=valid[r]))
        ts = [threading.Thread(target=submit, args=(r,)) for r in range(R)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        rows = [(tickets[r] & 0xFFFFF, r) for r in range(R)]
        outs = {r: b.wait(tickets[r]) for r in range(R)}
        b.close()
        # in batch order: row i of the flush is the request whose ticket index is i
        order = [r for _, r in sorted(rows)]
        p2 = np.zeros(R, np.int32)
        t2, q2 = np.zeros(R), np.zeros(R)
        pr2, va2 = [], []
        for i, r in enumerate(order):
            if r % 4:
                p2[i], t2[i], q2[i] = prio[r], ttft[r], tpot[r]
                pr2.append(None if preds[r] is None else [e[0] for e in preds[r]])
                va2.append(valid[r])
            else:
                pr2.append(None)
                va2.append(None)
        rej = am.rejects(model_cfg(acfg), pool, p2, t2, q2, pr2, va2, None, 0, 0)
        for i, r in enumerate(order):
            st = int(np.asarray(outs[r][0]["status"]).reshape(-1)[0])
            assert (st == -2) == bool(rej[i]), f"request {r}"


def test_scheduler_admitters_reference_table(epp):
    """latencyslo/plugin_test.go's rows through plugins.Scheduler(admitters=[...]): a rejected request raises
    AdmissionError ("request cannot be admitted"), every other one is scheduled."""
    P = epp.plugins
    prof = P.NewSchedulerProfile().WithScorers(P.NewWeightedScorer(P.QueueScorer(), 1)).WithPicker(P.NewMaxScorePicker(1))
    sched = P.Scheduler(P.SingleProfileHandler(), {"default": prof}, max_endpoints=4,
                        admitters=[P.LatencyAdmissionFactory("lat", None)])
    inv = lambda: P.NewLatencyPredictionInfo(False, False, -50, -10, 150, 40, 0)      # noqa: E731
    ok = lambda: P.NewLatencyPredictionInfo(True, True, 20, 5, 80, 25, 0)            # noqa: E731
    rows = [(1, "100", "30", [(0.5, 5, inv())], False),
            (-1, "", "", [(0.5, 5, None)], False),
            (-1, "100", "30", [(0.5, 5, inv()), (0.4, 3, inv())], True),
            (-1, "100", "30", [(0.5, 5, inv()), (0.4, 0, inv())], False),
            (-1, "100", "30", [(0.5, 5, inv()), (0.01, 3, inv())], False),
            (-1, "100", "30", [(0.5, 5, inv()), (0.4, 3, ok())], False),
            (-1, "100", "30", [(0.5, 5, None)], False)]
    for prio, ttft, tpot, eps, want in rows:
        pods = []
        for i, (kv, run, info) in enumerate(eps):
            pod = P.NewEndpoint(P.EndpointMetadata(f"pod{i}"), P.Metrics(0, kv, run))
            if info is not None:
                pod.Put(P.LatencyPredictionInfoKey, info)
            pods.append(pod)
        req = P.InferenceRequest(TargetModel="m", Objectives=P.RequestObjectives(prio),
                                 Headers={"x-slo-ttft-ms": ttft, "x-slo-tpot-ms": tpot})
        if want:
            with pytest.raises(P.AdmissionError, match="request cannot be admitted"):
                sched.Schedule(req, pods)
        else:
            assert sched.Schedule(req, pods).ProfileResults["default"].TargetEndpoints
