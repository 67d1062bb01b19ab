"""The micro-batcher (csrc/batcher.cu) on engines whose decisions depend on state that every flush moves forward: the
request ordinals (seeded ties, random draws), the prefix index (index_picks) and the in-flight counters.  Concurrent
submitters group the requests by timing; the tests read the flushes that actually ran back from the tickets
(tests/batcher_replay.py), replay them one by one on the models and compare bit for bit.  Each scenario also replays the
same rows as one call in request order and asserts that this wrong replay disagrees, so that it can fail.  Failed
flushes, ticket expiry and the drain of epp_batcher_destroy are covered too.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import batcher_replay as BR
import helpers

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


@pytest.fixture(scope="module")
def tg():
    from tools import tracegen
    tracegen.build()
    return tracegen


def _submit_wait(bt, prompt, **kw):
    t = bt.submit(prompt, **kw)
    d, dd = bt.wait(t)
    return t, d, dd


def _rows_agree(got, want):
    """got: {row: (ticket, decision, detail)}, want: {row: (oracle decision, total, match_blocks)} -> bool per row."""
    ok = []
    for r in sorted(want):
        _, d, dd = got[r]
        o, total, mb = want[r]
        same = int(d["status"]) == int(o["status"]) and int(d["total_blocks"]) == total
        if same and int(o["status"]) == 0:
            pf = -1 if int(d["prefill_pick"]) == NO else int(d["prefill_pick"])
            same = (int(d["pick"]) == int(o["pick"]) and np.float64(d["score"]).tobytes() == np.float64(o["score"]).tobytes()
                    and int(d["tie_count"]) == int(o["tie_count"]) and int(d["match_blocks"]) == mb
                    and pf == int(o["prefill_pick"]) and int(dd["prefill_ran"]) == int(o["prefill_ran"]))
            if same and int(o["prefill_pick"]) >= 0:
                same = (np.float64(dd["prefill_score"]).tobytes() == np.float64(o["prefill_score"]).tobytes()
                        and int(dd["prefill_tie_count"]) == int(o["prefill_tie_count"]))
        ok.append(same)
    return np.array(ok)


def _assert_replay(epp, got, want, where):
    rows = sorted(want)
    dec = np.array([got[r][1] for r in rows], dtype=epp.DECISION_DTYPE)
    det = np.array([got[r][2] for r in rows], dtype=epp.DETAIL_DTYPE)
    odec = np.array([want[r][0] for r in rows])
    ototal = np.array([want[r][1] for r in rows], np.int32)
    helpers.assert_decisions_equal(dec, det, odec, ototal, where=where)
    ok = odec["status"] == 0
    np.testing.assert_array_equal(dec["match_blocks"][ok], np.array([want[r][2] for r in rows])[ok], err_msg=where + " match_blocks")
    assert _rows_agree(got, want).all()


def _pd_engine(epp, w, pool, **kw):
    eng = helpers.make_engine(w, tie_seed=BR.SEED, **kw)
    from tools import tracegen as tg
    eng.register_model(tg.MODEL)
    eng.pool_set(np.arange(w.E, dtype=np.uint32), *pool)
    return eng


# ---- 1. seeded ties + index_picks, P/D ---------------------------------------------------------------------------------
def test_seeded_ties_with_prerequest_pd(epp, orc, tg):
    w, tokens, pool = BR.pd_landscape(tg)
    R = tokens.shape[0]
    with _pd_engine(epp, w, pool) as eng:
        base0 = eng.stats()["n_decisions"]
        with epp.Batcher(eng, max_batch=48, max_delay_us=200, index_picks=True) as bt:
            got = BR.run_threads(64, range(R), lambda r: _submit_wait(bt, tokens[r]))
            st = bt.stats()
        fl = BR.flushes({r: got[r][0] for r in got})
        sizes = BR.sizes(fl)
        print(f"seeded P/D + index_picks: {len(fl)} flushes, sizes min {min(sizes)} max {max(sizes)} "
              f"full {sum(s == 48 for s in sizes)}")
        assert st["n_flushes"] == len(fl) and st["n_requests"] == R and st["n_index_errors"] == 0
        assert eng.stats()["n_decisions"] == base0 + R
        assert any(s < 48 for s in sizes), "no flush was closed by the delay"
        want, ix = BR.pd_replay(orc, tg, w, tokens, pool, BR.with_bases(fl, base0))
        _assert_replay(epp, got, want, "seeded P/D replay")
        assert sum(want[r][2] > 0 for r in range(R)) > R // 10 and any(int(want[r][0]["prefill_ran"]) for r in range(R))
        wrong, _ = BR.pd_replay(orc, tg, w, tokens, pool, BR.single(range(R), base0))
        assert not _rows_agree(got, wrong).all(), "the single-flush replay agrees: the test cannot tell groupings apart"
        eng.index_commit()
        assert eng.stats()["index_pairs"] == len(ix.export()[0])


# ---- 2. random pickers on every flush-size path ------------------------------------------------------------------------
def _picker_engine(epp, world, picker):
    spec = lambda sc: epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, p) for k, wt, p in sc], picker=picker)   # noqa: E731
    eng = epp.Engine(world.E, spec(BR.PICKER_DECODE), spec(BR.PICKER_PREFILL), block_size_tokens=world.BST,
                     max_prefix_blocks=world.B, tie_seed=BR.SEED, always_disagg=True)
    world.load(eng)
    return eng


def _assert_picker_rows(got, want):
    """-> the rows whose decision differs from the picker model's."""
    bad = []
    for r, (p, s, n, mb, p1, s1, n1) in want.items():
        _, d, dd = got[r]
        if not (int(d["status"]) == 0 and int(d["pick"]) == p and np.float64(d["score"]).tobytes() == np.float64(s).tobytes()
                and int(d["tie_count"]) == n and int(d["match_blocks"]) == mb and int(d["prefill_pick"]) == p1
                and np.float64(dd["prefill_score"]).tobytes() == np.float64(s1).tobytes() and int(dd["prefill_tie_count"]) == n1):
            bad.append(r)
    return bad


@pytest.mark.parametrize("picker", [1, 2])
def test_random_pickers_every_flush_size(epp, orc, picker):
    from tools import picker_model as PM
    assert picker in (PM.RANDOM, PM.WEIGHTED_RANDOM)
    world = BR.PickerWorld(orc, R=1600)
    cls = lambda n: "<=8" if n <= 8 else "9-1024" if n <= 1024 else ">1024"      # noqa: E731
    phases = []                          # per batcher: {row: (ticket, decision, detail)}; its seqs start at 0
    with _picker_engine(epp, world, picker) as eng:
        # The size classes are told apart by flush size alone: this test takes no profiler trace.  Traces in the same
        # process as the batchers' flusher threads were followed by traces that lost device records in later tests.
        base0 = eng.stats()["n_decisions"]
        # zero-copy small flushes (<= 8 rows): one full flush from one submitter, then 32 submitters
        with epp.Batcher(eng, max_batch=8, max_delay_us=50) as bt:
            def full8():
                ts = [bt.submit(world.tokens[r]) for r in range(8)]
                return {r: (t, *bt.wait(t)) for r, t in zip(range(8), ts)}
            got = full8()
            got.update(BR.run_threads(32, range(8, 400), lambda r: _submit_wait(bt, world.tokens[r])))
            phases.append(got)
        # DMA-fed small flushes (9 .. 1024 rows): 32 submitters with 12 requests each in flight, and a delay long
        # enough for a flush to collect several submitters' requests
        with epp.Batcher(eng, max_batch=512, max_delay_us=3000) as bt:
            def twelve(t):
                rows = list(range(400 + 12 * t, 400 + 12 * t + 12))
                ts = [bt.submit(world.tokens[r]) for r in rows]
                return {r: (tk, *bt.wait(tk)) for r, tk in zip(rows, ts)}
            got = {}
            for part in BR.run_threads(32, range(32), twelve).values():
                got.update(part)
            phases.append(got)
        # the chunked sparse path (> 1024 rows): one submitter, one flush of 1500
        with epp.Batcher(eng, max_batch=1500, max_delay_us=20_000_000) as bt:
            def big():
                ts = {r: bt.submit(world.tokens[r]) for r in range(100, 1600)}
                return {r: (t, *bt.wait(t)) for r, t in ts.items()}
            phases.append(big())
        assert eng.stats()["n_decisions"] == base0 + sum(len(g) for g in phases)
    base, classes = base0, set()
    for k, got in enumerate(phases):
        fl = BR.flushes({r: got[r][0] for r in got})
        print(f"picker {picker}, batcher {k}: {len(fl)} flushes, sizes {sorted(BR.sizes(fl))}")
        classes.update(cls(n) for n in BR.sizes(fl))
        want = BR.picker_replay(world, picker, BR.with_bases(fl, base))
        bad = _assert_picker_rows(got, want)
        assert not bad, f"batcher {k}: {len(bad)} rows differ from the replay, first {bad[:4]}"
        if k < 2:                        # concurrent submitters: the request order is not the flushes' order
            wrong = BR.picker_replay(world, picker, BR.single(got.keys(), base))
            assert _assert_picker_rows(got, wrong), f"batcher {k}: the single-flush replay agrees"
        base += len(got)
    assert classes == {"<=8", "9-1024", ">1024"}, classes


# ---- 4. in-flight load feeding the scorers -----------------------------------------------------------------------------
def test_inflight_load_between_flushes(epp, orc, tg):
    from tools import inflight_model as M
    w, trace = BR.inflight_landscape(tg, R=640)
    tokens = trace.requests()[0]
    role, kv, waiting, running = trace.pool()
    _, ix, _, _, _ = helpers.setup_oracle(orc, w, trace)
    R1 = 384
    with helpers.make_engine(w, inflight_load=True) as eng:
        helpers.setup_engine(eng, w, trace)
        base0 = eng.stats()["n_decisions"]
        model = M.Counters(w.E)
        with epp.Batcher(eng, max_batch=40, max_delay_us=150) as bt:
            got = BR.run_threads(32, range(R1), lambda r: _submit_wait(bt, tokens[r]))
            fl1 = BR.flushes({r: got[r][0] for r in got})
            want = BR.inflight_replay(orc, tg, w, trace, ix, model, BR.with_bases(fl1, base0), tokens)
            # a release from the main thread while the batcher is idle: every third request of phase 1 finishes
            eps, lens = [], []
            for r in range(0, R1, 3):
                for e in model.targets(np.array([got[r][1]]), None, 0):
                    eps.append(e)
                    lens.append(w.prompt_bytes)
            eng.inflight_release(eps, lens)
            model.release(eps, lens)
            got2 = BR.run_threads(32, range(R1, w.R), lambda r: _submit_wait(bt, tokens[r]))
            got.update(got2)
            st = bt.stats()
        fl = BR.flushes({r: got[r][0] for r in got})
        fl2 = fl[len(fl1):]
        assert [r for _, rows in fl[:len(fl1)] for r in rows] == [r for _, rows in fl1 for r in rows]
        plan2 = BR.with_bases(fl, base0)[len(fl1):]
        want.update(BR.inflight_replay(orc, tg, w, trace, ix, model, plan2, tokens))
        print(f"in-flight load: phase 1 sizes {BR.sizes(fl1)}, phase 2 sizes {BR.sizes(fl2)}")
        assert st["n_flushes"] == len(fl) and st["n_requests"] == w.R
        _assert_replay(epp, got, want, "in-flight replay")
        req, tok = eng.inflight_get()
        np.testing.assert_array_equal(req, model.req)
        np.testing.assert_array_equal(tok, model.tok)
        wrong = BR.inflight_replay(orc, tg, w, trace, ix, M.Counters(w.E), BR.single(range(R1), base0), tokens)
        picks = [int(got[r][1]["pick"]) == int(wrong[r][0]["pick"]) for r in range(R1)]
        assert not all(picks), "the single-flush replay agrees"


# ---- 3. no-hit-lru: evictions between concurrent flushes ------------------------------------------------------------
@pytest.mark.parametrize("picker", [0, 2])
def test_nohit_lru_between_flushes(epp, orc, picker):
    """A max-score (seeded ties) and a weighted-random engine whose LRU holds 20 of 96 endpoints: far more cold picks
    than that, so every flush reads an LRU that earlier flushes filled and evicted from."""
    world = BR.PickerWorld(orc, E=96, R=480)
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(*sc) for sc in BR.NOHIT_SCORERS], picker=picker)
    with epp.Engine(world.E, spec, block_size_tokens=world.BST, max_prefix_blocks=world.B, tie_seed=BR.SEED) as eng:
        world.load(eng)
        base0 = eng.stats()["n_decisions"]
        with epp.Batcher(eng, max_batch=32, max_delay_us=200) as bt:
            got = BR.run_threads(16, range(world.R), lambda r: _submit_wait(bt, world.tokens[r]))
            st = bt.stats()
        fl = BR.flushes({r: got[r][0] for r in got})
        print(f"no-hit-lru picker {picker}: {len(fl)} flushes, sizes {sorted(BR.sizes(fl))}")
        assert st["n_flushes"] == len(fl) and st["n_requests"] == world.R
        model = BR.nohit_model(orc, world, picker)
        want = BR.nohit_replay(model, world, BR.with_bases(fl, base0))
        assert sum(want[r][5] for r in want) > 3 * BR.NOHIT_LRU

        def bad_rows(want):
            return [r for r, (status, pick, score, _, mb, _) in want.items()
                    if not (int(got[r][1]["status"]) == status and int(got[r][1]["pick"]) == pick
                            and np.float64(got[r][1]["score"]).tobytes() == np.float64(score).tobytes()
                            and int(got[r][1]["match_blocks"]) == mb)]
        bad = bad_rows(want)
        assert not bad, f"{len(bad)} rows differ from the replay, first {bad[:4]}"
        assert eng.nohit_lru_get() == model.lru.keys()
        assert bad_rows(BR.nohit_replay(BR.nohit_model(orc, world, picker), world, BR.single(range(world.R), base0))), \
            "the single-flush replay agrees"


# ---- 5. admitters under concurrency ----------------------------------------------------------------------------------
def test_admitters_between_flushes(epp, orc, tg):
    """The latency-slo-admitter and the probabilistic-admitter on an engine with index_picks and the in-flight
    producer: the probabilistic draws follow the flushes' ordinal bases, and rejected rows reach neither PreRequest nor
    the in-flight counters."""
    from tools import admission_model as am
    w, tokens, pool, cfg, rows = BR.admit_landscape(tg, orc)
    with helpers.make_engine(w, tie_seed=BR.SEED, inflight_load=True) as eng:
        eng.admission_set(latency_slo=True, probabilistic=True, power=cfg["power"], k=cfg["k"])
        eng.register_model(tg.MODEL)
        eng.pool_set(np.arange(w.E, dtype=np.uint32), np.zeros(w.E, np.uint8), pool["kv"], pool["waiting"], pool["running"])
        base0 = eng.stats()["n_decisions"]

        def one(r):
            adm = dict(priority=int(rows["priority"][r]), ttft_slo=float(rows["ttft"][r]), tpot_slo=float(rows["tpot"][r]))
            if rows["preds"][r] is not None:
                adm["pred_valid"] = rows["valid"][r]
            return _submit_wait(bt, tokens[r], predictions=rows["preds"][r], admission=adm)
        with epp.Batcher(eng, max_batch=32, max_delay_us=200, index_picks=True) as bt:
            got = BR.run_threads(16, range(w.R), one)
            st = bt.stats()
        fl = BR.flushes({r: got[r][0] for r in got})
        print(f"admitters: {len(fl)} flushes, sizes {sorted(BR.sizes(fl))}")
        assert st["n_flushes"] == len(fl) and st["n_requests"] == w.R and st["n_index_errors"] == 0
        want, ix, counters = BR.admit_replay(orc, tg, am, w, tokens, pool, cfg, rows, BR.with_bases(fl, base0))
        rej = [r for r in range(w.R) if int(want[r][0]["status"]) == am.STATUS_REJECTED]
        assert w.R // 8 < len(rej) < w.R // 2
        for r in rej:
            d = got[r][1]
            assert int(d["status"]) == am.STATUS_REJECTED and int(d["pick"]) == NO and int(d["match_blocks"]) == 0, r
        _assert_replay(epp, got, {r: want[r] for r in range(w.R) if r not in set(rej)}, "admitted rows")
        assert int((np.array([int(got[r][1]["status"]) for r in range(w.R)]) == am.STATUS_REJECTED).sum()) == len(rej)
        req, tok = eng.inflight_get()
        np.testing.assert_array_equal(req, counters.req)
        np.testing.assert_array_equal(tok, counters.tok)
        eng.index_commit()
        assert eng.stats()["index_pairs"] == len(ix.export()[0])
        wrong, _, _ = BR.admit_replay(orc, tg, am, w, tokens, pool, cfg, rows, BR.single(range(w.R), base0))
        assert any(int(wrong[r][0]["status"]) != int(got[r][1]["status"]) for r in range(w.R)), \
            "the single-flush replay agrees"


# ---- 6. first-k lists across staging laps ------------------------------------------------------------------------------
def test_first_k_lists_with_error_rows(epp, orc, tg):
    K = 4
    w = tg.baseline_configs()["config4"].scaled(E=96, R=16 * 40, T=256, name="config4")
    w.non_cached_tokens = 32
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests()
    pool, ix, primary, prefill, _ = helpers.setup_oracle(orc, w, trace)
    role = trace.pool()[0]
    kv, waiting, running = BR.flat_pool(w.E, 11)
    opool = orc.PoolState(role, kv, waiting, running)
    err = {r for r in range(w.R) if r % 4 == 1}               # an empty endpoint subset: status -1, no lists
    with helpers.make_engine(w, pick_k=K, tie_seed=BR.SEED) as eng:
        helpers.setup_engine(eng, w, trace)
        eng.pool_set(np.arange(w.E, dtype=np.uint32), role, kv, waiting, running)
        base0 = eng.stats()["n_decisions"]
        with epp.Batcher(eng, max_batch=24, max_delay_us=200) as bt:
            def one(r):
                t = bt.submit(tokens[r], subset=[] if r in err else None)
                return (t, *bt.wait_topk(t))
            got = BR.run_threads(16, range(w.R), one)
        fl = BR.flushes({r: got[r][0] for r in got})
        print(f"first-k: {len(fl)} flushes, sizes {sorted(BR.sizes(fl))}")
        assert len(fl) > 8                                     # the four staging buffers went round at least twice
        bad = []
        for _, rows, base in BR.with_bases(fl, base0):
            odec, ototal, olists = helpers.oracle_decisions(orc, w, opool, ix, primary, prefill, tokens[rows], 2, topk=K,
                                                            tie_seed=BR.SEED, tie_base=base)
            keep = [i for i, r in enumerate(rows) if r not in err]
            dec = np.array([got[rows[i]][1] for i in keep], dtype=epp.DECISION_DTYPE)
            det = np.array([got[rows[i]][2] for i in keep], dtype=epp.DETAIL_DTYPE)
            helpers.assert_decisions_equal(dec, det, odec[keep], ototal[keep], where=f"first-k flush at {base}")
            for i, r in enumerate(rows):
                lists = got[r][3]
                if r in err:
                    if int(got[r][1]["status"]) != -1 or any(lists.values()):
                        bad.append((r, int(got[r][1]["status"]), lists))
                    continue
                for name in ("primary", "prefill"):
                    assert lists[name] == [int(x) for x in olists[name][i] if x >= 0], (r, name)
                assert lists["encode"] == []
        assert not bad, f"error rows with a status other than -1 or with lists: {bad[:4]}"
        # the wrong replay: one flush in request order
        odec, _, olists = helpers.oracle_decisions(orc, w, opool, ix, primary, prefill, tokens, 2, topk=K,
                                                   tie_seed=BR.SEED, tie_base=base0)
        same = [got[r][3]["primary"] == [int(x) for x in olists["primary"][r] if x >= 0] for r in range(w.R) if r not in err]
        assert not all(same), "the single-flush replay agrees"


# ---- 7. a failed flush -------------------------------------------------------------------------------------------------
def test_failed_flush_takes_no_ordinals(epp, orc, tg):
    """The first flush of a batcher fails (no pool yet): each of its tickets raises the engine's error and no ordinal is
    taken.  pool_set then comes from the main thread, and the later flushes of the same batcher start at the unchanged
    ordinal base (the failed flush still counts as a flush)."""
    w, tokens, pool = BR.pd_landscape(tg, E=48, R=8 + 16 * 10, seed=4)
    R = tokens.shape[0]
    with helpers.make_engine(w, tie_seed=BR.SEED) as eng:
        eng.register_model(tg.MODEL)
        with pytest.raises(epp.EngineError) as ei:
            eng.schedule(tokens[:1], uniform_len=w.prompt_bytes)         # before pool_set: the engine refuses
        message = ei.value.message
        base0 = eng.stats()["n_decisions"]
        with epp.Batcher(eng, max_batch=8, max_delay_us=200) as bt:
            ts = [bt.submit(tokens[r]) for r in range(8)]              # one full flush of 8, before the pool
            for t in ts:
                with pytest.raises(epp.EngineError) as ei:
                    bt.wait(t)
                assert ei.value.message == message
            failed = {BR.split(t)[0] for t in ts}
            assert len(failed) == 1 and eng.stats()["n_decisions"] == base0
            eng.pool_set(np.arange(w.E, dtype=np.uint32), *pool)
            got = BR.run_threads(16, range(8, R), lambda r: _submit_wait(bt, tokens[r]))
            st = bt.stats()
        tickets = {r: got[r][0] for r in got}
        tickets.update({r: ts[r] for r in range(8)})
        fl = BR.flushes(tickets)
        assert fl[0][0] in failed and st["n_flushes"] == len(fl) and st["n_requests"] == R
        plan = BR.with_bases(fl, base0, failed=failed)[1:]
        assert plan[0][2] == base0
        want, _ = BR.pd_replay(orc, tg, w, tokens, pool, plan, index_picks=False)
        _assert_replay(epp, got, want, "same batcher after the failed flush")
        assert eng.stats()["n_decisions"] == base0 + R - 8
        wrong, _ = BR.pd_replay(orc, tg, w, tokens, pool, [(0, r, b + 8) for _, r, b in plan], index_picks=False)
        assert not _rows_agree(got, wrong).all(), "a replay whose ordinals count the failed flush agrees"


# ---- 8. ticket rules ---------------------------------------------------------------------------------------------------
def test_ticket_expiry_and_short_prompts(epp, orc):
    E, BST, B = 8, 4, 4
    rng = np.random.default_rng(8)
    fams = [rng.integers(0, 256, 16 * B, dtype=np.uint8) for _ in range(3)]
    lens = [0, 7, 15, 16, 33, 64, 100]
    prompts = []
    for r in range(4100):
        n = lens[r % len(lens)]
        p = rng.integers(0, 256, n, dtype=np.uint8)
        if r % 3 and n:
            k = min(n, 16 * B)
            p[:k] = fams[r % 3][:k]
        prompts.append(p.tobytes())
    kv = np.array([0.1, 0.3, 0.3, 0.5, 0.2, 0.2, 0.9, 0.4])
    waiting = np.array([0, 1, 2, 0, 3, 1, 0, 2], np.int32)
    sc = [(2, 2.0, 0.0), (1, 2.0, 0.0), (0, 3.0, 0.0)]
    hs, es = [], []
    for g, f in enumerate(fams):
        h = orc.hash_prompt(f.tobytes(), b"m", BST, B)
        for e in (g, g + 3):
            hs += h[:2 + g]
            es += [e] * (2 + g)
    ix = orc.Indexer()
    ix.load_pairs(np.array(hs, np.uint64), np.array(es, np.uint32))
    data = np.frombuffer(b"".join(prompts) or b"\0", np.uint8)
    offs = np.zeros(len(prompts) + 1, np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    opool = orc.PoolState(np.zeros(E, np.uint8), kv, waiting)
    odec, ototal = orc.cycle_batch(b"m", BST, B, 0, False, ix, orc.make_profile(0, sc), None, opool, data, offs, 4)
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in sc])
    with epp.Engine(E, spec, block_size_tokens=BST, max_prefix_blocks=B) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), kv, waiting, np.zeros(E, np.int32))
        eng.index_load_snapshot(np.array(hs, np.uint64), np.array(es, np.uint32))
        with epp.Batcher(eng, max_batch=1, max_delay_us=0) as bt:
            tickets, dec, det = [], [], []
            for p in prompts:
                t, d, dd = _submit_wait(bt, p)
                tickets.append(t)
                dec.append(d)
                det.append(dd)
            assert [BR.split(t) for t in tickets] == [(s, 0) for s in range(len(prompts))]
            with pytest.raises(epp.EngineError, match="expired"):
                bt.wait(tickets[0])                                  # flushed 4100 flushes ago
            with pytest.raises(epp.EngineError, match="expired"):
                bt.wait(tickets[3])                                  # the last one out of the ring
            for r in (4, 10, 2000, len(prompts) - 1):                # within the last 4096 flushes
                d, dd = bt.wait(tickets[r])
                assert d.tobytes() == dec[r].tobytes() and dd.tobytes() == det[r].tobytes(), r
            with pytest.raises(epp.EngineError, match="unknown ticket"):
                bt.wait(len(prompts) << 20)                          # the fill position: not reserved
            with pytest.raises(epp.EngineError, match="unknown ticket"):
                bt.wait(tickets[-1] + 1)                             # past the last row of a flushed batch
            st = bt.stats()
        assert st["n_flushes"] == len(prompts) and st["n_full_flushes"] == len(prompts)
    dec = np.array(dec, dtype=epp.DECISION_DTYPE)
    det = np.array(det, dtype=epp.DETAIL_DTYPE)
    helpers.assert_decisions_equal(dec, det, odec, ototal, where="max_batch 1")
    short = np.array([len(p) < 4 * BST for p in prompts])
    assert (dec["match_blocks"][short] == 0).all() and (dec["total_blocks"][short] == 0).all()
    assert (dec["match_blocks"][~short] > 0).any()


# ---- 9. destroy drains -------------------------------------------------------------------------------------------------
def test_destroy_drains_a_partial_batch(epp, orc, tg):
    w = tg.baseline_configs()["config3"].scaled(E=32, R=10, T=256, name="config3")
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests()
    role, kv, waiting, running = trace.pool()
    with helpers.make_engine(w) as eng:
        eng.register_model(tg.MODEL)
        eng.pool_set(np.arange(w.E, dtype=np.uint32), role, kv, waiting, running)
        base0 = eng.stats()["n_decisions"]
        bt = epp.Batcher(eng, max_batch=64, max_delay_us=60_000_000, index_picks=True)
        for r in range(w.R):
            bt.submit(tokens[r])
        st = bt.stats()
        assert st["n_pending"] == w.R and st["n_flushes"] == 0
        bt.close()                                            # no wait outstanding: destroy flushes the 10, then stops
        assert eng.stats()["n_decisions"] == base0 + w.R
        ix = orc.Indexer()
        odec, _ = helpers.oracle_decisions(orc, w, orc.PoolState(role, kv, waiting, running), ix,
                                           orc.make_profile(w.primary_filter, list(w.primary_scorers)), None, tokens)
        hs = [orc.hash_prompt(tokens[r].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks) for r in range(w.R)]
        for r in range(w.R):
            if odec["status"][r] == 0:
                ix.add(hs[r], int(odec["pick"][r]))
        eng.index_commit()
        assert eng.stats()["index_pairs"] == len(ix.export()[0]) > 0
        for r in range(w.R):
            for h in hs[r][:3]:
                assert eng.index_get(h) == ix.get(h), r
