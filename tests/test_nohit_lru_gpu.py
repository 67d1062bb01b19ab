"""GPU parity of the no-hit-lru scorer (csrc/nohit_lru.cu and the cold / warm sets of every pick kernel) against the CPU
restatement tools/nohit_lru_model.py, whose other scorer columns come from the C oracle.  Match rows come from the
engine's epp_prefix_match (checked against the oracle by test_gpu_parity.py), so every scheduling call here is compared
decision for decision, and the LRU (epp_nohit_lru_get) after every call.  Run on an H100: pytest -m gpu."""
import dataclasses

import numpy as np
import pytest

import helpers
from tools import nohit_lru_model as M

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


def _engine_1(epp, E, lru=0, weight=1.0):
    eng = epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(M.NO_HIT_LRU, weight, float(lru))]))
    eng.register_model(b"m")
    return eng


def _pool(eng, n):
    eng.pool_set(np.arange(n, dtype=np.uint32), [0] * n, [0.0] * n, [0] * n, [0] * n)


# ---- the reference's KATs (no_hit_lru_test.go) through epp_score and 1-request scheduling calls --------------------
def test_score_table(epp):
    with _engine_1(epp, 3) as eng:
        _pool(eng, 3)
        z = np.zeros((1, 3), dtype=np.int32)
        # :158-175 cold, all never used
        assert list(eng.score(z, [4], 0, 0)[0]) == [1.0, 0.5, 0.0]
        assert list(eng.score(z, [4], 0, -1)[0]) == [1.0, 0.5, 0.0]
        # :176-194 a cache hit anywhere: neutral 0.5
        assert list(eng.score(np.array([[3, 0, 0]], dtype=np.int32), [4], 0, 0)[0]) == [0.5, 0.5, 0.5]
        # :195-208 single endpoint
        eng.pool_set(np.array([1], dtype=np.uint32), [0], [0.0], [0], [0])
        assert list(eng.score(z, [4], 0, 0)[0]) == [0.0, 1.0, 0.0]


def test_prefer_least_recently_used_after_cold_requests(epp):
    """no_hit_lru_test.go:264-372, one request per call."""
    with _engine_1(epp, 3) as eng:
        _pool(eng, 3)
        cold = np.zeros((1, 3), dtype=np.int32)
        warm = np.array([[2, 0, 0]], dtype=np.int32)
        picks = []
        for m in (cold, cold, warm, cold, cold):
            dec, _ = eng.schedule_with_match(m, [4], [64], 16)
            picks.append(int(dec["pick"][0]))
        assert picks == [0, 1, 0, 2, 0]
        assert eng.nohit_lru_get() == [1, 2, 0]
        eng.score(cold, [4], 0, 0)                   # epp_score never updates
        assert eng.nohit_lru_get() == [1, 2, 0]


def test_sharded_mode_rejects_the_scorer(epp):
    with _engine_1(epp, 8) as eng:
        with pytest.raises(Exception):
            eng.shard_set(0, 4)


def test_lru_size_must_agree(epp):
    with pytest.raises(Exception):
        epp.Engine(8, epp.ProfileSpec(1, [epp.ScorerSpec(M.NO_HIT_LRU, 1.0, 4.0)]),
                   epp.ProfileSpec(2, [epp.ScorerSpec(M.NO_HIT_LRU, 1.0, 5.0)]))


# ---- multi-batch parity on the trace generator's workloads ---------------------------------------------------------
def _workload(name, E, R, lru, decode_and_prefill=True):
    from tools import tracegen as tg
    w = tg.baseline_configs()[name].scaled(E=E, R=R, T=512)
    nh = (M.NO_HIT_LRU, 1.0, float(lru))
    w = dataclasses.replace(w, primary_scorers=tuple(w.primary_scorers) + (nh,))
    if w.prefill_scorers is not None and decode_and_prefill:
        w = dataclasses.replace(w, prefill_scorers=tuple(w.prefill_scorers) + (nh,))
    return w


def _model(orc, w, trace, lru, tie_seed):
    from tools import tracegen as tg
    role, kv, waiting, running = trace.pool()
    pool = orc.PoolState(role, kv, waiting, running)
    profiles = [(w.primary_filter, list(w.primary_scorers))]
    if w.prefill_scorers is not None:
        profiles.append((tg.FILTER_PREFILL, list(w.prefill_scorers)))
    return M.Model(orc, pool, w.E, profiles, lru, nct=w.non_cached_tokens, block_size_tokens=w.block_size_tokens,
                   tie_seed=tie_seed)


def _compare(dec, want, where):
    st = np.array([x[0] for x in want])
    assert (dec["status"] == st).all(), where
    ok = st == 0
    assert (dec["pick"][ok] == np.array([x[1] for x in want])[ok]).all(), where
    assert (dec["score"][ok] == np.array([x[2] for x in want])[ok]).all(), where
    assert (dec["prefill_pick"] == np.array([x[3] for x in want], dtype=np.uint32)).all(), where


def _run(epp, orc, name, path, *, tie_seed=0, lru=0, E=64, R=256, batches=4, pool_change=False):
    import torch

    from tools import tracegen as tg
    w = _workload(name, E, R, lru)
    trace = tg.Trace(w)
    model = _model(orc, w, trace, lru, tie_seed)
    names_all = {}
    cold_total = 0
    with helpers.make_engine(w, tie_seed=tie_seed) as eng:
        helpers.setup_engine(eng, w, trace)
        for b in range(batches):
            tokens, _, _ = trace.requests(b * w.R, w.R)
            match, total = eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
            in_len = np.full(w.R, w.prompt_bytes, dtype=np.int64)
            want = model.schedule(match, total, in_len)
            cold_total += sum(1 for x in want if x[5])
            if path == "host":
                fn = lambda: eng.schedule(tokens, uniform_len=w.prompt_bytes)
            elif path == "device":
                dt = torch.from_numpy(tokens.view(np.int32)).cuda()
                fn = lambda: eng.schedule(dt, uniform_len=w.prompt_bytes)
            elif path == "zerocopy":                  # prompts in pinned memory, read by the kernel over PCIe (R <= 8)
                buf = epp.PinnedBuffer(tokens.nbytes + 64)
                buf.array[: tokens.nbytes] = tokens.reshape(-1).view(np.uint8)
                fn = lambda: eng.schedule(buf.array, uniform_len=w.prompt_bytes, n_requests=w.R)
            elif path == "async":
                dt = torch.from_numpy(tokens.view(np.int32)).cuda()

                def fn():
                    r = eng.schedule(dt, uniform_len=w.prompt_bytes, asynchronous=True)
                    eng.synchronize()
                    return r
            else:
                fn = lambda: eng.schedule_with_match(match, total, in_len, w.block_size_tokens)
            (dec, det), names = helpers.kernels_launched(fn, repeatable=False)
            for n, c in names.items():
                names_all[n] = names_all.get(n, 0) + c
            if path in ("device", "async"):
                torch.cuda.synchronize()
                dec = epp.decisions_from_torch(dec)
            _compare(dec, want, f"{name} {path} batch {b}")
            assert eng.nohit_lru_get() == model.lru.keys(), f"{name} {path} LRU after batch {b}"
            if pool_change and b == 1:
                role, kv, waiting, running = trace.pool()
                waiting = np.roll(waiting, 3)
                eng.pool_set(np.arange(w.E, dtype=np.uint32), role, kv, waiting, running)
                model.set_pool(orc.PoolState(role, kv, waiting, running))
    assert cold_total > 0 and model.lru.keys(), "the workload has cold requests"
    return names_all


def _launched(names, frag):
    return sum(c for n, c in names.items() if frag in n)


def _nohit_sparse(names):
    return _launched(names, "k_match_pick_sparse_nohit<")


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("lru", [0, 5])
@pytest.mark.parametrize("name", ["config3", "config4"])
def test_parity_device_batches(epp, orc, name, lru, tie_seed):
    names = _run(epp, orc, name, "device", tie_seed=tie_seed, lru=lru)
    if helpers.trace_complete(names):
        assert _launched(names, "k_nohit_touch") > 0
        assert _nohit_sparse(names) > 0


@pytest.mark.parametrize("name", ["config3", "config4"])
def test_parity_host_small_batches(epp, orc, name):
    names = _run(epp, orc, name, "host", tie_seed=0x77, lru=7)
    if helpers.trace_complete(names):
        assert _launched(names, "k_cycle_small_nohit<") > 0 and _launched(names, "k_nohit_touch") > 0


@pytest.mark.parametrize("name", ["config3", "config4"])
def test_parity_zero_copy_small_batches(epp, orc, name):
    names = _run(epp, orc, name, "zerocopy", lru=3, R=8, batches=8)
    if helpers.trace_complete(names):
        assert _launched(names, "k_cycle_small_nohit<") > 0


@pytest.mark.parametrize("name", ["config3", "config4"])
def test_parity_with_match(epp, orc, name):
    names = _run(epp, orc, name, "with_match", lru=9, pool_change=True)
    if helpers.trace_complete(names):
        assert _launched(names, "k_dense_pick") > 0


def test_engine_without_the_scorer_launches_no_new_kernel(epp):
    import torch

    from tools import tracegen as tg
    w = tg.baseline_configs()["config3"].scaled(E=64, R=256, T=512)
    trace = tg.Trace(w)
    with helpers.make_engine(w) as eng:
        helpers.setup_engine(eng, w, trace)
        tokens, _, _ = trace.requests(0, w.R)
        dt = torch.from_numpy(tokens.view(np.int32)).cuda()
        _, names = helpers.kernels_launched(lambda: eng.schedule(dt, uniform_len=w.prompt_bytes))
        assert helpers.trace_complete(names)
        assert _launched(names, "nohit") == 0 and _nohit_sparse(names) == 0
        assert _launched(names, "k_match_pick_sparse<8, false, false, 1>") > 0
        with pytest.raises(Exception):
            eng.nohit_lru_get()


# ---- the general evaluation: prefix-cache-affinity-filter + first k (pick_general.cuh) -------------------------------
@pytest.mark.parametrize("k", [1, 3])
def test_general_path_affinity_filter_and_topk(epp, orc, k):
    """The narrowed set holds sticky endpoints only, so the request is warm there and the scorer adds 0.5 · w
    (no_hit_lru.go:159-165); un-narrowed cold requests use the LRU column.  Expected: the C oracle with the scorer's
    column supplied as an external column (the same clamp(score) · weight term in the same position)."""
    E, R, w_nh = 16, 48, 1.5
    rng = np.random.default_rng(7)
    role = np.zeros(E, np.uint8)
    kv = rng.random(E)
    waiting = rng.integers(0, 6, E).astype(np.int32)
    running = rng.integers(0, 6, E).astype(np.int32)
    scorers = [(2, 2.0, 0.0), (1, 2.0, 0.0), (0, 3.0, 0.0)]
    aff = (0.5, 0.0, 0.0)
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in scorers] + [epp.ScorerSpec(M.NO_HIT_LRU, w_nh, 0.0)],
                           affinity=epp.AffinityFilterSpec(*aff))
    lru = M.GoLRU(0)
    with epp.Engine(E, spec, pick_k=k) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E, dtype=np.uint32), role, kv, waiting, running)
        for b in range(3):
            total = np.full(R, 8, np.int32)
            match = np.zeros((R, E), np.int32)
            for r in range(R):
                if r % 3:                                   # warm: a few holders, some of them sticky (>= 4 of 8)
                    hold = rng.choice(E, size=rng.integers(1, 4), replace=False)
                    match[r, hold] = rng.integers(1, 9, size=hold.shape[0])
            keys = lru.keys()
            if k > 1:
                (dec, _, lists), names = helpers.kernels_launched(lambda: eng.schedule_with_match(match, total, topk=True),
                                                                  repeatable=False)
            else:
                (dec, _), names = helpers.kernels_launched(lambda: eng.schedule_with_match(match, total), repeatable=False)
            if helpers.trace_complete(names):
                assert _launched(names, "k_dense_pick") > 0
            cold_picks = []
            for r in range(R):
                cold = M.is_cold(range(E), match[r])
                col = M.cold_column(list(range(E)), keys, E) if cold else np.full(E, 0.5)
                pool = orc.PoolState(role, kv, waiting, running, ext=col.reshape(1, E))
                prof = orc.make_profile(0, scorers + [(4, w_nh, 0.0)], affinity=aff)
                picks, sc, _, _ = orc.profile_run_topk(prof, pool, match[r], int(total[r]), max(k, 1))
                assert int(dec["pick"][r]) == picks[0] and dec["score"][r] == sc[0], f"batch {b} request {r}"
                if k > 1:
                    row = [int(x) for x in np.asarray(lists["primary"][r]).astype(np.int64) if int(x) != NO]
                    assert row == picks, f"batch {b} request {r}"
                    np.testing.assert_array_equal(np.asarray(lists["primary_scores"][r])[: len(sc)], sc)
                if cold:
                    cold_picks.append(picks[0])
            assert cold_picks
            for e in cold_picks:
                lru.add(e)
            assert eng.nohit_lru_get() == lru.keys(), f"LRU after batch {b}"


# ---- the encode stage overwrites the cold bit (decode -> encode -> prefill) -------------------------------------------
def test_parity_encode_stage(epp, orc):
    from tools import tracegen as tg
    w = _workload("config4", 64, 256, 0)
    trace = tg.Trace(w)
    nh = (M.NO_HIT_LRU, 1.0, 0.0)
    enc_scorers = [(2, 1.0, 0.0), (0, 2.0, 0.0), nh]
    role, kv, waiting, running = trace.pool()
    model = M.Model(orc, orc.PoolState(role, kv, waiting, running), w.E,
                    [(w.primary_filter, list(w.primary_scorers)), (tg.FILTER_PREFILL, list(w.prefill_scorers))], 0,
                    nct=w.non_cached_tokens, block_size_tokens=w.block_size_tokens, encode=(0, enc_scorers))
    rng = np.random.default_rng(3)
    with helpers.make_engine(w, encode=epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in enc_scorers])) as eng:
        helpers.setup_engine(eng, w, trace)
        for b in range(3):
            tokens, _, _ = trace.requests(b * w.R, w.R)
            mm = (rng.random(w.R) < 0.5).astype(np.uint8)
            match, total = eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
            want = model.schedule(match, total, np.full(w.R, w.prompt_bytes, np.int64), multimodal=mm)
            dec, det = eng.schedule(tokens, uniform_len=w.prompt_bytes, multimodal=mm)
            _compare(dec, want, f"encode batch {b}")
            assert eng.nohit_lru_get() == model.lru.keys(), f"encode LRU after batch {b}"


# ---- a prefix held by more than 32 endpoints: the dense-counter overflow pass decides (and writes the cold bit) -------
def test_parity_overflow_pass(epp, orc):
    import torch

    from tools import tracegen as tg
    w = _workload("config3", 64, 256, 0)
    trace = tg.Trace(w)
    model = _model(orc, w, trace, 0, 0)
    with helpers.make_engine(w) as eng:
        _, (hs, es) = helpers.setup_engine(eng, w, trace)
        tokens, _, _ = trace.requests(0, w.R)
        fh, nb = eng.hash_prompts(tokens, uniform_len=w.prompt_bytes)
        extra_h, extra_e = [], []
        for r in range(0, w.R, 4):                   # 40 holders of the first 3 blocks of every 4th prompt
            for e in range(40):
                extra_h += list(fh[r, :3])
                extra_e += [e] * 3
        eng.index_load_snapshot(np.concatenate([hs, np.array(extra_h, np.uint64)]),
                                np.concatenate([es, np.array(extra_e, np.uint32)]))
        for b in range(2):
            match, total = eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
            assert ((match > 0).sum(axis=1) > 32).any()
            want = model.schedule(match, total, np.full(w.R, w.prompt_bytes, np.int64))
            dt = torch.from_numpy(tokens.view(np.int32)).cuda()
            dec, _ = eng.schedule(dt, uniform_len=w.prompt_bytes)
            torch.cuda.synchronize()
            _compare(epp.decisions_from_torch(dec), want, f"overflow batch {b}")
            assert eng.nohit_lru_get() == model.lru.keys(), f"overflow LRU after batch {b}"
            tokens, _, _ = trace.requests((b + 1) * w.R, w.R)


# ---- one request per flush: the reference's sequence exactly ----------------------------------------------------------
def test_batcher_max_batch_1_is_sequential(epp, orc):
    from tools import tracegen as tg
    w = _workload("config3", 32, 48, 0)
    trace = tg.Trace(w)
    model = _model(orc, w, trace, 0, 0)
    with helpers.make_engine(w) as eng:
        helpers.setup_engine(eng, w, trace)
        tokens, _, _ = trace.requests(0, w.R)
        match, total = eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
        with epp.Batcher(eng, max_batch=1, max_delay_us=0) as bt:
            for r in range(w.R):
                want = model.schedule(match[r:r + 1], total[r:r + 1], np.array([w.prompt_bytes], np.int64))
                d, _ = bt.schedule(tokens[r].tobytes())
                assert (int(d["status"]), int(d["pick"]), float(d["score"])) == want[0][:3], f"request {r}"
        assert eng.nohit_lru_get() == model.lru.keys()
        assert len(model.lru.keys()) > 2                   # cold requests rotated through the pool


# ---- back-to-back pipelined async batches (two chunks on two streams) -------------------------------------------------
def test_pipelined_async_batches_back_to_back(epp, orc):
    import torch

    from tools import tracegen as tg
    w = _workload("config3", 64, 8192, 0)
    trace = tg.Trace(w)
    model = _model(orc, w, trace, 0, 0)
    with helpers.make_engine(w) as eng:
        helpers.setup_engine(eng, w, trace)
        batches = [trace.requests(b * w.R, w.R)[0] for b in range(3)]
        wants = []
        for tokens in batches:
            match, total = eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
            wants.append(model.schedule(match, total, np.full(w.R, w.prompt_bytes, np.int64)))
        dts = [torch.from_numpy(t.view(np.int32)).cuda() for t in batches]
        torch.cuda.synchronize()

        def run():
            outs = [eng.schedule(dt, uniform_len=w.prompt_bytes, asynchronous=True) for dt in dts]   # no wait between
            eng.synchronize()
            return outs
        outs, names = helpers.kernels_launched(run, repeatable=False)
        for b, (dec, _) in enumerate(outs):
            _compare(epp.decisions_from_torch(dec), wants[b], f"pipelined batch {b}")
        assert eng.nohit_lru_get() == model.lru.keys()
        if helpers.trace_complete(names):
            assert _launched(names, "k_hash_fused") == 6          # two chunks per call: the pipelined path ran
            assert _nohit_sparse(names) == 6 and _launched(names, "k_nohit_touch") == 3


def test_scheduler_prefer_least_recently_used(epp):
    """no_hit_lru_test.go:264-372 through plugins.Scheduler (one request per Schedule call, as the reference runs it):
    cold requests rotate a -> b -> c -> a, a warm request (a holds blocks) changes nothing."""
    from epp_b200 import plugins as P
    eps = [P.NewEndpoint(P.EndpointMetadata(n)) for n in ("endpoint-a", "endpoint-b", "endpoint-c")]
    prof = P.NewSchedulerProfile().WithScorers(P.NewWeightedScorer(P.NoHitLRU(), 1.0)).WithPicker(P.NewMaxScorePicker())
    sched = P.Scheduler(P.SingleProfileHandler(), {"default": prof}, max_endpoints=3)
    sched.engine.register_model(b"m")

    def pick(warm=False):
        for i, e in enumerate(eps):
            e.Put(P.PrefixCacheMatchInfoKey, P.NewPrefixCacheMatchInfo(2 if (warm and i == 0) else 0, 4, 16))
        res = sched.Schedule(P.InferenceRequest(Prompt=b"x" * 64), eps)
        return res.ProfileResults["default"].TargetEndpoints[0].GetMetadata().Name

    assert [pick(), pick(), pick(warm=True), pick(), pick()] == \
        ["endpoint-a", "endpoint-b", "endpoint-a", "endpoint-c", "endpoint-a"]
    assert sched.engine.nohit_lru_get() == [1, 2, 0]
    sched.engine.close()


def test_lora_affinity_in_the_same_profile(epp, orc):
    """lora-affinity adds the endpoints where the request's adapter is resident to the match map with count 0: they are
    not hits, so a request with no prefix match stays cold (no_hit_lru.go:140-155).  Expected: the C oracle with the
    scorer's column supplied as an external column and the request's adapter residency."""
    E, R, n_models = 16, 48, 3
    rng = np.random.default_rng(11)
    role, kv = np.zeros(E, np.uint8), rng.random(E)
    waiting, running = rng.integers(0, 5, E).astype(np.int32), np.zeros(E, np.int32)
    scorers = [(0, 2.0, 0.0), (8, 1.0, 0.0)]
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in scorers] + [epp.ScorerSpec(M.NO_HIT_LRU, 1.0, 0.0)])
    max_active = rng.integers(1, 3, E).astype(np.int32)
    members = [(int(e), int(m), int(rng.integers(1, 3))) for m in range(n_models)
               for e in rng.choice(E, size=4, replace=False)]
    loaded = np.zeros(E, np.int32)
    for e, _, _ in members:
        loaded[e] += 1
    lru = M.GoLRU(0)
    with epp.Engine(E, spec) as eng:
        for m in range(n_models):
            eng.register_model(b"adapter-%d" % m)
        eng.pool_set(np.arange(E, dtype=np.uint32), role, kv, waiting, running)
        eng.pool_set_lora(np.arange(E, dtype=np.uint32), max_active, loaded, members)
        for b in range(3):
            total = np.full(R, 8, np.int32)
            match = np.zeros((R, E), np.int32)
            for r in range(R):
                if r % 2:
                    hold = rng.choice(E, size=2, replace=False)
                    match[r, hold] = rng.integers(1, 9, size=2)
            mids = rng.integers(0, n_models, R).astype(np.uint32)
            keys = lru.keys()
            (dec, _), names = helpers.kernels_launched(lambda: eng.schedule_with_match(match, total, model_ids=mids),
                                                       repeatable=False)
            cold_picks = []
            for r in range(R):
                cold = M.is_cold(range(E), match[r])
                col = M.cold_column(list(range(E)), keys, E) if cold else np.full(E, 0.5)
                pool = orc.PoolState(role, kv, waiting, running, ext=col.reshape(1, E))
                st = np.zeros(E, np.uint8)
                for e, m, s in members:
                    if m == mids[r] and (st[e] == 0 or s == 1):
                        st[e] = s
                pool.set_lora(st, max_active, loaded)
                _, mx, pick, _ = orc.profile_run(orc.make_profile(0, scorers + [(4, 1.0, 0.0)]), pool, match[r],
                                                 int(total[r]))
                assert int(dec["pick"][r]) == pick and dec["score"][r] == mx, f"batch {b} request {r}"
                if cold:
                    cold_picks.append(pick)
            assert cold_picks
            for e in cold_picks:
                lru.add(e)
            assert eng.nohit_lru_get() == lru.keys(), f"LRU after batch {b}"
