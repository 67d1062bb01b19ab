"""The random-picker and the weighted-random-picker on the device, bit for bit against the CPU oracle's scores and the
draw restated in tools/picker_model.py: the sparse kernel (host, device and pipelined async batches), its > 32-holder
overflow pass (k_match_pick), the small-batch kernel (DMA and zero-copy), injected match rows (k_dense_pick), the
no-hit-lru build, P/D with a different picker per profile, and the affinity filter (gen::eval).  Every call proves from
its profiler trace that the kernel it is about ran.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import helpers
from helpers import assert_ran
from oracle import pyoracle as O
from tools import picker_model as PM

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
BST, B = 8, 12                      # 32-byte blocks: small host batches take k_cycle_small
BB = 4 * BST
L = BB * B
QUEUE, KV, PREFIX, NO_HIT = 2, 1, 0, 9
SEED = 0x5EED


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


class World:
    """E endpoints (some outside the pool), prompt families with hand-placed holders: family 0 has 40 holders (the
    sparse map overflows), the others a few at chosen depths; a share of cold prompts."""

    def __init__(self, E=70, R=1100, seed=1):
        rng = np.random.default_rng(seed)
        self.E, self.R = E, R
        self.ids = np.array([e for e in range(E) if e % 11 != 5], np.uint32)
        self.role = np.full(E, 0xFF, np.uint8)
        self.role[self.ids] = 0
        self.kv = rng.random(E).round(2)
        self.waiting = rng.integers(0, 6, E).astype(np.int32)
        self.running = np.zeros(E, np.int32)
        fams = [rng.integers(0, 256, L, dtype=np.uint8) for _ in range(6)]
        holders = [[(int(e), 2) for e in range(0, 40)],
                   [(0, 12), (69, 5)], [(33, 3), (34, 3), (35, 8)], [(64, 1)], [(1, 12)], [(68, 6), (2, 6)]]
        toks = rng.integers(0, 256, (R, L), dtype=np.uint8)
        kind = rng.integers(-1, len(fams), R)
        for r in range(R):
            if kind[r] >= 0:
                n = int(rng.integers(1, B + 1)) * BB
                toks[r, :n] = fams[kind[r]][:n]
        self.tokens = toks
        self.fams, self.holders = fams, holders

    def load(self, eng):
        eng.register_model(b"m")                       # model 0 of every request
        eng.pool_set(self.ids, self.role[self.ids], self.kv[self.ids], self.waiting[self.ids], self.running[self.ids])
        fam = np.stack(self.fams)
        h, _ = eng.hash_prompts(fam, uniform_len=L)
        hs, es = [], []
        for g, hl in enumerate(self.holders):
            for e, depth in hl:
                hs += [int(x) for x in h[g][:depth]]
                es += [e] * depth
        eng.index_load_snapshot(np.array(hs, np.uint64), np.array(es, np.uint32))

    def pool(self):
        return O.PoolState(self.role, self.kv, self.waiting, self.running)


def scorers(weights=(2.0, 2.0, 3.0)):
    return [(QUEUE, weights[0], 0.0), (KV, weights[1], 0.0), (PREFIX, weights[2], 0.0)]


def expect_profile(w, sc, picker, match_row, total, seed, key, filt=0):
    prof = O.make_profile(filt, sc)
    pool = w.pool()
    scores, _, _, _ = O.profile_run(prof, pool, match_row, total)
    base, _, _, _ = O.profile_run(prof, pool, np.zeros(w.E, np.int32), total)
    cands = [e for e in range(w.E) if O.lib().orc_role_filter_keeps(filt, int(w.role[e])) and w.role[e] != 0xFF]
    explicit = {e for e in cands if match_row[e] > 0}
    return PM.draw(picker, cands, base, scores, explicit, seed, key, [s[1] for s in sc])


def check(dec, det, w, match, total, specs, seed, ordinal0, where, in_len=None, always=False):
    """specs: [(scorers, picker)] of decode [, prefill]."""
    for r in range(len(dec)):
        key = 4 * (ordinal0 + r)
        sc, pk = specs[0]
        pick, score, n = expect_profile(w, sc, pk, match[r], int(total[r]), seed, key)
        d = dec[r]
        assert d["status"] == 0 and int(d["pick"]) == pick, (where, r, int(d["pick"]), pick)
        assert np.float64(d["score"]).tobytes() == np.float64(score).tobytes(), (where, r, d["score"], score)
        assert int(d["tie_count"]) == n and int(d["match_blocks"]) == int(match[r][pick]), (where, r)
        if len(specs) > 1 and always:
            sc1, pk1 = specs[1]
            p1, s1, n1 = expect_profile(w, sc1, pk1, match[r], int(total[r]), seed, key + 1)
            assert int(d["prefill_pick"]) == p1, (where, r, "prefill")
            assert np.float64(det[r]["prefill_score"]).tobytes() == np.float64(s1).tobytes()
            assert int(det[r]["prefill_tie_count"]) == n1


def decisions(epp, t):
    return t.cpu().numpy().view(epp.DECISION_DTYPE).reshape(-1)


@pytest.mark.parametrize("picker", [PM.RANDOM, PM.WEIGHTED_RANDOM])
@pytest.mark.parametrize("seed", [0, SEED])
def test_every_path_matches_the_model(epp, picker, seed):
    import torch
    w = World()
    sc = scorers()
    spec = epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, p) for k, wt, p in sc], picker=picker)
    with epp.Engine(w.E, spec, block_size_tokens=BST, max_prefix_blocks=B, tie_seed=seed) as eng:
        w.load(eng)
        match, total = eng.prefix_match(w.tokens, uniform_len=L)
        assert (np.count_nonzero(match > 0, axis=1) > 32).any(), "no request overflows the sparse map"
        # host batch above the small-batch limit: k_match_pick_sparse_rand + the overflow pass
        o0 = eng.stats()["n_decisions"]
        (dec, det), names = helpers.kernels_launched(lambda: eng.schedule(w.tokens, uniform_len=L), repeatable=False)
        assert_ran(names, "k_match_pick_sparse_rand", absent=("k_match_pick_sparse<",), where="host batch")
        assert_ran(names, "k_match_pick_rand(", where="overflow pass")
        check(dec, det, w, match, total, [(sc, picker)], seed, o0, "host")
        # device batch and three pipelined async batches
        dt = torch.from_numpy(w.tokens).cuda()
        o0 = eng.stats()["n_decisions"]
        d = decisions(epp, eng.schedule(dt, uniform_len=L)[0])
        check(d, None, w, match, total, [(sc, picker)], seed, o0, "device")
        o0 = eng.stats()["n_decisions"]
        outs = [eng.schedule(dt, uniform_len=L, asynchronous=True)[0] for _ in range(3)]
        eng.synchronize()
        for i, t in enumerate(outs):
            check(decisions(epp, t), None, w, match, total, [(sc, picker)], seed, o0 + i * w.R, f"async {i}")
        # small batches: zero-copy (<= 8) and DMA
        for n in (5, 300):
            o0 = eng.stats()["n_decisions"]
            (dec, det), names = helpers.kernels_launched(lambda: eng.schedule(w.tokens[:n].copy(), uniform_len=L),
                                                         repeatable=False)
            assert_ran(names, "k_cycle_small_rand", where=f"small {n}")
            check(dec, det, w, match[:n], total[:n], [(sc, picker)], seed, o0, f"small {n}")
        # injected match rows
        o0 = eng.stats()["n_decisions"]
        (dec, det), names = helpers.kernels_launched(lambda: eng.schedule_with_match(match, total), repeatable=False)
        assert_ran(names, "k_dense_pick_rand", where="with_match")
        check(dec, det, w, match, total, [(sc, picker)], seed, o0, "with_match")


def test_pd_with_a_picker_per_profile(epp):
    w = World(R=600, seed=3)
    sc0, sc1 = scorers((1.0, 0.5, 4.0)), scorers((0.0, 1.0, 1.0))
    dec_spec = epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, p) for k, wt, p in sc0], picker=PM.WEIGHTED_RANDOM)
    pre_spec = epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, p) for k, wt, p in sc1], picker=PM.RANDOM)
    with epp.Engine(w.E, dec_spec, pre_spec, block_size_tokens=BST, max_prefix_blocks=B, tie_seed=SEED,
                    always_disagg=True) as eng:
        w.load(eng)
        match, total = eng.prefix_match(w.tokens, uniform_len=L)
        for name, fn in (("sparse", lambda: eng.schedule(w.tokens, uniform_len=L)),
                         ("small", lambda: eng.schedule(w.tokens[:7].copy(), uniform_len=L)),
                         ("with_match", lambda: eng.schedule_with_match(match, total))):
            o0 = eng.stats()["n_decisions"]
            dec, det = fn()
            n = len(dec)
            check(dec, det, w, match[:n], total[:n], [(sc0, PM.WEIGHTED_RANDOM), (sc1, PM.RANDOM)], SEED, o0, name,
                  always=True)


def test_affinity_filter_and_rejections(epp):
    w = World(R=500, seed=5)
    sc = scorers()
    aff = epp.AffinityFilterSpec(0.5, 0.0, 0.0, -1)
    for picker in (PM.RANDOM, PM.WEIGHTED_RANDOM):
        spec = epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, p) for k, wt, p in sc], aff, picker)
        with epp.Engine(w.E, spec, block_size_tokens=BST, max_prefix_blocks=B, tie_seed=SEED) as eng:
            w.load(eng)
            match, total = eng.prefix_match(w.tokens, uniform_len=L)
            o0 = eng.stats()["n_decisions"]
            dec, _ = eng.schedule_with_match(match, total)
            prof = O.make_profile(0, sc, (0.5, 0.0, 0.0))
            pool = w.pool()
            for r in range(w.R):
                scores, _, _, _ = O.profile_run(prof, pool, match[r], int(total[r]))
                cands = [e for e in range(w.E) if w.role[e] != 0xFF and scores[e] != -1.0]   # -1.0: filtered out
                narrowed = len(cands) < len(w.ids)
                if narrowed:
                    want = PM.draw(picker, cands, None, scores, set(cands), SEED, 4 * (o0 + r), [s[1] for s in sc], gaps=False)
                else:
                    want = expect_profile(w, sc, picker, match[r], int(total[r]), SEED, 4 * (o0 + r))
                assert int(dec[r]["pick"]) == want[0], (picker, r)
                assert np.float64(dec[r]["score"]).tobytes() == np.float64(want[1]).tobytes()
                assert int(dec[r]["tie_count"]) == want[2]
            with pytest.raises(epp.EngineError):
                eng.shard_set(0, w.E)
    with pytest.raises(epp.EngineError):
        epp.Engine(8, epp.ProfileSpec(0, [], picker=3))


def test_frequencies_follow_the_scores(epp):
    """One large batch of cold requests: every request sees the same scores (epp_score rows), so the pick counts of the
    weighted picker follow s_i / W, and those of the random picker are uniform."""
    from scipy.stats import chisquare
    E, R = 40, 60000
    rng = np.random.default_rng(9)
    for picker in (PM.WEIGHTED_RANDOM, PM.RANDOM):
        spec = epp.ProfileSpec(0, [epp.ScorerSpec(QUEUE, 1.0, 0.0), epp.ScorerSpec(KV, 3.0, 0.0)], picker=picker)
        with epp.Engine(E, spec, block_size_tokens=BST, max_prefix_blocks=B, tie_seed=SEED) as eng:
            kv = rng.random(E)
            kv[:5] = 1.0                                           # some endpoints score 0 on the kv term
            eng.register_model(b"m")
            eng.pool_set(np.arange(E, dtype=np.uint32), [0] * E, kv, rng.integers(0, 9, E).astype(np.int32), [0] * E)
            match, total = np.zeros((1, E), np.int32), np.zeros(1, np.int32)
            s = eng.score(match, total)[0]
            dec, _ = eng.schedule(rng.integers(0, 256, (R, L), dtype=np.uint8), uniform_len=L)
            counts = np.bincount(dec["pick"].astype(np.int64), minlength=E)
            p = np.maximum(s, 0) / np.maximum(s, 0).sum() if picker == PM.WEIGHTED_RANDOM else np.full(E, 1.0 / E)
            keep = p > 0
            assert counts[~keep].sum() == 0
            assert chisquare(counts[keep], R * p[keep] / p[keep].sum()).pvalue > 1e-4


def _spec(epp, sc, picker, aff=None):
    return epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, p) for k, wt, p in sc], aff, picker)


def _base_score(w, sc, match_row, total, aff=None):
    prof = O.make_profile(0, sc, aff)
    pool = w.pool()
    scores, _, _, _ = O.profile_run(prof, pool, match_row, total)
    base, _, _, _ = O.profile_run(O.make_profile(0, sc), pool, np.zeros(w.E, np.int32), total)
    return scores, base


@pytest.mark.parametrize("picker", [PM.RANDOM, PM.WEIGHTED_RANDOM])
def test_first_k_lists(epp, picker):
    """pick_k > 1 (gen::eval on the dense-counter and injected-match kernels): successive draws without replacement, up
    to 64 and past the positive set, with and without a narrowing affinity filter."""
    w = World(R=300, seed=11)
    sc = scorers((2.0, 0.0, 3.0))                          # kv weight 0: plenty of candidates score 0 when cold
    for k, aff in ((64, None), (5, (0.5, 0.0, 0.0))):
        spec = _spec(epp, sc, picker, epp.AffinityFilterSpec(*aff, -1) if aff else None)
        with epp.Engine(w.E, spec, block_size_tokens=BST, max_prefix_blocks=B, tie_seed=SEED, pick_k=k) as eng:
            w.load(eng)
            match, total = eng.prefix_match(w.tokens, uniform_len=L)
            for name, fn in (("with_match", lambda: eng.schedule_with_match(match, total, topk=True)),
                             ("schedule", lambda: eng.schedule(w.tokens, uniform_len=L, topk=True))):
                o0 = eng.stats()["n_decisions"]
                dec, _, lists = fn()
                for r in range(w.R):
                    scores, base = _base_score(w, sc, match[r], int(total[r]), aff)
                    cands = [e for e in range(w.E) if w.role[e] != 0xFF and scores[e] != -1.0]
                    narrowed = len(cands) < len(w.ids)
                    explicit = set(cands) if narrowed else {e for e in cands if match[r][e] > 0}
                    want = PM.draw_k(picker, cands, base, scores, explicit, SEED, 4 * (o0 + r), [s[1] for s in sc], k,
                                     gaps=not narrowed)
                    got = [int(x) for x in lists["primary"][r]]
                    assert got[:len(want)] == [p for p, _ in want], (name, k, r)
                    assert all(x == NO for x in got[len(want):])
                    gs = np.asarray(lists["primary_scores"][r][:len(want)], np.float64)
                    assert gs.tobytes() == np.array([s for _, s in want], np.float64).tobytes(), (name, k, r)
                    assert int(dec[r]["pick"]) == want[0][0] and int(dec[r]["tie_count"]) == len(cands)


class _NoHitPickerModel:
    """tools/nohit_lru_model.Model with the profile's picker in place of max-score: the scores and the bases (match 0)
    of the warm or cold set, then the draw of tools/picker_model.py."""

    def __init__(self, M, picker, *a, **kw):
        base = M.Model

        class Model(base):
            def run_profile(self, pi, match_row, total, key, lru_keys):
                filt, scs = self.profiles[pi]
                cand = self.candidates(filt)
                if not cand:
                    return NO, 0.0, 0, None
                cold = M.is_cold(cand, match_row)
                mask = np.zeros(self.E, dtype=np.uint8)
                mask[cand] = 1
                idx = np.asarray(cand)

                def fold(mrow):
                    acc = np.zeros(self.E, np.float64)
                    for s, sc in enumerate(scs):
                        if sc[0] == M.NO_HIT_LRU:
                            col = M.cold_column(cand, lru_keys, self.E) if cold else np.full(self.E, 0.5)
                        elif sc[0] == 0:
                            col = (np.asarray(mrow, np.float64) / float(total)) if total else np.zeros(self.E)
                            col = np.minimum(np.maximum(col, 0.0), 1.0)
                        else:
                            col = self.column(pi, s, mask)
                        acc[idx] = acc[idx] + col[idx] * sc[1]
                    return acc

                score, base0 = fold(match_row), fold(np.zeros(self.E, np.int32))
                pick, s, n = PM.draw(picker, cand, base0, score, {e for e in cand if match_row[e] > 0}, self.tie_seed,
                                     key, [sc[1] for sc in scs])
                return pick, s, n, cold

        self.m = Model(*a, **kw)


def test_nohit_lru_with_a_weighted_picker(epp):
    """Several calls so that the LRU fills: the cold sets' cands / wcum / icum rebuilt after every update, read by
    eval_random_lanes (k_match_pick_sparse_rand, k_cycle_small_rand) -- pick and score bits against the model."""
    from tools import nohit_lru_model as M
    w = World(R=1100, seed=13)
    sc = scorers((1.0, 0.5, 4.0)) + [(NO_HIT, 2.0, 16.0)]
    with epp.Engine(w.E, _spec(epp, sc, PM.WEIGHTED_RANDOM), block_size_tokens=BST, max_prefix_blocks=B,
                    tie_seed=SEED) as eng:
        w.load(eng)
        model = _NoHitPickerModel(M, PM.WEIGHTED_RANDOM, O, w.pool(), w.E, [(0, sc)], 16, block_size_tokens=BST,
                                  tie_seed=SEED).m
        match, total = eng.prefix_match(w.tokens, uniform_len=L)
        assert ((match > 0).sum(axis=1) == 0).any()
        for call, (r0, r1, kern) in enumerate([(0, 1100, "k_match_pick_sparse_rand"), (0, 6, "k_cycle_small_rand"),
                                               (6, 400, "k_cycle_small_rand"), (0, 1100, "k_match_pick_sparse_rand"),
                                               (400, 405, "k_cycle_small_rand")]):
            model.n_decisions = eng.stats()["n_decisions"]
            want = model.schedule(match[r0:r1], total[r0:r1])
            (dec, _), names = helpers.kernels_launched(lambda: eng.schedule(w.tokens[r0:r1].copy(), uniform_len=L),
                                                       repeatable=False)
            assert_ran(names, kern, where=f"call {call}")
            for r, (st, pick, score, _, _, _) in enumerate(want):
                assert int(dec[r]["pick"]) == pick, (call, r)
                assert np.float64(dec[r]["score"]).tobytes() == np.float64(score).tobytes(), (call, r)
            assert eng.nohit_lru_get() == model.lru.keys(), call
        assert len(model.lru.keys()) > 4


def test_encode_stage_and_batcher(epp):
    """The encode profile (key + 2, its own candidate arrays) with a random picker, and a max_batch = 1 batcher."""
    w = World(R=400, seed=17)
    sc0, sc1, sc2 = scorers((1.0, 0.5, 4.0)), scorers((0.0, 1.0, 1.0)), scorers((3.0, 1.0, 0.5))
    mm = (np.arange(w.R) % 3 != 0).astype(np.uint8)
    with epp.Engine(w.E, _spec(epp, sc0, PM.RANDOM), _spec(epp, sc1, PM.MAX_SCORE), encode=_spec(epp, sc2, PM.WEIGHTED_RANDOM),
                    block_size_tokens=BST, max_prefix_blocks=B, tie_seed=SEED, always_disagg=True) as eng:
        w.load(eng)
        match, total = eng.prefix_match(w.tokens, uniform_len=L)
        for name, n in (("sparse", w.R), ("small", 7)):
            o0 = eng.stats()["n_decisions"]
            dec, det = eng.schedule(w.tokens[:n].copy(), uniform_len=L, multimodal=mm[:n])
            for r in range(n):
                key = 4 * (o0 + r)
                p0 = expect_profile(w, sc0, PM.RANDOM, match[r], int(total[r]), SEED, key)
                assert int(dec[r]["pick"]) == p0[0] and int(dec[r]["tie_count"]) == p0[2], (name, r)
                if mm[r]:
                    p2 = expect_profile(w, sc2, PM.WEIGHTED_RANDOM, match[r], int(total[r]), SEED, key + 2)
                    assert int(det[r]["encode_pick"]) == p2[0], (name, r)
                    assert np.float64(det[r]["encode_score"]).tobytes() == np.float64(p2[1]).tobytes()
                    assert int(det[r]["encode_tie_count"]) == p2[2]
                else:
                    assert int(det[r]["encode_pick"]) == NO
        o0 = eng.stats()["n_decisions"]
        with epp.Batcher(eng, max_batch=1, max_delay_us=0) as bt:
            for r in range(24):
                d, dd = bt.schedule(w.tokens[r].tobytes(), multimodal=bool(mm[r]))
                key = 4 * (o0 + r)
                p0 = expect_profile(w, sc0, PM.RANDOM, match[r], int(total[r]), SEED, key)
                assert int(d["pick"]) == p0[0], ("batcher", r)
                assert np.float64(d["score"]).tobytes() == np.float64(p0[1]).tobytes()
                if mm[r]:
                    p2 = expect_profile(w, sc2, PM.WEIGHTED_RANDOM, match[r], int(total[r]), SEED, key + 2)
                    assert int(dd["encode_pick"]) == p2[0], ("batcher encode", r)


def test_plugins_scheduler_with_the_pickers(epp):
    """plugins.SchedulerProfile.WithPicker(NewRandomPicker / NewWeightedRandomPicker) through Scheduler.Schedule."""
    P = epp.plugins
    assert P.NewRandomPicker(-3).maxNumOfEndpoints == 1 and P.NewWeightedRandomPicker(0).maxNumOfEndpoints == 1
    E = 12
    rng = np.random.default_rng(21)
    eps = [P.NewEndpoint(P.EndpointMetadata(f"pod{i}"), P.Metrics(int(rng.integers(0, 5)), round(float(rng.random()), 2)))
           for i in range(E)]
    for make, kind in ((P.NewRandomPicker, PM.RANDOM), (P.NewWeightedRandomPicker, PM.WEIGHTED_RANDOM)):
        prof = P.NewSchedulerProfile().WithScorers(P.NewWeightedScorer(P.QueueScorer(), 2.0),
                                                   P.NewWeightedScorer(P.KVCacheUtilizationScorer(), 1.0))
        prof = prof.WithPicker(make(1))
        assert prof.spec().picker == kind
        sched = P.Scheduler(P.SingleProfileHandler(), {"p": prof}, max_endpoints=E, tie_seed=SEED)
        reqs = [P.InferenceRequest(Prompt=bytes(40)) for _ in range(50)]
        res = sched.Schedule(reqs, eps)
        pool = O.PoolState(np.zeros(E, np.uint8), [e.metrics.KVCacheUsagePercent for e in eps],
                           [e.metrics.WaitingQueueSize for e in eps])
        sc = [(QUEUE, 2.0, 0.0), (KV, 1.0, 0.0)]
        scores, _, _, _ = O.profile_run(O.make_profile(0, sc), pool, np.zeros(E, np.int32), 0)
        for i, r in enumerate(res):
            want = PM.draw(kind, list(range(E)), scores, scores, set(), SEED, 4 * i, [2.0, 1.0])
            assert r.ProfileResults["p"].TargetEndpoints[0] is eps[want[0]], (kind, i)
            assert r.ProfileResults["p"].Score == want[1]
