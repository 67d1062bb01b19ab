"""GPU parity of the general profile evaluation (csrc/pick_general.cuh) vs the CPU oracle and the reference's own KATs:
the k best endpoints of the max-score picker (picker/maxscore/picker.go:87-115) and the prefix-cache-affinity-filter
(filter/prefixcacheaffinity/plugin.go:105-151).  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

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


def _pack(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    return np.frombuffer(b"".join(prompts), dtype=np.uint8).copy(), offs


def _lists_as_int(lists):
    out = {}
    for k, v in lists.items():
        v = np.asarray(v.cpu() if hasattr(v, "cpu") else v)
        if k.endswith("scores"):
            out[k] = v
        else:
            v = v.astype(np.int64) & 0xFFFFFFFF
            v[v == NO] = -1
            out[k] = v
    return out


# ------------------------------------------------------------------------------------------------
# KATs of picker/maxscore/picker_test.go:30-128 (TestPickMaxScorePicker)
# ------------------------------------------------------------------------------------------------
PICKER_KATS = [
    # name, k, scores of pod1..pod3, expected order (slot ids), number of tie-break candidates at the head
    ("Single max score", 1, [10, 25, 15], [1], 0),
    ("Multiple max scores, all are equally scored", 2, [50, 50, 30], [0, 1], 2),
    ("Multiple results sorted by highest score, more pods than needed", 2, [20, 25, 30], [2, 1], 0),
    ("Multiple results sorted by highest score, less pods than needed", 4, [20, 25, 30], [2, 1, 0], 0),
    ("Multiple results sorted by highest score, num of pods exactly needed", 3, [30, 25, 30], [0, 2, 1], 2),
]


@pytest.mark.parametrize("tie_seed", [0, 77])
@pytest.mark.parametrize("name,k,scores,want,n_tie", PICKER_KATS, ids=[c[0] for c in PICKER_KATS])
def test_reference_TestPickMaxScorePicker(epp, name, k, scores, want, n_tie, tie_seed):
    """The scores are injected through an external scorer column (score / 100, weight 1)."""
    E = 3
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(4, 1.0, 0.0)]), n_ext_cols=1, pick_k=k, tie_seed=tie_seed) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E), np.zeros(E, np.uint8), np.zeros(E), np.zeros(E, np.int32), ext=np.array([scores]) / 100.0)
        match, total = np.zeros((1, E), np.int32), np.zeros(1, np.int32)
        if k == 1:
            dec, det = eng.schedule_with_match(match, total)
            got = [int(dec["pick"][0])]
        else:
            dec, det, lists = eng.schedule_with_match(match, total, topk=True)
            row = _lists_as_int(lists)["primary"][0]
            got = [int(x) for x in row if x >= 0]
            assert int(dec["pick"][0]) == got[0]
            np.testing.assert_array_equal(lists["primary_scores"][0][: len(got)], np.array([scores[e] for e in got]) / 100.0)
            assert (row[len(got):] == -1).all()
        assert len(got) == len(want)
        assert sorted(got[:n_tie]) == sorted(want[:n_tie])          # random order inside the tied head
        assert got[n_tie:] == want[n_tie:]
        if n_tie and tie_seed == 0:
            assert got[:n_tie] == sorted(want[:n_tie])              # deterministic mode: ascending slots


# ------------------------------------------------------------------------------------------------
# KATs of filter/prefixcacheaffinity/plugin_test.go:50-118
# ------------------------------------------------------------------------------------------------
AFFINITY_KATS = [
    # name, (threshold, exploration, maxTTFTPenaltyMs), [(prefixMatch of 100, ttft)], endpoints kept
    ("AffinityThresholdDisabled", (0.0, 0.0, 0.0), [(0, 10), (90, 20)], 2),
    ("SingleEndpoint", (0.80, 0.0, 0.0), [(90, 10)], 1),
    ("NoStickyEndpoints", (0.80, 0.0, 0.0), [(10, 10), (20, 20), (50, 30)], 3),
    ("NarrowToSticky", (0.80, 0.0, 5000.0), [(90, 100), (85, 120), (10, 50)], 2),
    ("TTFTPenaltyBreaksStickiness", (0.80, 0.0, 100.0), [(90, 500), (10, 50)], 2),
    ("ExplorationProbability", (0.80, 1.0, 0.0), [(90, 100), (10, 50)], 2),
]


@pytest.mark.parametrize("name,cfg,eps,kept", AFFINITY_KATS, ids=[c[0] for c in AFFINITY_KATS])
def test_reference_affinity_filter_kats(epp, orc, name, cfg, eps, kept):
    """A profile with NO scorer scores every surviving candidate 0.0, so tie_count is the size of the filtered set."""
    E = len(eps)
    spec = epp.ProfileSpec(0, [], affinity=epp.AffinityFilterSpec(cfg[0], cfg[1], cfg[2], ttft_column=0))
    with epp.Engine(E, spec, n_ext_cols=1, tie_seed=5) as eng:
        eng.register_model(b"m")
        ttft = np.array([[t for _, t in eps]], dtype=np.float64)
        eng.pool_set(np.arange(E), np.zeros(E, np.uint8), np.zeros(E), np.zeros(E, np.int32), ext=ttft)
        match = np.array([[m for m, _ in eps]], np.int32)
        dec, det = eng.schedule_with_match(match, np.array([100], np.int32))
        assert int(dec["tie_count"][0]) == kept, name
        pool = orc.PoolState(np.zeros(E, np.uint8), np.zeros(E), np.zeros(E, np.int32), ext=ttft)
        prof = orc.make_profile(0, [], affinity=(cfg[0], cfg[1], cfg[2], 0))
        picks, _, ties, _ = orc.profile_run_topk(prof, pool, match[0], 100, 1, tie_seed=5, tie_key=0)
        assert ties == kept and picks == [int(dec["pick"][0])]


def test_affinity_config_validation(epp):
    """Config.validate, plugin.go:87-98."""
    for bad in (epp.AffinityFilterSpec(1.5), epp.AffinityFilterSpec(0.8, -0.1), epp.AffinityFilterSpec(0.8, 1.1),
                epp.AffinityFilterSpec(0.8, 0.01, -1.0), epp.AffinityFilterSpec(0.8, 0.01, 10.0, ttft_column=3)):
        with pytest.raises(epp.EngineError):
            epp.Engine(4, epp.ProfileSpec(0, [epp.ScorerSpec(0, 1.0)], affinity=bad))
    with epp.Engine(4, epp.ProfileSpec(0, [epp.ScorerSpec(0, 1.0)], affinity=epp.AffinityFilterSpec()), pick_k=2) as eng:
        with pytest.raises(epp.EngineError):
            eng.shard_set(0, 2)                     # neither feature exists in the endpoint-sharded mode
    with epp.Engine(4, epp.ProfileSpec(0, [epp.ScorerSpec(0, 1.0)])) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(4), np.zeros(4, np.uint8), np.zeros(4), np.zeros(4, np.int32))
        with pytest.raises(epp.EngineError):
            eng.schedule_with_match(np.zeros((1, 4), np.int32), np.zeros(1, np.int32), topk=True)   # pick_k <= 1


# ------------------------------------------------------------------------------------------------
# whole cycle vs the oracle
# ------------------------------------------------------------------------------------------------
def _workload(orc, rng, E, bst, B, n_req, holders=(2, 5, 9, 20, 40)):
    fam = [bytes(rng.integers(0, 256, 4 * bst * B, dtype=np.uint8)) for _ in range(len(holders))]
    pairs_h, pairs_e = [], []
    for g, p in enumerate(fam):
        h = orc.hash_prompt(p, b"m", bst, B)
        for e in rng.choice(E, size=holders[g], replace=False):
            depth = int(rng.choice([len(h) // 2, (3 * len(h)) // 4, len(h)]))
            pairs_h += h[:depth]
            pairs_e += [int(e)] * depth
    prompts = []
    for _ in range(n_req):
        g = int(rng.integers(0, len(fam) + 1))
        if g >= len(fam):
            prompts.append(bytes(rng.integers(0, 256, 4 * bst * B, dtype=np.uint8)))
        else:
            keep = int(rng.integers(1, B + 1)) * 4 * bst
            prompts.append(fam[g][:keep] + bytes(rng.integers(0, 256, 4 * bst * B - keep, dtype=np.uint8)))
    return pairs_h, pairs_e, prompts


@pytest.mark.parametrize("tie_seed", [0, 0xC0FFEE])
def test_topk_vs_oracle(epp, orc, tie_seed):
    """pick_k = 5 on a pool with few load levels (large groups of equal scores), disagg handler with an encode stage:
    the three lists of every request equal the oracle's, through host and device batches; list[0] is the pick."""
    import helpers
    import torch
    E, bst, B, K, R = 96, 2, 16, 5, 300
    rng = np.random.default_rng(51)
    kv = rng.integers(0, 3, E) / 3.0
    waiting = rng.integers(0, 2, E).astype(np.int32)
    role = rng.choice([1, 2, 3, 5, 7, 0], size=E).astype(np.uint8)
    prim = [(2, 1.0, 0), (1, 1.0, 0), (0, 2.0, 0)]
    pref = [(2, 1.0, 0), (0, 1.0, 0)]
    enc = [(1, 1.0, 0)]
    spec = lambda f, sc: epp.ProfileSpec(f, [epp.ScorerSpec(k, w, p) for k, w, p in sc])
    pairs_h, pairs_e, prompts = _workload(orc, rng, E, bst, B, R)
    d, offs = _pack(prompts)
    mm = (rng.random(R) < 0.5).astype(np.uint8)
    with epp.Engine(E, spec(1, prim), spec(2, pref), block_size_tokens=bst, max_prefix_blocks=B, non_cached_tokens=4,
                    encode=spec(3, enc), pick_k=K, tie_seed=tie_seed) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E), role, kv, waiting)
        eng.index_load_snapshot(pairs_h, pairs_e)
        ix = orc.Indexer()
        ix.load_pairs(pairs_h, pairs_e)
        pool = orc.PoolState(role, kv, waiting)
        for batch in range(2):
            base = eng.stats()["n_decisions"]
            dec, det, lists = eng.schedule(d, offsets=offs, multimodal=mm, topk=True)
            odec, ototal, olists = orc.cycle_batch(b"m", bst, B, 4, False, ix, orc.make_profile(1, prim), orc.make_profile(2, pref),
                                                   pool, d, offs, 2, tie_seed=tie_seed, tie_base=base,
                                                   encode=orc.make_profile(3, enc), multimodal=mm, topk=K)
            helpers.assert_decisions_equal(dec, det, odec, ototal, where=f"top-k batch {batch}")
            got = _lists_as_int(lists)
            for name in ("primary", "prefill", "encode"):
                np.testing.assert_array_equal(got[name], olists[name], err_msg=name)
            np.testing.assert_array_equal(got["primary_scores"].view(np.uint64), olists["primary_scores"].view(np.uint64))
            ok = dec["status"] == 0
            np.testing.assert_array_equal(got["primary"][ok, 0], dec["pick"][ok].astype(np.int64))
            pf = dec["prefill_pick"].astype(np.int64); pf[pf == NO] = -1
            np.testing.assert_array_equal(got["prefill"][:, 0], pf)
            en = det["encode_pick"].astype(np.int64); en[en == NO] = -1
            np.testing.assert_array_equal(got["encode"][:, 0], en)
            assert (got["primary"][ok] >= 0).all() and (got["prefill"][:, 1] >= 0).any() and (got["encode"][:, 1] >= 0).any()
            for r in np.nonzero(ok)[0][:50]:                     # a list never repeats an endpoint
                row = got["primary"][r]
                assert len(set(row.tolist())) == K
        # the same batch through device pointers (the ordinals moved on, so compare against a fresh oracle run)
        base = eng.stats()["n_decisions"]
        dd, do = torch.from_numpy(d).cuda(), torch.from_numpy(offs.view(np.int64)).cuda()
        ddec, ddet, dlists = eng.schedule(dd, offsets=do, multimodal=torch.from_numpy(mm).cuda(), topk=True)
        torch.cuda.synchronize()
        odec, ototal, olists = orc.cycle_batch(b"m", bst, B, 4, False, ix, orc.make_profile(1, prim), orc.make_profile(2, pref),
                                               pool, d, offs, 2, tie_seed=tie_seed, tie_base=base,
                                               encode=orc.make_profile(3, enc), multimodal=mm, topk=K)
        helpers.assert_decisions_equal(epp.decisions_from_torch(ddec), ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1),
                                       odec, ototal, where="top-k device batch")
        got = _lists_as_int(dlists)
        for name in ("primary", "prefill", "encode"):
            np.testing.assert_array_equal(got[name], olists[name], err_msg="device " + name)
        # plain epp_schedule on a pick_k > 1 engine: the pick alone, same rule
        base = eng.stats()["n_decisions"]
        dec1, det1 = eng.schedule(d, offsets=offs, multimodal=mm)
        odec1, ototal1 = orc.cycle_batch(b"m", bst, B, 4, False, ix, orc.make_profile(1, prim), orc.make_profile(2, pref),
                                         pool, d, offs, 2, tie_seed=tie_seed, tie_base=base,
                                         encode=orc.make_profile(3, enc), multimodal=mm)
        helpers.assert_decisions_equal(dec1, det1, odec1, ototal1, where="pick only on a top-k engine")


@pytest.mark.parametrize("tie_seed", [0, 0xABCD])
def test_affinity_filter_vs_oracle(epp, orc, tie_seed):
    """Affinity filter on the decode profile (threshold 0.5, exploration 0.3, TTFT gate 40 ms on an ext column) in front
    of queue / running / active-request / prefix scorers, whose normalisation must follow the narrowed set; the prefill
    profile keeps the plain evaluation.  Every outcome of the filter occurs in the batch."""
    import helpers
    E, bst, B, R = 96, 2, 16, 500
    rng = np.random.default_rng(61)
    kv = rng.integers(0, 4, E) / 4.0
    waiting = rng.integers(0, 6, E).astype(np.int32)
    running = rng.integers(0, 9, E).astype(np.int32)
    role = np.where(np.arange(E) % 4 == 0, 2, 1).astype(np.uint8)
    ext = np.stack([rng.integers(0, 100, E).astype(np.float64),          # column 0: predicted TTFT (ms)
                    rng.integers(0, 12, E).astype(np.float64)])          # column 1: in-flight requests
    prim = [(2, 1.0, 0), (5, 1.0, 0), (7, 1.0, 1.0, 1, 2.0), (1, 1.0, 0), (0, 2.0, 0)]
    pref = [(2, 1.0, 0), (0, 1.0, 0)]
    aff = (0.5, 0.3, 40.0, 0)
    pairs_h, pairs_e, prompts = _workload(orc, rng, E, bst, B, R)
    d, offs = _pack(prompts)
    pspec = epp.ProfileSpec(1, [epp.ScorerSpec(2, 1.0), epp.ScorerSpec(5, 1.0), epp.ScorerSpec(7, 1.0, 1.0, 1, 2.0),
                                epp.ScorerSpec(1, 1.0), epp.ScorerSpec(0, 2.0)],
                            affinity=epp.AffinityFilterSpec(*aff))
    with epp.Engine(E, pspec, epp.ProfileSpec(2, [epp.ScorerSpec(2, 1.0), epp.ScorerSpec(0, 1.0)]), block_size_tokens=bst,
                    max_prefix_blocks=B, non_cached_tokens=4, n_ext_cols=2, tie_seed=tie_seed) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E), role, kv, waiting, running, ext=ext)
        eng.index_load_snapshot(pairs_h, pairs_e)
        ix = orc.Indexer()
        ix.load_pairs(pairs_h, pairs_e)
        pool = orc.PoolState(role, kv, waiting, running, ext=ext)
        oprim = orc.make_profile(1, prim, affinity=aff)
        oplain = orc.make_profile(1, prim)
        opref = orc.make_profile(2, pref)
        base = eng.stats()["n_decisions"]
        dec, det = eng.schedule(d, offsets=offs)
        odec, ototal = orc.cycle_batch(b"m", bst, B, 4, False, ix, oprim, opref, pool, d, offs, 2, tie_seed=tie_seed, tie_base=base)
        helpers.assert_decisions_equal(dec, det, odec, ototal, where="affinity filter")
        plain, _ = orc.cycle_batch(b"m", bst, B, 4, False, ix, oplain, opref, pool, d, offs, 2, tie_seed=tie_seed, tie_base=base)
        changed = (plain["pick"] != odec["pick"]) | (plain["score"] != odec["score"])
        assert changed.sum() > 20                     # the filter matters on this workload ...
        assert (~changed).sum() > 20                  # ... and does not always narrow (no sticky endpoint / gate / exploration)
        # device-pointer batch: same kernel path, ordinals moved on
        import torch
        base = eng.stats()["n_decisions"]
        ddec, ddet = eng.schedule(torch.from_numpy(d).cuda(), offsets=torch.from_numpy(offs.view(np.int64)).cuda())
        torch.cuda.synchronize()
        odec2, ototal2 = orc.cycle_batch(b"m", bst, B, 4, False, ix, oprim, opref, pool, d, offs, 2, tie_seed=tie_seed, tie_base=base)
        helpers.assert_decisions_equal(epp.decisions_from_torch(ddec), ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1),
                                       odec2, ototal2, where="affinity filter, device batch")
        # injected match rows (dense pick kernel)
        match = (rng.integers(0, 5, size=(64, E)) * 4).astype(np.int32)
        match[:, rng.random(E) < 0.7] = 0
        base = eng.stats()["n_decisions"]
        dec3, det3 = eng.schedule_with_match(match, np.full(64, B, np.int32), input_len_bytes=np.full(64, 8 * B, np.int64))
        for r in range(64):
            picks, scores, ties, _ = orc.profile_run_topk(oprim, pool, match[r], B, 1, tie_seed=tie_seed, tie_key=4 * (base + r))
            assert picks == [int(dec3["pick"][r])] and ties == int(dec3["tie_count"][r])
            assert np.float64(scores[0]).view(np.uint64) == dec3["score"][r].view(np.uint64)


def test_mirror_scheduler_with_affinity_filter_and_two_targets(epp):
    """Through the reference-interface mirror (plugins.py), written like filter/prefixcacheaffinity/plugin_test.go:
    endpoints a / b hold 90 % / 85 % of the prompt, c 10 %; the filter narrows to {a, b}, the queue scorer then
    normalises over those two only (b has the shorter queue), and the picker returns both in score order."""
    P = epp.plugins
    def make_endpoint(name, prefix_match, waiting):
        ep = P.NewEndpoint(P.EndpointMetadata(name), P.Metrics(WaitingQueueSize=waiting))
        ep.Put(P.PrefixCacheMatchInfoKey, P.NewPrefixCacheMatchInfo(prefix_match, 100, 16))
        return ep
    endpoints = [make_endpoint("a", 90, 7), make_endpoint("b", 85, 3), make_endpoint("c", 10, 0)]
    profile = P.NewSchedulerProfile().WithFilters(P.PrefixCacheAffinityFilter(0.80, 0.0, 5000.0)) \
        .WithScorers(P.NewWeightedScorer(P.QueueScorer(), 1.0)).WithPicker(P.NewMaxScorePicker(2))
    sched = P.Scheduler(P.SingleProfileHandler(), {"default": profile}, max_endpoints=3)
    got = sched.Schedule(P.InferenceRequest(RequestID="r", TargetModel="m", Prompt=b"x" * 64), endpoints)
    res = got.ProfileResults["default"]
    assert [e.GetMetadata().Name for e in res.TargetEndpoints] == ["b", "a"]
    assert res.Score == 1.0 and res.TieCount == 1
    # without the filter c (empty queue) wins and b, a follow
    plain = P.NewSchedulerProfile().WithScorers(P.NewWeightedScorer(P.QueueScorer(), 1.0)).WithPicker(P.NewMaxScorePicker(3))
    got = P.Scheduler(P.SingleProfileHandler(), {"default": plain}, max_endpoints=3).Schedule(
        P.InferenceRequest(RequestID="r", TargetModel="m", Prompt=b"x" * 64), endpoints)
    assert [e.GetMetadata().Name for e in got.ProfileResults["default"].TargetEndpoints] == ["c", "b", "a"]
