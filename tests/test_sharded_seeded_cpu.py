"""Seeded ties in the endpoint-sharded mode without a GPU: sharded.resolve_records_host against a brute-force global
rank, the seeded protocol (three exchanges) over gloo at world 2 with the oracle standing in for each rank's kernels,
and the cases of test_sharded_seeded_gpu.py reaching the edges they name, from their builders and the oracle alone."""
import os

import numpy as np
import pytest

import test_sharded as T
import test_sharded_disagg_gpu as D
import test_sharded_landscapes_gpu as L
import test_sharded_seeded_gpu as SD

SEED = SD.SEED


def sh():
    return L.sharded()


# ------------------------------------------------------------------------------------------------
# resolve_records_host
# ------------------------------------------------------------------------------------------------
def records_of(scores, ranges):
    """Per-rank records of one stage from global scores ([R, E], NaN = not a candidate): local max, lowest tied slot,
    tied count."""
    R = scores.shape[0]
    recs = np.zeros((len(ranges), R), sh().SHARD_BEST_DTYPE)
    for g, (lo, hi) in enumerate(ranges):
        for r in range(R):
            loc = scores[r, lo:hi]
            ok = ~np.isnan(loc)
            if not ok.any():
                recs[g, r] = (0.0, sh().NO_ENDPOINT, 0, 0, -1)
                continue
            mx = loc[ok].max()
            idx = lo + np.flatnonzero(ok & (loc == mx))
            recs[g, r] = (mx, idx[0], len(idx), r % 7, 0)
    return recs


@pytest.mark.parametrize("case", ["random", "empty-shards", "single", "inf", "neg-inf", "descending"])
def test_resolve_matches_brute_force(orc, case):
    rng = np.random.default_rng(L.seed_of("resolve", case))
    E, R = 90, 200
    cuts = {"empty-shards": [0, 30, 30, 90], "single": [44, 45]}.get(case, sorted(rng.choice(np.arange(1, E), 3, replace=False)))
    ranges = L.ranges_of(cuts, E)
    if case == "descending":
        ranges = ranges[::-1]
    vals = {"inf": [np.inf, 1.0], "neg-inf": [-np.inf]}.get(case, [0.5, 1.0, 1.5])
    scores = rng.choice(vals, (R, E))
    scores[rng.random((R, E)) < 0.1] = np.nan
    if case == "single":
        scores[:, :] = np.nan
        scores[::2, 44] = 2.0                               # N == 1 on the one-slot shard
        scores[1::2, 60] = 2.0
    scores[7, :] = np.nan                                   # no candidate anywhere
    recs = records_of(scores, ranges)
    base = 12345
    merged, owner, local = sh().resolve_records_host(recs, SEED, base)
    for r in range(R):
        ok = ~np.isnan(scores[r])
        if not ok.any():
            assert owner[r] == -1 and merged["status"][r] == -1
            continue
        group = np.flatnonzero(ok & (scores[r] == scores[r][ok].max()))
        assert merged["tie_count"][r] == len(group)
        member = group[orc.tie_rank(SEED, 4 * (base + r), len(group))] if len(group) > 1 else group[0]
        lo, hi = ranges[owner[r]]
        assert lo <= member < hi, (case, r)
        assert group[(group >= lo) & (group < hi)][local[r]] == member
        assert sh().tie_rank_host(SEED, 4 * (base + r), len(group)) == orc.tie_rank(SEED, 4 * (base + r), len(group))
    assert (merged["tie_count"] > 1).any() or case == "single"
    if case == "single":
        assert (merged["tie_count"][merged["status"] == 0] == 1).all()


# ------------------------------------------------------------------------------------------------
# the protocol over gloo
# ------------------------------------------------------------------------------------------------
def _seeded_rank(orc, w, pool, ix, primary, hashes, gmasks, lo, hi):
    """Phase 2 restated (T._oracle_rank_pick) plus each request's local arg-max set."""
    best = T._oracle_rank_pick(orc, sh(), w, pool, ix, primary, hashes, gmasks, lo, hi)
    sets = []
    for r, h in enumerate(hashes):
        stop = next((i for i in range(len(h)) if not (gmasks[r, i // 32] >> (i % 32)) & 1), len(h))
        counts = np.zeros(w.E, np.int32)
        for i in range(stop):
            for s in ix.get(h[i]):
                counts[s] += 1
        scores, _, _, _ = orc.profile_run(primary, pool, counts, len(h))
        idx = np.flatnonzero((scores >= 0) & (np.arange(w.E) >= lo) & (np.arange(w.E) < hi))
        mx = scores[idx].max() if len(idx) else None
        sets.append((idx[scores[idx] == mx] if len(idx) else idx, counts))
    return best, sets


def _gloo_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import pyoracle as orc
        from tools import tracegen as tg
        s = sh()
        w = T._workload()
        trace = tg.Trace(w, n_threads=1)
        tokens, _, _ = trace.requests()
        lo, hi = s.shard_range(rank, world, w.E)
        pool, ix, primary, masks, hashes = T._oracle_rank_outputs(orc, w, trace, tokens, lo, hi)
        gm = s.or_allgather(torch.from_numpy(masks.view(np.int32)), dist).numpy().view(np.uint32)
        best, sets = _seeded_rank(orc, w, pool, ix, primary, hashes, gm, lo, hi)
        allb = s.allgather_records(torch.from_numpy(best.view(np.uint8).reshape(-1, 24)), dist).numpy()
        allb = allb.reshape(world, -1).view(s.SHARD_BEST_DTYPE).reshape(world, -1)
        merged, owner, local = s.resolve_records_host(allb, SEED, 0)
        sel = np.zeros(len(hashes), s.SHARD_SEL_DTYPE)
        sel["pick"] = s.NO_ENDPOINT
        for r, (grp, counts) in enumerate(sets):
            if owner[r] == rank:
                sel[r] = (grp[local[r]], counts[grp[local[r]]])
        alls = s.allgather_records(torch.from_numpy(sel.view(np.uint8).reshape(-1, 8)), dist).numpy()
        alls = alls.reshape(world, -1).view(s.SHARD_SEL_DTYPE).reshape(world, -1)
        final = merged.copy()
        for r in range(len(hashes)):
            if owner[r] >= 0:
                final["pick"][r], final["match_blocks"][r] = alls[owner[r], r]["pick"], alls[owner[r], r]["match_blocks"]
        q.put((rank, final.tobytes(), int((merged["pick"] != final["pick"]).sum())))
    finally:
        dist.destroy_process_group()


def test_seeded_protocol_gloo_world2(orc):
    import torch.multiprocessing as mp
    import helpers
    from tools import tracegen as tg
    s = sh()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = T._free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        rank, final, moved = q.get(timeout=240)
        res[rank] = (np.frombuffer(final, dtype=s.SHARD_BEST_DTYPE), moved)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    np.testing.assert_array_equal(res[0][0], res[1][0])
    w = T._workload()
    trace = tg.Trace(w, n_threads=1)
    tokens, _, _ = trace.requests()
    pool, ix, primary, _, _ = helpers.setup_oracle(orc, w, trace)
    d, offs = tokens.reshape(-1), np.arange(0, tokens.size + 1, tokens.shape[1], dtype=np.uint64)
    odec, _ = orc.cycle_batch(tg.MODEL, w.block_size_tokens, w.max_prefix_blocks, 0, False, ix, primary, None, pool,
                              d.view(np.uint8), offs * tokens.itemsize, 1, tie_seed=SEED, tie_base=0)
    m = res[0][0]
    np.testing.assert_array_equal(m["status"], odec["status"])
    np.testing.assert_array_equal(m["pick"].astype(np.int64), odec["pick"].astype(np.int64))
    np.testing.assert_array_equal(m["score"].view(np.uint64), odec["score"].view(np.uint64))
    np.testing.assert_array_equal(m["tie_count"].astype(np.int64), odec["tie_count"].astype(np.int64))


# ------------------------------------------------------------------------------------------------
# the GPU cases reach their edges
# ------------------------------------------------------------------------------------------------
def decisions(orc, S, base=0, tie_seed=SEED):
    """The oracle's decisions (status, pick, ... in pyoracle.DECISION_DTYPE: no pick = -1) and the picks' match counts."""
    out, _, mb = SD.expected(orc, S, S.prompts, base, tie_seed)
    return out, mb


def owners(dec, ranges, picks=None):
    p = dec["pick"] if picks is None else picks
    return np.array([next((g for g, (lo, hi) in enumerate(ranges) if lo <= x < hi), -1) for x in p])


@pytest.mark.parametrize("world", [2, 3, 5])
def test_A_seeded_picks_leave_the_lowest_shard(orc, world):
    """In descending ranges the tie group spans every shard and the seeded member often lies on another shard than the
    lowest slot."""
    S = L.scene_cross("tie-prefix", world)
    seeded, plain = decisions(orc, S)[0], decisions(orc, S, tie_seed=0)[0]
    ranges = S.ranges[::-1]
    tied = seeded["tie_count"] > 1
    assert len(set(owners(seeded, ranges)[tied])) == world
    assert (owners(seeded, ranges)[tied] != owners(plain, ranges)[tied]).any()


def test_B_cold_ties_the_whole_pool(orc):
    S = SD.scene_cold(2)
    dec = decisions(orc, S)[0]
    assert (dec["tie_count"] == S.E).all() and len(set(dec["pick"].tolist())) > 20


def test_B_edges(orc):
    # matched candidates inside the equal-base group: prefix weight 0 and group members matched
    S = L.scene_cross("tie-zero", 4)
    dec, mb = decisions(orc, S)
    assert ((mb > 0) & (dec["tie_count"] >= 20)).any()
    # +inf ties on several shards
    S = L.scene_cross("inf", 4)
    dec = decisions(orc, S)[0]
    assert np.isinf(dec["score"]).all() and (dec["tie_count"] > 1).all()
    sets = [g for g, _, _ in __import__("test_sharded_landscapes_cpu").argmax_sets(orc, S)]
    assert max(len(set(owners(None, S.ranges, g))) for g in sets) >= 2
    # -inf on every candidate
    S = L.scene_cross("neg-inf", 4)
    dec = decisions(orc, S)[0]
    assert (dec["score"] == -np.inf).all() and (dec["tie_count"] == S.E).all()


def test_B_dense_select_is_needed(orc):
    S = SD.scene_dense()
    ranges = SD.even(2, S.E)
    assert L.overflow_ranks(orc, S, S.prompts, ranges) == {0}
    dec = decisions(orc, S)[0]
    g = np.array(S.group)
    # requests whose seeded member is a slot of the overflowing shard other than its lowest group member
    on0 = (dec["tie_count"] == len(g)) & (dec["pick"] < ranges[0][1]) & (dec["pick"] != g[0])
    assert on0.sum() >= 10


def test_C_ordinal_changes_the_picks(orc):
    S = L.scene_cross("tie-prefix", 3)
    a, b = decisions(orc, S, 0)[0], decisions(orc, S, len(S.prompts))[0]
    assert (a["pick"] != b["pick"]).any()
    S = L.scene_lora()
    dec = decisions(orc, S)[0]
    assert len(set(S.adapters(len(S.prompts)).tolist())) == 3 and (dec["tie_count"] > 1).any()


def test_D_decider_flips(orc):
    S = SD.scene_pd_flip()
    (seeded, smb), (plain, pmb) = decisions(orc, S), decisions(orc, S, tie_seed=0)
    assert (smb != pmb).any()
    assert (seeded["prefill_ran"] != plain["prefill_ran"]).any()


@pytest.mark.parametrize("world", [2, 3])
def test_D_prefill_owner_has_no_decode(orc, world):
    S = D.scene_roles("split")
    dec = decisions(orc, S)[0]
    ranges = SD.even(world, S.E)
    decode_ranks = {g for g, (lo, hi) in enumerate(ranges) if (S.role[lo:hi] == D.R_DECODE).any()}
    ran = (dec["prefill_ran"] == 1) & (dec["prefill_pick"] >= 0)
    pre = owners(dec, ranges, dec["prefill_pick"])
    assert (ran & ~np.isin(pre, list(decode_ranks))).any()


def test_D_encode_seeded(orc):
    S = D.scene_encode("all", 2)
    seeded, plain = decisions(orc, S)[0], decisions(orc, S, tie_seed=0)[0]
    enc = seeded["encode_ran"] == 1
    assert enc.any() and (seeded["encode_pick"][enc] != plain["encode_pick"][enc]).any()


def test_F_spread_reaches_every_shard(orc):
    S = L.scene_cross("tie-prefix", 4)
    dec = decisions(orc, S)[0]
    grp = dec["tie_count"] >= 20
    assert grp.sum() >= 20 and set(owners(dec, S.ranges)[grp].tolist()) == set(range(4))
    assert set(owners(decisions(orc, S, tie_seed=0)[0], S.ranges)[grp].tolist()) == {0}
