"""The staged merge of the endpoint-sharded mode under the disagg handler, without a GPU:
  * sharded.merge_stage_records_host (the host statement of epp_shard_merge with S records per request) on hand-written
    [n_ranks][R][S] records: the P/D decider on both sides of its boundary, its other early outs, a decode tie whose lowest
    slot sits on a later rank, stages empty everywhere, +-inf scores, mixed multimodal flags;
  * a gloo world-2 run of the staged protocol with the oracle standing in for each rank's kernels, one profile at a time;
  * from the builders of test_sharded_disagg_gpu.py and the oracle alone: each GPU case reaches the edge it names."""
import importlib
import os

import numpy as np
import pytest

import test_sharded as TS
import test_sharded_disagg_gpu as G

NO = 0xFFFFFFFF
BST = 16


def sh():
    return importlib.import_module("llm-d-inference-scheduler_b200.sharded")


def recs(world, R, S):
    a = np.zeros((world, R, S), dtype=sh().SHARD_BEST_DTYPE)
    a["status"] = -1
    a["pick"] = NO
    return a


def merge(a, in_len, mm=None, **kw):
    kw.setdefault("block_size_tokens", BST)
    return sh().merge_stage_records_host(a, np.asarray(in_len, np.int64), mm, **kw)


# ------------------------------------------------------------------------------------------------
# merge_stage_records_host
# ------------------------------------------------------------------------------------------------
def test_decider_boundary(orc):
    """tokens - match_blocks * bst == nct runs prefill, nct - 1 does not; the decider is the oracle's."""
    nct, mb = 20, 3
    a = recs(2, 2, 2)
    a[0, :, 0] = (1.0, 5, 1, mb, 0)
    a[1, :, 1] = (0.5, 40, 2, 0, 0)
    in_len = [4 * (mb * BST + nct), 4 * (mb * BST + nct - 1)]
    dec, det = merge(a, in_len, non_cached_tokens=nct)
    assert list(det["prefill_ran"]) == [1, 0]
    assert det["prefill_pick"][0] == 40 and det["prefill_tie_count"][0] == 2 and det["prefill_score"][0] == 0.5
    assert det["prefill_pick"][1] == NO and det["prefill_tie_count"][1] == 0
    for L in in_len:
        assert sh().pd_decide_host(nct, L, mb, BST) == orc.pd_decide(nct, L, mb, BST)
    for L in range(0, 4 * 200, 3):
        for m in (0, 1, 5):
            for n in (0, 1, 17, 64):
                assert sh().pd_decide_host(n, L, m, BST) == orc.pd_decide(n, L, m, BST)


@pytest.mark.parametrize("case", ["short", "nct0", "always"])
def test_decider_early_outs(case):
    a = recs(1, 1, 2)
    a[0, 0, 0] = (1.0, 2, 1, 0, 0)
    a[0, 0, 1] = (0.25, 9, 1, 0, 0)
    kw = {"short": dict(non_cached_tokens=100), "nct0": dict(non_cached_tokens=0),
          "always": dict(non_cached_tokens=0, always_disagg=True)}[case]
    dec, det = merge(a, [4 * 99], **kw)
    assert det["prefill_ran"][0] == (case == "always")
    assert det["prefill_pick"][0] == (9 if case == "always" else NO)


def test_decode_tie_on_later_rank_sets_match_blocks():
    """The tie's lowest slot sits on rank 2 and its match_blocks (6) decides against prefill, rank 0's (1) would not."""
    nct = 10
    a = recs(3, 1, 2)
    a[0, 0, 0] = (2.0, 30, 2, 1, 0)
    a[1, 0, 0] = (1.0, 1, 1, 9, 0)
    a[2, 0, 0] = (2.0, 12, 3, 6, 0)
    a[0, 0, 1] = (0.75, 31, 1, 0, 0)
    in_len = [4 * (6 * BST + nct - 1)]
    dec, det = merge(a, in_len, non_cached_tokens=nct)
    assert (dec["pick"][0], dec["tie_count"][0], dec["match_blocks"][0]) == (12, 5, 6)
    assert det["prefill_ran"][0] == 0
    a[2, 0, 0]["match_blocks"] = 1
    dec, det = merge(a, in_len, non_cached_tokens=nct)
    assert det["prefill_ran"][0] == 1 and det["prefill_pick"][0] == 31


def test_stage0_empty_everywhere():
    a = recs(2, 1, 3)
    a[0, 0, 1] = (1.0, 3, 1, 0, 0)
    a[1, 0, 2] = (1.0, 4, 1, 0, 0)
    dec, det = merge(a, [4000], [1], always_disagg=True, encode_enabled=True)
    assert dec["status"][0] == -1 and dec["pick"][0] == NO
    assert det["prefill_ran"][0] == 0 and det["encode_ran"][0] == 0
    assert det["prefill_pick"][0] == NO and det["encode_pick"][0] == NO


def test_other_stages_empty_everywhere():
    a = recs(2, 1, 3)
    a[1, 0, 0] = (0.5, 7, 1, 0, 0)
    dec, det = merge(a, [4000], [1], always_disagg=True, encode_enabled=True)
    assert dec["status"][0] == 0 and dec["pick"][0] == 7
    assert det["prefill_ran"][0] == 1 and det["prefill_pick"][0] == NO and det["prefill_tie_count"][0] == 0
    assert det["encode_ran"][0] == 1 and det["encode_pick"][0] == NO


def test_infinite_scores_per_stage():
    inf = np.inf
    a = recs(3, 1, 3)
    a[0, 0, 0] = (inf, 9, 1, 2, 0)
    a[2, 0, 0] = (inf, 4, 2, 3, 0)
    a[1, 0, 1] = (-inf, 20, 4, 0, 0)
    a[2, 0, 1] = (-inf, 15, 1, 0, 0)
    a[0, 0, 2] = (1.0, 1, 1, 0, 0)
    a[1, 0, 2] = (inf, 22, 1, 0, 0)
    dec, det = merge(a, [40], [1], always_disagg=True, encode_enabled=True)
    assert dec["score"][0] == inf and dec["pick"][0] == 4 and dec["tie_count"][0] == 3 and dec["match_blocks"][0] == 3
    assert det["prefill_score"][0] == -inf and det["prefill_pick"][0] == 15 and det["prefill_tie_count"][0] == 5
    assert det["encode_score"][0] == inf and det["encode_pick"][0] == 22


def test_multimodal_mixed():
    a = recs(2, 4, 3)
    a[0, :, 0] = (1.0, 0, 1, 0, 0)
    a[1, :, 2] = (0.5, 33, 1, 0, 0)
    mm = np.array([1, 0, 1, 0], np.uint8)
    dec, det = merge(a, [400] * 4, mm, encode_enabled=True)
    assert list(det["encode_ran"]) == [1, 0, 1, 0]
    assert list(det["encode_pick"]) == [33, NO, 33, NO]
    _, det = merge(a, [400] * 4, None, encode_enabled=True)
    assert not det["encode_ran"].any()


def test_single_stage_is_merge_records_host():
    rng = np.random.default_rng(3)
    a = recs(4, 50, 1)
    ok = rng.random((4, 50)) < 0.7
    a[..., 0]["status"] = np.where(ok, 0, -1)
    a[..., 0]["score"] = rng.integers(0, 3, (4, 50)) * 0.5
    a[..., 0]["pick"] = np.where(ok, np.arange(4)[:, None] * 100 + rng.integers(0, 100, (4, 50)), NO)
    a[..., 0]["tie_count"] = rng.integers(1, 4, (4, 50))
    dec, det = merge(a, np.full(50, 4000), non_cached_tokens=1, always_disagg=True)
    np.testing.assert_array_equal(dec, sh().merge_records_host(a[..., 0]))
    assert not det["prefill_ran"].any() and not det["encode_ran"].any()


# ------------------------------------------------------------------------------------------------
# gloo world 2: the staged protocol with the oracle as each rank's kernels
# ------------------------------------------------------------------------------------------------
def _workload():
    from tools import tracegen as tg
    return tg.baseline_configs()["config4"].scaled(E=96, R=96, T=512, name="config4-tiny")


def _rank_records(orc, w, trace, tokens, lo, hi, gmasks):
    """Phase 2 of the staged protocol restated: per stage, the best of this shard's candidates under the global stop
    (test_sharded._oracle_rank_pick, one profile at a time); prefill evaluated when the decider may say yes."""
    import helpers
    s = sh()
    pool, ix, primary, prefill, (hs, es) = helpers.setup_oracle(orc, w, trace)
    keep = (es >= lo) & (es < hi)
    lix = orc.Indexer()
    lix.load_pairs(hs[keep], es[keep])
    from tools import tracegen as tg
    hashes = [orc.hash_prompt(tokens[r].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks)
              for r in range(tokens.shape[0])]
    d = TS._oracle_rank_pick(orc, s, w, pool, lix, primary, hashes, gmasks, lo, hi)
    p = TS._oracle_rank_pick(orc, s, w, pool, lix, prefill, hashes, gmasks, lo, hi)
    nct = w.non_cached_tokens
    if not (nct != 0 and tokens.shape[1] >= nct):           # every prompt is T tokens long
        p["status"] = -1
    out = np.zeros((tokens.shape[0], 2), dtype=s.SHARD_BEST_DTYPE)
    out[:, 0], out[:, 1] = d, p
    return out, hashes, lix


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
        w = _workload()
        trace = tg.Trace(w, n_threads=1)
        tokens, _, _ = trace.requests()
        lo, hi = s.shard_range(rank, world, w.E)
        _, _, _, masks, _ = TS._oracle_rank_outputs(orc, w, trace, tokens, lo, hi)
        gm = s.or_allgather(torch.from_numpy(masks.view(np.int32)), dist).numpy().view(np.uint32)
        best, _, _ = _rank_records(orc, w, trace, tokens, lo, hi, gm)
        allb = s.allgather_records(torch.from_numpy(best.view(np.uint8).reshape(tokens.shape[0], -1)), dist).numpy()
        allb = allb.reshape(world, tokens.shape[0], -1).view(s.SHARD_BEST_DTYPE).reshape(world, tokens.shape[0], 2)
        dec, det = s.merge_stage_records_host(allb, np.full(tokens.shape[0], w.prompt_bytes, np.int64),
                                              non_cached_tokens=w.non_cached_tokens,
                                              block_size_tokens=w.block_size_tokens)
        q.put((rank, dec.tobytes(), det.tobytes()))
    finally:
        dist.destroy_process_group()


def test_staged_protocol_gloo_world2(orc):
    import torch.multiprocessing as mp
    import helpers
    from tools import tracegen as tg
    s = sh()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = TS._free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        rank, dec, det = q.get(timeout=240)
        res[rank] = (np.frombuffer(dec, s.SHARD_BEST_DTYPE), np.frombuffer(det, s.STAGE_DETAIL_DTYPE))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    np.testing.assert_array_equal(res[0][0], res[1][0])
    np.testing.assert_array_equal(res[0][1], res[1][1])
    w = _workload()
    trace = tg.Trace(w, n_threads=1)
    tokens, _, _ = trace.requests()
    pool, ix, primary, prefill, _ = helpers.setup_oracle(orc, w, trace)
    odec, _ = helpers.oracle_decisions(orc, w, pool, ix, primary, prefill, tokens, 1)
    dec, det = res[0]
    np.testing.assert_array_equal(dec["status"], odec["status"])
    ok = odec["status"] == 0
    np.testing.assert_array_equal(dec["pick"][ok].astype(np.int64), odec["pick"][ok].astype(np.int64))
    np.testing.assert_array_equal(dec["score"][ok].view(np.uint64), odec["score"][ok].view(np.uint64))
    np.testing.assert_array_equal(det["prefill_ran"][ok].astype(np.int64), odec["prefill_ran"][ok].astype(np.int64))
    pf = det["prefill_pick"].astype(np.int64)
    pf[pf == NO] = -1
    np.testing.assert_array_equal(pf[ok], odec["prefill_pick"][ok].astype(np.int64))
    has = ok & (odec["prefill_pick"] >= 0)
    np.testing.assert_array_equal(det["prefill_score"][has].view(np.uint64), odec["prefill_score"][has].view(np.uint64))
    assert has.any()


# ------------------------------------------------------------------------------------------------
# the GPU cases reach their edges (builders + oracle only)
# ------------------------------------------------------------------------------------------------
def _exp(orc, S):
    return G.expected(orc, S, S.prompts)


@pytest.mark.parametrize("kind", ["interleaved", "split", "no-prefill", "no-decode"])
def test_edges_roles(orc, kind):
    S = G.scene_roles(kind)
    odec, _, _ = _exp(orc, S)
    ok = odec["status"] == 0
    if kind == "no-decode":
        assert not ok.any()
    elif kind == "no-prefill":
        assert ok.all() and (odec["prefill_ran"] == 1).any() and (odec["prefill_pick"] == -1).all()
    else:
        assert (odec["prefill_pick"][ok] >= 0).any() and (odec["prefill_ran"][ok] == 0).any()
    if kind == "split":          # the decode pick on the lower half, the prefill pick on the upper
        has = ok & (odec["prefill_pick"] >= 0)
        assert (odec["pick"][ok] < S.E // 2).all() and (odec["prefill_pick"][has] >= S.E // 2).all() and has.any()


@pytest.mark.parametrize("kind", ["boundary", "always", "nct0", "short", "long"])
def test_edges_decider(orc, kind):
    S = G.scene_decider(kind)
    odec, _, mb = _exp(orc, S)
    ok = odec["status"] == 0
    assert ok.all() and (odec["pick"] < 20).all()
    ran = odec["prefill_ran"] == 1
    tokens = np.array([len(p) // 4 for p in S.prompts])
    if kind in ("boundary", "long"):
        gap = tokens - mb * G.BST
        assert ((gap == S.nct) & ran).any() and ((gap == S.nct - 1) & ~ran).any()
        assert (odec["prefill_pick"][ran] >= 20).all()       # the prefill best on the other rank than the decode pick
    if kind == "long":
        cap = S.B * G.BB
        assert (np.array([len(p) for p in S.prompts]) > cap + 4 * S.nct).any()
        assert ((tokens - mb * G.BST > S.nct) & ran).any()  # only the bytes behind the hashed rows make it run
    if kind == "always":
        assert ran.all()
    if kind == "nct0":
        assert not ran.any()
    if kind == "short":
        assert (tokens < S.nct).any() and (tokens >= S.nct).any() and not ran[tokens < S.nct].any()


@pytest.mark.parametrize("kind", ["all", "some", "none"])
def test_edges_encode(orc, kind):
    S = G.scene_encode(kind, 2)
    odec, _, _ = _exp(orc, S)
    ok = odec["status"] == 0
    mm = S.mm.astype(bool)
    assert (ok & mm).any() and (ok & ~mm).any()
    if kind == "none":
        assert (odec["encode_pick"][ok & mm] == -1).all()
    else:
        assert (odec["encode_pick"][ok & mm] >= 0).all()
    if kind == "some":
        cut = sh().shard_range(0, 2, S.E)[1]
        assert (odec["encode_pick"][ok & mm] < cut).all()


def test_edges_dense_and_lora(orc):
    S = G.scene_overflow()
    assert G.dense_ranks(orc, S, S.prompts, G.even(2, S.E)) == {0}
    S = G.scene_lora()
    odec, _, _ = _exp(orc, S)
    assert set(S.adapters(len(S.prompts)).tolist()) == {0, 1, 2}
    assert (odec["prefill_pick"] >= 0).any()
