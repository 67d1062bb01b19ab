"""Chain profiles on the whole-pool match kernels (k_match_pick_lat[_rand] behind Schedule, k_dense_pick_lat[_rand]
behind the injected-match entry points) against tools/latency_model.py and tools/context_length_model.py, bit for bit:
status, pick, score bytes, tie count, match_blocks, total_blocks, the stage fields and the first-k lists with their
scores.  The landscapes come from tests/test_chain_pool_cpu.py, which asserts that each reaches its edge:
  - pools on both sides of the shared-memory limit of the per-warp counters (12 536 in shared memory, 12 537 on the
    zeroed global scratch);
  - a populated index with prompts of up to 128 blocks, global stops on the 32-block probe chunk edges and holders with
    holes, through every batch path;
  - one launch in which every warp decides several requests, some with more than 128 matched endpoints, against a
    second engine that decides the same rows one per warp;
  - tie groups of more than 32 at the top of the first-k lists, and random pickers drawing past 32;
  - the admitters behind the chain kernel, decided by entries past the first 32 of a subset or a prediction list."""
from __future__ import annotations

import functools

import numpy as np
import pytest

import test_chain_pool_cpu as cases
from test_chain_pool_cpu import (BLOCK_BYTES, CTX, FILTER_DECODE, KEY, KINDS, MAXB, POOL_SIZES, PRED_DT, PROFILES, TIE_PROFILES,
                                 check_row, counts_of, decide, info_of)
from tools import admission_model as am
from tools import context_length_model as cm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _spec(epp, p):
    lat = None
    if p["lcfg"] is not None:
        lat = dict(p["lcfg"])
        if "strategy" in lat:
            lat["strategy"] = epp.capi.HEADROOM_MOST if lat["strategy"] == "most" else epp.capi.HEADROOM_LEAST
    aff = None if p["a2"] is None else epp.AffinityFilterSpec(*p["a2"])
    return epp.ProfileSpec(FILTER_DECODE, [epp.ScorerSpec(k, w, pa) for k, w, pa in p["scorers"]], aff, p["picker"],
                           latency=lat, context_length=p["cl"])


def engine(epp, E, p, seed, k):
    eng = epp.Engine(E, _spec(epp, p), tie_seed=seed, pick_k=k, block_size_tokens=16, max_prefix_blocks=MAXB)
    eng.register_model(b"m")
    return eng


def set_pool(eng, pool, labels=None):
    role, kv, waiting, running = pool
    ids = np.flatnonzero(role != 0xFF).astype(np.uint32)
    eng.pool_set(ids, role[ids], kv[ids], waiting[ids], running[ids])
    if labels is not None:
        eng.pool_set_labels(np.arange(len(role), dtype=np.uint32), labels)


def prompts_of(nbytes, seed):
    offs = np.zeros(len(nbytes) + 1, np.uint64)
    offs[1:] = np.cumsum(nbytes)
    data = np.random.default_rng(seed).integers(0, 256, int(offs[-1])).astype(np.uint8)
    return data, offs


def load_index(eng, data, offs, holders):
    """The snapshot in which request r's block b is held by holders[r][b]; -> the expected match counts [R][E], which
    prefix_match must return."""
    E = eng.E
    h, nb = eng.hash_prompts(data, offsets=offs)
    assert list(nb) == [len(x) for x in holders]
    hs, eps = [], []
    for r, blocks in enumerate(holders):
        if not blocks:
            continue
        hs.append(np.repeat(h[r, :len(blocks)], [b.size for b in blocks]))
        eps.append(np.concatenate(blocks))
    eng.index_load_snapshot(np.concatenate(hs).astype(np.uint64), np.concatenate(eps).astype(np.uint32))
    counts = np.stack([counts_of(E, b) for b in holders])
    got, total = eng.prefix_match(data, offsets=offs)
    assert np.array_equal(got, counts)
    assert list(total) == [len(x) for x in holders]
    return counts


def host_out(epp, out, topk):
    """Device outputs (torch) of a synchronized call -> numpy decisions, details, first-k lists."""
    dec = epp.decisions_from_torch(out[0])
    det = out[1].cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
    lists = None
    if topk:
        lists = {n: v.cpu().numpy().view(np.uint32 if n != "primary_scores" else np.float64) for n, v in out[2].items()}
    return dec, det, lists


def same_rows(a, b, n, what):
    assert a[0][:n].tobytes() == b[0][:n].tobytes(), f"{what}: decisions"
    assert a[1][:n].tobytes() == b[1][:n].tobytes(), f"{what}: details"
    if a[2] is not None:
        for name in ("primary", "primary_scores"):
            assert a[2][name][:n].tobytes() == b[2][name][:n].tobytes(), f"{what}: {name}"


def inputs(p, preds, R):
    kw = dict(predictions=list(preds) if p["lcfg"] is not None else None)
    if p["cl"] is not None:
        kw["context_tokens"] = np.array([CTX[r % len(CTX)] for r in range(R)], np.int64)
    return kw


# ---- 1. pool sizes on both sides of the shared-memory limit --------------------------------------------------------
@pytest.mark.parametrize("E", POOL_SIZES)
@pytest.mark.parametrize("prof", list(PROFILES))
@pytest.mark.parametrize("seed", [0, 0x5EED])
@pytest.mark.parametrize("k", [1, 4, 64])
def test_pool_sizes(epp, orc, E, prof, seed, k):
    p = PROFILES[prof]
    pool = cases.make_pool(E, 3)
    labels = cases.make_labels(E, 4) if p["cl"] else None
    ranges = [cm.endpoint_state(lb, KEY) for lb in labels] if labels else None
    R = len(KINDS) + 5
    nbytes, holders, preds = cases.deep_rows(E, R, 100 + k)
    data, offs = prompts_of(nbytes, 7)
    kw = inputs(p, preds, R)
    with engine(epp, E, p, seed, k) as a, engine(epp, E, p, seed, k) as b:
        set_pool(a, pool, labels)
        set_pool(b, pool, labels)
        counts = load_index(a, data, offs, holders)
        totals = np.array([len(x) for x in holders], np.int32)
        got = a.schedule(data, offsets=offs, topk=k > 1, **kw)
        inj = b.schedule_with_match(counts, totals, topk=k > 1, **kw)
    for r in range(R):
        m = decide(orc, p, pool, counts[r], totals[r], info_of(preds[r]) if p["lcfg"] else {},
                   kw.get("context_tokens", [-1] * R)[r], ranges, seed, 4 * r, k)
        for out in (got, inj):
            check_row(m, r, counts[r], totals[r], out[0], out[1], out[2] if k > 1 else None)


@functools.lru_cache(maxsize=1)
def deep_rows_8512():
    return cases.deep_rows(4096, 8192 + 320, 23)


# ---- 2. a populated index, deep prompts and holes, through every batch path ---------------------------------------
@pytest.mark.parametrize("prof,k", [("chart", 64), ("context_length", 4), ("random_chain", 4)])
def test_deep_prompts_every_path(epp, orc, prof, k):
    import torch
    p = PROFILES[prof]
    E, seed = 4096, 0x5EED
    R = 8192 + 320                                    # an asynchronous device batch of two pipelined chunks
    pool = cases.make_pool(E, 21)
    labels = cases.make_labels(E, 22) if p["cl"] else None
    ranges = [cm.endpoint_state(lb, KEY) for lb in labels] if labels else None
    nbytes, holders, preds = deep_rows_8512()
    data, offs = prompts_of(nbytes, 24)
    kw = inputs(p, preds, R)
    ddata, doffs = torch.from_numpy(data).cuda(), torch.from_numpy(offs.astype(np.int64)).cuda()
    outs = {}
    for path in ("host", "device", "async", "pipelined", "with_match"):
        with engine(epp, E, p, seed, k) as eng:
            set_pool(eng, pool, labels)
            counts = load_index(eng, data, offs, holders)
            totals = np.array([len(x) for x in holders], np.int32)
            if path == "host":
                outs[path] = eng.schedule(data, offsets=offs, topk=True, **kw)
            elif path == "with_match":
                outs[path] = eng.schedule_with_match(counts, totals, topk=True, **kw)
            else:
                n = 4096 if path == "async" else R           # below two 4096-row chunks: one launch sequence
                sub = dict(kw)
                if "predictions" in sub and sub["predictions"] is not None:
                    sub["predictions"] = sub["predictions"][:n]
                if "context_tokens" in sub:
                    sub["context_tokens"] = sub["context_tokens"][:n]
                o = doffs[:n + 1]
                out = eng.schedule(ddata, offsets=o, topk=True, asynchronous=path != "device", **sub)
                eng.synchronize()
                torch.cuda.synchronize()
                outs[path] = host_out(epp, out, True)
    host = outs["host"]
    for path in ("device", "pipelined", "with_match"):
        same_rows(outs[path], host, R, path)
    same_rows(outs["async"], host, 4096, "async")
    rng = np.random.default_rng(25)
    rows = sorted(set(range(2 * len(KINDS))) | set(range(4224, 4288)) | set(rng.choice(R, 60, replace=False).tolist()))
    for r in rows:
        m = decide(orc, p, pool, counts[r], totals[r], info_of(preds[r]) if p["lcfg"] else {},
                   kw.get("context_tokens", [-1] * R)[r], ranges, seed, 4 * r, k)
        check_row(m, r, counts[r], totals[r], host[0], host[1], host[2])


# ---- 3. warps that decide more than one request ------------------------------------------------------------------
@pytest.mark.parametrize("E", [12536, 12537])
def test_warps_decide_many_requests(epp, orc, E):
    import torch
    p = PROFILES["max_score_mix"]
    seed, k = 0x5EED, 4
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    W = cases.pick_warps(E, sm)
    R = 2 * cases.pick_warps(12537, sm) + 300
    pool = cases.make_pool(E, 31)
    holders, big = cases.warp_rows(E, R, W, 32)
    rng = np.random.default_rng(33)
    preds = []
    for r in range(R):
        if r % 5:
            preds.append(None)
            continue
        pr = np.zeros(32, PRED_DT)
        pr["slot"] = np.sort(rng.choice(E, 32, replace=False))
        pr["ttft"] = rng.integers(1, 400, 32)
        pr["ttft_headroom"] = rng.integers(-60, 150, 32)
        pr["tpot_headroom"] = rng.integers(-5, 20, 32)
        preds.append(pr)
    data, offs = prompts_of(np.full(R, 4 * BLOCK_BYTES, np.int64), 34)
    rows2d = data.reshape(R, 4 * BLOCK_BYTES)
    step = sm * 8                                     # the warps of one launch at E = 12 536: one request each
    with engine(epp, E, p, seed, k) as a, engine(epp, E, p, seed, k) as b:
        set_pool(a, pool)
        set_pool(b, pool)
        counts = load_index(a, data, offs, holders)
        load_index(b, data, offs, holders)
        got = a.schedule(rows2d, uniform_len=4 * BLOCK_BYTES, topk=True, predictions=preds)
        parts = [b.schedule(rows2d[r0:r0 + step], uniform_len=4 * BLOCK_BYTES, topk=True, predictions=preds[r0:r0 + step])
                 for r0 in range(0, R, step)]
        want = (np.concatenate([x[0] for x in parts]), np.concatenate([x[1] for x in parts]),
                {n: np.concatenate([x[2][n] for x in parts]) for n in ("primary", "primary_scores")})
    same_rows(got, want, R, f"E={E}: one launch vs one request per warp")
    nh = (counts > 0).sum(axis=1)
    assert (nh > cases.LIST_CAP).sum() >= 10
    for r in cases.warp_sample(R, W, big):
        m = decide(orc, p, pool, counts[r], 4, info_of(preds[r]), seed=seed, key=4 * r, k=k)
        check_row(m, r, counts[r], 4, got[0], got[1], got[2])


# ---- 4. tie groups past 32 in the first-k lists -----------------------------------------------------------------
@pytest.mark.parametrize("E", [4096, 12537])
@pytest.mark.parametrize("kind", list(TIE_PROFILES))
def test_ties_past_32(epp, orc, E, kind):
    p = TIE_PROFILES[kind]
    seed, k, R = 0x5EED, 64, 4
    pool, holders, preds = cases.tie_landscape(E, kind, R, 41)
    data, offs = prompts_of(np.full(R, 4 * BLOCK_BYTES, np.int64), 42)
    kw = dict(predictions=list(preds) if kind == "headroom" else None)
    with engine(epp, E, p, seed, k) as a, engine(epp, E, p, seed, k) as b:
        set_pool(a, pool)
        set_pool(b, pool)
        counts = load_index(a, data, offs, holders)
        got = a.schedule(data, offsets=offs, topk=True, **kw)
        inj = b.schedule_with_match(counts, np.full(R, 4, np.int32), topk=True, **kw)
    for r in range(R):
        m = decide(orc, p, pool, counts[r], 4, info_of(preds[r]), seed=seed, key=4 * r, k=k)
        if p["picker"] == 0:
            assert m["ties"] >= 40
        for out in (got, inj):
            check_row(m, r, counts[r], 4, out[0], out[1], out[2])


# ---- 5. admission behind the chain kernel, past one 32-entry chunk ---------------------------------------------
def adm_engines(epp, probabilistic):
    prof = lambda: epp.ProfileSpec(0, [epp.ScorerSpec(2, 2.0), epp.ScorerSpec(1, 2.0), epp.ScorerSpec(0, 3.0),  # noqa: E731
                                       epp.ScorerSpec(10, 1.0)], latency=dict(tier_filter=1))
    base = epp.Engine(cases.ADM_E, prof(), tie_seed=3)
    adm = epp.Engine(cases.ADM_E, prof(), tie_seed=3)
    adm.admission_set(latency_slo=True, probabilistic=probabilistic, queue_depth_threshold=30, kv_cache_util_threshold=2.0,
                      k=1000.0)
    return base, adm


def adm_set_pool(eng, pool):
    eng.register_model(b"m")
    ids = np.flatnonzero(pool["present"]).astype(np.uint32)
    eng.pool_set(ids, np.zeros(ids.size, np.uint8), pool["kv"][ids], pool["waiting"][ids], pool["running"][ids])


def adm_same(got, want, what):
    for a, b, name in zip(got, want, ("decisions", "details")):
        assert a.tobytes() == b.tobytes(), f"{what}: {name} differ"


@pytest.mark.parametrize("idle_cold", [False, True])
def test_admission_past_one_chunk(epp, idle_cold):
    R = 600
    pool = cases.adm_pool(51, idle_cold)
    prio, ttft, tpot, subs, preds, valid = cases.adm_rows(pool, R, 52, subsets=idle_cold)
    cfg = cases.adm_cfg(idle_cold)
    ad = dict(priority=prio, ttft_slo=ttft, tpot_slo=tpot, pred_valid=valid)
    prompts = np.random.default_rng(53).integers(0, 256, (R, 256)).astype(np.uint8)
    base, adm = adm_engines(epp, idle_cold)
    with base, adm:
        for e in (base, adm):
            adm_set_pool(e, pool)
        if not idle_cold:
            # whole-pool rows on the injected-match kernel
            match = np.random.default_rng(54).integers(0, 4, (R, cases.ADM_E)).astype(np.int32)
            total = np.full(R, 8, np.int32)
            ord_base = base.stats()["n_decisions"]
            want = base.schedule_with_match(match, total, predictions=preds)
            got = adm.schedule_with_match(match, total, predictions=preds, admission=ad)
            rej = am.rejects(cfg, pool, prio, ttft, tpot, cases.slots_of(preds), valid, None, 3, ord_base)
            assert rej.any() and (~rej).any()
            adm_same(got, am.apply(want[0], want[1], rej), "with_match")
        # the hash + dense-counter path, with the subset rows on the subset kernel
        ord_base = base.stats()["n_decisions"]
        want = base.schedule(prompts, uniform_len=256, subsets=subs, predictions=preds)
        got = adm.schedule(prompts, uniform_len=256, subsets=subs, predictions=preds, admission=ad)
        rej = am.rejects(cfg, pool, prio, ttft, tpot, cases.slots_of(preds), valid, subs, 3, ord_base)
        assert rej.any() and (~rej).any()
        adm_same(got, am.apply(want[0], want[1], rej), f"schedule idle_cold={idle_cold}")
