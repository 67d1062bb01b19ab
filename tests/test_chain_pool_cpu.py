"""Landscapes of the chain-profile pool tests (tests/test_chain_pool_gpu.py), run through the models only: each edge the
GPU tests rely on is asserted to occur here, so a landscape that stops reaching its edge fails on any machine.

A chain profile lists the latency scorer, the slo-headroom-tier-filter or the context-length-aware plugin; on such an
engine every batch is decided by k_match_pick_lat[_rand] (Schedule) or k_dense_pick_lat[_rand] (injected match counts).
The builders below are shared with the GPU tests: pools on both sides of the dense-counter kernel's shared-memory limit,
prompts whose global stop falls on the 32-block probe chunk edges, holders with holes, requests with more than 128
matched endpoints, tie groups of more than 32 at the top of the final set, and admission inputs that only a second
32-entry chunk decides."""
from __future__ import annotations

import numpy as np
import pytest

from tools import admission_model as am
from tools import context_length_model as cm
from tools import latency_model as lm

NO = 0xFFFFFFFF
LAT, QUEUE, KV, PREFIX, RUNNING, CL = 10, 2, 1, 0, 5, 11
FILTER_DECODE = 1
KEY = cm.DEFAULT_LABEL
BLOCK_BYTES = 64                 # 16 tokens of 4 bytes
MAXB = 128                       # max_prefix_blocks
LIST_CAP, PICK_WARPS = 128, 8    # kListCap, kPickWarps (csrc/pick_kernels.cu)
SMEM_CAP = 200 * 1024            # the dense-counter kernel's shared-memory opt-in on an H100
POOL_SIZES = (4096, 12536, 12537)
STOPS = (0, 31, 32, 33, 63, 64, 65)
PRED_DT = np.dtype([("slot", "<u4"), ("dispatched", "<i4"), ("ttft", "<f8"), ("ttft_headroom", "<f8"),
                    ("tpot_headroom", "<f8")])


# ---- launch geometry of the dense-counter kernel, restated from engine.cu / pick_kernels.cu -------------------------
def smem_bytes(E, global_counts):
    """match_pick_smem_bytes: per warp (E + 1) / 2 counter words (none on global scratch) + the list + 4 words."""
    return ((0 if global_counts else (E + 1) // 2) + LIST_CAP + 4) * 4 * PICK_WARPS


def on_global_scratch(E):
    return smem_bytes(E, False) > SMEM_CAP


def pick_warps(E, sm_count):
    """pick_grid * kPickWarps: 4 CTAs per SM on global scratch, else as many as 220 KiB hold (1..8)."""
    if on_global_scratch(E):
        ctas = 4
    else:
        ctas = min(8, max(1, (220 * 1024) // (smem_bytes(E, False) + 1024)))
    return sm_count * ctas * PICK_WARPS


# ---- pools and profiles -------------------------------------------------------------------------------------------
def make_pool(E, seed, absent=5):
    """role (0xFF = absent; role 2, prefill, is dropped by the decode filter), kv, waiting, running.  The last slot is
    present, the one before it absent."""
    rng = np.random.default_rng(seed)
    role = rng.choice(np.array([1, 1, 1, 3, 4, 2], np.uint8), E)
    role[rng.choice(E - 2, absent - 1, replace=False)] = 0xFF
    role[E - 2] = 0xFF
    role[E - 1] = 1
    return role, rng.choice([0.0, 0.25, 0.5, 0.75], E), rng.integers(0, 6, E), rng.integers(0, 6, E)


def make_labels(E, seed):
    """Every slot carries a range (or an invalid one), so a context length outside all ranges empties the set."""
    rng = np.random.default_rng(seed)
    vals = ["0-1000", "500-4000", "4000-9000", "100-100000", "abc"]
    return [{KEY: vals[i]} for i in rng.choice(len(vals), E, p=[0.3, 0.3, 0.2, 0.15, 0.05])]


CTX = (50, 800, 3000, 5000, 20000, 200000)         # 200000: outside every range


CHART = dict(scorers=[(LAT, 1.0, 0.0)], picker=2, a2=(0.80, 0.3, 5000.0), cl=None,
             lcfg=dict(tier_filter=1, epsilon_explore_neg=0.3, a1_affinity_threshold=0.99,
                       a1_exploration_probability=0.3, a1_max_ttft_penalty_ms=5000.0))
PROFILES = {
    "chart": CHART,
    "max_score_mix": dict(scorers=[(QUEUE, 2.0, 0.0), (KV, 2.0, 0.0), (PREFIX, 3.0, 0.0), (LAT, 1.5, 0.0)], picker=0,
                          a2=(0.80, 0.2, 100.0), cl=None,
                          lcfg=dict(tier_filter=1, epsilon_explore_neg=0.5, strategy="most")),
    "context_length": dict(scorers=[(CL, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=0, a2=None,
                           cl=dict(enable_filtering=True), lcfg=None),
    "random_chain": dict(scorers=[(LAT, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=1, a2=None, cl=None,
                         lcfg=dict(tier_filter=1, epsilon_explore_neg=0.4)),
}


def decide(orc, p, pool, counts, total, info, ctx=-1, ranges=None, seed=0, key=0, k=1):
    """The model's decision of one request on profile p (tools/context_length_model.py, which is
    tools/latency_model.py's when the profile does not list the context-length plugin)."""
    role, kv, waiting, running = pool
    E = len(role)
    filt = bool(p["cl"] and p["cl"]["enable_filtering"])
    return cm.profile_decide(orc, FILTER_DECODE, p["scorers"], p["picker"], role, kv, waiting, running,
                             np.asarray(counts, np.int32), int(total), ranges if ranges is not None else [None] * E,
                             int(ctx), filt, info or {}, p["lcfg"], p["a2"], seed, key, k)


def info_of(pred):
    """PRED_DT entries -> the model's slot -> Info."""
    if pred is None:
        return {}
    return {int(x["slot"]): lm.Info(float(x["ttft"]), float(x["ttft_headroom"]), float(x["tpot_headroom"]),
                                    int(x["dispatched"])) for x in pred}


def check_row(m, r, counts, total, dec, det, lists):
    """Engine row r against the model's decision m, bit for bit."""
    ok = bool(m["picks"])
    assert dec["status"][r] == (0 if ok else -1), r
    assert dec["tie_count"][r] == (m["ties"] if ok else 0), r
    assert int(dec["total_blocks"][r]) == int(total), r
    if lists is not None:
        n = len(m["picks"])
        assert list(lists["primary"][r, :n]) == m["picks"], (r, m["final"][:8])
        assert lists["primary_scores"][r, :n].tobytes() == np.asarray(m["scores"], np.float64).tobytes(), r
        assert (lists["primary"][r, n:] == NO).all(), r
    if det is not None:
        assert det["prefill_ran"][r] == 0 and det["encode_ran"][r] == 0, r
    if not ok:
        return
    assert dec["pick"][r] == m["picks"][0], (r, m["final"][:8])
    assert np.float64(dec["score"][r]).tobytes() == np.float64(m["scores"][0]).tobytes(), r
    assert dec["match_blocks"][r] == counts[m["picks"][0]], r
    assert dec["prefill_pick"][r] == NO, r


# ---- the chain's stages, for the edge checks --------------------------------------------------------------------
def stages(orc, p, pool, counts, total, info, seed, key):
    """(A1 narrowed, tier took the negative side while positives existed, A2 narrowed) of profile p's chain."""
    role = pool[0]
    lcfg = dict(lm.DEFAULT_CFG, **(p["lcfg"] or {}))
    cands = [e for e in range(len(role)) if role[e] != 0xFF and orc.lib().orc_role_filter_keeps(FILTER_DECODE, int(role[e]))]
    never = lambda: 1.0  # noqa: E731
    s, a1, flip, a2 = cands, False, False, False
    if lcfg["tier_filter"]:
        if lcfg["a1_affinity_threshold"] > 0:
            s1 = lm.affinity_filter(s, counts, total, lcfg["a1_affinity_threshold"], lcfg["a1_exploration_probability"],
                                    lcfg["a1_max_ttft_penalty_ms"], info,
                                    (lambda: lm.draw_u(seed, lm.A1_DOMAIN, key)) if seed else never)
            a1, s = s1 != s, s1
        pos = [e for e in s if e in info and info[e].ttft_headroom >= 0 and info[e].tpot_headroom >= 0]
        s2 = lm.tier_filter(s, info, lcfg["epsilon_explore_neg"],
                            (lambda: lm.draw_u(seed, lm.TIER_DOMAIN, key)) if seed else never)
        flip = bool(pos) and len(s2) > 0 and not set(s2) & set(pos)
        s = s2
    if p["a2"] is not None:
        s3 = lm.affinity_filter(s, counts, total, p["a2"][0], p["a2"][1], p["a2"][2], info,
                                (lambda: lm.draw_u(seed, lm.EXPLORE_DOMAIN, key)) if seed else never)
        a2 = s3 != s
    return a1, flip, a2


# ---- deep prompts over a populated index --------------------------------------------------------------------------
KINDS = STOPS + ("full", "last", "trunc", "empty")


def deep_rows(E, R, seed):
    """R requests -> (prompt bytes [R], holders [R][total] of ascending slot arrays, predictions [R] of PRED_DT).
    Row r's kind is KINDS[r % len(KINDS)]: a global stop at that block; "full": every block held, total at a
    32-block edge; "last": only the last block unheld; "trunc": a prompt past max_prefix_blocks, every kept block held;
    "empty": a prompt shorter than one block.  Deep holders hold every block before the stop, hole holders all but
    one or two of them, short holders a prefix, and late holders only blocks at and after the stop."""
    rng = np.random.default_rng(seed)
    nbytes = np.zeros(R, np.int64)
    holders, preds = [], []
    for r in range(R):
        kind = KINDS[r % len(KINDS)]
        if kind == "empty":
            T, s = 0, 0
            nbytes[r] = 40
        elif kind in ("full", "trunc"):
            T = MAXB if kind == "trunc" else int(rng.choice([32, 64, 96, 128]))
            s = T
            nbytes[r] = (150 if kind == "trunc" else T) * BLOCK_BYTES
        elif kind == "last":
            T = int(rng.integers(34, MAXB + 1))
            s = T - 1
            nbytes[r] = T * BLOCK_BYTES
        else:
            s = kind
            T = min(MAXB, s + int(rng.choice([1, 2, 5, 20, 60])))
            # the last block may be partial; a prompt shorter than one block has none
            nbytes[r] = T * BLOCK_BYTES if T == 1 else (T - 1) * BLOCK_BYTES + int(rng.integers(1, BLOCK_BYTES + 1))
        pool_pick = lambda n: rng.choice(E, n, replace=False)  # noqa: E731
        ids = pool_pick(40)
        ids[0] = E - 1 if r % 3 == 0 else ids[0]                                     # the last slot holds blocks
        ids = np.unique(ids)
        rng.shuffle(ids)
        deep, hole, short, late = ids[:2], ids[2:5], ids[5:20], ids[20:24]
        blocks = [set() for _ in range(T)]
        for b in range(s):
            blocks[b].update(int(e) for e in deep)
        for e in hole:
            if s >= 3:
                gaps = set(rng.choice(np.arange(1, s - 1), min(2, s - 2), replace=False).tolist())
                for b in range(s):
                    if b not in gaps:
                        blocks[b].add(int(e))
        for e in short:
            for b in range(int(rng.integers(0, s + 1))):
                blocks[b].add(int(e))
        for e in late:
            for b in range(s + 1, T):
                blocks[b].add(int(e))
        holders.append([np.array(sorted(x), np.uint32) for x in blocks])
        # predictions on the holders and on a few dozen other slots: mixed headrooms, so the tier filter splits
        ps = np.unique(np.concatenate([ids, pool_pick(40)]))
        pr = np.zeros(ps.size, PRED_DT)
        pr["slot"] = ps
        pr["ttft"] = rng.integers(1, 400, ps.size)
        pr["ttft_headroom"] = rng.integers(-60, 150, ps.size)
        pr["tpot_headroom"] = rng.integers(-5, 20, ps.size)
        pr["dispatched"] = rng.integers(0, 3, ps.size)
        preds.append(None if r % 7 == 6 else pr)
    return nbytes, holders, preds


def counts_of(E, blocks):
    """matchLongestPrefix over one request's blocks: in block order, stop at the first block nobody holds."""
    c = np.zeros(E, np.int32)
    for h in blocks:
        if h.size == 0:
            break
        c[h] += 1
    return c


def stop_of(blocks):
    for b, h in enumerate(blocks):
        if h.size == 0:
            return b
    return len(blocks)


def prefix_len(blocks, e):
    for b, h in enumerate(blocks):
        if e not in h:
            return b
    return len(blocks)


# ---- many requests per warp ----------------------------------------------------------------------------------------
BIG = (127, 128, 129, 300, 129, 700, 128, 129, 450, 127)


def warp_rows(E, R, W, seed):
    """R requests of 4 blocks for a kernel of W warps (request r and r + W are decided by one warp, in turn) ->
    (holders [R][4], big rows).  Big rows hold BIG's numbers of distinct holders; the row after each and the row one
    warp stride after each have few or none, and no row shares a holder with the row one warp stride earlier."""
    rng = np.random.default_rng(seed)
    big = {}
    step = max(1, (R - W - 2) // (2 * len(BIG)))
    for i in range(2 * len(BIG)):
        big[i * step + (i % 3)] = BIG[i % len(BIG)]
    holders = []
    for r in range(R):
        prev = set()
        if r >= W:
            prev = {int(e) for b in holders[r - W] for e in b}
        n = big.get(r)
        if n is None:
            n = 0 if (r - W in big or r - 1 in big) and r % 2 else int(rng.integers(0, 4 if (r - W in big or r - 1 in big) else 9))
        ids = [int(e) for e in rng.choice(E, min(E, n + len(prev) + 8), replace=False) if int(e) not in prev][:n]
        blocks = [set(), set(), set(), set()]
        for j, e in enumerate(ids):
            depth = 1 + (j % 4) if n > 8 else int(rng.integers(1, 5))
            for b in range(depth):
                blocks[b].add(int(e))
        holders.append([np.array(sorted(x), np.uint32) for x in blocks])
    return holders, sorted(big)


def warp_sample(R, W, big, n_min=200, seed=0):
    """Rows checked against the model: every big row, the row after it, the row one warp stride after it, and others."""
    rows = set()
    for p in big:
        rows.update((p, p + 1, p + W))
    rng = np.random.default_rng(seed)
    while len(rows) < n_min:
        rows.add(int(rng.integers(0, R)))
    return sorted(r for r in rows if r < R)


# ---- tie groups past 32 ---------------------------------------------------------------------------------------------
TIE_PROFILES = {
    "composite": dict(scorers=[(LAT, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=0, a2=None, cl=None,
                      lcfg=dict(tier_filter=1, epsilon_explore_neg=0.0)),
    "headroom": dict(scorers=[(LAT, 1.0, 0.0)], picker=0, a2=None, cl=None,
                     lcfg=dict(tier_filter=1, epsilon_explore_neg=0.0)),
    "random": dict(scorers=[(LAT, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=1, a2=None, cl=None, lcfg=None),
    "weighted": dict(scorers=[(LAT, 1.0, 0.0), (PREFIX, 1.0, 0.0)], picker=2, a2=None, cl=None, lcfg=None),
}
TIE_BLOCK = 48


def tie_landscape(E, kind, R, seed):
    """-> (pool, holders [R][4], predictions [R]).  "composite": a block of 48 slots with kv 0, no queue and the same
    3-block match, no predictions: they top the composite bucket together.  "headroom": the block's predictions share
    the smallest positive headrooms.  "random" / "weighted": about a hundred members of mixed scores."""
    rng = np.random.default_rng(seed)
    role, kv, waiting, running = make_pool(E, seed)
    kv = np.maximum(kv, 0.25)
    waiting = np.maximum(waiting, 1)
    holders, preds = [], []
    for r in range(R):
        b0 = int(rng.integers(0, E - TIE_BLOCK - 2))
        blk = np.arange(b0, b0 + TIE_BLOCK)
        role[blk] = 1
        kv[blk] = 0.0
        waiting[blk] = 0
        blocks = [set(blk.tolist()), set(blk.tolist()), set(blk.tolist()), set()]
        others = rng.choice(np.setdiff1d(np.arange(E), blk), 60, replace=False)
        for e in others[:20]:
            blocks[0].add(int(e))
        holders.append([np.array(sorted(x), np.uint32) for x in blocks])
        if kind == "headroom":
            ps = np.union1d(blk, others)
            pr = np.zeros(ps.size, PRED_DT)
            pr["slot"] = ps
            isb = np.isin(ps, blk)
            pr["ttft"] = 100.0
            pr["ttft_headroom"] = np.where(isb, 5.0, rng.integers(20, 200, ps.size))
            pr["tpot_headroom"] = np.where(isb, 1.0, rng.integers(2, 30, ps.size))
            pr["tpot_headroom"][~isb & (np.arange(ps.size) % 5 == 0)] = -3.0               # a negative tier as well
            preds.append(pr)
        else:
            preds.append(None)
    if kind in ("random", "weighted"):
        # about a hundred members: the rest of the pool is dropped by the decode filter
        keep = np.zeros(E, bool)
        for h in holders:
            keep[h[0]] = True
        keep[rng.choice(E, 40, replace=False)] = True
        role = np.where(keep, np.where(role == 0xFF, 1, role), np.uint8(2)).astype(np.uint8)
        role[E - 2] = 0xFF
    return (role, kv, waiting, running), holders, preds


# ---- admission past one 32-entry chunk -----------------------------------------------------------------------------
ADM_E = 4096
SUB_SIZES = (33, 64, 100, 1024)


def adm_pool(seed, idle_cold):
    """Present slots are busy and warm except, with idle_cold, the idle slots 2000-2003 and the cold slots 3000-3003;
    40 absent slots lie below 200, and 3500-3503 and the last slot are absent too."""
    rng = np.random.default_rng(seed)
    present = np.ones(ADM_E, bool)
    present[rng.choice(200, 40, replace=False)] = False
    present[3500:3504] = False
    present[ADM_E - 1] = False
    kv = rng.choice([0.05, 0.1, 0.2, 0.3, 0.5], ADM_E)
    waiting = rng.integers(0, 8, ADM_E).astype(np.int32)
    running = rng.integers(1, 6, ADM_E).astype(np.int32)
    if idle_cold:
        running[2000:2004] = 0
        kv[3000:3004] = 0.01
    return dict(present=present, kv=kv, waiting=waiting, running=running)


def adm_rows(pool, R, seed, subsets):
    """-> (priority, ttft_slo, tpot_slo, subsets, predictions [R] of PRED_DT, validity bytes [R]).
    Kinds (r % 6): 0 the only candidate entry lies past index 32; 1 the only valid entry lies past index 32; 2 every
    entry invalid; 3 a subset whose only idle or cold slot lies past position 32; 4 absent subset entries, the last
    slot among them, after position 32; 5 no predictions."""
    rng = np.random.default_rng(seed)
    present = pool["present"]
    absent = np.flatnonzero(~present)
    busy = np.flatnonzero(present & (pool["running"] > 0) & (pool["kv"] >= 0.02))
    prio = np.where(np.arange(R) % 11 == 10, 0, -1).astype(np.int32)
    ttft = np.full(R, 100.0)
    tpot = np.where(np.arange(R) % 4 == 0, 30.0, 0.0)
    subs, preds, valid = [], [], []
    for r in range(R):
        kind = r % 6
        n_sub = SUB_SIZES[(r // 6) % len(SUB_SIZES)]
        sub = None
        if subsets and kind in (0, 1, 2):
            sub = sorted(rng.choice(busy, n_sub, replace=False).tolist())
        elif subsets and kind == 3:
            special = int(rng.choice([2000, 2001, 3000, 3002])) if pool["running"][2000] == 0 else int(busy[-1])
            lo = sorted(rng.choice(busy[busy < special], n_sub - 1, replace=False).tolist())
            sub = sorted(lo + [special])
            assert sub.index(special) >= 32
        elif subsets and kind == 4:
            lo = sorted(rng.choice(busy[busy < 3500], max(32, n_sub - 4), replace=False).tolist())
            sub = lo + [3500, 3502, ADM_E - 1]         # a slot >= max_endpoints is refused before any kernel runs
        subs.append(sub)
        cand = np.array(sorted(sub), np.int64) if sub is not None else busy
        cand = cand[(cand < ADM_E)]
        cand = cand[present[cand]]
        n = int(rng.integers(33, 201))
        if kind == 0:
            # 32+ non-candidate entries (absent slots, or pool slots outside the subset) below one candidate entry
            below = absent[absent < 200] if sub is None else np.setdiff1d(np.arange(ADM_E), cand)
            top = int(cand[cand > below[min(n - 2, below.size - 1)]][0])
            nb = min(n - 1, int((below < top).sum()))
            slots = np.concatenate([below[below < top][:nb], [top]])
            bits = np.zeros(slots.size, np.uint8)
            bits[:-1] = rng.integers(0, 4, slots.size - 1)                # the non-candidates' bits do not count
            bits[-1] = int(rng.choice([0, 1, 2]))
        elif kind in (1, 2, 3, 4):
            slots = np.sort(rng.choice(cand, min(n, cand.size), replace=False))
            bits = rng.choice(np.array([0, 1, 2], np.uint8), slots.size)
            if kind == 1:
                bits[int(rng.integers(32, slots.size))] = 3
        else:
            slots, bits = None, None
        if slots is None:
            preds.append(None)
            valid.append(None)
            continue
        pr = np.zeros(slots.size, PRED_DT)
        pr["slot"] = slots
        pr["ttft"] = 10.0
        pr["ttft_headroom"] = 1.0 - (bits & 1)
        pr["tpot_headroom"] = 1.0 - (bits >> 1)
        preds.append(pr)
        valid.append(bits.astype(np.uint8))
    return prio, ttft, tpot, (subs if subsets else None), preds, valid


def adm_cfg(probabilistic):
    c = dict(am.DEFAULTS)
    c.update(queue_depth_threshold=30, kv_cache_util_threshold=2.0, k=1000.0)
    c.update(latency_slo=True, probabilistic=probabilistic)
    return c


def slots_of(preds):
    return [None if p is None else [int(s) for s in p["slot"]] for p in preds]


# ==== the tests: every edge is reached ===============================================================================
def test_shared_memory_limit():
    assert smem_bytes(12536, False) == SMEM_CAP and not on_global_scratch(12536)
    assert on_global_scratch(12537) and smem_bytes(12537, True) == (LIST_CAP + 4) * 4 * PICK_WARPS
    assert not on_global_scratch(4096)
    for sm in (132, 114):
        assert pick_warps(12536, sm) == sm * 8          # one CTA per SM
        assert pick_warps(12537, sm) == sm * 32         # the most warps any pool size gets
        assert pick_warps(4096, sm) == sm * 24
    # once the counters no longer fit two CTAs per SM, no pool size gets more warps than the global-scratch build
    assert max(pick_warps(E, 132) for E in range(6400, 40000, 7)) == 132 * 32


def test_deep_rows_reach_every_stop(orc):
    E = 4096
    nbytes, holders, _ = deep_rows(E, 3 * len(KINDS), 1)
    stops = [stop_of(h) for h in holders]
    totals = [len(h) for h in holders]
    for s in STOPS:
        assert s in stops
    assert any(s == t and t == MAXB for s, t in zip(stops, totals))                # every kept block held
    assert any(s == t and t % 32 == 0 and t < MAXB for s, t in zip(stops, totals))
    assert any(s == t - 1 for s, t in zip(stops, totals))
    assert any(t == 0 for t in totals)
    assert all(t == (0 if n < BLOCK_BYTES else min(MAXB, -(-n // BLOCK_BYTES))) for t, n in zip(totals, nbytes))
    assert any(n % BLOCK_BYTES for n, t in zip(nbytes, totals) if 0 < t < MAXB)
    holes = late = 0
    for h in holders:
        c = counts_of(E, h)
        s = stop_of(h)
        for e in np.flatnonzero(c):
            holes += int(c[e]) != min(prefix_len(h, int(e)), s)
        late += any(int(e) not in h[b] for b in range(s) for e in (h[s + 1] if s + 1 < len(h) else []))
    assert holes > 0 and late > 0


@pytest.mark.parametrize("prof", list(PROFILES))
def test_deep_rows_reach_the_chain_edges(orc, prof):
    E = 4096
    p = PROFILES[prof]
    pool = make_pool(E, 3)
    ranges = [cm.endpoint_state(lb, KEY) for lb in make_labels(E, 4)]
    _, holders, preds = deep_rows(E, 2 * len(KINDS), 5)
    seen = dict(a1=set(), a2=set(), flip=set(), empty=0, status0=0, unsorted=0)
    for r, h in enumerate(holders):
        c = counts_of(E, h)
        info = info_of(preds[r])
        if p["lcfg"] is not None:
            a1, flip, a2 = stages(orc, p, pool, c, len(h), info, 0x5EED, 4 * r)
            seen["a1"].add(a1)
            seen["a2"].add(a2)
            seen["flip"].add(flip)
        m = decide(orc, p, pool, c, len(h), info, CTX[r % len(CTX)], ranges, 0x5EED, 4 * r, 4)
        seen["empty"] += not m["picks"]
        seen["unsorted"] += m["final"] != sorted(m["final"])
        seen["status0"] += bool(m["picks"])
    assert seen["status0"] > 0
    if prof == "chart":
        assert seen["a1"] == {True, False} and seen["a2"] == {True, False} and True in seen["flip"]
    if prof == "max_score_mix":
        assert seen["a2"] == {True, False} and True in seen["flip"]
    if prof == "context_length":
        assert seen["empty"] > 0                       # the filter empties the requests whose context fits no range
    if prof == "random_chain":
        assert seen["unsorted"] > 0                    # the tier's negative side lists endpoints without a prediction last


def test_warp_rows_reach_the_list_cap():
    E, sm = 12536, 132
    W = pick_warps(E, sm)
    R = 2 * pick_warps(12537, sm) + 300
    holders, big = warp_rows(E, R, W, 7)
    nh = [int((counts_of(E, h) > 0).sum()) for h in holders]
    assert {127, 128, 129} <= {nh[p] for p in big} and max(nh) >= 300
    assert sum(n > LIST_CAP for n in nh) >= 10
    for p in big:
        assert nh[p + 1] <= 3 and nh[p + W] <= 3
    for r in range(W, R):
        a = set(np.concatenate(holders[r]).tolist())
        b = set(np.concatenate(holders[r - W]).tolist())
        assert not a & b, r
    assert any(nh[p + W] == 0 for p in big) and any(nh[p + W] > 0 for p in big)
    rows = warp_sample(R, W, big)
    assert len(rows) >= 200 and all(p + W in rows for p in big)


@pytest.mark.parametrize("kind", list(TIE_PROFILES))
def test_tie_groups_past_32(orc, kind):
    E = 4096
    p = TIE_PROFILES[kind]
    pool, holders, preds = tie_landscape(E, kind, 3, 11)
    for r, h in enumerate(holders):
        c = counts_of(E, h)
        m = decide(orc, p, pool, c, len(h), info_of(preds[r]), seed=0x5EED, key=4 * r, k=64)
        assert len(m["picks"]) == 64 and len(set(m["picks"])) == 64
        if p["picker"] == 0:
            assert m["ties"] >= 40 and m["scores"][39] == m["scores"][0]
        else:
            assert len(m["final"]) > 64


@pytest.mark.parametrize("idle_cold", [False, True])
def test_admission_rows_need_the_second_chunk(idle_cold):
    pool = adm_pool(13, idle_cold)
    cfg = adm_cfg(False)
    prio, ttft, tpot, subs, preds, valid = adm_rows(pool, 240, 17, subsets=idle_cold)
    full = am.rejects(cfg, pool, prio, ttft, tpot, slots_of(preds), valid, subs)
    # the same rows with every list cut to its first 32 entries
    cut_p = [None if p is None else p[:32] for p in preds]
    cut_v = [None if v is None else v[:32] for v in valid]
    cut_s = None if subs is None else [None if s is None else s[:32] for s in subs]
    cut = am.rejects(cfg, pool, prio, ttft, tpot, slots_of(cut_p), cut_v, cut_s)
    kinds = np.arange(240) % 6
    assert full.any() and (~full).any()
    differ = full != cut
    assert differ[kinds == 0].any() and differ[kinds == 1].any()
    if idle_cold:
        assert differ[kinds == 3].any()
        assert {len(s) for s in subs if s is not None} >= set(SUB_SIZES)
        assert all(s.index(3500) >= 32 for s in subs if s is not None and 3500 in s)
    lens = [len(p) for r, p in enumerate(preds) if p is not None and kinds[r] < 3]
    assert min(lens) >= 33 and max(lens) > 64
