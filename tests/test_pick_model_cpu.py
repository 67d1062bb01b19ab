"""CPU check of the ALGORITHM behind the sparse match/pick kernel (csrc/match_sparse.cu, DESIGN.md 4.2-4.3).

The reference scores EVERY candidate endpoint for every request (runScorerPlugins, scheduler_profile.go:151-174) and
picks a member of the arg-max set.  The kernel instead evaluates only the endpoints that hold part of the prompt's
prefix and takes everyone else from a per-pool precomputation:

  * an endpoint with zero matched blocks has exactly the ordered weighted sum `base[e]` = the same left-to-right
    accumulation with every prefix term replaced by clamp(0) * w -- request independent, bit for bit;
  * candidates sorted once by (base desc, slot asc) with the size of every equal-base group; the best unmatched
    endpoint is the first unmatched entry of that order, and the number of unmatched endpoints tied with it is its
    group size minus the matched endpoints of the same base.

`sparse_pick` restates that in Python floats (IEEE double, no fusion) and is compared with the oracle's full scan:
max score bits, lowest slot id of the arg-max set and the size of the set.  `eval_lanes` / `select_tied` restate the
kernel's tie selection (match_sparse.cuh eval_profile_lanes / select_tied): every rank of the arg-max set must be the
oracle's member of that rank.  No GPU involved."""
from __future__ import annotations

import numpy as np
import pytest


def clamp01(x):
    return 0.0 if x < 0.0 else (1.0 if x > 1.0 else x)


def pool_precompute(orc, scorers, pool, cand):
    """k_pool_terms / k_pool_sort / k_pool_groups: contrib[s][e], base[e], order, group sizes."""
    n = pool.n
    zeros = np.zeros(n, np.int32)
    contrib = []
    for sc in scorers:
        if sc[0] == orc.SCORER_PREFIX:
            contrib.append(None)
        else:
            col = orc.score_column(sc, pool, cand, zeros, 0)
            contrib.append([clamp01(float(col[e])) * sc[1] for e in range(n)])
    base = []
    for e in range(n):
        acc = 0.0
        for s, sc in enumerate(scorers):
            acc = acc + (clamp01(0.0) * sc[1] if contrib[s] is None else contrib[s][e])
        base.append(acc)
    order = sorted((e for e in range(n) if cand[e]), key=lambda e: (-base[e], e))
    grp = {}
    for e in order:
        grp[base[e]] = grp.get(base[e], 0) + 1
    return contrib, base, order, grp


def sparse_pick(scorers, contrib, base, order, grp, cand, matched: dict, total: int):
    """eval_profile_lanes: matched = {endpoint: blocks}.  -> (max score, lowest slot id, tie count) or None."""
    best = None

    def add(val, e, ties):
        nonlocal best
        if best is None or val > best[0]:
            best = (val, e, ties)
        elif val == best[0]:
            best = (val, min(e, best[1]), best[2] + ties)

    for e, m in matched.items():
        if not cand[e]:
            continue
        acc = 0.0
        for s, sc in enumerate(scorers):
            if contrib[s] is None:
                raw = 0.0 if total == 0 else float(m) / float(total)
                acc = acc + clamp01(raw) * sc[1]
            else:
                acc = acc + contrib[s][e]
        add(acc, e, 1)
    for e in order:
        if e in matched:
            continue
        same = sum(1 for me in matched if cand[me] and base[me] == base[e])
        add(base[e], e, grp[base[e]] - same)
        break
    return best


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_sparse_pick_equals_full_scan(orc, seed):
    rng = np.random.default_rng(seed)
    n = 61
    for trial in range(30):
        role = rng.choice([0, 1, 2, 3, 4, 8], n).astype(np.uint8)
        # coarse metric values on purpose: many endpoints share a base, so the tie bookkeeping is exercised
        kv = rng.choice([0.0, 0.25, 0.5, 0.75, 1.0, 1.25], n)
        waiting = rng.choice([0, 0, 0, 3, 7, 200], n).astype(np.int32)
        running = rng.choice([0, 1, 5], n).astype(np.int32)
        ext = np.stack([rng.choice([-0.5, 0.0, 0.4, 1.0, 1.7], n), rng.choice([0, 100, 6000], n).astype(np.float64)])
        pool = orc.PoolState(role, kv, waiting, running, ext)
        scorers = [(orc.SCORER_QUEUE, 2.0, 0.0), (orc.SCORER_KV_UTIL, 2.0, 0.0), (orc.SCORER_PREFIX, 3.0, 0.0),
                   (orc.SCORER_LOAD_AWARE, 1.0, 10.0), (orc.SCORER_EXTERNAL, 0.5, 0), (orc.SCORER_TOKEN_LOAD, 1.0, 5000.0, 1)]
        k = int(rng.integers(1, len(scorers) + 1))
        scorers = [scorers[i] for i in rng.permutation(len(scorers))[:k]]
        filt = int(rng.choice([orc.FILTER_NONE, orc.FILTER_DECODE, orc.FILTER_PREFILL]))
        prof = orc.make_profile(filt, scorers)
        cand = np.array([orc.lib().orc_role_filter_keeps(filt, int(r)) for r in role], np.uint8)
        contrib, base, order, grp = pool_precompute(orc, scorers, pool, cand)
        for _ in range(8):
            total = int(rng.choice([0, 1, 16, 256]))
            match = np.zeros(n, np.int32)
            if total:
                idx = rng.choice(n, int(rng.integers(0, 9)), replace=False)
                match[idx] = rng.integers(1, total + 1, len(idx))
            matched = {int(e): int(match[e]) for e in np.flatnonzero(match)}
            scores, mx, pick, argmax = orc.profile_run(prof, pool, match, total)
            got = sparse_pick(scorers, contrib, base, order, grp, cand, matched, total)
            if not argmax:
                assert got is None
                continue
            assert got is not None
            assert np.float64(got[0]).view(np.uint64) == np.float64(mx).view(np.uint64), (seed, trial, scorers)
            assert got[1] == pick and got[2] == len(argmax), (seed, trial, scorers, got, pick, len(argmax))


# ------------------------------------------------------------------------------------------------
# the tie selection of eval_profile_lanes / select_tied, every rank of the arg-max set
# ------------------------------------------------------------------------------------------------
def _lower_bound(a, lo, hi, x):
    while lo < hi:
        mid = (lo + hi) >> 1
        if a[mid] < x:
            lo = mid + 1
        else:
            hi = mid
    return lo


def select_tied(order, grp_pos, lanes, in_a, in_x_all, have_u, gpos, ue, k):
    """select_tied: the member of rank k (ascending slot) of S = A u (G \\ X).  lanes = the endpoints of the lane map;
    in_a / in_x_all are per lane; have_u = the group G of the first unmatched entry holds the maximum."""
    in_x = [x and have_u for x in in_x_all]
    below = lambda mask, x: sum(1 for i, f in enumerate(lanes) if mask[i] and f < x)
    gs = gpos - below(in_x, ue) if have_u else 0
    gsz = grp_pos[gpos] if have_u else 0
    for j, e in enumerate(lanes):                # one lower bound per A lane; the lowest lane of rank k answers
        if not in_a[j]:
            continue
        pos = _lower_bound(order, gs, gs + gsz, e) - gs if have_u else 0
        if below(in_a, e) + pos - (below(in_x, e) if have_u else 0) == k:
            return e
    lo, hi = 0, gsz - 1                          # an unmatched entry of G: the largest position of rank <= k
    while lo < hi:
        mid = (lo + hi + 1) >> 1
        x = order[gs + mid]
        if mid - below(in_x, x) + below(in_a, x) <= k:
            lo = mid
        else:
            hi = mid - 1
    return order[gs + lo]


def eval_lanes(scorers, contrib, base, order, grp_pos, cand, lanes, counts, total):
    """eval_profile_lanes<kTie>: lanes / counts = the lane map (count 0 = an entry lora-affinity added, scored like a
    holder).  -> None (no candidate) or dict(val, pick, ties, chunk of the first unmatched entry, select(rank), and the
    A / X flags per lane for the coverage checks)."""
    if not order:
        return None
    if not lanes:
        return dict(val=base[order[0]], pick=order[0], ties=grp_pos[0], chunk=0, select=lambda k: order[k], a=[], x=[],
                    gs=0, gsz=grp_pos[0], have_u=True)
    best = None

    def add(v, e, n):
        nonlocal best
        if best is None or v > best[0]:
            best = [v, e, n]
        elif v == best[0]:
            best = [v, min(e, best[1]), best[2] + n]

    mine = [bool(cand[e]) for e in lanes]
    myv = [None] * len(lanes)
    for j, e in enumerate(lanes):
        if mine[j]:
            acc = 0.0
            for s, sc in enumerate(scorers):
                if contrib[s] is None:
                    acc = acc + clamp01(0.0 if total == 0 else float(counts[j]) / float(total)) * sc[1]
                else:
                    acc = acc + contrib[s][e]
            myv[j] = acc
            add(acc, e, 1)
    in_map = set(lanes)
    have_u, in_x, chunk, gpos, ue, ubase = False, [False] * len(lanes), None, 0, None, None
    for k0 in range(0, len(order), 32):          # the first unmatched entry, 32 entries of the order at a time
        un = [k for k in range(k0, min(k0 + 32, len(order))) if order[k] not in in_map]
        if un:
            gpos = un[0]
            ue = order[gpos]
            ubase = base[ue]
            in_x = [mine[j] and base[e] == ubase for j, e in enumerate(lanes)]
            add(ubase, ue, grp_pos[gpos] - sum(in_x))
            have_u, chunk = True, k0 // 32
            break
    if best is None:
        return None
    in_a = [mine[j] and myv[j] == best[0] for j in range(len(lanes))]
    hu = have_u and ubase == best[0]
    gs = gpos - sum(1 for j, e in enumerate(lanes) if in_x[j] and e < ue) if hu else 0
    return dict(val=best[0], pick=best[1], ties=best[2], chunk=chunk, a=in_a, x=[v and hu for v in in_x], gs=gs,
                gsz=grp_pos[gpos] if hu else 0, have_u=hu,
                select=lambda k: select_tied(order, grp_pos, lanes, in_a, in_x, hu, gpos, ue, k))


def _tie_profiles(orc):
    third = 1.0 / 3.0
    return {
        # TestPDSchedule's decode profile weighs the prefix scorer 0: a holder scores exactly its base (A and X)
        "zero prefix weight": [(orc.SCORER_PREFIX, 0.0, 0.0), (orc.SCORER_KV_UTIL, 1.0, 0.0), (orc.SCORER_QUEUE, 1.0, 0.0)],
        "negative load weight": [(orc.SCORER_LOAD_AWARE, -1.0, 10.0), (orc.SCORER_KV_UTIL, 0.5, 0.0),
                                 (orc.SCORER_PREFIX, 2.0, 0.0)],
        "negative prefix weight": [(orc.SCORER_KV_UTIL, 1.0, 0.0), (orc.SCORER_PREFIX, -1.5, 0.0),
                                   (orc.SCORER_QUEUE, 0.5, 0.0)],
        "rounding": [(orc.SCORER_KV_UTIL, 0.1, 0.0), (orc.SCORER_QUEUE, 0.7, 0.0), (orc.SCORER_PREFIX, third, 0.0),
                     (orc.SCORER_LOAD_AWARE, 0.1, 10.0), (orc.SCORER_EXTERNAL, third, 0.0)],
    }


@pytest.mark.parametrize("name", ["zero prefix weight", "negative load weight", "negative prefix weight", "rounding"])
def test_select_tied_every_rank_equals_full_scan(orc, name):
    """Pools with few metric levels (groups of up to ~50 equal bases), slots outside the pool, and lane maps that hold
    random slots (candidates or not, counts 0..total), the first and the last slot of a group, or the 32 entries at the
    head of the order (the first unmatched entry is then in the second chunk).  Every rank k of the arg-max set must be
    the oracle's k-th member in ascending slot order."""
    scorers = _tie_profiles(orc)[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    n = 70
    seen = dict(second_chunk=0, a_and_x=0, x_first=0, x_last=0, u_and_a=0)
    for trial in range(40):
        role = rng.choice([0, 1, 2, 3, 0xFF], n, p=[0.4, 0.2, 0.15, 0.15, 0.1]).astype(np.uint8)
        kv = rng.choice([0.0, 0.5, 1.0] if trial % 2 else [0.0, 0.1, 0.3, 0.7, 1.0], n)
        waiting = rng.choice([0, 0, 0, 3, 12], n).astype(np.int32)
        if trial % 4 == 3:                              # one group of ~50: 32 holders at its head leave it in chunk 2
            kv = np.where(rng.random(n) < 0.9, 0.0, 0.5)
            waiting = np.where(rng.random(n) < 0.9, 0, 3).astype(np.int32)
        ext = rng.choice([0.0, 0.3, 1.0, 1.5], n).reshape(1, n)
        pool = orc.PoolState(role, kv, waiting, np.zeros(n, np.int32), ext)
        filt = int(rng.choice([orc.FILTER_NONE, orc.FILTER_DECODE]))
        prof = orc.make_profile(filt, scorers)
        cand = np.array([orc.lib().orc_role_filter_keeps(filt, int(r)) for r in role], np.uint8)
        contrib, base, order, grp = pool_precompute(orc, scorers, pool, cand)
        grp_pos = [grp[base[e]] for e in order]
        starts = [k for k in range(len(order)) if k == 0 or base[order[k]] != base[order[k - 1]]]
        for shape in range(12):
            total = int(rng.choice([0, 1, 16])) if shape % 4 == 0 else int(rng.choice([1, 16]))
            if shape % 3 == 0:                          # random slots, candidates or not
                lanes = [int(e) for e in rng.choice(n, int(rng.integers(0, 33)), replace=False)]
            elif shape % 3 == 1 and len(order) > 32:    # the head of the order
                lanes = list(order[:32])
            else:                                       # the first and the last slot of a group, and a few others
                g = starts[int(rng.integers(0, min(3, len(starts))))]
                gl = [order[k] for k in range(g, g + grp_pos[g])]
                lanes = sorted({gl[0], gl[-1]} | {int(e) for e in rng.choice(n, int(rng.integers(0, 6)), replace=False)})
            counts = [int(rng.integers(0, total + 1)) for _ in lanes]
            match = np.zeros(n, np.int32)
            for e, c in zip(lanes, counts):
                match[e] = c
            _, mx, pick, amax = orc.profile_run(prof, pool, match, total)
            got = eval_lanes(scorers, contrib, base, order, grp_pos, cand, lanes, counts, total)
            where = (name, trial, shape, lanes, counts, total)
            if not amax:
                assert got is None, where
                continue
            assert np.float64(got["val"]).view(np.uint64) == np.float64(mx).view(np.uint64), where
            assert got["pick"] == pick == amax[0] and got["ties"] == len(amax), (where, got["pick"], got["ties"], amax)
            if got["ties"] > 1:
                assert [got["select"](k) for k in range(len(amax))] == amax, where
                seen["second_chunk"] += got["chunk"] == 1 and got["have_u"]
                seen["a_and_x"] += any(a and x for a, x in zip(got["a"], got["x"]))
                seen["u_and_a"] += got["have_u"] and any(got["a"])
                if got["have_u"] and got["gsz"] > 1:
                    xs = {e for e, x in zip(lanes, got["x"]) if x}
                    seen["x_first"] += order[got["gs"]] in xs
                    seen["x_last"] += order[got["gs"] + got["gsz"] - 1] in xs
    # the shapes the kernel's select_tied has special cases for occurred with a tie
    assert seen["x_first"] and seen["x_last"] and seen["u_and_a"], seen
    if name == "zero prefix weight":
        assert seen["a_and_x"] and seen["second_chunk"], seen
