"""The cases of test_sharded_landscapes_gpu.py reach the edges they name, checked from their builders and the CPU oracle
alone (no GPU): a later change to a scene cannot quietly drop the edge the GPU test claims to cover."""
import numpy as np
import pytest

import test_pick_paths_gpu as PP
import test_sharded_landscapes_gpu as SL


def argmax_sets(orc, S, prompts=None, a=0):
    """Per request: (argmax set of the unsharded profile run, its max, the walk's match counts)."""
    ix = S.oracle_index(orc)
    prof = orc.make_profile(S.prof[0], list(S.prof[1]))
    out = []
    for r, p in enumerate(S.prompts if prompts is None else prompts):
        h = orc.hash_prompt(p, S.models[a], SL.BST, S.B)
        m, _ = ix.match_longest_prefix(h, S.E)
        _, mx, _, group = orc.profile_run(prof, S.oracle_pool(orc, a), m, len(h))
        out.append((group, mx, m))
    return out


def shard_of(ranges, e):
    return next(g for g, (lo, hi) in enumerate(ranges) if lo <= e < hi)


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("layout", SL.A_LAYOUTS)
def test_A_layouts_cover_the_pool(layout, world):
    ranges = SL.layout_ranges(layout, world)
    assert len(ranges) == world
    assert sorted(ranges) == SL.ranges_of(sorted({x for r in ranges for x in r} - {0, SL.A_E}), SL.A_E) or layout == "empty"
    assert sum(hi - lo for lo, hi in ranges) == SL.A_E and all(lo <= hi for lo, hi in ranges)
    if layout == "ragged":
        assert any(lo % 32 or hi % 32 for lo, hi in ranges[:-1])
    if layout == "empty":
        assert any(lo == hi for lo, hi in ranges)
    if layout == "single":
        assert any(hi - lo == 1 for lo, hi in ranges)
    if layout == "dropped":
        assert any(set(range(lo, hi)) and set(range(lo, hi)) <= set(SL.A_DROPPED) for lo, hi in ranges)
    if layout == "descending":
        assert [lo for lo, _ in ranges] == sorted((lo for lo, _ in ranges), reverse=True)
    if layout == "outside":
        assert any(set(SL.A_OUTSIDE) & set(range(lo, hi)) for lo, hi in ranges)


def test_A_tie_group_spans_the_shards(orc):
    S = SL.scene_layout()
    sets = argmax_sets(orc, S)
    spread = max(len({shard_of(SL.layout_ranges("split", 5), e) for e in g}) for g, _, _ in sets)
    assert spread >= 4
    ix = S.oracle_index(orc)
    assert 42 in ix.get(S.chain(S.prompts[0])[0]) or any(42 in SL.walk_holders(orc, S, ix, p) for p in S.prompts)


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["tie-zero", "tie-prefix", "inf", "neg-inf", "lone"])
def test_B_cross_shard_edges(orc, kind, world):
    S = SL.scene_cross(kind, world)
    sh = SL.sharded()
    ranges = [sh.shard_range(g, world, S.E) for g in range(world)]
    sets = argmax_sets(orc, S)
    spans = [len({shard_of(ranges, e) for e in g}) for g, _, _ in sets]
    if kind.startswith("tie"):
        assert max(spans) == world, "a max-score tie group over every shard"
        if kind == "tie-zero":        # the lowest member does not match as much as some other member
            assert any(m[min(g)] != m[g].max() for g, _, m in sets)
    if kind == "inf":
        inf = [g for g, mx, _ in sets if np.isposinf(mx)]
        assert inf and max(len({shard_of(ranges, e) for e in g}) for g in inf) >= 2
    if kind == "neg-inf":
        assert all(np.isneginf(mx) for _, mx, _ in sets)
    if kind == "lone":
        lone = [g for g, _, _ in sets if g == [S.E - 1]]
        assert lone, "the lone deep holder wins some request"
        assert len(S.group) == 40 // world * (world - 1) and all(shard_of(ranges, e) != world - 1 for e in S.group)
        assert shard_of(ranges, S.E - 1) == world - 1


@pytest.mark.parametrize("world", [2, 3, 5])
def test_C_extremes_on_different_shards(world):
    S = SL.scene_norm(world)
    sh = SL.sharded()
    ranges = [sh.shard_range(g, world, S.E) for g in range(world)]
    for key, vals in (("queue", S.waiting), ("running", S.running)):
        lo, hi = S.marks[key]
        assert vals[lo] == vals.min() and vals[hi] == vals.max() and (vals == vals.max()).sum() == 1
        assert shard_of(ranges, lo) != shard_of(ranges, hi)
    act = S.ext[2]
    e = S.marks["active"]
    assert act[e] == act.max() and (act == act.max()).sum() == 1
    assert shard_of(ranges, e) != shard_of(ranges, S.marks["queue"][0])
    assert {k for k, *_ in S.prof[1]} == set(range(8))


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("B", [20, 32, 33, 64, 70, 96])
def test_D_stop_blocks(orc, B, world):
    S = SL.scene_stop(B, world)
    assert {(B + 31) // 32 for B in (20, 32, 33, 64, 70, 96)} == {1, 2, 3}
    sh = SL.sharded()
    ranges = [sh.shard_range(g, world, S.E) for g in range(world)]
    ix = S.oracle_index(orc)
    seen = set()
    for k, (s, mode, a, b, c) in enumerate(S.families):
        seen.add(s)
        assert shard_of(ranges, a) == 0 and shard_of(ranges, b) == world - 1
        if s == B:
            continue
        f = [p for p in S.prompts if len(p) >= (s + 1) * SL.BB]
        h = S.chain(S.fams[k])
        assert len(h) == B and len(S.chain(S.prompts[2 * k])) > s
        holders = ix.get(h[s])
        if mode == "other":           # held by another rank only; a's own blocks go on past it
            assert holders == {b} and all(a in ix.get(x) for x in h[s + 1:]) and (s + 1 < B or s == B - 1)
        else:
            assert holders == set() and all({a, b} <= ix.get(x) for x in h[s + 1:])
        assert f
    assert seen == set(SL.d_stops(B))
    assert any(len(p) % SL.BB for p in S.prompts) and sum(len(p) < SL.BB for p in S.prompts) >= 4


@pytest.mark.parametrize("kind", ["dense", "split", "global"])
def test_E_overflow_edges(orc, kind):
    S = SL.scene_overflow(kind)
    sh = SL.sharded()
    ranges = [sh.shard_range(g, 2, S.E) for g in range(2)]
    per = [sum(lo <= e < hi for e in S.holders) for lo, hi in ranges]
    assert per == ([17, 16] if kind == "split" else [40, 0])
    assert SL.overflow_ranks(orc, S, S.prompts, ranges) == (set() if kind == "split" else {0})
    if kind == "split":             # the unsharded pool would overflow
        assert SL.overflow_ranks(orc, S, S.prompts, [(0, S.E)]) == {0}
    if kind == "global":
        assert S.E == 131073


@pytest.mark.parametrize("world", [2, 3])
def test_F_incremental_tables_leave_tombstones(orc, world):
    """Replayed commit by commit: some rank's table held a block at an earlier commit that none of the rank's slots
    holds after the last one (a tombstone once the commit patches the table), and that block lies in the middle of a
    prompt whose later blocks are still held."""
    S = SL.scene_incremental(world)
    sh = SL.sharded()
    ranges = [sh.shard_range(g, world, S.E) for g in range(world)]
    ix = orc.Indexer(S.lru)
    seen = set()                       # (rank, hash) held by the rank at some commit before the last
    for k, step in enumerate(S.steps):
        for e, h in step:
            ix.add(np.array(h, np.uint64), int(e))
        if k < len(S.steps) - 1:
            for e, h in (x for st in S.steps[: k + 1] for x in st):
                for x in h:
                    seen |= {(shard_of(ranges, s), x) for s in ix.get(x)}
    final = S.oracle_index(orc)
    gone = {(g, x) for g, x in seen if not any(shard_of(ranges, s) == g for s in final.get(x))}
    assert gone, "a block an earlier commit held is gone from its rank's table"
    mid = 0
    for p in S.prompts:
        h = S.chain(p)
        held = [bool(final.get(x)) for x in h]
        mid += any((g, x) in gone and any(held[i + 1:]) for i, x in enumerate(h) for g in range(world))
    assert mid, "a tombstone in the middle of a prompt whose later blocks are held"


def test_G_lora_adapters_decide(orc):
    """Scoring every request as adapter 0 (what a pick that loses the model ids does) changes some decision."""
    S = SL.scene_lora()
    mo = S.adapters(len(S.prompts))
    assert set(mo.tolist()) == {0, 1, 2}
    want = SL.expected(orc, S, S.prompts)[0]
    S0 = SL.scene_lora()
    S0.model_of = None
    ix = S0.oracle_index(orc)
    prof = orc.make_profile(S0.prof[0], list(S0.prof[1]))
    differ = 0
    for r, p in enumerate(S.prompts):
        a = int(mo[r])
        h = orc.hash_prompt(p, S.models[a], SL.BST, S.B)
        m, _ = ix.match_longest_prefix(h, S.E)
        sc, _, pick, _ = orc.profile_run(prof, S0.oracle_pool(orc, 0), m, len(h))
        differ += pick != want["pick"][r] or sc.max() != want["score"][r]
    assert differ >= 5


@pytest.mark.parametrize("layout", SL.LAYOUTS)
def test_G_layouts(layout):
    rng = np.random.default_rng(0)
    S = SL.scene_lora()
    ps, buf, offs, lens, T = SL.layout_batch(S.prompts, layout, rng)
    assert len(ps) == len(S.prompts)
    if layout == "uniform":
        assert T and len(buf) >= T * len(ps) and all(len(p) == T for p in ps)
        return
    starts = offs[:-1].astype(np.int64)
    if layout == "offsets0":
        assert (starts % 32 == 0).all()
    if layout == "offsets16":
        assert (starts % 32 == 16).all()
    if layout == "odd":
        assert (starts % 2 == 1).any()
    if layout == "lengths":
        assert (lens < np.diff(offs)).all() and ps == S.prompts
    for r, p in enumerate(ps):
        assert buf[int(offs[r]): int(offs[r]) + len(p)] == p


def test_J_merge_records_edges():
    sh = SL.sharded()
    for n, R in ((2, 257), (5, 1000), (64, 300)):
        a = SL.merge_records(n, R, n * 1000 + R)
        m = sh.merge_records_host(a)
        ok = m["status"] == 0
        assert (~ok).any() and np.isneginf(m["score"][ok]).any() and R % 256
        later_lower = 0
        for r in range(R):
            v = a[:, r][a[:, r]["status"] == 0]
            if len(v) and (v["score"] == v["score"].max()).sum() > 1:
                top = np.flatnonzero((a[:, r]["status"] == 0) & (a[:, r]["score"] == m["score"][r]))
                later_lower += a[top[-1], r]["pick"] < a[top[0], r]["pick"]
        assert later_lower > 0, "equal scores with a lower slot on a later rank"
