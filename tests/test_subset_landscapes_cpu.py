"""The cases of test_subset_landscapes_gpu.py reach the edges they name, checked from their builders and the CPU oracle
alone (no GPU): a later change to a landscape cannot quietly drop the edge the GPU test claims to cover."""
import numpy as np
import pytest

import test_pick_paths_gpu as PP
import test_subset_landscapes_gpu as SL
from tools import inflight_model as IM
from tools import picker_model as PM


@pytest.mark.parametrize("path", ["device", "host", "pipelined"])
@pytest.mark.parametrize("name", SL.A_LANDS)
def test_A_subset_shapes(orc, name, path):
    L, ix, prompts, mm, subsets, rows = SL.a_case(orc, name, path)
    sizes = {len(subsets[r]) for r in rows if subsets[r] is not None}
    assert {0, 1, 31, 32, 33}.issubset(sizes) or L.E < 33
    assert any(subsets[r] is None for r in rows)
    ids = set(L.ids.tolist())
    drops = set(SL.filter_drops(orc, L, L.prim))
    stale = [r for r in rows if subsets[r] and (set(subsets[r]) - ids or set(subsets[r]) & drops)]
    assert stale or (ids == set(range(L.E)) and not drops)
    straddles = 0
    for r in rows[:200]:
        s = subsets[r]
        if not s or len(s) < 33:
            continue
        m, total = SL.whole_match(orc, ix, prompts[r], L.E)
        _, _, _, group = orc.profile_run(PP._oprof(orc, L.prim), SL.narrowed(L, s).oracle_pool(orc), m, total)
        pos = np.searchsorted(np.array(s), np.array(group))
        straddles += bool(len(group) > 1 and pos.min() < 32 <= pos.max())
    # (a pool of one slot, and L3's continuous metrics, have no tie group to place)
    assert straddles > 0 or name == "L6-one-candidate" or name.startswith("L3")
    if path == "pipelined":
        h = len(prompts) // 2
        assert subsets[h - 1] is not None and subsets[h] is not None
        assert min(rows) < h <= max(rows)
    if path == "host":
        _, offs, _ = SL.host_layout(prompts)
        assert SL.restricted_host_chunks(prompts, subsets) >= 3, "restricted rows in several host chunks"


@pytest.mark.parametrize("inf", [False, True])
@pytest.mark.parametrize("K", [33, 64])
def test_B_head_groups_past_k(orc, K, inf):
    L, ix, prompts, subsets, rows = SL.b_case(orc, K, inf, "device")
    big = 0
    for r in rows:
        m, total = SL.whole_match(orc, ix, prompts[r], L.E)
        _, mx, _, group = orc.profile_run(PP._oprof(orc, L.prim), SL.narrowed(L, subsets[r]).oracle_pool(orc), m, total)
        if len(group) >= K + (6 if K == 64 else 7):
            big += 1
            assert not inf or np.isposinf(mx)
    assert big >= 5, "subsets whose head group holds 40 / 70 candidates"
    pre_only = [r for r in rows if subsets[r] == L.pre]
    assert pre_only and all(not set(subsets[r]) & set(L.head) for r in pre_only)


@pytest.mark.parametrize("mass", list(SL.MASSES))
@pytest.mark.parametrize("k", [33, 64])
@pytest.mark.parametrize("picker", [PM.RANDOM, PM.WEIGHTED_RANDOM])
def test_B_random_draws_past_32(orc, picker, k, mass):
    L, ix, subsets = SL.random_case(orc, picker, k, mass)
    assert all(40 <= len(s) <= 100 for s in subsets)
    long = 0
    for r, s in enumerate(subsets[:12]):
        cands, sc, draws = SL.random_expect(orc, L, ix, L.prompts[r], s, picker, 0x1234, r, k)
        long += len(draws) > 32
        v = np.array(list(sc.values()))
        if mass == "inf":
            assert np.isposinf(v).any()
        if mass == "zero":
            assert (v == 0).all()
    assert long == 12
    if mass == "scaled":
        assert sum(abs(w) for _, w, _ in L.prim[1]) > 2.0 ** 960


@pytest.mark.parametrize("E", [256, 4096])
def test_C_walk_edges(orc, E):
    W = SL.Walk(orc, E, SL.seed_of("C", E, "fused"), heavy=(6, 33, 1100) if E >= 4096 else (6, 33))
    ix = SL.oracle_index(orc, W.hs, W.es)
    walked, short = set(), 0
    noncontig = 0
    for p, f, s in W.requests:
        h = orc.hash_prompt(p, PP.MODEL, SL.WBST, SL.WB)
        m, n = ix.match_longest_prefix(h, E)
        if not h:
            short += 1
            continue
        walked.add(min(n, len(h)))
        a0 = W.A[f][0]
        if a0 in s and 0 < m[a0] < n - 1:
            noncontig += 1
    assert {31, 32, 33, 63, 64, SL.WB}.issubset(walked) and 0 in walked
    assert short > 0 and noncontig > 0
    counts = {}
    for hsh in W.hs.tolist():
        counts[hsh] = counts.get(hsh, 0) + 1
    need = (6, 33, 1100) if E >= 4096 else (6, 33)
    assert all(any(c >= k + 1 for c in counts.values()) for k in need)
    # the slot that alone holds the blocks a0 / a1 skip is listed by some requests and not by others
    assert any(W.x in s for _, _, s in W.requests) and any(W.x not in s for _, _, s in W.requests)


def test_C_stale_rows_would_be_counted(orc):
    """The batch after the deep one lists the deep family's holders, which hold every block of the stale rows."""
    W = SL.Walk(orc, 256, SL.seed_of("C-stale"))
    deep = SL.STOPS.index(SL.WB)
    assert len(W.H[deep]) > 0 and all(0 < SL.STOPS[f] < SL.WB for f in range(1, 6))


def test_D_cold_ranks_span_chunks(orc):
    C = SL.NohitCase(orc, 20, SL.seed_of("D", 20))
    spanning, one, no_prefill = 0, 0, 0
    for b in range(3):
        prompts, subsets = C.batch(b)
        outs, info = C.expect(prompts, subsets, 64 * b)
        for (out, _), (dc, pc, cd, cp, keys) in zip(outs, info):
            never = [i for i, e in enumerate(dc) if e not in set(keys)]
            if cd and len(dc) > 32 and never and never[0] < 32 <= never[-1] and len(set(dc) & set(keys)):
                spanning += 1
            one += len(dc) == 1 and cd and float(out[0]["score"][0]) >= 1.0
            no_prefill += not pc and len(dc) > 0
        assert len(C.lru.keys()) <= 20
    assert spanning > 10 and one and no_prefill
    assert len(C.lru.keys()) == 20                           # the LRU is smaller than the subsets and full


def test_E_min_max_only_inside_the_subset(orc):
    L, ix, subsets = SL.edge_case(orc)
    assert len(set(L.waiting.tolist())) > 1 and len(set(L.running.tolist())) > 1
    for s in subsets:
        assert len(s) >= 2 and len(set(L.waiting[s].tolist())) == 1 and len(set(L.running[s].tolist())) == 1
    L, neg, releases = SL.inflight_case(61)
    cnt = IM.Counters(L.E)
    cnt.req[:] = 5
    cnt.reset(neg)
    cnt.release(releases, [64] * len(releases))
    assert (cnt.req[neg] < 0).all() and max(0, cnt.req[neg].max()) == 0


@pytest.mark.parametrize("path", ["host", "pipelined"])
def test_F_nonzero_adapters_in_later_chunks(orc, path):
    R = 8192 if path == "pipelined" else 96
    C = SL.LoraCase(orc, SL.seed_of("F", path), R)
    if path == "host":
        _, offs, _ = SL.host_layout(C.prompts)
        chunks = SL.host_chunks(offs)
        assert len(chunks) >= 3
        second = range(*chunks[1]) if chunks[1][1] - chunks[1][0] > 1 else range(*chunks[2])
    else:
        second = range(R // 2, R)
    assert any(C.mids[r] != 0 for r in second)
    held = 0
    for r in list(second)[:30]:
        m = SL.whole_match(orc, C.ix, C.prompts[r], C.E, model=SL.LORA_MODELS[int(C.mids[r])])[0]
        held += C.mids[r] != 0 and (m > 0).any()
    assert held > 0, "requests of adapters other than 0 match their own families"
    assert any(mi != 0 for _, mi, _ in C.members)
