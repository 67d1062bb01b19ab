"""Every path of the index write side (csrc/index_store.cu: indexer.Add, LRU eviction, RemovePod, PreRequest) and of
the incremental patch of the read table, against the CPU oracle's indexer running the same calls one at a time.

index_add only queues, so each test profiles the call that applies the queue (index_commit) and first proves from the
torch.profiler trace, and from last_index_patched, that the path it is about ran.  Then index_get of every hash of the
test's universe (the all-ones hash included) and the number of pairs of the inverted map must equal the oracle's; the
read-table tests also compare prefix_match rows and schedule decisions with orc.cycle_batch, so that run detection sees
interned, un-interned and tombstoned lists next to each other.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import assert_ran, kernels_launched, ran, trace_complete

pytestmark = pytest.mark.gpu

ALL1 = 0xFFFFFFFFFFFFFFFF
BST, B = 4, 8                                  # tokens per block and prefix cap of the engines that also match prompts
PROF = [(0, 3.0, 0), (2, 2.0, 0), (1, 2.0, 0)]
SUB = 1 << 18                                  # queued calls per store batch (flush_add_queue, engine.cu)


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    _load_kernels(epp_b200)
    return epp_b200


def _load_kernels(epp):
    """Launches every write-side and read-table kernel once, in a throwaway engine: traces that contained a kernel's
    first launch in the process have lost their device records, and the commits these tests profile cannot be
    repeated."""
    with epp.Engine(8, lru_capacity_per_server=2) as eng:
        eng.index_add(0, _keys(0, 600))            # a new LRU (compaction + repack), a leak, evictions, a rehash
        eng.index_add(1, [ALL1])
        eng.index_commit()                         # bulk build
        for e in range(1, 8):
            eng.index_add(e, _keys(0, 2))
        eng.index_commit()                         # patch with spilled lists
        eng.index_remove_endpoint(1)
        eng.index_retain_endpoints([2, 3])
        eng.index_get(ALL1)


def _keys(start, n):
    """n distinct hashes, keyed by start .. start + n - 1 (an odd multiplier is a bijection of 64-bit words)."""
    k = (np.arange(start, start + n, dtype=np.uint64) + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)
    assert not (k == np.uint64(ALL1)).any()
    return [int(x) for x in k]


class Both:
    """The engine and the oracle's indexer, driven by the same calls."""

    def __init__(self, eng, ix):
        self.eng, self.ix = eng, ix
        self.universe = {ALL1}

    def add(self, e, hs, nb=0):
        hs = [int(h) for h in hs]
        self.eng.index_add(e, hs, nb)
        self.ix.add(hs, e, nb)
        self.universe.update(hs)

    def remove(self, e):
        self.eng.index_remove_endpoint(e)
        self.ix.remove_pod(e)

    def retain(self, active):
        self.eng.index_retain_endpoints(active)
        for p in self.ix.pods():
            if p not in active:
                self.ix.remove_pod(p)

    def commit(self, where, ran_=(), absent=(), patched=None):
        """index_commit under the profiler: asserts the kernels that must / must not have run and the commit path."""
        _, names = kernels_launched(self.eng.index_commit, repeatable=False)
        for k in ran_:
            assert_ran(names, k, where=where)
        if absent:
            assert trace_complete(names), f"{where}: the trace lost its device records; kernels: {sorted(names)}"
        for k in absent:
            assert not ran(names, k), f"{where}: {k} ran; kernels: {sorted(names)}"
        if patched is not None:
            assert self.eng.stats()["last_index_patched"] == patched, f"{where}: last_index_patched"
        return names

    def check(self, where, sample=None, rng=None):
        """index_get of the universe (or of `sample` random members and the all-ones hash) and the pair count."""
        hs = sorted(self.universe)
        if sample is not None and sample < len(hs):
            hs = [ALL1] + [hs[i] for i in rng.choice(len(hs), sample, replace=False)]
        for h in hs:
            assert self.eng.index_get(h) == self.ix.get(h), f"{where}: index_get({h:#x})"
        assert self.eng.stats()["index_pairs"] == len(self.ix.export()[0]), f"{where}: index_pairs"


def _pack(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    return np.frombuffer(b"".join(prompts) + b"\0" * 16, dtype=np.uint8).copy(), offs


def _prompts(orc, rng, n):
    """n prompts of B blocks -> (prompts, their block hashes)."""
    ps = [rng.integers(0, 256, 4 * BST * B, dtype=np.uint8).tobytes() for _ in range(n)]
    return ps, [orc.hash_prompt(p, b"m", BST, B) for p in ps]


def _reader(epp, E, **kw):
    """An engine that also matches and schedules prompts (model b"m", a fixed pool)."""
    eng = epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(k, w, p) for k, w, p in PROF]), block_size_tokens=BST,
                     max_prefix_blocks=B, **kw)
    eng.register_model(b"m")
    eng.pool_set(np.arange(E), np.zeros(E, np.uint8), (np.arange(E) % 4) / 4.0, (np.arange(E) % 3).astype(np.int32))
    return eng


def _check_reads(orc, both, prompts, E, where):
    """prefix_match rows and schedule decisions against the oracle."""
    import helpers
    d, o = _pack(prompts)
    match, total = both.eng.prefix_match(d, offsets=o)
    for r, p in enumerate(prompts):
        want, _ = both.ix.match_longest_prefix(orc.hash_prompt(p, b"m", BST, B), E)
        np.testing.assert_array_equal(match[r], want, err_msg=f"{where}: prefix_match row {r}")
    dec, det = both.eng.schedule(d, offsets=o)
    pool = orc.PoolState(np.zeros(E, np.uint8), (np.arange(E) % 4) / 4.0, (np.arange(E) % 3).astype(np.int32))
    odec, ototal = orc.cycle_batch(b"m", BST, B, 0, False, both.ix, orc.make_profile(0, PROF), None, pool, d, o, 4)
    helpers.assert_decisions_equal(dec, det, odec, ototal, where=where)


# ------------------------------------------------------------------------------------------------
# 1. store paths
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("repack", [False, True])
def test_log_compaction_vs_oracle(epp, orc, repack):
    """k_compact_count / scan / scatter / copyback / finish: three endpoints whose logs run out of segment in the same
    apply, with tails mid-block (earlier evictions), dead entries from re-adds and live entries spread over several
    256-entry blocks.  Without repack the batch fits the compacted segment; with it (a batch several times the LRU)
    k_store_repack follows in the same apply.  Later rounds evict through the compacted logs."""
    rng = np.random.default_rng(41 + repack)
    caps = {0: 1000, 3: 700, 5: 1500}          # segments of 4 352, 3 072 and 6 400 entries after the creating batch
    nxt = [0]

    def fresh(n):
        nxt[0] += n
        return _keys(nxt[0] - n, n)

    with epp.Engine(8, lru_capacity_per_server=64) as eng:
        both = Both(eng, orc.Indexer(64))
        hist = {}
        for e, c in caps.items():
            hist[e] = fresh(c)
            both.add(e, hist[e], c)
        both.commit("creating batch")
        both.check("creating batch")
        compacted = None
        for rnd in range(9):
            big = repack and rnd == 2 and compacted is None
            for e, c in caps.items():
                calls = 5 if big else 3
                for _ in range(calls):
                    n = c * 8 // 10 if big else c * 7 // 30
                    recent = hist[e][-c:]
                    re_add = [recent[i] for i in rng.choice(len(recent), n // 2, replace=False)]
                    hs = re_add + fresh(n - n // 2)
                    rng.shuffle(hs)
                    both.add(e, hs)
                    hist[e] += hs
            where = f"repack={repack} round {rnd}"
            names = both.commit(where)
            if compacted is None and ran(names, "k_compact_scatter"):
                compacted = rnd
                assert_ran(names, "k_compact_copyback", where=where)
                if repack:
                    assert_ran(names, "k_store_repack", where=where)
                else:
                    assert trace_complete(names) and not ran(names, "k_store_repack"), f"{where}: {sorted(names)}"
                both.check(where)
            else:
                both.check(where, sample=1500, rng=rng)
        assert compacted is not None and compacted < 7, compacted
        both.check("final")


def test_eviction_cut_far_past_the_tail_vs_oracle(epp, orc):
    """k_evict_cut beyond its first 32 x 8-block strip: 40 000 distinct hashes, the same 40 000 again, then 30 000 new
    ones with an LRU of 40 000 put the cut 70 000 entries (273 blocks) past the tail.  Then one apply that evicts from
    48 endpoints with different LRU sizes and block counts (evict_locate over a long endpoint list)."""
    rng = np.random.default_rng(5)
    with epp.Engine(64, lru_capacity_per_server=40000) as eng:
        both = Both(eng, orc.Indexer(40000))
        a, c = _keys(0, 40000), _keys(40000, 30000)
        both.add(0, a)
        both.add(0, a)
        both.add(0, c)
        both.commit("cut 273 blocks past the tail", ran_=("k_evict_count", "k_evict_cut", "k_evict_apply"))
        assert eng.index_get(a[29999]) == set() and eng.index_get(a[30000]) == {0}
        both.check("cut 273 blocks past the tail")
        nxt = 70000
        caps = {e: 40 + 97 * e for e in range(1, 49)}
        for e, cap in caps.items():
            both.add(e, _keys(nxt, cap), cap)
            nxt += cap
        both.commit("many endpoints: creating calls")
        for e, cap in caps.items():
            for _ in range(1 + e % 3):
                n = int(rng.integers(1, cap + 1))
                both.add(e, _keys(nxt, n))
                nxt += n
        both.commit("many endpoints: evictions", ran_=("k_evict_count", "k_evict_cut", "k_evict_apply"))
        both.check("many endpoints: evictions", sample=20000, rng=rng)


def test_pair_table_rehash_keeps_leaked_pairs_vs_oracle(epp, orc):
    """k_store_rehash while leaked pairs (in_map = 1, seq = 0) and all-ones-hash records exist: after the rehash the
    leaked pairs are still visible, still survive RemovePod, and disappear once re-added and evicted normally."""
    rng = np.random.default_rng(9)
    with epp.Engine(16, lru_capacity_per_server=4) as eng:
        both = Both(eng, orc.Indexer(4))
        leaked = {}
        for e in range(8):
            hs = _keys(100 * e, 12)
            if e < 3:
                hs[0] = ALL1                       # leaks
            elif e < 5:
                hs[-1] = ALL1                      # stays in the LRU
            both.add(e, hs)
            leaked[e] = hs[:8]
        both.commit("leaks")
        both.check("leaks")
        assert eng.index_get(ALL1) == {0, 1, 2, 3, 4}
        for e in range(8, 16):                     # churn: 24 000 new pairs outgrow the 1 024-entry pair table
            both.add(e, _keys(10000 + 3000 * e, 3000), 5000)
        both.commit("rehash", ran_=("k_store_count_alive", "k_store_rehash"))
        both.check("after rehash", sample=3000, rng=rng)
        for e in range(8):
            for h in leaked[e]:
                assert e in eng.index_get(h), (e, h)
        for e in range(4):
            both.remove(e)
        both.commit("RemovePod")
        both.check("leaked pairs survive RemovePod", sample=3000, rng=rng)
        for e in range(4):
            assert all(e in eng.index_get(h) for h in leaked[e]), e
        for e in range(4):                         # a new LRU of 4: re-add the leaked hashes, then push them out
            for i in range(0, 8, 4):
                both.add(e, leaked[e][i:i + 4])
            both.add(e, _keys(900 + 100 * e, 4))
        both.commit("re-added and evicted")
        both.check("re-added and evicted", sample=3000, rng=rng)
        for e in range(4):
            assert not any(e in eng.index_get(h) for h in leaked[e]), e


K = _keys(1 << 40, 64)                             # hashes of the leak-boundary cases


def _leak_case(name):
    """(default LRU size, steps): a step is ("add", ep, hashes, num_gpu_blocks), ("rm", ep), ("retain", eps) or
    ("commit",)."""
    a, b, c, d, x, y = K[:6]
    if name == "lru1":
        return 1, [("add", 0, [a], 0), ("add", 0, [a, b], 0), ("add", 1, [a, b, c], 0), ("add", 2, [a, a, b, b], 0),
                   ("commit",), ("add", 0, [c, a, c], 0), ("add", 1, [ALL1, d], 0), ("add", 2, [b, ALL1], 0), ("commit",)]
    if name == "cap_and_cap_plus_1":
        return 5, [("add", 0, K[:5], 0), ("add", 1, K[:6], 0), ("add", 2, K[10:16], 0), ("add", 2, K[:5], 0),
                   ("commit",), ("add", 3, K[20:25] + K[20:21], 0), ("add", 0, K[30:36], 0), ("commit",)]
    if name == "cap_minus_1_or_cap_distinct_follow":
        return 4, [("add", 0, [x, a, b, c, a, b], 0),          # 3 distinct after the last x: kept in the LRU
                   ("add", 1, [x, a, b, c, d, a], 0),          # 4: x leaks
                   ("add", 2, [a, x, b, c, d, b, c], 0),       # a leaks, x does not
                   ("add", 3, [x, y, a, x, b, c, d, y], 0),    # last x followed by exactly 4: leaks
                   ("commit",), ("add", 1, [y, K[9], K[10], K[11]], 0), ("add", 3, K[12:16], 0), ("commit",)]
    if name == "leak_then_readd_same_batch":
        return 3, [("add", 0, [a, b, c, d, x], 0), ("add", 0, [a], 0), ("add", 0, [y, K[8], K[9]], 0),
                   ("add", 1, [a, b, c, d, x], 0), ("add", 1, [b], 0), ("commit",)]
    if name == "retain_with_leaks":
        return 3, [("add", e, K[8 * e: 8 * e + 8], 0) for e in range(4)] + [
                   ("commit",), ("retain", [0, 2]), ("commit",), ("add", 1, K[:3], 0), ("commit",)]
    if name == "lru_recreated_after_removepod":
        return 4, [("add", 0, K[:3], 3), ("add", 0, K[3:9], 0), ("commit",), ("rm", 0), ("add", 0, K[20:27], 7),
                   ("add", 0, K[30:33], 0), ("commit",), ("rm", 0), ("add", 0, K[40:42], 0), ("add", 0, K[42:50], 0),
                   ("commit",)]
    raise KeyError(name)


@pytest.mark.parametrize("case", ["lru1", "cap_and_cap_plus_1", "cap_minus_1_or_cap_distinct_follow",
                                  "leak_then_readd_same_batch", "retain_with_leaks", "lru_recreated_after_removepod"])
def test_leak_boundaries_vs_oracle(epp, orc, case):
    """k_store_leak at its edges (an Add of more hashes than the LRU holds evicts hashes of the same call and leaves
    them in the inverted map), and the leaked pairs under later Adds, CleanUpInactivePods and a re-created LRU."""
    cap, steps = _leak_case(case)
    with epp.Engine(8, lru_capacity_per_server=cap) as eng:
        both = Both(eng, orc.Indexer(cap))
        queued = False                                 # RemovePod and CleanUpInactivePods apply the queue themselves
        for i, st in enumerate(steps):
            if st[0] == "add":
                both.add(st[1], st[2], st[3])
                queued = True
                continue
            if st[0] == "rm":
                both.remove(st[1])
            elif st[0] == "retain":
                both.retain(st[1])
            else:
                both.commit(f"{case} step {i}", ran_=("k_store_upsert", "k_store_leak") if queued else ())
                both.check(f"{case} step {i}")
            queued = False


def test_queue_split_into_sub_batches_vs_oracle(epp, orc):
    """More than 2^18 queued calls in one flush: flush_add_queue applies them as two store batches, in order.  Calls on
    both sides of the boundary depend on each other: endpoint 61 adds the same hash last before and first after it
    (LRU of 3, so the order decides what is evicted), endpoint 62 is created by a call of the second sub-batch with its
    own num_gpu_blocks, and endpoint 63, created in the first one, passes another size in the second (ignored)."""
    rng = np.random.default_rng(3)
    n_calls = SUB + 3000
    u = _keys(0, 4000)
    ep = rng.integers(0, 61, n_calls)
    pick = rng.integers(0, len(u), n_calls)
    special = {SUB - 3: (61, u[0], 0), SUB - 2: (61, u[1], 0), SUB - 1: (61, u[2], 0), SUB: (61, u[2], 0),
               SUB + 1: (61, u[3], 0), SUB + 2: (61, u[0], 0),
               SUB + 5: (62, u[4], 2), SUB + 6: (62, u[5], 0), SUB + 7: (62, u[6], 0),
               SUB - 10: (63, u[7], 0), SUB + 8: (63, u[8], 9), SUB + 9: (63, u[9], 0), SUB + 10: (63, u[10], 0),
               SUB + 11: (63, u[11], 0)}
    with epp.Engine(64, lru_capacity_per_server=3) as eng:
        both = Both(eng, orc.Indexer(3))
        for i in range(n_calls):
            e, h, nb = special.get(i, (int(ep[i]), u[pick[i]], 0))
            if i % 5000 == 4999:
                both.add(e, [h, u[(pick[i] + 1) % len(u)], u[(pick[i] + 7) % len(u)], ALL1], nb)
            else:
                both.add(e, [h], nb)
        names = both.commit("two sub-batches")
        upserts = sum(c for n, c in names.items() if "k_store_upsert" in n)
        assert upserts == 2, upserts
        both.check("two sub-batches")
        assert eng.index_get(u[2]) & {61} and not eng.index_get(u[1]) & {61}


# ------------------------------------------------------------------------------------------------
# 2. read-table paths
# ------------------------------------------------------------------------------------------------
PATCH = ("k_patch_group", "k_patch_apply", "k_patch_intern_claim", "k_patch_intern_apply")


def test_patch_apply_branches_vs_oracle(epp, orc):
    """Every branch of k_patch_apply in one patched commit -- inline to inline, inline to spilled, more than 16 entries
    at once from an inline list, spilled to spilled (copy-on-write), spilled to inline, down to a tombstone -- then a
    tombstone revived, and a commit whose change log is empty (re-adds of cached pairs): patched with no k_patch_* or
    k_index_* launch.  Prompts whose blocks carry interned lists (bulk build), lists the patch re-interned and
    tombstones next to each other check run detection through prefix_match and schedule."""
    E = 128
    rng = np.random.default_rng(17)
    prompts, ph = _prompts(orc, rng, 6)
    with _reader(epp, E) as eng:
        both = Both(eng, orc.Indexer())
        lists = {}                                 # block hash -> initial holders
        p0, p1, p2 = ph[0], ph[1], ph[2]
        for h in p0:                               # one interned list over a whole prompt
            lists[h] = list(range(60, 68))
        lists[p1[0]], lists[p1[1]], lists[p1[2]] = [0, 1], [0, 1, 2, 3], [4, 5, 6]
        lists[p1[3]], lists[p1[4]], lists[p1[5]] = list(range(7, 15)), list(range(40, 47)), [50, 51]
        lists[p1[6]] = lists[p1[7]] = list(range(7, 15))
        for h in p2:
            lists[h] = [int(x) for x in rng.choice(E, int(rng.integers(1, 9)), replace=False)]
        for h, eps in lists.items():
            for e in eps:
                both.add(e, [h])
        both.add(100, ph[3][:5])
        both.commit("bulk build", ran_=("k_index_insert", "k_intern_claim"), patched=0)
        both.check("bulk build")
        _check_reads(orc, both, prompts, E, "bulk build")

        both.add(2, [p1[0]])                                       # inline -> inline (3)
        for e in (4, 5, 6):
            both.add(e, [p1[1]])                                   # inline -> spilled (7)
        for e in range(70, 85):
            both.add(e, [p1[2]])                                   # 15 at once onto an inline list (18)
        for e in (90, 91):
            both.add(e, [p1[3], p1[6]])                            # spilled -> spilled, copy-on-write (10)
        for e in (41, 42, 43, 44, 50, 51):
            both.remove(e)                                         # spilled -> inline (3); p1[5] -> tombstone
        for h in p0[2:4]:
            both.add(68, [h])                                      # two equal new lists inside an interned run
        both.commit("patch branches", ran_=PATCH, absent=("k_index_insert",), patched=1)
        assert eng.index_get(p1[5]) == set() and len(eng.index_get(p1[2])) == 18
        both.check("patch branches")
        _check_reads(orc, both, prompts, E, "patch branches")

        both.add(52, [p1[5]])                                      # tombstone revived
        both.add(101, ph[4])
        both.commit("revive", ran_=("k_patch_group", "k_patch_apply"), absent=("k_index_insert",), patched=1)
        assert eng.index_get(p1[5]) == {52}
        both.check("revive")
        _check_reads(orc, both, prompts, E, "revive")

        both.add(101, ph[4])                                       # cached pairs again: nothing enters or leaves the map
        both.add(60, [p0[0]])
        both.commit("empty change log", ran_=("k_store_upsert",), absent=("k_patch_", "k_index_"), patched=1)
        both.check("empty change log")
        _check_reads(orc, both, prompts, E, "empty change log")


@pytest.mark.parametrize("rule", ["change_set", "load_factor"])
def test_patch_size_rules_vs_oracle(epp, orc, rule):
    """One commit on each side of a rule of patch_read_table: the change set (at most max(2^16, pairs / 2) logged
    changes) and the table's load factor (used slots + changes <= 6/10 of the slots).  The first commit is exactly at
    the bound and patches, the second is one over it and takes the bulk build."""
    rng = np.random.default_rng(23)
    if rule == "change_set":
        D, slots, first, second = 70000, 1 << 19, [(2, 70000)], [(3, 70000), (4, 35001)]   # 70 000 <= 140 000 / 2
    else:
        D, slots, first, second = 4096, 1 << 14, [(2, 4096), (3, 1638)], [(4, 4096), (5, 1639)]  # 4 096 + 5 734 <= 9 830.4
    hs = _keys(7, D)
    with epp.Engine(8, lru_capacity_per_server=200000) as eng:
        both = Both(eng, orc.Indexer(200000))
        both.add(0, hs)
        both.add(1, hs)
        both.commit("bulk build", patched=0)
        assert eng.stats()["index_slots"] == slots
        for e, n in first:
            both.add(e, hs[:n])
        both.commit(f"{rule}: at the bound", ran_=("k_patch_apply",), absent=("k_index_insert",), patched=1)
        both.check(f"{rule}: at the bound", sample=3000, rng=rng)
        for e, n in second:
            both.add(e, hs[:n])
        both.commit(f"{rule}: one over", ran_=("k_index_insert",), absent=("k_patch_group",), patched=0)
        both.check(f"{rule}: one over", sample=3000, rng=rng)


def test_patch_falls_back_on_the_all_ones_hash_vs_oracle(epp, orc):
    """A change log that names the all-ones hash (kept in the side record of the bulk build): k_patch_group sees it,
    k_patch_apply does not run, and the commit takes the bulk build."""
    E = 16
    rng = np.random.default_rng(29)
    prompts, ph = _prompts(orc, rng, 3)
    with _reader(epp, E) as eng:
        both = Both(eng, orc.Indexer())
        for e in range(8):
            both.add(e, ph[e % 3][: 2 + e % 6])
        both.commit("bulk build", patched=0)
        both.add(3, ph[1])
        both.commit("patch", ran_=("k_patch_apply",), patched=1)
        both.add(9, [ph[2][0], ALL1])
        both.commit("all-ones hash", ran_=("k_patch_group", "k_index_insert"), absent=("k_patch_apply",), patched=0)
        both.check("all-ones hash")
        _check_reads(orc, both, prompts, E, "all-ones hash")
        both.add(10, [ph[0][0]])
        both.commit("patch after the rebuild", ran_=("k_patch_apply",), patched=1)
        both.check("patch after the rebuild")


def test_patch_runs_out_of_posting_space_vs_oracle(epp, orc):
    """Lists of 200 endpoints copied on write use up the posting space a bulk build leaves for patches (2^20 entries)
    within a few commits; the commit whose k_patch_apply runs out partway takes the bulk build in the same commit.  The
    lists stay identical to one another, so that the interning bound never trips first."""
    E, L = 208, 1000
    hs = _keys(11, L)
    with epp.Engine(E) as eng:
        both = Both(eng, orc.Indexer())
        for e in range(200):
            both.add(e, hs)
        both.commit("bulk build", patched=0)
        fell_back = None
        for rnd in range(12):
            x = 200 + rnd % 2
            if rnd % 4 < 2:
                both.add(x, hs)
            else:
                both.remove(x)
            where = f"round {rnd}"
            names = both.commit(where, ran_=("k_patch_group", "k_patch_apply"))
            both.check(where)
            if eng.stats()["last_index_patched"] == 0:
                assert_ran(names, "k_index_insert", where=where)
                fell_back = rnd
                break
            assert trace_complete(names) and not ran(names, "k_index_insert"), f"{where}: {sorted(names)}"
        assert fell_back is not None and fell_back >= 2, fell_back
        both.add(205, hs[:10])
        both.commit("patch after the rebuild", ran_=("k_patch_apply",), patched=1)
        both.check("patch after the rebuild")


def test_every_257th_commit_is_a_bulk_build_vs_oracle(epp, orc):
    """commit_locked patches at most 256 times between bulk builds: 256 patched commits in a row, then a bulk build."""
    E = 32
    rng = np.random.default_rng(37)
    prompts, ph = _prompts(orc, rng, 4)
    flat = [h for p in ph for h in p]
    with _reader(epp, E, lru_capacity_per_server=1000) as eng:
        both = Both(eng, orc.Indexer(1000))
        both.add(0, flat + _keys(0, 400))          # every later commit changes lists of these hashes: no new slots
        both.commit("bulk build", patched=0)
        for i in range(1, 258):
            both.add(1 + i % 31, [flat[i % len(flat)]])
            where = f"commit {i}"
            if i in (1, 256, 257):
                both.commit(where, ran_=("k_patch_apply",) if i < 257 else ("k_index_insert",),
                            absent=("k_index_insert",) if i < 257 else ("k_patch_group",), patched=int(i < 257))
                both.check(where)
                _check_reads(orc, both, prompts, E, where)
            else:
                eng.index_commit()
                assert eng.stats()["last_index_patched"] == 1, where
                if i % 32 == 0:
                    both.check(where)


def test_patches_never_fill_the_interning_table_vs_oracle(epp, orc):
    """Regression: every spilled list a patch writes claims a key in the interning table, which only the bulk build
    empties, and a full table would make the next claim probe forever.  16 hashes held by 6 endpoints each (16 keys in
    a 64-slot table); every commit adds one new endpoint to all 16 lists (16 more keys).  patch_read_table must refuse
    a patch that could leave the table more than 6/10 full, so the commits alternate patch, bulk build, patch ... --
    the second commit, with at most 48 of 64 keys taken, is the first bulk build.  300 commits, parity after each."""
    E, n_commits = 400, 300
    rng = np.random.default_rng(43)
    prompts, ph = _prompts(orc, rng, 2)
    hs = [h for p in ph for h in p]                       # 16 distinct block hashes
    with _reader(epp, E) as eng:
        both = Both(eng, orc.Indexer())
        for i, h in enumerate(hs):
            for j in range(6):
                both.add(i + 16 * j, [h])                     # a different set of 6 endpoints per hash
        both.commit("bulk build", ran_=("k_intern_claim",), patched=0)
        assert eng.stats()["index_slots"] == 64
        for c in range(1, n_commits + 1):
            both.add(95 + c, hs)
            where = f"commit {c}"
            if c <= 4:
                both.commit(where, ran_=("k_patch_apply",) if c % 2 else ("k_index_insert",), patched=c % 2)
            else:
                eng.index_commit()
                assert eng.stats()["last_index_patched"] == c % 2, where
            both.check(where)
            if c <= 4 or c % 25 == 0:
                _check_reads(orc, both, prompts, E, where)
