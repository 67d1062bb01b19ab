"""The subset pick kernel (k_subset_pick, csrc/subset_pick.cu) on hand-built landscapes, against the CPU oracle bit for bit:
every landscape of test_pick_paths_gpu.py under restricted requests of every list shape, first-k lists past 32 entries,
random draws past 32, a match walk over prompts of more than 32 blocks (global stops in later chunks, non-contiguous
holders, blocks with 6 / 33 / 1100 holders, trimmed and whole rows, the hash kernels' switches), no-hit-lru cold ranks
over lists of more than one 32-entry chunk, the scorers' edges inside the subset, LoRA adapters other than 0 on the
chunked host and pipelined device paths, and pools of 4096 and 131 073 slots.

A restricted request's expected decision is orc_cycle_batch of that request alone, on the pool with every slot outside
its subset absent (role 0xFF), with tie_base = its ordinal: Schedule called with the subset's endpoints.  No-hit-lru cold
columns come from tools/nohit_lru_model.py over the restricted candidates (fed as ext columns), random draws from
tools/picker_model.py with every candidate explicit.  The builders are plain functions of the oracle:
test_subset_landscapes_cpu.py checks from them alone that each case reaches the edge it names.
Run on an H100: pytest -m gpu."""
import copy
import zlib

import numpy as np
import pytest

import helpers
import test_pick_paths_gpu as PP
from tools import inflight_model as IM
from tools import nohit_lru_model as NH
from tools import picker_model as PM

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
ABSENT = 0xFF
SUBSET = "k_subset_pick"
LORA = 8
HOST_GAP = 49 << 20                 # > the host path's 48 MiB chunk: every gap in a host batch starts a new chunk


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


# ------------------------------------------------------------------------------------------------
# oracle side
# ------------------------------------------------------------------------------------------------
def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


def narrowed(L, subset):
    """L with its pool narrowed to `subset` (None: the whole pool)."""
    if subset is None:
        return L
    N = copy.copy(L)
    N.ids = np.intersect1d(L.ids, np.asarray(subset, np.int64))
    return N


def narrowed_pool(orc, L, subset, ext):
    """The oracle pool of L narrowed to `subset`, with the given ext columns."""
    role = np.full(L.E, ABSENT, np.uint8)
    ids = narrowed(L, subset).ids
    role[ids] = L.role[ids]
    return orc.PoolState(role, L.kv, L.waiting, L.running, ext)


def oracle_index(orc, hs, es):
    ix = orc.Indexer()
    if len(hs):
        ix.load_pairs(hs, es)
    return ix


def expect(orc, L, ix, prompt, subset, tie_seed, ordinal, *, mm=None, topk=0, prim=None, pref="same", pool=None,
           model=PP.MODEL, bst=PP.BST, B=PP.B, always=False):
    """orc_cycle_batch of one request on L's pool narrowed to `subset`."""
    N = narrowed(L, subset)
    d, o = PP._pack([prompt])
    pf = L.pref if pref == "same" else pref
    return orc.cycle_batch(model, bst, B, L.nct, always, ix, PP._oprof(orc, prim or L.prim), PP._oprof(orc, pf),
                           pool if pool is not None else N.oracle_pool(orc), d, o, 1, tie_seed=tie_seed, tie_base=ordinal,
                           encode=PP._oprof(orc, L.enc), multimodal=None if mm is None else np.array([mm], np.uint8),
                           topk=topk)


def whole_match(orc, ix, prompt, E, model=PP.MODEL, bst=PP.BST, B=PP.B):
    h = orc.hash_prompt(prompt, model, bst, B)
    m, _ = ix.match_longest_prefix(h, E)
    return m, len(h)


def check_row(dec, det, lists, r, out, m, where):
    """One engine row against one oracle row: decision, detail, matchBlocks of the pick, first-k lists and score bits."""
    helpers.assert_decisions_equal(dec[r:r + 1], None if det is None else det[r:r + 1], out[0], out[1], where=where)
    if out[0]["status"][0] == 0:
        assert int(dec["match_blocks"][r]) == int(m[int(out[0]["pick"][0])]), f"{where}: match_blocks"
    if lists is not None:
        ol = out[2]
        for name in ("primary", "prefill", "encode"):
            np.testing.assert_array_equal(lists[name][r], ol[name][0], err_msg=f"{where}: {name} list")
        np.testing.assert_array_equal(lists["primary_scores"][r].view(np.uint64), ol["primary_scores"][0].view(np.uint64),
                                      err_msg=f"{where}: primary list scores")


def filter_drops(orc, L, prof):
    """Slots of L's pool that the profile's role filter drops."""
    s = orc.profile_run(orc.make_profile(prof[0], [(PP.QUEUE, 0.0, 0.0)]), L.oracle_pool(orc), np.zeros(L.E, np.int32), 0)[0]
    return [int(e) for e in L.ids if s[e] == -1.0]


def straddle(group, E):
    """A list holding exactly the tie group `group` and the lowest other slots, so that the group has members on both
    sides of list entry 32 (None: no such list)."""
    g = np.array(sorted(group), np.int64)
    if len(g) < 2:
        return None
    rest = np.setdiff1d(np.arange(E), g)
    for f in range(len(rest) + 1):
        s = np.union1d(g, rest[:f])
        pos = np.searchsorted(s, g)
        if pos[0] < 32 <= pos[-1]:
            return s.tolist()
    return None


KINDS = ["all", "holders", "non-holders", "tie-group", 1, 31, 32, 33, 63, 64, 65, "E", "empty", "stale"]


def land_subset(orc, L, ix, prompt, kind, rng, drops):
    """A request's subset of the given kind, chosen from the landscape."""
    E = L.E
    if kind == "all":
        return None
    m, total = whole_match(orc, ix, prompt, E)
    if kind == "holders":
        return sorted(set(np.flatnonzero(m > 0).tolist()) | set(rng.choice(E, size=min(3, E), replace=False).tolist()))
    if kind == "non-holders":
        free = np.flatnonzero(m == 0)
        return sorted(rng.choice(free, size=min(10, len(free)), replace=False).tolist())
    if kind == "tie-group":
        _, _, _, group = orc.profile_run(PP._oprof(orc, L.prim), L.oracle_pool(orc), m, total)
        s = straddle(group, E)
        return s if s is not None else sorted(rng.choice(E, size=min(33, E), replace=False).tolist())
    if kind == "empty":
        return []
    if kind == "stale":
        extra = sorted(set(range(E)) - set(L.ids.tolist())) + list(drops)
        s = set(rng.choice(L.ids, size=min(8, len(L.ids)), replace=False).tolist())
        if extra:
            s |= set(rng.choice(extra, size=min(8, len(extra)), replace=False).tolist())
        return sorted(s)
    n = E if kind == "E" else min(int(kind), E)
    return sorted(rng.choice(E, size=n, replace=False).tolist())


A_LANDS = list(PP.LANDS) + ["L3-forward", "L3-shuffled"]


def a_land(orc, name):
    if name == "L3-forward":
        return PP.land_rounding(orc, 3, list(range(len(PP.ROUNDING))))
    if name == "L3-shuffled":
        return PP.land_rounding(orc, 3, [3, 6, 1, 4, 0, 5, 2])
    return PP.LANDS[name]()


def pipelined_rows(R, rng, n=300):
    h = R // 2
    return sorted(set(rng.choice(R, size=n, replace=False).tolist()) | {0, 1, h - 2, h - 1, h, h + 1, R - 1})


def a_case(orc, name, path):
    """Case A: landscape, oracle index, prompts (tiled for the pipelined path), multimodal flags, subsets, checked rows."""
    L = a_land(orc, name)
    ix = oracle_index(orc, L.hs, L.es)
    rng = np.random.default_rng(seed_of("A", name, path))
    prompts, mm = list(L.prompts), L.mm
    if path == "pipelined":
        reps = -(-8192 // len(prompts))
        prompts = prompts * reps
        mm = None if mm is None else np.tile(mm, reps)
        rows = pipelined_rows(len(prompts), rng)
    else:
        rows = list(range(len(prompts)))
    drops = filter_drops(orc, L, L.prim)
    subsets = [None] * len(prompts)
    h = len(prompts) // 2
    for i, r in enumerate(rows):
        kind = KINDS[i % len(KINDS)]
        if kind == "all" and path == "pipelined" and r in (h - 1, h):      # both sides of the chunk boundary restricted
            kind = "tie-group"
        subsets[r] = land_subset(orc, L, ix, prompts[r], kind, rng, drops)
    return L, ix, prompts, mm, subsets, rows


# ------------------------------------------------------------------------------------------------
# engine side
# ------------------------------------------------------------------------------------------------
def host_layout(prompts, groups=4):
    """32-byte aligned rows in `groups` runs separated by gaps wider than a host chunk -> (bytes, starts, lengths)."""
    starts, pos = [], 0
    per = -(-len(prompts) // groups)
    for i, p in enumerate(prompts):
        if i and i % per == 0:
            pos += HOST_GAP
        starts.append(pos)
        pos += max(32, (len(p) + 31) // 32 * 32)
    buf = np.zeros(pos + 64, np.uint8)
    for s, p in zip(starts, prompts):
        buf[s: s + len(p)] = np.frombuffer(p, np.uint8)
    return buf, np.array(starts + [pos], np.uint64), np.array([len(p) for p in prompts], np.uint64)


def host_chunks(offsets):
    """The host path's chunk plan over offsets (run_batch: about 48 MiB of prompt bytes, at least one request each)."""
    R, out, r = len(offsets) - 1, [], 0
    while r < R:
        e = r
        while e < R and (e == r or int(offsets[e + 1]) - int(offsets[r]) <= 48 << 20):
            e += 1
        out.append((r, e))
        r = e
    return out


def aligned_rows(prompts, align=64):
    """Rows at multiples of `align` bytes with exact lengths (the fused hash kernel's layout) -> (bytes, starts, lengths)."""
    starts = np.zeros(len(prompts) + 1, np.uint64)
    np.cumsum([(len(p) + align - 1) // align * align + align for p in prompts], out=starts[1:])
    data = np.zeros(int(starts[-1]) + 64, np.uint8)
    for s, p in zip(starts, prompts):
        data[int(s): int(s) + len(p)] = np.frombuffer(p, np.uint8)
    return data, starts, np.array([len(p) for p in prompts], np.uint64)


def odd_packed(prompts):
    """Prompts packed back to back after one leading byte: odd offsets (the generic hash kernel)."""
    offs = np.zeros(len(prompts) + 1, np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    offs += 1
    return np.frombuffer(b"\x00" + b"".join(prompts) + b"\0" * 16, np.uint8).copy(), offs


def run(epp, eng, prompts, subsets, path, *, mm=None, topk=False, model_ids=None, layout=None, keep_hashes=False):
    """One batch on the given path -> (decisions, details, first-k lists or None, kernel names)."""
    import torch
    if path == "host":
        data, offs, lens = host_layout(prompts)
        kw = dict(offsets=offs, lengths=lens)
    elif layout == "aligned":
        data, offs, lens = aligned_rows(prompts)
        kw = dict(offsets=offs, lengths=lens)
    elif layout == "odd":
        data, offs = odd_packed(prompts)
        kw = dict(offsets=offs)
    else:
        data, offs = PP._pack(prompts)
        kw = dict(offsets=offs)
    if path != "host":
        data = torch.from_numpy(data).cuda()
        kw = {k: torch.from_numpy(np.asarray(v).view(np.int64)).cuda() for k, v in kw.items()}
        if mm is not None:
            mm = torch.from_numpy(np.asarray(mm, np.uint8)).cuda()
        if model_ids is not None:
            model_ids = torch.from_numpy(np.asarray(model_ids, np.uint32).view(np.int32)).cuda()
    asyn = path == "pipelined"

    def call():
        r = eng.schedule(data, multimodal=mm, model_ids=model_ids, subsets=subsets, topk=topk, asynchronous=asyn,
                         keep_hashes=keep_hashes, **kw)
        if asyn:
            eng.synchronize()
        return r
    out, names = helpers.kernels_launched(call, repeatable=False)
    if path != "host":
        torch.cuda.synchronize()
        dec, det = epp.decisions_from_torch(out[0]), PP._det(epp, out[1])
    else:
        dec, det = out[0], out[1]
    return dec, det, (PP._lists(out[2]) if topk else None), names


def assert_subset_ran(names, path, where, n_chunks=None):
    if not helpers.trace_complete(names):
        return
    helpers.assert_ran(names, SUBSET, absent=("k_cycle_small",), where=where)
    launches = sum(c for n, c in names.items() if SUBSET in n)
    if path == "pipelined":
        assert launches == 2, f"{where}: {launches} subset launches"
    elif path == "host" and n_chunks:
        assert launches == n_chunks, f"{where}: {launches} subset launches for {n_chunks} chunks with restricted rows"


def restricted_host_chunks(prompts, subsets):
    _, offs, _ = host_layout(prompts)
    return sum(1 for r0, r1 in host_chunks(offs) if any(s is not None for s in subsets[r0:r1]))


# ------------------------------------------------------------------------------------------------
# A. every landscape through the subset kernel
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["device", "host", "pipelined"])
@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("name", A_LANDS)
def test_landscape_subsets(epp, orc, name, tie_seed, path):
    L, ix, prompts, mm, subsets, rows = a_case(orc, name, path)
    where = f"{name} tie_seed={tie_seed} {path}"
    with PP._engine(epp, L, tie_seed) as eng:
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, prompts, subsets, path, mm=mm)
    assert_subset_ran(names, path, where, restricted_host_chunks(prompts, subsets) if path == "host" else None)
    for i, r in enumerate(rows):
        out = expect(orc, L, ix, prompts[r], subsets[r], tie_seed, base + r, mm=None if mm is None else int(mm[r]))
        m, _ = whole_match(orc, ix, prompts[r], L.E)
        check_row(dec, det, None, r, out, m, f"{where} request {r} ({KINDS[i % len(KINDS)]})")
    empty = [r for r in rows if subsets[r] == []]
    assert empty and (dec["status"][empty] == -1).all()


# ------------------------------------------------------------------------------------------------
# B. first-k lists and random draws past 32 entries
# ------------------------------------------------------------------------------------------------
def land_deep(seed, head, inf):
    """A P/D pool of 120: 100 decode slots of which `head` form the head group (kv 0, waiting 0; with inf the decode
    weights near 1e308 make its sums +inf), 20 prefill slots; few holders, most prompts cold."""
    rng = np.random.default_rng(seed)
    E = 120
    role = np.ones(E, np.uint8)
    pre = rng.choice(E, 20, replace=False)
    role[pre] = 2
    hd = rng.choice(np.flatnonzero(role == 1), head, replace=False)
    kv, waiting = np.full(E, 0.5), np.full(E, 3, np.int32)
    kv[hd], waiting[hd] = 0.0, 0
    kv[pre[:8]], waiting[pre[:8]] = 0.0, 0
    w1, w2 = (1e308, 1.7e308) if inf else (1.0, 1.0)
    L = PP.Land(E, role, kv, waiting, (PP.F_DECODE, [(PP.KV, w1, 0.0), (PP.QUEUE, w2, 0.0), (PP.PREFIX, 1.0, 0.0)]),
                pref=(PP.F_PREFILL, [(PP.KV, 1.0, 0.0), (PP.PREFIX, 1.0, 0.0)]),
                holders=PP._holders(rng, np.arange(E), [2, 5]), nct=4, seed=seed, cold_share=0.6, R=64)
    L.head, L.pre = sorted(hd.tolist()), sorted(pre.tolist())
    return L


DEEP_KINDS = ["E", "head+5", "head", "prefill-only", "random-90"]


def deep_subset(L, kind, rng):
    E = L.E
    if kind == "E":
        return list(range(E))
    if kind == "head":
        return L.head
    if kind == "head+5":
        return sorted(set(L.head) | set(rng.choice(E, 5, replace=False).tolist()))
    if kind == "prefill-only":
        return L.pre
    return sorted(rng.choice(E, 90, replace=False).tolist())


def b_case(orc, K, inf, path):
    L = land_deep(seed_of("B", K, inf), 40 if K == 33 else 70, inf)
    ix = oracle_index(orc, L.hs, L.es)
    rng = np.random.default_rng(seed_of("B-subsets", K, inf, path))
    prompts = list(L.prompts)
    if path == "pipelined":
        prompts = prompts * -(-8192 // len(prompts))
        rows = pipelined_rows(len(prompts), rng, n=200)
    else:
        rows = list(range(len(prompts)))
    subsets = [None] * len(prompts)
    for i, r in enumerate(rows):
        subsets[r] = deep_subset(L, DEEP_KINDS[i % len(DEEP_KINDS)], rng)
    return L, ix, prompts, subsets, rows


@pytest.mark.parametrize("path", ["device", "pipelined"])
@pytest.mark.parametrize("inf", [False, True])
@pytest.mark.parametrize("K", [33, 64])
def test_deep_first_k_lists(epp, orc, K, inf, path):
    """Max-score lists of 33 / 64 entries over subsets whose head group has 40 / 70 candidates (+inf-headed with inf),
    a P/D prefill list, and prefill-only subsets (no decode candidate: every list of the row stays empty)."""
    tie_seed = 0xAB
    L, ix, prompts, subsets, rows = b_case(orc, K, inf, path)
    where = f"K={K} inf={inf} {path}"
    with PP._engine(epp, L, tie_seed, pick_k=K) as eng:
        base = eng.stats()["n_decisions"]
        dec, det, lists, names = run(epp, eng, prompts, subsets, path, topk=True)
    assert_subset_ran(names, path, where)
    for i, r in enumerate(rows):
        out = expect(orc, L, ix, prompts[r], subsets[r], tie_seed, base + r, topk=K)
        m, _ = whole_match(orc, ix, prompts[r], L.E)
        check_row(dec, det, lists, r, out, m, f"{where} request {r} ({DEEP_KINDS[i % len(DEEP_KINDS)]})")
        row = lists["primary"][r]
        assert len(set(row[row >= 0].tolist())) == int((row >= 0).sum()), f"{where} request {r}: repeated endpoint"


MASSES = {
    "inf": [(PP.KV, 1e308, 0.0), (PP.QUEUE, 1.7e308, 0.0), (PP.PREFIX, 1.0, 0.0)],       # +inf scores
    "zero": [(PP.KV, 0.0, 0.0), (PP.QUEUE, 0.0, 0.0), (PP.PREFIX, 0.0, 0.0)],           # W = 0
    "scaled": [(PP.KV, 1e300, 0.0), (PP.QUEUE, 6e299, 0.0), (PP.PREFIX, 2e299, 0.0)],   # sum |w| > 2^960
}


def random_case(orc, picker, k, mass):
    """Case B (random pickers): a pool of 120, subsets of 40-100 candidates -> (L, ix, subsets, expected draws)."""
    rng = np.random.default_rng(seed_of("Brnd", picker, k, mass))
    E = 120
    kv = rng.choice([0.0, 0.25, 0.5, 1.0], E)
    waiting = rng.integers(0, 6, E).astype(np.int32)
    L = PP.Land(E, np.zeros(E, np.uint8), kv, waiting, (PP.F_NONE, MASSES[mass]),
                holders=PP._holders(rng, np.arange(E), [3, 12, 45]), R=48, seed=seed_of("Brnd-land", mass))
    ix = oracle_index(orc, L.hs, L.es)
    subsets = [sorted(rng.choice(E, size=int(rng.integers(40, 101)), replace=False).tolist()) for _ in L.prompts]
    return L, ix, subsets


def random_expect(orc, L, ix, prompt, s, picker, tie_seed, ordinal, k):
    """-> (candidates, their scores, picker_model draws)."""
    m, total = whole_match(orc, ix, prompt, L.E)
    scores, _, _, _ = orc.profile_run(PP._oprof(orc, L.prim), narrowed(L, s).oracle_pool(orc), m, total)
    cands = [e for e in s if scores[e] != -1.0]
    sc = {e: float(scores[e]) for e in cands}
    draws = PM.draw_k(picker, cands, None, sc, set(), tie_seed, 4 * ordinal, [w for _, w, _ in L.prim[1]], k, gaps=False)
    return cands, sc, draws


@pytest.mark.parametrize("mass", list(MASSES))
@pytest.mark.parametrize("k", [33, 64])
@pytest.mark.parametrize("picker", [PM.RANDOM, PM.WEIGHTED_RANDOM])
def test_deep_random_lists(epp, orc, picker, k, mass):
    tie_seed = 0x1234
    L, ix, subsets = random_case(orc, picker, k, mass)
    spec = epp.ProfileSpec(PP.F_NONE, [epp.ScorerSpec(*s) for s in L.prim[1]], picker=picker)
    with epp.Engine(L.E, spec, block_size_tokens=PP.BST, max_prefix_blocks=PP.B, tie_seed=tie_seed, pick_k=k) as eng:
        eng.register_model(PP.MODEL)
        eng.pool_set(*L.pool_arrays())
        eng.index_load_snapshot(np.array(L.hs, np.uint64), np.array(L.es, np.uint32))
        base = eng.stats()["n_decisions"]
        dec, _, lists, names = run(epp, eng, L.prompts, subsets, "device", topk=True)
    assert_subset_ran(names, "device", f"picker {picker} k={k} {mass}")
    for r, s in enumerate(subsets):
        cands, _, draws = random_expect(orc, L, ix, L.prompts[r], s, picker, tie_seed, base + r, k)
        where = f"picker {picker} k={k} {mass} request {r}"
        assert int(dec["status"][r]) == 0 and int(dec["pick"][r]) == draws[0][0], where
        assert dec["score"][r:r + 1].view(np.uint64)[0] == np.array([draws[0][1]]).view(np.uint64)[0], where
        assert int(dec["tie_count"][r]) == len(cands), where
        got = [int(x) for x in lists["primary"][r] if x >= 0]
        assert got == [p for p, _ in draws], where
        np.testing.assert_array_equal(lists["primary_scores"][r][: len(draws)].view(np.uint64),
                                      np.array([s for _, s in draws]).view(np.uint64), err_msg=where)


# ------------------------------------------------------------------------------------------------
# C. the match walk over prompts of more than 32 blocks
# ------------------------------------------------------------------------------------------------
WB, WBST = 128, 16                  # 128-block cap, 64-byte blocks (the fused hash kernel's block size)
WBB = 4 * WBST
STOPS = [0, 31, 32, 33, 63, 64, WB]


class Walk:
    """Families of prompts whose global stop (the first block no endpoint holds) falls on each of STOPS.  Family f has a
    holder set H (6 / 33 / 1100 slots, in turn) holding every block before its stop; slots a0 and a1 hold only the even
    blocks and the multiples of 3; a slot x outside every subset holds the other blocks, so the index holds each block up
    to the stop and a0 / a1 hold non-contiguous blocks."""

    def __init__(self, orc, E, seed, heavy=(6, 33), R=96):
        rng = np.random.default_rng(seed)
        self.E, self.rng = E, rng
        self.x = E - 1
        free = list(rng.permutation(E - 1))
        self.fam, self.H, self.A = [], [], []
        hs, es = [], []
        for f, stop in enumerate(STOPS):
            fam = rng.integers(0, 256, WBB * (WB + 2), dtype=np.uint8).tobytes()
            h = orc.hash_prompt(fam, PP.MODEL, WBST, WB)
            H = sorted(int(free.pop()) for _ in range(heavy[f % len(heavy)]))
            A = [int(free.pop()), int(free.pop())]
            for i in range(stop):
                holders = set(H)
                if i % 2 == 0:
                    holders.add(A[0])
                if i % 3 == 0:
                    holders.add(A[1])
                if i % 2 and i % 3:
                    holders.add(self.x)
                hs += [h[i]] * len(holders)
                es += sorted(holders)
            self.fam.append(fam)
            self.H.append(H)
            self.A.append(A)
        self.hs, self.es = np.array(hs, np.uint64), np.array(es, np.uint32)
        self.free = free
        self.role = np.zeros(E, np.uint8)
        self.kv = np.zeros(E)
        self.waiting = rng.integers(0, 4, E).astype(np.int32)
        self.prim = (PP.F_NONE, [(PP.PREFIX, 1.0, 0.0), (PP.KV, 1.0, 0.0)])
        self.requests = [self.request(r) for r in range(R)]

    def request(self, r):
        """(prompt, family or None, subset) of request r."""
        rng = self.rng
        if r % 16 == 15:                                     # shorter than one block: no hash at all
            return rng.integers(0, 256, int(rng.integers(1, WBB)), dtype=np.uint8).tobytes(), None, \
                sorted(rng.choice(self.E, 5, replace=False).tolist())
        f = r % len(STOPS)
        stop = STOPS[f]
        n = WB + 2 if r % 3 == 0 else int(rng.integers(min(stop + 1, WB), WB + 1))
        prompt = self.fam[f][: n * WBB - int(rng.integers(0, WBB))]
        H, A = self.H[f], self.A[f]
        kind = (r // len(STOPS)) % 4
        others = [int(e) for e in rng.choice(self.free, 3, replace=False)]
        if kind == 0:                                        # every holder listed
            s = set(H) | set(A) | set(others)
        elif kind == 1:                                      # only the non-contiguous holders
            s = set(A) | set(others)
        elif kind == 2:                                      # part of H and a0
            s = set(H[: max(1, len(H) // 2)]) | {A[0]} | set(others)
        else:                                                # the outside holder listed too
            s = set(H[:3]) | set(A) | {self.x}
        return prompt, f, sorted(s)

    def land(self):
        L = PP.Land(self.E, self.role, self.kv, self.waiting, self.prim, R=0)
        return L


def walk_expect(orc, W, L, ix, prompt, s, tie_seed, ordinal):
    return expect(orc, L, ix, prompt, s, tie_seed, ordinal, bst=WBST, B=WB, pref=None)


def walk_engine(epp, W, tie_seed, hs=None, es=None):
    eng = epp.Engine(W.E, PP._spec(epp, W.prim), block_size_tokens=WBST, max_prefix_blocks=WB, tie_seed=tie_seed)
    eng.register_model(PP.MODEL)
    eng.pool_set(np.arange(W.E), W.role, W.kv, W.waiting)
    if hs is None:
        hs, es = W.hs, W.es
    if len(hs):
        eng.index_load_snapshot(hs, es)
    return eng


def check_walk(orc, W, ix, dec, det, prompts, subsets, tie_seed, base, where):
    L = W.land()
    for r, s in enumerate(subsets):
        out = walk_expect(orc, W, L, ix, prompts[r], s, tie_seed, base + r)
        m, _ = whole_match(orc, ix, prompts[r], W.E, bst=WBST, B=WB)
        check_row(dec, det, None, r, out, m, f"{where} request {r}")


@pytest.mark.parametrize("E,variant", [(256, "fused"), (256, "odd-packed"), (256, "EPP_HASH_TRIM=0"),
                                       (256, "EPP_HASH_SKIP=0"), (4096, "fused")])
def test_match_walk(epp, orc, monkeypatch, E, variant):
    """Global stops at blocks 0, 31, 32, 33, 63, 64 and the cap, non-contiguous holders, 6 / 33 (/ 1100) holders of a
    block, prompts shorter than a block; aligned rows through the fused kernel (trimmed) or an odd-offset blob through
    the generic one (untrimmed), and the hash kernels' switches."""
    if variant.startswith("EPP_"):
        k, v = variant.split("=")
        monkeypatch.setenv(k, v)
    tie_seed = 0x3C
    W = Walk(orc, E, seed_of("C", E, variant), heavy=(6, 33, 1100) if E >= 4096 else (6, 33))
    ix = oracle_index(orc, W.hs, W.es)
    prompts = [p for p, _, _ in W.requests]
    subsets = [s for _, _, s in W.requests]
    with walk_engine(epp, W, tie_seed) as eng:
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, prompts, subsets, "device", layout="odd" if variant == "odd-packed" else "aligned")
    where = f"walk E={E} {variant}"
    assert_subset_ran(names, "device", where)
    if helpers.trace_complete(names):
        want = {"fused": "k_hash_fused(", "odd-packed": "k_hash_generic("}
        if variant in want:
            helpers.assert_ran(names, want[variant], where=where)
    check_walk(orc, W, ix, dec, det, prompts, subsets, tie_seed, base, where)


def test_trimmed_batch_after_a_deep_batch(epp, orc):
    """A batch of prompts held to the cap leaves whole hash rows behind; the next batch, at the same rows, stops at
    blocks 31-64 and lists the deep family's holders: the walk must not read the stale hashes past each row's bound."""
    tie_seed = 0
    W = Walk(orc, 256, seed_of("C-stale"))
    ix = oracle_index(orc, W.hs, W.es)
    deep = STOPS.index(WB)
    R = 64
    first = [W.fam[deep]] * R
    shallow = [f for f, st in enumerate(STOPS) if 0 < st < WB]
    second = [W.fam[shallow[r % len(shallow)]] for r in range(R)]
    subsets = [sorted(set(W.H[deep]) | set(W.H[shallow[r % len(shallow)]]) | set(W.A[deep])) for r in range(R)]
    with walk_engine(epp, W, tie_seed) as eng:
        run(epp, eng, first, None, "device", layout="aligned")
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, second, subsets, "device", layout="aligned")
    assert_subset_ran(names, "device", "after a deep batch")
    check_walk(orc, W, ix, dec, det, second, subsets, tie_seed, base, "after a deep batch")


def test_walk_over_an_incrementally_built_index(epp, orc):
    """PreRequest adds (epp_index_add_picked) and commits patch the read table: single-slot subsets place each family's
    prefixes, at several depths, on chosen slots; restricted requests then walk the patched table."""
    tie_seed = 0x51
    W = Walk(orc, 256, seed_of("C-incremental"), R=0)
    rng = np.random.default_rng(7)
    ix = oracle_index(orc, [], [])
    with walk_engine(epp, W, tie_seed, hs=[], es=[]) as eng:
        for rnd in range(2):
            prompts, subsets = [], []
            for f in range(1, len(STOPS)):
                for e in rng.choice(W.E - 1, 6, replace=False):
                    prompts.append(W.fam[f][: int(rng.integers(33, WB + 1)) * WBB])
                    subsets.append([int(e)])
            dec, _, _, _ = run(epp, eng, prompts, subsets, "device", layout="aligned", keep_hashes=True)
            eng.index_add_picked()
            eng.index_commit()
            for p, s in zip(prompts, subsets):
                ix.add(orc.hash_prompt(p, PP.MODEL, WBST, WB), s[0])
            assert (dec["pick"] == np.array([s[0] for s in subsets], np.uint32)).all()
        prompts = [W.fam[1 + r % (len(STOPS) - 1)][: (WB + 2) * WBB] for r in range(64)]
        held = sorted(set(ix.pods()))
        subsets = [sorted(rng.choice(held, size=[3, 9, 40][r % 3], replace=False).tolist()) for r in range(64)]
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, prompts, subsets, "device", layout="aligned")
    assert_subset_ran(names, "device", "incremental index")
    check_walk(orc, W, ix, dec, det, prompts, subsets, tie_seed, base, "incremental index")
    assert (dec["match_blocks"] > 32).any()


# ------------------------------------------------------------------------------------------------
# D. no-hit-lru over long subsets
# ------------------------------------------------------------------------------------------------
class NohitCase:
    """A P/D pool of 256 (prefill slots 0 mod 5) whose decode and prefill profiles both carry the no-hit-lru scorer
    beside a queue scorer over a wide waiting range, so the cold ranks of every list entry move the pick.  Three calls of
    cold subsets of 33-200 slots; the LRU (size below the subsets) fills with the picks between them.  The model:
    tools/nohit_lru_model.py cold columns as ext columns 0 (decode) and 1 (prefill) of the oracle."""

    E, W_NH = 256, 1.0

    def __init__(self, orc, lru, seed):
        rng = np.random.default_rng(seed)
        self.orc, self.lru_size, self.rng = orc, lru, rng
        E = self.E
        self.role = np.where(np.arange(E) % 5 == 0, 2, 1).astype(np.uint8)
        self.waiting = rng.integers(0, 400, E).astype(np.int32)
        self.prim = (PP.F_DECODE, [(PP.QUEUE, 1.0, 0.0), (NH.NO_HIT_LRU, self.W_NH, float(lru))])
        self.pref = (PP.F_PREFILL, [(PP.QUEUE, 1.0, 0.0), (NH.NO_HIT_LRU, self.W_NH, float(lru))])
        self.L = PP.Land(E, self.role, np.zeros(E), self.waiting, self.prim, pref=self.pref,
                         holders=PP._holders(rng, np.arange(E), [3, 6]), R=0, seed=seed)
        self.ix = oracle_index(orc, self.L.hs, self.L.es)
        self.lru = NH.GoLRU(lru)
        self.dec = [e for e in range(E) if self.role[e] == 1]
        self.pre = [e for e in range(E) if self.role[e] == 2]

    def batch(self, b, R=64):
        rng = self.rng
        prompts, subsets = [], []
        for r in range(R):
            prompts.append(self.L.prompt(rng, 0.5))
            if r == 0:
                subsets.append([self.dec[int(rng.integers(len(self.dec)))]])            # one candidate (score 1.0)
            elif r == 1:
                subsets.append(sorted(rng.choice(self.dec, 40, replace=False).tolist()))   # no prefill candidate
            else:
                n = int(rng.integers(33, 201))
                subsets.append(sorted(rng.choice(self.E, n, replace=False).tolist()))
        return prompts, subsets

    def expect(self, prompts, subsets, base):
        """Expected decisions of one call (the LRU as it stood at its start), then PreRequest's Adds."""
        orc, E = self.orc, self.E
        keys = self.lru.keys()
        ext_prim = (PP.F_DECODE, [(PP.QUEUE, 1.0, 0.0), (PP.EXT, self.W_NH, 0.0)])
        ext_pref = (PP.F_PREFILL, [(PP.QUEUE, 1.0, 0.0), (PP.EXT, self.W_NH, 1.0)])
        outs, info = [], []
        for r, (p, s) in enumerate(zip(prompts, subsets)):
            m, _ = whole_match(orc, self.ix, p, E)
            dc = [e for e in self.dec if e in set(s)]
            pc = [e for e in self.pre if e in set(s)]
            cd, cp = NH.is_cold(dc, m), NH.is_cold(pc, m)
            col = np.stack([NH.cold_column(dc, keys, E) if cd else np.full(E, 0.5),
                            NH.cold_column(pc, keys, E) if cp else np.full(E, 0.5)])
            N = narrowed(self.L, s)
            role = np.full(E, ABSENT, np.uint8)
            role[N.ids] = self.role[N.ids]
            pool = orc.PoolState(role, np.zeros(E), self.waiting, np.zeros(E), col)
            L = copy.copy(self.L)
            L.prim, L.pref = ext_prim, ext_pref
            out = expect(orc, L, self.ix, p, s, 0, base + r, pool=pool, always=True)
            outs.append((out, m))
            info.append((dc, pc, cd, cp, keys))
        for (out, _), (dc, pc, cd, cp, _) in zip(outs, info):
            d = out[0]
            cold = cp if pc else cd
            if d["status"][0] == 0 and cold:
                self.lru.add(int(d["pick"][0]))
                if int(d["prefill_pick"][0]) >= 0:
                    self.lru.add(int(d["prefill_pick"][0]))
        return outs, info


@pytest.mark.parametrize("lru", [20, 100])
def test_nohit_lru_long_subsets(epp, orc, lru):
    C = NohitCase(orc, lru, seed_of("D", lru))
    with epp.Engine(C.E, PP._spec(epp, C.prim), PP._spec(epp, C.pref), block_size_tokens=PP.BST, max_prefix_blocks=PP.B,
                    always_disagg=True) as eng:
        eng.register_model(PP.MODEL)
        eng.pool_set(np.arange(C.E), C.role, np.zeros(C.E), C.waiting)
        eng.index_load_snapshot(np.array(C.L.hs, np.uint64), np.array(C.L.es, np.uint32))
        for b in range(3):
            prompts, subsets = C.batch(b)
            base = eng.stats()["n_decisions"]
            dec, det, _, names = run(epp, eng, prompts, subsets, "device")
            outs, _ = C.expect(prompts, subsets, base)
            for r, (out, m) in enumerate(outs):
                check_row(dec, det, None, r, out, m, f"nohit lru={lru} batch {b} request {r}")
            assert eng.nohit_lru_get() == C.lru.keys(), f"nohit lru={lru}: LRU after batch {b}"
            assert_subset_ran(names, "device", f"nohit lru={lru} batch {b}")


# ------------------------------------------------------------------------------------------------
# E. scorer edges inside the subset
# ------------------------------------------------------------------------------------------------
def edge_case(orc):
    """L4 with running spread over the pool; subsets of one (waiting, running) class: min = max holds only inside the
    subset (and the active-request max is taken over it)."""
    L = PP.land_edges(4)
    rng = np.random.default_rng(44)
    L.running = rng.choice([1, 3, 5], L.E).astype(np.int32)
    ix = oracle_index(orc, L.hs, L.es)
    classes = {}
    for e in range(L.E):
        classes.setdefault((int(L.waiting[e]), int(L.running[e])), []).append(e)
    big = [c for c in classes.values() if len(c) >= 3]
    subsets = []
    for r in range(len(L.prompts)):
        c = big[r % len(big)]
        subsets.append(sorted(rng.choice(c, size=int(rng.integers(2, len(c) + 1)), replace=False).tolist()))
    return L, ix, subsets


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
def test_clamp_edges_inside_the_subset(epp, orc, tie_seed):
    L, ix, subsets = edge_case(orc)
    with PP._engine(epp, L, tie_seed) as eng:
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, L.prompts, subsets, "device")
    assert_subset_ran(names, "device", "L4 edges")
    for r, s in enumerate(subsets):
        out = expect(orc, L, ix, L.prompts[r], s, tie_seed, base + r)
        m, _ = whole_match(orc, ix, L.prompts[r], L.E)
        check_row(dec, det, None, r, out, m, f"L4 edges request {r}")


INFLIGHT_PRIM = [(PP.QUEUE, 1.0, 0.0), (IM.TOKEN_LOAD, 1.0, 4096.0, IM.TOKEN_COL, 0.0),
                 (IM.ACTIVE_REQUEST, 2.0, 1.0, IM.REQUEST_COL, 0.0), (PP.PREFIX, 1.0, 0.0)]


def inflight_case(seed):
    """A pool of 64 and the slots whose counters a reset followed by two releases leaves at -2 / -1 (the subsets of the
    second call list only those: their active-request max is 0)."""
    rng = np.random.default_rng(seed)
    E = 64
    L = PP.Land(E, np.zeros(E, np.uint8), rng.choice([0.0, 0.5], E), rng.integers(0, 4, E), (PP.F_NONE, INFLIGHT_PRIM),
                holders=PP._holders(rng, np.arange(E), [4, 9]), R=48, seed=seed)
    neg = sorted(rng.choice(E, 12, replace=False).tolist())
    releases = neg + neg[::2]
    return L, neg, releases


def test_inflight_negative_counts_inside_the_subset(epp, orc):
    L, neg, releases = inflight_case(61)
    ix = oracle_index(orc, L.hs, L.es)
    cnt = IM.Counters(L.E)
    rng = np.random.default_rng(3)
    with epp.Engine(L.E, PP._spec(epp, L.prim), block_size_tokens=PP.BST, max_prefix_blocks=PP.B, inflight_load=True,
                    tie_seed=0x17) as eng:
        eng.register_model(PP.MODEL)
        eng.pool_set(*L.pool_arrays())
        eng.index_load_snapshot(np.array(L.hs, np.uint64), np.array(L.es, np.uint32))
        lens = np.array([len(p) for p in L.prompts], np.uint64)
        for b in range(2):
            if b == 0:
                subsets = [None] * len(L.prompts)
            else:
                subsets = [sorted(rng.choice(neg, size=int(rng.integers(1, len(neg) + 1)), replace=False).tolist())
                           for _ in L.prompts]
            ext = cnt.ext()
            base = eng.stats()["n_decisions"]
            dec, det, _, names = run(epp, eng, L.prompts, subsets, "device")
            for r, s in enumerate(subsets):
                out = expect(orc, L, ix, L.prompts[r], s, 0x17, base + r, pool=narrowed_pool(orc, L, s, ext))
                m, _ = whole_match(orc, ix, L.prompts[r], L.E)
                check_row(dec, det, None, r, out, m, f"inflight batch {b} request {r}")
            cnt.pre_request(dec, lens)
            if b == 0:
                eng.inflight_reset(np.array(neg, np.uint32))
                cnt.reset(neg)
                rl = np.array(releases, np.uint32)
                eng.inflight_release(rl, np.full(len(rl), 64, np.uint64))
                cnt.release(releases, [64] * len(releases))
                assert (cnt.req[neg] < 0).all()
                got_req, got_tok = eng.inflight_get()
                np.testing.assert_array_equal(got_req, cnt.req)
                np.testing.assert_array_equal(got_tok, cnt.tok)
            else:
                assert_subset_ran(names, "device", "inflight")


# ------------------------------------------------------------------------------------------------
# F. LoRA adapters other than 0
# ------------------------------------------------------------------------------------------------
LORA_MODELS = [PP.MODEL, b"adapter-1", b"adapter-2"]


class LoraCase:
    """A pool of 48 with LoRA residency for three adapters; index families hashed under each adapter; requests of every
    adapter, restricted in every chunk of the batch."""

    def __init__(self, orc, seed, R):
        rng = np.random.default_rng(seed)
        E = self.E = 48
        self.prim = (PP.F_NONE, [(PP.PREFIX, 2.0, 0.0), (LORA, 1.0, 0.0), (PP.QUEUE, 0.5, 0.0)])
        self.L = PP.Land(E, np.zeros(E, np.uint8), np.zeros(E), rng.integers(0, 3, E), self.prim, R=0, seed=seed)
        self.fam = {m: [rng.integers(0, 256, PP.B * PP.BB, dtype=np.uint8).tobytes() for _ in range(3)] for m in LORA_MODELS}
        hs, es = [], []
        for m in LORA_MODELS:
            for f in self.fam[m]:
                h = orc.hash_prompt(f, m, PP.BST, PP.B)
                for e in rng.choice(E, 5, replace=False):
                    d = int(rng.integers(1, PP.B + 1))
                    hs += h[:d]
                    es += [int(e)] * d
        self.hs, self.es = hs, es
        self.ix = oracle_index(orc, hs, es)
        self.max_active = rng.integers(1, 3, E).astype(np.int32)
        self.members = [(int(e), mi, int(rng.integers(1, 3))) for mi in range(len(LORA_MODELS))
                        for e in rng.choice(E, 10, replace=False)]
        self.loaded = np.zeros(E, np.int32)
        for e, _, _ in self.members:
            self.loaded[e] += 1
        self.mids = (np.arange(R) % len(LORA_MODELS)).astype(np.uint32)
        rng.shuffle(self.mids)
        self.prompts = []
        for r in range(R):
            f = self.fam[LORA_MODELS[self.mids[r]]][int(rng.integers(0, 3))]
            self.prompts.append(f[: PP.BB * int(rng.integers(1, PP.B + 1))] + rng.integers(0, 256, 7, dtype=np.uint8).tobytes())
        self.rng = rng

    def state(self, mi):
        st = np.zeros(self.E, np.uint8)
        for e, m, x in self.members:
            if m == mi and (st[e] == 0 or x == 1):
                st[e] = x
        return st

    def expect(self, orc, r, s, ordinal):
        N = narrowed(self.L, s)
        pool = N.oracle_pool(orc).set_lora(self.state(int(self.mids[r])), self.max_active, self.loaded)
        m = LORA_MODELS[int(self.mids[r])]
        out = expect(orc, self.L, self.ix, self.prompts[r], s, 0, ordinal, pool=pool, model=m)
        return out, whole_match(orc, self.ix, self.prompts[r], self.E, model=m)[0]


@pytest.mark.parametrize("path", ["host", "pipelined"])
def test_lora_adapters_per_chunk(epp, orc, path):
    R = 8192 if path == "pipelined" else 96
    C = LoraCase(orc, seed_of("F", path), R)
    rng = C.rng
    rows = pipelined_rows(R, rng, n=240) if path == "pipelined" else list(range(R))
    subsets = [None] * R
    for r in rows:
        subsets[r] = sorted(rng.choice(C.E, size=[4, 11, 40][r % 3], replace=False).tolist())
    with epp.Engine(C.E, PP._spec(epp, C.prim), block_size_tokens=PP.BST, max_prefix_blocks=PP.B) as eng:
        for m in LORA_MODELS:
            eng.register_model(m)
        eng.pool_set(*C.L.pool_arrays())
        eng.pool_set_lora(np.arange(C.E, dtype=np.uint32), C.max_active, C.loaded, C.members)
        eng.index_load_snapshot(np.array(C.hs, np.uint64), np.array(C.es, np.uint32))
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, C.prompts, subsets, path, model_ids=C.mids)
    assert_subset_ran(names, path, f"lora {path}", restricted_host_chunks(C.prompts, subsets) if path == "host" else None)
    for r in rows:
        out, m = C.expect(orc, r, subsets[r], base + r)
        check_row(dec, det, None, r, out, m, f"lora {path} request {r} model {C.mids[r]}")


# ------------------------------------------------------------------------------------------------
# G. large pools
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,sizes", [(4096, (1, 33, 1024, 4096)), (131073, (131073, 65537))])
def test_large_pools(epp, orc, E, sizes):
    L = PP.land_pool(E, 80 + E % 89)
    L.prompts = L.prompts[: 4 * len(sizes)]
    ix = oracle_index(orc, L.hs, L.es)
    rng = np.random.default_rng(E)
    subsets = [sorted(rng.choice(E, size=sizes[r % len(sizes)], replace=False).tolist()) for r in range(len(L.prompts))]
    tie_seed = 0x99
    with PP._engine(epp, L, tie_seed) as eng:
        base = eng.stats()["n_decisions"]
        dec, det, _, names = run(epp, eng, L.prompts, subsets, "device")
    assert_subset_ran(names, "device", f"E={E}")
    for r, s in enumerate(subsets):
        out = expect(orc, L, ix, L.prompts[r], s, tie_seed, base + r)
        m, _ = whole_match(orc, ix, L.prompts[r], E)
        check_row(dec, det, None, r, out, m, f"E={E} request {r} subset {len(s)}")
