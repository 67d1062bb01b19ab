"""The endpoint-sharded mode (DESIGN §7: epp_shard_*, csrc/shard_p2p.cu) on one GPU, on hand-built landscapes, against
the CPU oracle run unsharded on the whole pool, bit for bit: status, pick, score bits, tie count, match_blocks and
total_blocks.

Every rank is its own engine on the one GPU: epp_shard_set(lo, hi), the full pool, and the rank's own postings (a
snapshot, the full index, or index_add + index_commit with LRU eviction).  Both exchanges are driven from the host
(probe -> OR of the masks in torch -> pick -> stack of the records -> merge), or stepped phase by phase over peer memory
(epp_shard_p2p_phase), or run by one rank alone (epp_shard_schedule_p2p, world 1).  The cases:
  A  shard layouts: even splits, ragged ranges, an empty shard, a one-slot shard, a shard the role filter empties, ranges
     handed out in descending slot order, out-of-pool slots inside a shard; worlds of 1, 2, 3 and 5
  B  cross-shard landscapes: tie groups over 2-5 shards, +inf sums on several shards, -inf on every candidate, a lone
     winner against a large tie group elsewhere
  C  normalisers that span the pool (queue / running min-max, the active-request maximum) placed on different shards
  D  the global stop: blocks that only another rank holds, blocks nobody holds, stops at 0 / 31 / 32 / 33 / 63 / 64 / the
     cap under 1, 2 and 3 mask words, partial trailing blocks, prompts shorter than one block
  E  more than 32 in-shard holders (the dense-counter pass with global masks), 33 holders split 17 / 16, a 131 073-slot pool
  F  local tables: own postings, the full index on every rank, incremental tables with LRU tombstones (EPP_INDEX_PATCH 0/1)
  G  lora-affinity with per-request adapters 0 / 1 / 2 under every batch layout, on both exchanges
  H  the peer-memory exchange stepped over 2-4 ranks and consecutive batches of different R; one rank's own exchange
     over R >= 8192 (the two halves on the engine's two streams)
  I  the contract: lowest-slot ties whatever tie_seed, and the configurations and calls the mode rejects
  J  epp_shard_merge alone against sharded.merge_records_host
Every protocol call proves from its profiler trace that its kernels ran.  The builders are plain functions of the
oracle: test_sharded_landscapes_cpu.py checks from them alone that each case reaches the edge it names.
Run on an H100: pytest -m gpu."""
import importlib
import zlib

import numpy as np
import pytest

import helpers
import test_pick_paths_gpu as PP
from helpers import assert_ran, kernels_launched, ran
from tools import nohit_lru_model as NH

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
MODEL, BST, BB = PP.MODEL, PP.BST, PP.BB
(PREFIX, KV, QUEUE, LOAD, EXT, RUNNING, TOKEN, ACTIVE) = range(8)
LORA = 8
F_NONE, F_DECODE = 0, 1
PROBE, SPARSE, MERGE, DENSE = "k_shard_probe", "k_match_pick_sparse<6, true, false, 1>", "k_shard_merge", "k_match_pick("
P2P = ("k_p2p_wait", "k_p2p_or_masks", "k_p2p_gather", "k_p2p_signal")
LAYOUTS = ("uniform", "offsets0", "offsets16", "odd", "lengths")


def sharded():
    return importlib.import_module("llm-d-inference-scheduler_b200.sharded")


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode())


# ------------------------------------------------------------------------------------------------
# scenes: a pool, one profile, a hand-placed index and a batch of prompts (no GPU needed)
# ------------------------------------------------------------------------------------------------
class Scene:
    """E slots (ids: the pool; the others are outside it, role 0xFF, and may hold postings), one profile of
    max_prefix_blocks B.  The index is (hs, es) pairs, or `adds` = [(slot, hashes), ...] replayed through index_add with
    an LRU of `lru` blocks per slot.  models[a] is adapter a; lora = (max_active, loaded, state[a][e])."""

    def __init__(self, E, B, role, kv, waiting, prof, *, running=None, ext=None, ids=None, models=(MODEL,), lora=None,
                 lru=None):
        self.E, self.B, self.prof, self.models, self.lora, self.lru = E, B, prof, list(models), lora, lru
        self.role = np.asarray(role, np.uint8)
        self.kv = np.asarray(kv, np.float64)
        self.waiting = np.asarray(waiting, np.int32)
        self.running = np.zeros(E, np.int32) if running is None else np.asarray(running, np.int32)
        self.ext = None if ext is None else np.asarray(ext, np.float64).reshape(-1, E)
        self.ids = np.arange(E) if ids is None else np.asarray(sorted(ids))
        self.hs, self.es, self.adds = [], [], None
        self.steps, self.expect_patched = None, None     # adds per commit; last_index_patched after a later commit
        self.prompts, self.model_of = [], None

    def chain(self, fam, a=0):
        from oracle import pyoracle as orc
        return orc.hash_prompt(fam, self.models[a], BST, self.B)

    def hold(self, fam, slot, blocks, a=0):
        """slot holds the given block indices of family fam (hashed for adapter a)."""
        h = self.chain(fam, a)
        for i in blocks:
            self.hs.append(h[i])
            self.es.append(int(slot))

    def n_ext(self):
        return 0 if self.ext is None else self.ext.shape[0]

    def pool_arrays(self):
        i = self.ids
        return i, self.role[i], self.kv[i], self.waiting[i], self.running[i], None if self.ext is None else self.ext[:, i]

    def oracle_pool(self, orc, a=0):
        keep = np.zeros(self.E, bool)
        keep[self.ids] = True
        role = np.where(keep, self.role, 0xFF).astype(np.uint8)
        z = lambda x: np.where(keep, x, 0)
        ext = None if self.ext is None else np.where(keep[None, :], self.ext, 0.0)
        pool = orc.PoolState(role, z(self.kv), z(self.waiting), z(self.running), ext)
        if self.lora is not None:
            mx, loaded, state = self.lora
            pool.set_lora(state[a], mx, loaded)
        return pool

    def oracle_index(self, orc):
        ix = orc.Indexer(self.lru or 31250)
        if self.adds is not None:
            for e, h in self.adds:
                ix.add(np.array(h, np.uint64), int(e))
        elif self.hs:
            ix.load_pairs(self.hs, self.es)
        return ix

    def adapters(self, R):
        return np.zeros(R, np.int64) if self.model_of is None else np.asarray(self.model_of[:R], np.int64)


def fam_bytes(rng, blocks):
    return rng.integers(0, 256, blocks * BB, dtype=np.uint8).tobytes()


def tail(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def family_prompts(rng, fams, R, B, cold_share=0.15):
    """Prefixes of the families at random depths (partial trailing blocks included), and cold prompts."""
    out = []
    for _ in range(R):
        t = tail(rng, int(rng.integers(0, BB)))
        if rng.random() < cold_share:
            out.append(tail(rng, BB * int(rng.integers(1, B + 1))) + t)
        else:
            f = fams[int(rng.integers(0, len(fams)))]
            out.append(f[: BB * int(rng.integers(1, B + 1))] + t)
    return out


def ranges_of(cuts, E):
    c = [0] + list(cuts) + [E]
    return [(c[i], c[i + 1]) for i in range(len(c) - 1)]


# ---- A: shard layouts -------------------------------------------------------------------------------------------
A_E = 100
A_DROPPED = range(90, 100)        # role 2: the decode filter drops them
A_OUTSIDE = range(40, 46)         # outside the pool
A_TIES = [3, 27, 43, 58, 71, 88, 95]


def scene_layout(seed=11):
    """Decode profile (queue, kv, prefix); slots 90-99 prefill-only, 40-45 outside the pool.  Family 0 is held in full by
    a tie group spread over the whole slot range (with an out-of-pool and a dropped member), family 1 by six slots at
    random depths, family 2 only by out-of-pool slot 42 past block 4 (the walk goes on through it)."""
    rng = np.random.default_rng(seed)
    E, B = A_E, 40
    role = np.ones(E, np.uint8)
    role[list(A_DROPPED)] = 2
    kv = rng.choice([0.25, 0.5], E)
    waiting = rng.choice([1, 3], E).astype(np.int32)
    kv[A_TIES] = 0.0
    waiting[A_TIES] = 0
    S = Scene(E, B, role, kv, waiting, (F_DECODE, [(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0), (PREFIX, 2.0, 0.0)]),
              ids=np.setdiff1d(np.arange(E), list(A_OUTSIDE)))
    fams = [fam_bytes(rng, B) for _ in range(3)]
    for e in A_TIES:
        S.hold(fams[0], e, range(B))
    for e in rng.choice(E, 6, replace=False):
        S.hold(fams[1], e, range(int(rng.integers(1, B + 1))))
    S.hold(fams[2], 42, range(B))
    S.hold(fams[2], 10, range(5))
    S.hold(fams[2], 97, range(12))
    S.prompts = family_prompts(rng, fams, 96, B)
    return S


A_LAYOUTS = ("split", "ragged", "empty", "single", "dropped", "descending", "outside")


def layout_ranges(layout, world, E=A_E):
    """The shard ranges of a layout, in the order the ranks are stacked for the merge."""
    sh = sharded()
    if world == 1:
        return [(0, E)]
    if layout in ("split", "descending"):
        r = [sh.shard_range(g, world, E) for g in range(world)]
        return r[::-1] if layout == "descending" else r
    cuts = {
        "ragged": {2: [61], 3: [37, 77], 4: [13, 37, 77], 5: [13, 37, 61, 77]},
        "empty": {2: [0], 3: [37, 37], 5: [13, 37, 37, 77]},
        "single": {2: [1], 3: [58, 59], 5: [3, 4, 58, 59]},
        "dropped": {2: [90], 3: [45, 90], 5: [20, 45, 70, 90]},
        "outside": {2: [46], 3: [40, 46], 5: [20, 40, 46, 80]},
    }[layout][world]
    return ranges_of(cuts, E)


# ---- B: cross-shard landscapes -----------------------------------------------------------------------------------
def scene_cross(kind, world, seed=0):
    """tie-zero: the prefix weighs 0, so 40 equal-base slots spread over every shard tie whatever they match (the lowest
    slot must win with ITS match count); tie-prefix: 40 slots hold family 0 to the same depth; inf: weights near 1e308
    whose sums overflow to +inf on part of every shard; neg-inf: every candidate's sum is -inf; lone: one slot on the
    last shard, which holds no member of the tie group, matches deeper than the tie group spread over the other shards."""
    rng = np.random.default_rng(seed_of("cross", kind, world, seed))
    E, B = 150, 24
    sh = sharded()
    rs = [sh.shard_range(g, world, E) for g in range(world)]
    kv = rng.choice([0.25, 0.5], E)
    waiting = rng.choice([1, 2], E).astype(np.int32)
    src = rs[:-1] if kind == "lone" else rs                 # lone: the winner's shard (the last) holds no group member
    group = np.sort(np.concatenate([rng.choice(np.arange(lo, hi), 40 // world, replace=False) for lo, hi in src]))
    if kind in ("tie-zero", "tie-prefix", "lone"):
        kv[group] = 0.0
        waiting[group] = 0
    prof = {
        "tie-zero": (F_NONE, [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 0.0, 0.0)]),
        "tie-prefix": (F_NONE, [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 1.0, 0.0)]),
        "lone": (F_NONE, [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 4.0, 0.0)]),
        "inf": (F_NONE, [(KV, 1e308, 0.0), (QUEUE, 1.7e308, 0.0), (PREFIX, 1.0, 0.0)]),
        "neg-inf": (F_NONE, [(KV, -1e308, 0.0), (QUEUE, -1.7e308, 0.0), (PREFIX, 1.0, 0.0)]),
    }[kind]
    if kind == "inf":
        kv = np.where(rng.random(E) < 0.3, 0.0, 0.5)
        waiting = np.where(kv == 0.0, 0, 3).astype(np.int32)
    if kind == "neg-inf":
        kv = np.zeros(E)
        waiting = np.zeros(E, np.int32)
    S = Scene(E, B, np.zeros(E, np.uint8), kv, waiting, prof)
    fams = [fam_bytes(rng, B) for _ in range(3)]
    for e in group:
        S.hold(fams[0], e, range(B // 2 if kind == "lone" else (int(rng.integers(1, B + 1)) if kind == "tie-zero" else B)))
    if kind == "lone":
        S.hold(fams[0], E - 1, range(B))
        kv[E - 1], waiting[E - 1] = 0.0, 0
    for e in rng.choice(E, 8, replace=False):
        S.hold(fams[1], e, range(int(rng.integers(1, B + 1))))
    S.prompts = family_prompts(rng, fams[:2], 80, B, cold_share=0.1)
    S.group, S.ranges = [int(e) for e in group], rs
    return S


# ---- C: normalisers over the whole pool ---------------------------------------------------------------------------
C_SCORERS = [(QUEUE, 0.7, 0.0), (RUNNING, 0.7, 0.0), (ACTIVE, 1.0, 0.5, 2, 0.0), (KV, 0.1, 0.0), (LOAD, 1.0 / 3.0, 10.0),
             (EXT, 0.1, 0.0), (TOKEN, 1.0 / 3.0, 5000.0, 1), (PREFIX, 1.0, 0.0)]


def scene_norm(world, seed=0):
    """Queue and running minimum on the first shard, their maximum on the last, the active-request maximum on a middle
    one; every other value sits strictly inside, so no shard alone sees the pool's range."""
    rng = np.random.default_rng(seed_of("norm", world, seed))
    E, B = 120, 16
    sh = sharded()
    rs = [sh.shard_range(g, world, E) for g in range(world)]
    waiting = rng.integers(3, 12, E).astype(np.int32)
    running = rng.integers(2, 8, E).astype(np.int32)
    active = rng.integers(1, 6, E).astype(np.float64)       # above idle (0): every score reads the maximum
    lo0, hi_last = rs[0][0] + 1, rs[-1][1] - 2
    waiting[lo0], waiting[hi_last] = 0, 40
    running[lo0 + 1], running[hi_last] = 0, 30
    mid = rs[len(rs) // 2] if world > 2 else rs[1]
    active[mid[0] + 3] = 25.0
    ext = np.stack([rng.random(E) * 1.4 - 0.2, rng.integers(0, 9000, E).astype(np.float64), active])
    S = Scene(E, B, np.zeros(E, np.uint8), rng.random(E), waiting, (F_NONE, C_SCORERS), running=running, ext=ext)
    fams = [fam_bytes(rng, B) for _ in range(4)]
    for f in fams:
        for e in rng.choice(E, 10, replace=False):
            S.hold(f, e, range(int(rng.integers(1, B + 1))))
    S.prompts = family_prompts(rng, fams, 96, B)
    S.marks = {"queue": (lo0, hi_last), "running": (lo0 + 1, hi_last), "active": mid[0] + 3}
    return S


# ---- D: the global stop ------------------------------------------------------------------------------------------
D_STOPS = (0, 31, 32, 33, 63, 64)


def d_stops(B):
    return [s for s in D_STOPS if s < B] + [B - 1, B]


def scene_stop(B, world, seed=0):
    """Per stop block s two families: "other" -- slot a (first shard) holds every block but s, slot b (last shard) holds
    block s only, slot c (first shard) holds [0, s): the walk goes on past s, which a's own table lacks; "nobody" -- a and
    b hold every block but s: the walk stops at s for everyone.  s = B: no stop inside the cap.  Prompts reach past s,
    with partial trailing blocks, plus prompts shorter than one block."""
    rng = np.random.default_rng(seed_of("stop", B, world, seed))
    E = 64
    sh = sharded()
    rs = [sh.shard_range(g, world, E) for g in range(world)]
    S = Scene(E, B, np.zeros(E, np.uint8), rng.choice([0.0, 0.5], E), rng.integers(0, 3, E),
              (F_NONE, [(PREFIX, 1.0, 0.0), (KV, 0.5, 0.0), (QUEUE, 0.25, 0.0)]))
    S.families, fams = [], []
    first, last = list(range(*rs[0])), list(range(*rs[-1]))
    for s in d_stops(B):
        for mode in ("other", "nobody"):
            f = fam_bytes(rng, B)
            a, c = rng.choice(first, 2, replace=False)
            b = int(rng.choice(last))
            every_but = [i for i in range(B) if i != s]
            S.hold(f, a, every_but)
            S.hold(f, b, [s] if mode == "other" and s < B else every_but)
            if mode == "other":
                S.hold(f, c, range(s))
            S.families.append((s, mode, int(a), int(b), int(c)))
            fams.append(f)
    prompts = []
    for k, f in enumerate(fams):
        s = S.families[k][0]
        for _ in range(2):
            depth = int(rng.integers(min(s + 2, B), B + 1))
            prompts.append(f[: depth * BB] + tail(rng, int(rng.integers(0, BB))))
    prompts += [tail(rng, int(rng.integers(0, BB))) for _ in range(4)]           # shorter than one block
    S.prompts, S.fams = prompts, fams
    return S


# ---- E: overflow ---------------------------------------------------------------------------------------------------
def scene_overflow(kind, seed=0):
    """dense: 40 holders of family 0 on the first of two shards (its sparse map overflows); split: 33 holders, 17 on
    each side of the cut and 16 on the other (no rank overflows, the pool would); global: 40 holders in a pool of 131 073
    slots, whose dense counters live in global scratch."""
    rng = np.random.default_rng(seed_of("overflow", kind, seed))
    E = 131073 if kind == "global" else 96
    B = 12
    cut = sharded().shard_range(0, 2, E)[1]
    kv = rng.choice([0.0, 0.25, 0.5], E)
    S = Scene(E, B, np.zeros(E, np.uint8), kv, rng.integers(0, 2, E), (F_NONE, [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0),
                                                                              (PREFIX, 2.0, 0.0)]))
    fams = [fam_bytes(rng, B) for _ in range(3)]
    if kind == "split":
        hold = list(rng.choice(cut, 17, replace=False)) + list(rng.choice(np.arange(cut, E), 16, replace=False))
    else:
        hold = list(rng.choice(min(cut, 200), 40, replace=False))
    for e in hold:
        S.hold(fams[0], e, range(int(rng.integers(1, B + 1))))
    for e in rng.choice(min(E, 300), 6, replace=False):
        S.hold(fams[1], e, range(B))
    S.prompts = family_prompts(rng, fams[:2], 48, B, cold_share=0.1)
    S.holders = [int(e) for e in hold]
    return S


# ---- F: incremental local tables ----------------------------------------------------------------------------------
def scene_incremental(seed=0):
    """In three steps (one index_commit after each), 40 slots, then 8 of them, then 8 others, add a stretch of a family
    through an LRU of 10 blocks, out of block order.  Eviction in a later step empties blocks that an earlier commit held: the table keeps them
    as tombstones (cnt 0) when the commit patches it, and the holes lie in the middle of held prefixes."""
    rng = np.random.default_rng(seed_of("incremental", seed))
    E, B = 48, 24
    S = Scene(E, B, np.zeros(E, np.uint8), rng.choice([0.0, 0.5], E), rng.integers(0, 3, E),
              (F_NONE, [(PREFIX, 2.0, 0.0), (KV, 1.0, 0.0)]), lru=10)
    fams = [fam_bytes(rng, B) for _ in range(4)]
    S.steps = []
    first = rng.permutation(E)[:40]
    for step, (slots, lo) in enumerate(((first, 1), (first[:8], 6), (first[8:16], 6))):
        # the later steps are small next to the table the first builds, so that a commit can patch it
        S.steps.append([])
        for e in slots:
            f = S.chain(fams[int(rng.integers(0, 4))])
            a = int(rng.integers(0, B - 9))
            b = a + int(rng.integers(lo, 10))
            S.steps[-1].append((int(e), f[a:b]))
    S.adds = [x for st in S.steps for x in st]
    S.prompts = family_prompts(rng, fams, 96, B, cold_share=0.05)
    return S


# ---- G: LoRA --------------------------------------------------------------------------------------------------------
def scene_lora(seed=0):
    """Three adapters resident on 6 / 14 / 24 slots (active or waiting), families cached under each adapter's own hash
    chain, prefix + queue + lora-affinity; requests of adapters 0, 1 and 2."""
    rng = np.random.default_rng(seed_of("lora", seed))
    E, B, A = 64, 16, 3
    models = [MODEL] + [MODEL + b"-lora%d" % a for a in range(1, A)]
    mx = rng.integers(0, 5, E).astype(np.int32)
    state = np.zeros((A, E), np.uint8)
    for a, k in enumerate((6, 14, 24)):
        idx = rng.choice(E, k, replace=False)
        state[a, idx] = rng.choice([1, 2], k)
    loaded = (state != 0).sum(axis=0).astype(np.int32) + rng.integers(0, 2, E).astype(np.int32)
    S = Scene(E, B, np.zeros(E, np.uint8), rng.choice([0.0, 0.5], E), rng.integers(0, 3, E),
              (F_NONE, [(PREFIX, 2.0, 0.0), (QUEUE, 1.0, 0.0), (LORA, 1.5, 0.0)]), models=models, lora=(mx, loaded, state))
    fams = [fam_bytes(rng, B) for _ in range(3)]
    for a in range(A):
        for f in fams:
            for e in rng.choice(E, 5, replace=False):
                S.hold(f, e, range(int(rng.integers(1, B + 1))), a=a)
    S.prompts = family_prompts(rng, fams, 120, B, cold_share=0.1)
    S.model_of = rng.integers(0, A, len(S.prompts))
    return S


# ------------------------------------------------------------------------------------------------
# oracle side
# ------------------------------------------------------------------------------------------------
def expected(orc, S, prompts):
    """orc_cycle_batch on the whole pool and the whole index (tie_seed 0), per adapter; match_blocks = the pick's count in
    the unsharded walk."""
    from oracle import pyoracle
    ix = S.oracle_index(orc)
    R = len(prompts)
    out = np.zeros(R, pyoracle.DECISION_DTYPE)
    tot = np.zeros(R, np.int32)
    mb = np.zeros(R, np.int64)
    mo = S.adapters(R)
    o = orc.make_profile(S.prof[0], list(S.prof[1]))
    for a in sorted(set(mo.tolist())):
        sel = np.flatnonzero(mo == a)
        ps = [prompts[i] for i in sel]
        d, offs = PP._pack(ps)
        od, ot = orc.cycle_batch(S.models[a], BST, S.B, 0, False, ix, o, None, S.oracle_pool(orc, a), d, offs, 4)
        out[sel], tot[sel] = od, ot
        for j, i in enumerate(sel):
            if od["status"][j] == 0:
                m, _ = ix.match_longest_prefix(orc.hash_prompt(ps[j], S.models[a], BST, S.B), S.E)
                mb[i] = m[od["pick"][j]]
    return out, tot, mb


def check(dec, exp, where):
    odec, ototal, mb = exp
    helpers.assert_decisions_equal(dec, None, odec, ototal, where=where)
    ok = odec["status"] == 0
    np.testing.assert_array_equal(dec["match_blocks"][ok].astype(np.int64), mb[ok], err_msg=f"{where}: match_blocks")


def walk_holders(orc, S, ix, prompt, a=0):
    """Slots holding some block before the unsharded global stop (the ones a rank's lane map counts)."""
    h = orc.hash_prompt(prompt, S.models[a], BST, S.B)
    eps = set()
    for x in h:
        got = ix.get(x)
        if not got:
            break
        eps |= got
    return eps


def overflow_ranks(orc, S, prompts, ranges):
    """Ranks whose sparse lane map overflows (> 32 in-shard slots: block holders and lora entries) on some request."""
    ix = S.oracle_index(orc)
    mo = S.adapters(len(prompts))
    over = set()
    for r, p in enumerate(prompts):
        eps = walk_holders(orc, S, ix, p, int(mo[r]))
        if S.lora is not None:
            eps |= set(np.flatnonzero(S.lora[2][int(mo[r])]).tolist())
        for g, (lo, hi) in enumerate(ranges):
            if sum(lo <= e < min(hi, S.E) for e in eps) > 32:
                over.add(g)
    return over


# ------------------------------------------------------------------------------------------------
# engine side
# ------------------------------------------------------------------------------------------------
def traced(fn, want=(), absent=(), where="", repeatable=True):
    """fn() under the profiler -> (its first result, kernel names); when the trace kept its device records, every kernel
    of `want` ran and none of `absent`."""
    r, names = kernels_launched(fn, repeatable=repeatable)
    if helpers.trace_complete(names):
        for k in want:
            assert_ran(names, k, absent, where=where)
        for k in absent:
            assert not ran(names, k), f"{where}: {k} ran"
    return r, names


def shard_engine(epp, S, lo, hi, *, tie_seed=0, full=False):
    kw = {"lru_capacity_per_server": S.lru} if S.lru else {}
    eng = epp.Engine(S.E, epp.ProfileSpec(S.prof[0], [epp.ScorerSpec(*s) for s in S.prof[1]]), block_size_tokens=BST,
                     max_prefix_blocks=S.B, n_ext_cols=S.n_ext(), tie_seed=tie_seed, **kw)
    for m in S.models:
        eng.register_model(m)
    eng.shard_set(lo, hi)
    eng.pool_set(*S.pool_arrays())
    if S.lora is not None:
        mx, loaded, state = S.lora
        eng.pool_set_lora(np.arange(S.E), mx, loaded,
                          [(e, a, int(state[a, e])) for a in range(len(S.models)) for e in range(S.E) if state[a, e]])
    keep = lambda e: full or lo <= e < hi
    if S.adds is not None:
        built = False
        for step in (S.steps if S.steps is not None else [S.adds]):
            mine = [(e, h) for e, h in step if keep(e)]
            for e, h in mine:
                eng.index_add(e, np.array(h, np.uint64))
            eng.index_commit()
            if mine and built and S.expect_patched is not None:       # the first commit builds the table in bulk
                assert eng.stats()["last_index_patched"] == S.expect_patched, f"shard [{lo}, {hi}): commit path"
            built = built or bool(mine)
    elif S.hs:
        hs, es = np.array(S.hs, np.uint64), np.array(S.es, np.uint32)
        k = np.array([keep(int(e)) for e in es])
        if k.any():
            eng.index_load_snapshot(hs[k], es[k])
    return eng


def layout_batch(prompts, layout, rng):
    """-> (the prompts as the engine reads them, host bytes, offsets, lengths, uniform_len) of a batch layout: uniform
    rows; offsets at 0 / 16 mod 32 (rows padded with random bytes, which are part of the prompt); packed rows from an odd
    start (the generic hash kernel); rows with lengths shorter than the row (the bytes behind are not read)."""
    if layout == "uniform":
        T = max(1, max(len(p) for p in prompts))
        ps = [p + tail(rng, T - len(p)) for p in prompts]
        return ps, b"".join(ps) + b"\0" * 64, None, None, T
    start = {"offsets0": 0, "offsets16": 16, "odd": 7, "lengths": 0}[layout]
    offs, pos = [], start
    for p in prompts:
        offs.append(pos)
        n = len(p)
        pos += n if layout == "odd" else (n + 31) // 32 * 32 + (32 if layout == "lengths" else 0)
    offs.append(pos)
    buf = bytearray(tail(rng, pos + 64))
    for o, p in zip(offs, prompts):
        buf[o: o + len(p)] = p
    buf = bytes(buf)
    offs = np.array(offs, np.uint64)
    if layout == "lengths":
        return list(prompts), buf, offs, np.array([len(p) for p in prompts], np.uint64), None
    return [buf[offs[r]: offs[r + 1]] for r in range(len(prompts))], buf, offs, None, None


def device_kw(buf, offs, lens, T, model_ids=None):
    import torch
    kw = {}
    data = torch.from_numpy(np.frombuffer(buf, np.uint8).copy()).cuda()
    if offs is not None:
        kw["offsets"] = torch.from_numpy(offs.view(np.int64)).cuda()
    else:
        kw["uniform_len"] = T
    if lens is not None:
        kw["lengths"] = torch.from_numpy(lens.view(np.int64)).cuda()
    if model_ids is not None:
        kw["model_ids"] = torch.from_numpy(np.asarray(model_ids, np.uint32).view(np.int32)).cuda()
    return data, kw


def run_protocol(epp, orc, S, ranges, *, prompts=None, layout="offsets0", tie_seed=0, full=False, where=""):
    """The host-driven protocol over one engine per range (stacked in the given order) -> (decisions, masks, records);
    checked against the oracle here."""
    import torch
    rng = np.random.default_rng(seed_of("layout", where))
    ps, buf, offs, lens, T = layout_batch(S.prompts if prompts is None else prompts, layout, rng)
    R = len(ps)
    mo = S.adapters(R)
    data, kw = device_kw(buf, offs, lens, T, None if S.model_of is None else mo)
    over = overflow_ranks(orc, S, ps, ranges)
    W = (S.B + 31) // 32
    engines = [shard_engine(epp, S, lo, hi, tie_seed=tie_seed, full=full) for lo, hi in ranges]
    try:
        masks, bests = [], []
        for g, eng in enumerate(engines):
            m = torch.zeros((R, W), dtype=torch.int32, device="cuda")
            traced(lambda: eng.shard_probe(data, m, **kw), (PROBE,), where=f"{where} probe rank {g}")
            masks.append(m)
        gm = masks[0].clone()
        for m in masks[1:]:
            gm |= m
        torch.cuda.synchronize()                 # torch-produced masks are complete before an engine reads them
        for g, eng in enumerate(engines):
            b = torch.zeros((R, 24), dtype=torch.uint8, device="cuda")
            traced(lambda: eng.shard_pick(R, gm, b), (SPARSE, DENSE) if g in over else (SPARSE,),
                   where=f"{where} pick rank {g} {ranges[g]}")
            bests.append(b)
        allb = torch.stack(bests)
        dec = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        traced(lambda: engines[0].shard_merge(R, len(engines), allb, dec), (MERGE,), where=f"{where} merge")
        torch.cuda.synchronize()
        out = epp.decisions_from_torch(dec)
    finally:
        for e in engines:
            e.close()
    check(out, expected(orc, S, ps), where)
    recs = [b.cpu().numpy().view(epp.SHARD_BEST_DTYPE).reshape(-1) for b in bests]
    return out, [m.cpu().numpy().view(np.uint32) for m in masks], recs


def p2p_engines(epp, S, ranges, R_max, tie_seed=0):
    engines, ptrs = [], []
    for lo, hi in ranges:
        eng = shard_engine(epp, S, lo, hi, tie_seed=tie_seed)
        _, ptr = eng.shard_p2p_export(R_max)
        engines.append(eng)
        ptrs.append(ptr)
    for g, eng in enumerate(engines):
        eng.shard_p2p_connect(len(engines), g, np.array(ptrs, dtype=np.uint64), ipc_handles=False)
    return engines


def run_p2p_stepped(epp, orc, engines, S, prompts, layout, where):
    """One batch through epp_shard_p2p_phase: every rank through phase 0, then 1, then 2 (ranks that share a GPU never
    wait for each other on the device).  Traced once: the phases advance the exchange epoch."""
    import torch
    rng = np.random.default_rng(seed_of("p2p", where))
    ps, buf, offs, lens, T = layout_batch(prompts, layout, rng)
    R = len(ps)
    data, kw = device_kw(buf, offs, lens, T, None if S.model_of is None else S.adapters(R))
    outs = [torch.zeros((R, 32), dtype=torch.uint8, device="cuda") for _ in engines]
    torch.cuda.synchronize()

    def phases():
        for phase in range(3):
            for g, eng in enumerate(engines):
                eng.shard_p2p_phase(data, outs[g], phase, **kw)
    traced(phases, (PROBE, SPARSE, MERGE) + P2P, where=where, repeatable=False)
    torch.cuda.synchronize()
    decs = [epp.decisions_from_torch(o) for o in outs]
    for d in decs[1:]:
        np.testing.assert_array_equal(d, decs[0], err_msg=f"{where}: ranks disagree")
    check(decs[0], expected(orc, S, ps), where)
    return decs[0]


# ------------------------------------------------------------------------------------------------
# A: shard layouts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout,world", [("split", 1)] + [(x, w) for x in A_LAYOUTS for w in (2, 3, 5)])
def test_A_shard_layouts(epp, orc, layout, world):
    S = scene_layout()
    ranges = layout_ranges(layout, world)
    dec, masks, recs = run_protocol(epp, orc, S, ranges, where=f"A {layout} x{world}")
    assert (dec["match_blocks"] > 0).any() and (dec["tie_count"] > 1).any()
    for g, (lo, hi) in enumerate(ranges):
        ok = recs[g]["status"] == 0
        assert ((recs[g]["pick"][ok] >= lo) & (recs[g]["pick"][ok] < hi)).all(), f"rank {g} picked outside its shard"
        cand = [e for e in range(lo, hi) if e in set(S.ids.tolist()) and e not in A_DROPPED]
        assert ok.all() if cand else not ok.any(), f"rank {g} {lo, hi}: a shard without candidates has no record"


# ------------------------------------------------------------------------------------------------
# B: cross-shard landscapes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["tie-zero", "tie-prefix", "inf", "neg-inf", "lone"])
def test_B_cross_shard(epp, orc, kind, world):
    S = scene_cross(kind, world)
    sh = sharded()
    ranges = [sh.shard_range(g, world, S.E) for g in range(world)][::-1]          # the lowest slots on the last rank
    # sharded engines decide by the lowest slot whatever their tie_seed (the oracle runs with tie_seed 0)
    dec, _, recs = run_protocol(epp, orc, S, ranges, tie_seed=0x5EED if world != 3 else 0, where=f"B {kind} x{world}")
    ok = dec["status"] == 0
    if kind == "neg-inf":
        assert ok.all() and np.isneginf(dec["score"]).all()
    if kind == "inf":
        assert np.isposinf(dec["score"][ok]).any()
        assert sum(np.isposinf(r["score"]).any() for r in recs) >= 2
    if kind.startswith("tie"):
        assert (dec["tie_count"] >= 40 // world * world).any()


# ------------------------------------------------------------------------------------------------
# C: normalisers that span the shards
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 5])
def test_C_pool_wide_normalisers(epp, orc, world):
    S = scene_norm(world)
    sh = sharded()
    run_protocol(epp, orc, S, [sh.shard_range(g, world, S.E) for g in range(world)], where=f"C x{world}")


# ------------------------------------------------------------------------------------------------
# D: the global stop
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("B", [20, 32, 33, 64, 70, 96])
def test_D_global_stop(epp, orc, B, world):
    S = scene_stop(B, world)
    sh = sharded()
    dec, masks, _ = run_protocol(epp, orc, S, [sh.shard_range(g, world, S.E) for g in range(world)],
                                 layout="lengths" if B % 2 else "odd", where=f"D B={B} x{world}")
    assert (dec["match_blocks"] > 32).any() or B < 33
    assert (dec["total_blocks"] == 0).sum() >= 4


# ------------------------------------------------------------------------------------------------
# E: overflow
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["dense", "split", "global"])
def test_E_overflow(epp, orc, kind):
    S = scene_overflow(kind)
    sh = sharded()
    ranges = [sh.shard_range(g, 2, S.E) for g in range(2)]
    dec, _, _ = run_protocol(epp, orc, S, ranges, where=f"E {kind}")
    want = {0} if kind != "split" else set()
    assert overflow_ranks(orc, S, S.prompts, ranges) == want
    assert (dec["match_blocks"] > 0).any()


# ------------------------------------------------------------------------------------------------
# F: local tables
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 5])
def test_F_full_index_on_every_rank(epp, orc, world):
    """Each rank loads every posting; those outside its range keep the walk alive but are never counted."""
    S = scene_layout(12)
    run_protocol(epp, orc, S, layout_ranges("ragged", world), full=True, where=f"F full x{world}")
    if world == 2:                      # the overflowing rank's table holds the other rank's holders too
        S = scene_overflow("dense", 3)
        run_protocol(epp, orc, S, [(48, 96), (0, 48)], full=True, where="F full overflow")


@pytest.mark.parametrize("patch", ["0", "1"])
@pytest.mark.parametrize("world", [2, 3])
def test_F_incremental_tables(epp, orc, monkeypatch, world, patch):
    monkeypatch.setenv("EPP_INDEX_PATCH", patch)
    S = scene_incremental(world)
    S.expect_patched = int(patch)                # commits 2 and 3 patch the table (or rebuild it under patch=0)
    sh = sharded()
    dec, _, _ = run_protocol(epp, orc, S, [sh.shard_range(g, world, S.E) for g in range(world)],
                             where=f"F incremental x{world} patch={patch}")
    assert (dec["match_blocks"] > 0).any()


# ------------------------------------------------------------------------------------------------
# G: LoRA adapters under every layout
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("exchange", ["protocol", "p2p"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_G_lora_adapters(epp, orc, layout, exchange):
    """Per-request model ids 0 / 1 / 2: epp_shard_pick scores lora-affinity with the adapters the probe was given."""
    S = scene_lora()
    sh = sharded()
    ranges = [sh.shard_range(g, 3, S.E) for g in range(3)]
    if exchange == "protocol":
        dec, _, _ = run_protocol(epp, orc, S, ranges, layout=layout, where=f"G lora {layout}")
    else:
        engines = p2p_engines(epp, S, ranges, len(S.prompts))
        try:
            dec = run_p2p_stepped(epp, orc, engines, S, S.prompts, layout, f"G lora p2p {layout}")
        finally:
            for e in engines:
                e.close()
    assert (dec["match_blocks"] > 0).any()


# ------------------------------------------------------------------------------------------------
# H: the exchanges
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 4])
def test_H_p2p_stepped_batches(epp, orc, world):
    """Consecutive batches of 57, 1, 200 (the exported maximum), 33 and 120 requests through the same exchange buffers."""
    S = scene_layout(13)
    S.B = 24                                     # one mask word
    S.hs, S.es = [], []
    rng = np.random.default_rng(world)
    fams = [fam_bytes(rng, S.B) for _ in range(3)]
    for e in A_TIES:
        S.hold(fams[0], e, range(S.B))
    for e in rng.choice(S.E, 40, replace=False):
        S.hold(fams[1 + int(e) % 2], e, range(int(rng.integers(1, S.B + 1))))
    prompts = family_prompts(rng, fams, 200, S.B)
    engines = p2p_engines(epp, S, layout_ranges("ragged", world), 200)
    try:
        for k, R in enumerate((57, 1, 200, 33, 120)):
            run_p2p_stepped(epp, orc, engines, S, prompts[k: k + R] if R < 200 else prompts,
                            LAYOUTS[k % len(LAYOUTS)], f"H p2p x{world} batch {k} R={R}")
    finally:
        for e in engines:
            e.close()


@pytest.mark.parametrize("world", [2, 3])
def test_H_p2p_stepped_global_stop(epp, orc, world):
    """The peer-memory OR of the masks on prefixes that are not closed per shard (scene D): a rank that ORed only its own
    masks would stop at a block only another rank holds."""
    S = scene_stop(70, world)
    sh = sharded()
    engines = p2p_engines(epp, S, [sh.shard_range(g, world, S.E) for g in range(world)], len(S.prompts))
    try:
        dec = run_p2p_stepped(epp, orc, engines, S, S.prompts, "lengths", f"H p2p stop x{world}")
        assert (dec["match_blocks"] > 32).any()
    finally:
        for e in engines:
            e.close()


@pytest.mark.parametrize("chunks", ["2", "1"])
def test_H_p2p_world_one_large_batch(epp, orc, monkeypatch, chunks):
    """epp_shard_schedule_p2p with one rank (shard [0, E)): its waits are on its own flags, raised before them in stream
    order.  R = 8 257 >= 8 192 splits the batch into two halves on the engine's two streams under EPP_DEV_CHUNKS=2."""
    import torch
    monkeypatch.setenv("EPP_DEV_CHUNKS", chunks)
    S = scene_layout(14)
    R = 8257
    rng = np.random.default_rng(int(chunks))
    prompts = [S.prompts[int(i)] for i in rng.integers(0, len(S.prompts), R)]
    ps, buf, offs, lens, T = layout_batch(prompts, "offsets0", rng)
    data, kw = device_kw(buf, offs, lens, T)
    eng = shard_engine(epp, S, 0, S.E)
    try:
        _, ptr = eng.shard_p2p_export(R)
        eng.shard_p2p_connect(1, 0, np.array([ptr], np.uint64), ipc_handles=False)
        out = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        _, names = traced(lambda: eng.shard_schedule_p2p(data, out, **kw), (PROBE, SPARSE, MERGE) + P2P,
                          where=f"H world 1 chunks={chunks}", repeatable=False)
        torch.cuda.synchronize()
        if helpers.trace_complete(names):
            n = sum(c for k, c in names.items() if SPARSE in k)
            assert n == (2 if chunks == "2" else 1), sorted(names.items())
        check(epp.decisions_from_torch(out), expected(orc, S, ps), f"H world 1 chunks={chunks}")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# I: contract pins
# ------------------------------------------------------------------------------------------------
def test_I_rejected_configurations(epp):
    P, Sp, capi = epp.ProfileSpec, epp.ScorerSpec, epp.capi
    base = [Sp(QUEUE, 1.0, 0.0), Sp(PREFIX, 1.0, 0.0)]
    cases = {
        "no-hit-lru": dict(primary=P(0, base + [Sp(NH.NO_HIT_LRU, 1.0, 4.0)])),
        "random picker": dict(primary=P(0, base, picker=capi.PICKER_RANDOM)),
        "weighted random picker": dict(primary=P(0, base, picker=capi.PICKER_WEIGHTED_RANDOM)),
        "inflight producer": dict(primary=P(0, base), inflight_load=True),
        "pick_k > 1": dict(primary=P(0, base), pick_k=2),
        "affinity filter": dict(primary=P(0, base, affinity=epp.AffinityFilterSpec())),
        "P/D handler": dict(primary=P(1, base), prefill=P(2, base)),
    }
    for name, kw in cases.items():
        with epp.Engine(16, max_prefix_blocks=8, block_size_tokens=BST, **kw) as eng:
            with pytest.raises(epp.EngineError, match="endpoint-sharded"):
                eng.shard_set(0, 8)


def test_I_rejected_calls(epp):
    import torch
    S = scene_stop(20, 2)
    ps, buf, offs, lens, T = layout_batch([S.prompts[i % len(S.prompts)] for i in range(40)], "offsets0", np.random.default_rng(0))
    data, kw = device_kw(buf, offs, lens, T)
    with shard_engine(epp, S, 0, 32) as eng:
        m = torch.zeros((40, 1), dtype=torch.int32, device="cuda")
        eng.shard_probe(data, m, **kw)
        torch.cuda.synchronize()
        b = torch.zeros((41, 24), dtype=torch.uint8, device="cuda")
        with pytest.raises(epp.EngineError, match="does not match"):
            eng.shard_pick(39, m, b)
        with pytest.raises(epp.EngineError, match="does not match"):
            eng.shard_merge(41, 1, b.unsqueeze(0), torch.zeros((41, 32), dtype=torch.uint8, device="cuda"))
    with shard_engine(epp, S, 0, S.E) as eng:
        _, ptr = eng.shard_p2p_export(39)
        eng.shard_p2p_connect(1, 0, np.array([ptr], np.uint64), ipc_handles=False)
        with pytest.raises(epp.EngineError, match="exceeds the exported exchange buffer"):
            eng.shard_schedule_p2p(data, torch.zeros((40, 32), dtype=torch.uint8, device="cuda"), **kw)
        with pytest.raises(epp.EngineError, match="exceeds the exported exchange buffer"):
            eng.shard_p2p_phase(data, torch.zeros((40, 32), dtype=torch.uint8, device="cuda"), 0, **kw)


# ------------------------------------------------------------------------------------------------
# J: epp_shard_merge alone
# ------------------------------------------------------------------------------------------------
def merge_records(n_ranks, R, seed):
    """Hand-written [n_ranks][R] records: scores from a small set with -inf and +inf (equal scores on many ranks), status
    -1 ranks, distinct slots drawn at random (a lower slot often on a later rank)."""
    sh = sharded()
    rng = np.random.default_rng(seed)
    a = np.zeros((n_ranks, R), dtype=sh.SHARD_BEST_DTYPE)
    a["score"] = rng.choice([-np.inf, -2.5, 0.0, 0.75, 0.75, 3.0, np.inf], (n_ranks, R))
    a["pick"] = rng.permutation(n_ranks * R).astype(np.uint32).reshape(n_ranks, R)     # disjoint, like the shards' slots
    a["tie_count"] = rng.integers(1, 50, (n_ranks, R))
    a["match_blocks"] = rng.integers(0, 20, (n_ranks, R))
    a["status"] = np.where(rng.random((n_ranks, R)) < 0.3, -1, 0)
    a["status"][:, :3] = -1                                       # no rank has a candidate
    a["status"][:, 3:6], a["score"][:, 3:6] = 0, -np.inf          # every rank's best is -inf
    bad = a["status"] == -1
    a["pick"][bad], a["score"][bad], a["tie_count"][bad], a["match_blocks"][bad] = NO, 0.0, 0, 0
    return a


@pytest.mark.parametrize("n_ranks,R", [(1, 300), (2, 257), (5, 1000), (64, 300)])
def test_J_merge_records(epp, n_ranks, R):
    import torch
    sh = sharded()
    a = merge_records(n_ranks, R, n_ranks * 1000 + R)
    want = sh.merge_records_host(a)
    S = scene_stop(20, 2)
    prompts = [S.prompts[i % len(S.prompts)] for i in range(R)]
    ps, buf, offs, lens, T = layout_batch(prompts, "offsets0", np.random.default_rng(R))
    data, kw = device_kw(buf, offs, lens, T)
    with shard_engine(epp, S, 0, 32) as eng:
        eng.shard_probe(data, torch.zeros((R, 1), dtype=torch.int32, device="cuda"), **kw)
        allb = torch.from_numpy(a.view(np.uint8).reshape(n_ranks, R, 24).copy()).cuda()
        dec = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        traced(lambda: eng.shard_merge(R, n_ranks, allb, dec), (MERGE,), where=f"J {n_ranks}x{R}")
        torch.cuda.synchronize()
        d = epp.decisions_from_torch(dec)
    totals = np.array([len(orc_chain(p, S.B)) for p in ps])
    np.testing.assert_array_equal(d["total_blocks"], totals)
    np.testing.assert_array_equal(d["status"], want["status"])
    ok = want["status"] == 0
    np.testing.assert_array_equal(d["pick"][ok], want["pick"][ok])
    np.testing.assert_array_equal(d["score"][ok].view(np.uint64), want["score"][ok].view(np.uint64))
    np.testing.assert_array_equal(d["tie_count"][ok], want["tie_count"][ok])
    np.testing.assert_array_equal(d["match_blocks"][ok], want["match_blocks"][ok])
    assert (d["pick"][~ok] == NO).all() and (d["prefill_pick"] == NO).all()
    assert np.isneginf(d["score"][ok]).any() and np.isposinf(d["score"][ok]).any() and (~ok).any()


def orc_chain(p, B):
    from oracle import pyoracle as orc
    return orc.hash_prompt(p, MODEL, BST, B)
