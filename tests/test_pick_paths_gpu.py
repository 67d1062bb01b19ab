"""Pool preparation (k_pool_candidates / k_pool_aux / k_pool_terms / k_pool_sort / k_pool_groups, and the no-hit-lru
rank / trim / column kernels) and the evaluation of every pick path, against the CPU oracle, on hand-built landscapes:
zero, negative and rounding-sensitive weights, every request-independent scorer at its clamp edges, weighted sums that
overflow to +-inf, tie groups placed across the 32-entry chunks of the order, pools from 1 to 131 073 slots, partial
pools and pool churn, top-k lists longer than 32, and a no-hit-lru scorer whose LRU spans several 1024-slot chunks.

Each landscape is one pool (roles, metrics, ext columns), one to three profiles and an index placed by hand: every
prompt family has chosen holders at chosen depths, so the matched sets and tie groups are the ones the landscape names.
One batch then runs through every path -- device batch, pipelined two-chunk async batch, host batch (k_cycle_small) and
zero-copy batch, injected match rows (k_dense_pick), epp_score rows, the dense-counter overflow pass for families with
more than 32 holders, and a pick_k > 1 engine (gen::eval) -- under both tie rules, and each result is compared with the
oracle bit for bit.  Every call proves from its profiler trace that the kernel it is about ran.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import helpers
from helpers import assert_ran, kernels_launched, ran
from tools import nohit_lru_model as M

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
MODEL = b"m"
BST, B = 8, 12                      # 32-byte blocks: host batches take the single-launch kernel
BB = 4 * BST
(PREFIX, KV, QUEUE, LOAD, EXT, RUNNING, TOKEN, ACTIVE) = range(8)
F_NONE, F_DECODE, F_PREFILL, F_ENCODE = range(4)
SPARSE, DENSE, SMALL = "k_match_pick_sparse<", "k_match_pick(", "k_cycle_small<"
POOL_KERNELS = ("k_pool_candidates", "k_pool_terms", "k_pool_sort", "k_pool_groups")
THIRD = 1.0 / 3.0


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


# ------------------------------------------------------------------------------------------------
# landscape builder
# ------------------------------------------------------------------------------------------------
class Land:
    """A pool, its profiles and a hand-placed index.  holders[g] = [(slot, depth in blocks), ...] of family g; every
    request is a prefix of a family (or a cold prompt) with a random tail.  ids = the slots in the pool (the others
    are outside it, role 0xFF, and may still hold index entries)."""

    def __init__(self, E, role, kv, waiting, prim, *, running=None, ext=None, pref=None, enc=None, holders=(), R=96,
                 ids=None, nct=0, seed=0, cold_share=0.2):
        self.E, self.prim, self.pref, self.enc, self.nct = E, prim, pref, enc, nct
        self.role = np.asarray(role, np.uint8)
        self.kv = np.asarray(kv, np.float64)
        self.waiting = np.asarray(waiting, np.int32)
        self.running = np.zeros(E, np.int32) if running is None else np.asarray(running, np.int32)
        self.ext = None if ext is None else np.asarray(ext, np.float64).reshape(-1, E)
        self.ids = np.arange(E) if ids is None else np.asarray(sorted(ids))
        rng = np.random.default_rng(seed)
        self.rng = rng
        self.fam = [rng.integers(0, 256, B * BB, dtype=np.uint8).tobytes() for _ in holders]
        self.hs, self.es = [], []
        for g, hl in enumerate(holders):
            h = _hash(self.fam[g])
            for e, depth in hl:
                self.hs += h[:depth]
                self.es += [int(e)] * depth
        self.prompts = [self.prompt(rng, cold_share) for _ in range(R)]
        self.mm = (rng.random(R) < 0.5).astype(np.uint8) if enc else None

    def prompt(self, rng, cold_share):
        tail = rng.integers(0, 256, int(rng.integers(0, 3 * BB)), dtype=np.uint8).tobytes()
        if not self.fam or rng.random() < cold_share:
            return rng.integers(0, 256, BB * int(rng.integers(1, B)), dtype=np.uint8).tobytes() + tail
        g = int(rng.integers(0, len(self.fam)))
        return self.fam[g][: BB * int(rng.integers(1, B + 1))] + tail

    def pool_arrays(self):
        """Engine pool_set arguments (the slots in the pool only)."""
        i = self.ids
        ext = None if self.ext is None else self.ext[:, i]
        return i, self.role[i], self.kv[i], self.waiting[i], self.running[i], ext

    def oracle_pool(self, orc):
        role = np.full(self.E, 0xFF, np.uint8)
        role[self.ids] = self.role[self.ids]
        keep = np.zeros(self.E, bool)
        keep[self.ids] = True
        z = lambda a: np.where(keep, a, 0)
        ext = None if self.ext is None else np.where(keep[None, :], self.ext, 0.0)
        return orc.PoolState(role, z(self.kv), z(self.waiting), z(self.running), ext)

    def n_ext(self):
        return 0 if self.ext is None else self.ext.shape[0]

    def stages(self):
        return 3 if self.enc else (2 if self.pref else 1)


def _hash(p):
    from oracle import pyoracle as orc
    return orc.hash_prompt(p, MODEL, BST, B)


def _spec(epp, prof):
    return None if prof is None else epp.ProfileSpec(prof[0], [epp.ScorerSpec(*s) for s in prof[1]])


def _oprof(orc, prof):
    return None if prof is None else orc.make_profile(prof[0], list(prof[1]))


def _pack(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    return np.frombuffer(b"".join(prompts) + b"\0" * 16, dtype=np.uint8).copy(), offs


def _rows(prompts):
    """32-byte aligned rows + lengths (the host layouts of the single-launch kernel)."""
    starts, pos = [], 0
    for p in prompts:
        starts.append(pos)
        pos += max(32, (len(p) + 31) // 32 * 32)
    return starts, pos, np.array([len(p) for p in prompts], dtype=np.uint64)


def _traced(fn, want, absent=(), where=""):
    """fn() under the profiler -> (its first result, kernel names); asserts that every kernel of `want` ran and none of
    `absent`.  A trace that lost kernel records is taken again with one more call of fn (every call here can be
    repeated: it changes nothing the test checks later); a trace without device records proves nothing either way."""
    out = None
    for attempt in range(3):
        r, names = kernels_launched(fn)
        out = r if attempt == 0 else out
        if all(ran(names, k) for k in want):
            break
    if helpers.trace_complete(names) or all(ran(names, k) for k in want):
        for k in want:
            assert_ran(names, k, absent, where=where)
    return out, names


def _engine(epp, L, tie_seed, pick_k=0, prim=None):
    eng = epp.Engine(L.E, _spec(epp, prim or L.prim), _spec(epp, L.pref), encode=_spec(epp, L.enc),
                     block_size_tokens=BST, max_prefix_blocks=B, non_cached_tokens=L.nct, n_ext_cols=L.n_ext(),
                     tie_seed=tie_seed, pick_k=pick_k)
    eng.register_model(MODEL)
    profs = [p for p in (prim or L.prim, L.pref, L.enc) if p is not None]
    aux = ("k_pool_aux",) if any(s[0] == ACTIVE for p in profs for s in p[1]) else ()
    _traced(lambda: eng.pool_set(*L.pool_arrays()), POOL_KERNELS + aux, where="pool_set")
    if L.hs:
        eng.index_load_snapshot(np.array(L.hs, np.uint64), np.array(L.es, np.uint32))
    return eng


def _oracle(orc, L, prompts, tie_seed, base, mm=None, topk=0, prim=None):
    ix = orc.Indexer()
    if L.hs:
        ix.load_pairs(L.hs, L.es)
    d, o = _pack(prompts)
    return orc.cycle_batch(MODEL, BST, B, L.nct, False, ix, _oprof(orc, prim or L.prim), _oprof(orc, L.pref),
                           L.oracle_pool(orc), d, o, 4, tie_seed=tie_seed, tie_base=base, encode=_oprof(orc, L.enc),
                           multimodal=mm, topk=topk)


def _sparse_name(L, tie_seed):
    st = L.stages()
    mincta = 8 if st == 1 and not tie_seed else 6
    return f"k_match_pick_sparse<{mincta}, false, {'true' if tie_seed else 'false'}, {st}>"


def _det(epp, det):
    return det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1) if hasattr(det, "cpu") else det


def _lists(lists):
    out = {}
    for k, v in lists.items():
        v = np.asarray(v.cpu() if hasattr(v, "cpu") else v)
        if not k.endswith("scores"):
            v = v.astype(np.int64) & 0xFFFFFFFF
            v[v == NO] = -1
        out[k] = v
    return out


def _overflows(L, prompts):
    """Some request matches a family held by more than 32 slots of the pool."""
    for fam in L.fam:                   # (the lane map holds every holder, in the pool or not)
        h0 = _hash(fam)[0]
        if len({e for h, e in zip(L.hs, L.es) if h == h0}) > 32:
            if any(p[:BB] == fam[:BB] for p in prompts):
                return True
    return False


def run_paths(epp, orc, L, tie_seed, *, asynchronous=True, host=True, topk=3, where=""):
    """One batch through every path; returns the device batch's decisions."""
    import torch
    prompts, mm = L.prompts, L.mm
    R = len(prompts)
    d, o = _pack(prompts)
    over = _overflows(L, prompts)
    sparse = _sparse_name(L, tie_seed)
    with _engine(epp, L, tie_seed) as eng:
        # (a) device batch, synchronous: the sparse kernel (+ the dense-counter overflow pass)
        dd, do = torch.from_numpy(d).cuda(), torch.from_numpy(o.view(np.int64)).cuda()
        dmm = None if mm is None else torch.from_numpy(mm).cuda()
        base = eng.stats()["n_decisions"]
        (dec, det), names = _traced(lambda: eng.schedule(dd, offsets=do, multimodal=dmm), (sparse,) + ((DENSE,) if over else ()),
                                    where=f"{where} device batch (overflow pass: {over})")
        torch.cuda.synchronize()
        dev_dec = epp.decisions_from_torch(dec)
        odec, ototal = _oracle(orc, L, prompts, tie_seed, base, mm)
        helpers.assert_decisions_equal(dev_dec, _det(epp, det), odec, ototal, where=f"{where} device batch")
        # (b) two-chunk async batch (>= 8192 requests: the batch tiled)
        if asynchronous:
            reps = -(-8192 // R)
            big = prompts * reps
            bmm = None if mm is None else np.tile(mm, reps)
            bd, bo = _pack(big)
            tbd, tbo = torch.from_numpy(bd).cuda(), torch.from_numpy(bo.view(np.int64)).cuda()
            tmm = None if bmm is None else torch.from_numpy(bmm).cuda()
            base = eng.stats()["n_decisions"]

            def run_async():
                r = eng.schedule(tbd, offsets=tbo, multimodal=tmm, asynchronous=True)
                eng.synchronize()
                return r
            (adec, adet), names = _traced(run_async, (sparse,), where=f"{where} async")
            if ran(names, sparse):
                assert sum(c for n, c in names.items() if sparse in n) == 2, f"{where} async: {sorted(names)}"
            odec2, ototal2 = _oracle(orc, L, big, tie_seed, base, bmm)
            helpers.assert_decisions_equal(epp.decisions_from_torch(adec), _det(epp, adet), odec2, ototal2,
                                           where=f"{where} async two-chunk batch")
        # (c) host batch (k_cycle_small, copied) and a zero-copy batch of 8 from pinned memory
        if host:
            for sub in (list(range(R)), list(range(min(8, R)))):
                sp = [prompts[i] for i in sub]
                starts, end, lens = _rows(sp)
                buf = epp.PinnedBuffer(end + 64)
                for s0, p in zip(starts, sp):
                    buf.array[s0: s0 + len(p)] = np.frombuffer(p, np.uint8)
                offs = np.array(starts + [end], dtype=np.uint64)
                smm = None if mm is None else mm[sub]
                src = buf.array if len(sub) <= 8 else buf.array.copy()
                base = eng.stats()["n_decisions"]
                (hdec, hdet), names = _traced(
                    lambda: eng.schedule(src, offsets=offs, lengths=lens, multimodal=smm, n_requests=len(sub)), (SMALL,),
                    (sparse,), where=f"{where} host batch of {len(sub)}")
                odec3, ototal3 = _oracle(orc, L, sp, tie_seed, base, smm)
                helpers.assert_decisions_equal(hdec, hdet, odec3, ototal3, where=f"{where} host batch of {len(sub)}")
                buf.close()
        # (d) the engine's own match rows through k_dense_pick
        (match, total), names = _traced(lambda: eng.prefix_match(d, offsets=o), (DENSE,), where=f"{where} prefix_match")
        in_len = np.array([len(p) for p in prompts], np.int64)
        base = eng.stats()["n_decisions"]
        (wdec, wdet), names = _traced(lambda: eng.schedule_with_match(match, total, in_len, BST), ("k_dense_pick",),
                                      where=f"{where} schedule_with_match")
        odec4, ototal4 = _oracle(orc, L, prompts, tie_seed, base)       # (no multimodal flags: no encode stage)
        helpers.assert_decisions_equal(wdec, wdet, odec4, ototal4, where=f"{where} schedule_with_match")
        # (e) epp_score rows (ordered weighted sum, -1 outside the candidates) against the oracle's scores
        pool = L.oracle_pool(orc)
        for pi, prof in enumerate((L.prim, L.pref, L.enc)):
            if prof is None:
                continue
            rows, names = _traced(lambda: eng.score(match, total, pi, -1), ("k_score_dense",), where=f"{where} score")
            op = _oprof(orc, prof)
            for r in range(0, R, max(1, R // 24)):
                want, _, _, _ = orc.profile_run(op, pool, match[r], int(total[r]))
                np.testing.assert_array_equal(rows[r].view(np.uint64), want.view(np.uint64),
                                              err_msg=f"{where} score profile {pi} row {r}")
    # (g) a pick_k > 1 engine: gen::eval through k_match_pick (batches) and k_dense_pick (injected rows)
    if topk:
        check_topk(epp, orc, L, tie_seed, topk, where=where)
    return dev_dec, odec


def check_topk(epp, orc, L, tie_seed, K, *, where=""):
    import torch
    prompts, mm = L.prompts, L.mm
    d, o = _pack(prompts)
    with _engine(epp, L, tie_seed, pick_k=K) as eng:
        for kind in ("host", "device"):
            base = eng.stats()["n_decisions"]
            if kind == "host":
                call = lambda: eng.schedule(d, offsets=o, multimodal=mm, topk=True)
            else:
                dd, do = torch.from_numpy(d).cuda(), torch.from_numpy(o.view(np.int64)).cuda()
                dmm = None if mm is None else torch.from_numpy(mm).cuda()
                call = lambda: eng.schedule(dd, offsets=do, multimodal=dmm, topk=True)
            (dec, det, lists), names = _traced(call, (DENSE,), (SPARSE, SMALL), where=f"{where} top-{K} {kind}")
            torch.cuda.synchronize()
            if kind == "device":
                dec, det = epp.decisions_from_torch(dec), _det(epp, det)
            odec, ototal, olists = _oracle(orc, L, prompts, tie_seed, base, mm, topk=K)
            helpers.assert_decisions_equal(dec, det, odec, ototal, where=f"{where} top-{K} {kind}")
            got = _lists(lists)
            for name in ("primary", "prefill", "encode"):
                np.testing.assert_array_equal(got[name], olists[name], err_msg=f"{where} top-{K} {kind} {name}")
                for row in got[name]:
                    row = row[row >= 0]
                    assert len(set(row.tolist())) == len(row), f"{where} top-{K} {kind} {name}: repeated endpoint"
            np.testing.assert_array_equal(got["primary_scores"].view(np.uint64), olists["primary_scores"].view(np.uint64),
                                          err_msg=f"{where} top-{K} {kind} scores")
        if mm is None:
            match, total = eng.prefix_match(d, offsets=o)
            base = eng.stats()["n_decisions"]
            in_len = np.array([len(p) for p in prompts], np.int64)
            (dec, det, lists), names = _traced(lambda: eng.schedule_with_match(match, total, in_len, BST, topk=True),
                                               ("k_dense_pick",), where=f"{where} top-{K} with match")
            odec, ototal, olists = _oracle(orc, L, prompts, tie_seed, base, topk=K)
            helpers.assert_decisions_equal(dec, det, odec, ototal, where=f"{where} top-{K} with match")
            got = _lists(lists)
            np.testing.assert_array_equal(got["primary"], olists["primary"], err_msg=f"{where} top-{K} with match")


# ------------------------------------------------------------------------------------------------
# landscapes
# ------------------------------------------------------------------------------------------------
def _holders(rng, slots, sizes, full=False):
    slots = np.asarray(slots)
    return [[(int(e), B if full else int(rng.integers(1, B + 1))) for e in rng.choice(slots, size=n, replace=False)]
            for n in sizes]


def land_zero_prefix(seed):
    """L1: the decode profile weighs the prefix scorer 0 (every holder scores its base), a P/D prefill profile and an
    encode profile; large equal-base groups, one family with 40 holders."""
    rng = np.random.default_rng(seed)
    E = 96
    role = rng.choice([1, 1, 1, 2, 3, 5, 7], E).astype(np.uint8)
    kv = np.where(rng.random(E) < 0.8, 0.0, 0.5)
    waiting = np.where(rng.random(E) < 0.8, 0, 2).astype(np.int32)
    dec = np.flatnonzero(np.isin(role, [1, 3, 7]))
    return Land(E, role, kv, waiting, (F_DECODE, [(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0), (PREFIX, 0.0, 0.0)]),
                pref=(F_PREFILL, [(QUEUE, 1.0, 0.0), (PREFIX, 1.0, 0.0)]), enc=(F_ENCODE, [(KV, 1.0, 0.0)]),
                holders=_holders(rng, dec, [3, 12, 40]) + _holders(rng, np.arange(E), [20]), nct=8, seed=seed)


def land_negative(seed):
    """L2: a negative load weight (every decode base is negative) and a negative prefix weight in prefill."""
    rng = np.random.default_rng(seed)
    E = 80
    role = np.where(np.arange(E) % 3 == 0, 2, 1).astype(np.uint8)
    kv = rng.choice([0.0, 0.5, 1.0], E)
    waiting = rng.choice([0, 0, 4, 8], E).astype(np.int32)
    return Land(E, role, kv, waiting, (F_DECODE, [(LOAD, -1.0, 10.0), (KV, 0.05, 0.0), (PREFIX, 2.0, 0.0)]),
                pref=(F_PREFILL, [(KV, 1.0, 0.0), (PREFIX, -1.5, 0.0), (QUEUE, 0.5, 0.0)]),
                holders=_holders(rng, np.arange(E), [4, 9, 36]), nct=8, seed=seed)


ROUNDING = [(KV, 0.1, 0.0), (QUEUE, 0.7, 0.0), (LOAD, THIRD, 10.0), (EXT, 0.1, 0.0), (PREFIX, -THIRD, 0.0),
            (RUNNING, 0.7, 0.0), (TOKEN, THIRD, 5000.0, 1)]


def land_rounding(orc, seed, order):
    """L3: weights 0.1, 0.7 and +-1/3 over 7 scorers with continuous metrics, in the given scorer order.  The prefix
    weight is negative and family g is held by the g + 1 best endpoints of the order, so the winners walk down the
    order: many bases, not only the head's, decide a pick."""
    rng = np.random.default_rng(seed)
    E = 64
    ext = np.stack([rng.random(E), rng.integers(0, 8000, E).astype(np.float64)])
    kv, waiting, running = rng.random(E), rng.integers(0, 14, E), rng.integers(0, 9, E)
    prof = (F_NONE, [ROUNDING[i] for i in order])
    base, _, _, _ = orc.profile_run(_oprof(orc, prof), orc.PoolState(np.zeros(E, np.uint8), kv, waiting, running, ext),
                                    np.zeros(E, np.int32), 0)
    head = sorted(range(E), key=lambda e: (-base[e], e))
    return Land(E, np.zeros(E, np.uint8), kv, waiting, prof, running=running, ext=ext,
                holders=[[(e, B) for e in head[: g + 1]] for g in range(24)], R=128, seed=seed, cold_share=0.05)


def land_edges(seed):
    """L4: every request-independent kind in one profile, at its clamp edges: kv in {0, 1, -0.25, 1.5}, waiting equal to
    the load-aware threshold, token load equal to its threshold, active requests equal to idle, running equal on every
    candidate (min = max), external values outside [0, 1]."""
    rng = np.random.default_rng(seed)
    E = 70
    kv = rng.choice([0.0, 1.0, -0.25, 1.5], E)
    waiting = rng.choice([0, 10, 25], E).astype(np.int32)
    ext = np.stack([rng.choice([-0.5, 0.0, 1.0, 1.5], E), rng.choice([0.0, 2500.0, 5000.0, 9000.0], E),
                    rng.choice([0.0, 2.0, 5.0], E)])
    prim = [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0), (LOAD, 1.0, 10.0), (EXT, 0.5, 0.0), (RUNNING, 1.0, 0.0),
            (TOKEN, 1.0, 5000.0, 1), (ACTIVE, 1.0, 0.5, 2, 2.0), (PREFIX, 2.0, 0.0)]
    return Land(E, np.zeros(E, np.uint8), kv, waiting, (F_NONE, prim), running=np.full(E, 3), ext=ext,
                holders=_holders(rng, np.arange(E), [3, 8, 33]), seed=seed)


def land_overflow_sum(seed):
    """L5: finite weights near 1e308 whose ordered sums overflow: +inf for part of decode (finite sums below it),
    -inf for every prefill candidate."""
    rng = np.random.default_rng(seed)
    E = 64
    role = np.where(np.arange(E) % 4 == 0, 2, 1).astype(np.uint8)
    kv = np.where(role == 2, 0.0, rng.choice([0.0, 0.0, 0.5], E))
    waiting = np.where(role == 2, 0, rng.choice([0, 0, 3], E)).astype(np.int32)
    return Land(E, role, kv, waiting, (F_DECODE, [(KV, 1e308, 0.0), (QUEUE, 1.7e308, 0.0), (PREFIX, 1.0, 0.0)]),
                pref=(F_PREFILL, [(KV, -1e308, 0.0), (QUEUE, -1.7e308, 0.0), (PREFIX, 1.0, 0.0)]),
                holders=_holders(rng, np.arange(E), [3, 10]), nct=8, seed=seed)


def land_whole_group(seed):
    """L6: one group spanning the whole pool of 100; 32 holders at the head of the order (slots 0-31: the first
    unmatched entry is in the second chunk) and 32 holders straddling it (slots 20-51)."""
    E = 100
    return Land(E, np.zeros(E, np.uint8), np.full(E, 0.5), np.zeros(E), (F_NONE, [(KV, 1.0, 0.0), (PREFIX, 1.0, 0.0)]),
                holders=[[(e, B) for e in range(32)], [(e, B) for e in range(20, 52)], [(e, 3) for e in range(5)]],
                seed=seed, cold_share=0.1)


def land_straddle(seed):
    """L6: groups of 40 / 30 / 30 (the first straddles the 32-entry chunk), a holder set covering 32 slots of the head
    group, and a prefill profile without candidates while decode has all of them."""
    E = 100
    kv = np.array([0.0] * 40 + [0.5] * 30 + [1.0] * 30)
    rng = np.random.default_rng(seed)
    perm = rng.permutation(E)
    return Land(E, np.ones(E, np.uint8), kv[perm], np.zeros(E), (F_DECODE, [(KV, 1.0, 0.0), (PREFIX, 0.5, 0.0)]),
                pref=(F_PREFILL, [(KV, 1.0, 0.0)]),
                holders=[[(int(e), B) for e in np.flatnonzero(kv[perm] == 0.0)[:32]],
                         [(int(e), int(rng.integers(1, B + 1))) for e in np.flatnonzero(kv[perm] == 0.5)[5:25]]],
                nct=4, seed=seed)


def land_single(seed):
    """L6 / L8: n_cand = 1 -- one slot in a pool of 33, the other slots (outside the pool) hold index entries."""
    E = 33
    return Land(E, np.zeros(E, np.uint8), np.zeros(E), np.zeros(E), (F_NONE, [(QUEUE, 1.0, 0.0), (PREFIX, 2.0, 0.0)]),
                holders=[[(e, B) for e in range(E)], [(3, 4), (17, 2)]], ids=[17], seed=seed)


def land_pool(E, seed):
    """L7: pools of E slots, few load levels, R small."""
    rng = np.random.default_rng(seed)
    kv = rng.choice([0.0, 0.25, 0.5], E)
    waiting = rng.choice([0, 0, 1], E).astype(np.int32)
    sizes = [min(E, n) for n in (1, 5, 40)]
    return Land(E, np.zeros(E, np.uint8), kv, waiting, (F_NONE, [(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0), (PREFIX, 2.0, 0.0)]),
                holders=_holders(rng, np.arange(E), sizes), R=48, seed=seed)


def land_partial(seed, ids=None, role=None):
    """L8: every fifth slot is outside the pool and holds index entries (some prefixes are held only there)."""
    rng = np.random.default_rng(seed)
    E = 64
    out = np.arange(0, E, 5)
    if ids is None:
        ids = np.setdiff1d(np.arange(E), out)
    role = rng.choice([1, 2, 3], E).astype(np.uint8) if role is None else role
    return Land(E, role, rng.choice([0.0, 0.5], E), rng.choice([0, 2], E),
                (F_DECODE, [(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0), (PREFIX, 2.0, 0.0)]),
                pref=(F_PREFILL, [(KV, 1.0, 0.0), (PREFIX, 1.0, 0.0)]),
                holders=[[(int(e), B) for e in out[:6]], [(int(e), 5) for e in out] + [(7, 2), (8, 3)],
                         _holders(rng, np.arange(E), [36])[0]],
                ids=ids, nct=8, seed=seed)


LANDS = {
    "L1-zero-prefix-weight": lambda: land_zero_prefix(1),
    "L2-negative-weights": lambda: land_negative(2),
    "L4-clamp-edges": lambda: land_edges(4),
    "L5-sums-overflow": lambda: land_overflow_sum(5),
    "L6-whole-pool-group": lambda: land_whole_group(6),
    "L6-groups-straddle-chunks": lambda: land_straddle(7),
    "L6-one-candidate": lambda: land_single(8),
    "L8-partial-pool": lambda: land_partial(9),
}


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("name", list(LANDS))
def test_landscape_every_path(epp, orc, name, tie_seed):
    L = LANDS[name]()
    dec, odec = run_paths(epp, orc, L, tie_seed, where=f"{name} tie_seed={tie_seed}")
    ok = odec["status"] == 0
    # (L5: the lowest slot of the +inf group wins, and it need not hold a block)
    assert ok.any() and ((dec["match_blocks"] > 0).any() or (name.startswith("L5") and not tie_seed)), name
    if name.startswith("L5"):
        assert np.isposinf(odec["score"][ok]).any() and np.isneginf(odec["prefill_score"][odec["prefill_pick"] >= 0]).all()
    if name.startswith("L2"):
        cold = ok & (dec["match_blocks"] == 0)
        assert cold.any() and (odec["score"][cold] < 0).all()
    if name.startswith("L6") or name.startswith("L1"):
        assert (odec["tie_count"][ok] > (32 if name.startswith("L6") else 8)).any() or name == "L6-one-candidate"
    if name == "L6-one-candidate":
        assert (odec["tie_count"][ok] == 1).all() and (odec["pick"][ok] == 17).all()


def test_L3_rounding_two_scorer_orders(epp, orc):
    """The same scorers in two orders round differently somewhere; each order equals the oracle bit for bit."""
    fwd = list(range(len(ROUNDING)))
    rev = [3, 6, 1, 4, 0, 5, 2]
    got = {}
    for tag, order in (("forward", fwd), ("shuffled", rev)):
        L = land_rounding(orc, 3, order)
        got[tag] = run_paths(epp, orc, L, 0x77 if tag == "shuffled" else 0, asynchronous=False, topk=2, where=f"L3 {tag}")
    a, b = got["forward"][1], got["shuffled"][1]
    assert (a["score"].view(np.uint64) != b["score"].view(np.uint64)).any(), "the orders never round differently"
    np.testing.assert_allclose(a["score"], b["score"], rtol=1e-14)


@pytest.mark.parametrize("E", [1, 33, 1025, 4096, 131073])
def test_L7_pool_sizes(epp, orc, E):
    """Many sort entries per thread of the one-CTA bitonic sort and long group walks in k_pool_groups."""
    L = land_pool(E, 70 + E % 97)
    run_paths(epp, orc, L, 0x1234 if E % 2 else 0, asynchronous=E <= 1025, topk=2 if E <= 4096 else 0, where=f"L7 E={E}")


def test_L8_pool_churn(epp, orc):
    """A second pool_set between batches drops slots, re-adds others and changes roles; decisions follow the new pool."""
    import copy

    import torch
    L1 = land_partial(9)
    rng = np.random.default_rng(19)
    ids2 = np.setdiff1d(np.arange(L1.E), np.arange(2, L1.E, 7))           # other slots out, the old ones back
    role2 = L1.role.copy()
    flip = rng.choice(L1.E, 20, replace=False)
    role2[flip] = np.where(role2[flip] == 1, 2, 1)
    L2 = copy.copy(L1)                                                    # the same index, another pool
    L2.ids, L2.role, L2.waiting = ids2, role2, np.roll(L1.waiting, 5)
    d, o = _pack(L1.prompts)
    with _engine(epp, L1, 0x99) as eng:
        for L in (L1, L2, L1):
            if L is not L1 or eng.stats()["n_decisions"]:
                _traced(lambda: eng.pool_set(*L.pool_arrays()), POOL_KERNELS, where="churn pool_set")
            base = eng.stats()["n_decisions"]
            dd, do = torch.from_numpy(d).cuda(), torch.from_numpy(o.view(np.int64)).cuda()
            dec, det = eng.schedule(dd, offsets=do)
            torch.cuda.synchronize()
            odec, ototal = _oracle(orc, L, L1.prompts, 0x99, base)
            helpers.assert_decisions_equal(epp.decisions_from_torch(dec), _det(epp, det), odec, ototal, where="churn")
            base = eng.stats()["n_decisions"]
            sp = L1.prompts[:40]
            starts, end, lens = _rows(sp)
            buf = np.zeros(end + 64, np.uint8)
            for s0, p in zip(starts, sp):
                buf[s0: s0 + len(p)] = np.frombuffer(p, np.uint8)
            (hdec, hdet), names = _traced(lambda: eng.schedule(buf, offsets=np.array(starts + [end], np.uint64), lengths=lens),
                                          (SMALL,), where="churn host batch")
            odec, ototal = _oracle(orc, L, sp, 0x99, base)
            helpers.assert_decisions_equal(hdec, hdet, odec, ototal, where="churn host batch")


@pytest.mark.parametrize("K", [33, 64])
@pytest.mark.parametrize("tie_seed", [0, 0xAB])
def test_L9_topk_past_32(epp, orc, K, tie_seed):
    """Groups of 40 and 70 equal scores, a prefill profile with fewer candidates than k; lists equal the oracle's and
    never repeat an endpoint (members 32-63 of a group are tracked in gen::eval's second register)."""
    rng = np.random.default_rng(K + tie_seed)
    E = 120
    kv = np.array([0.0] * 40 + [0.5] * 70 + [1.0] * 10)[rng.permutation(E)]
    role = np.where(rng.random(E) < 0.15, 3, 1).astype(np.uint8)
    L = Land(E, role, kv, np.zeros(E), (F_DECODE, [(KV, 1.0, 0.0), (PREFIX, 1.0, 0.0)]),
             pref=(F_PREFILL, [(KV, 1.0, 0.0), (PREFIX, 1.0, 0.0)]),
             holders=_holders(rng, np.arange(E), [2, 7, 50]), nct=4, seed=K)
    check_topk(epp, orc, L, tie_seed, K, where=f"L9 k={K}")


def test_L5_topk_with_infinite_sums(epp, orc):
    """gen::eval's first group is +inf: it must be emitted, and the groups after it strictly below."""
    L = land_overflow_sum(55)
    check_topk(epp, orc, L, 0, 5, where="L5 top-5")


# ------------------------------------------------------------------------------------------------
# L10: no-hit-lru with an LRU spanning several 1024-slot chunks
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,lru", [(4096, 1), (4096, 1023), (4096, 1025), (4096, 4096), (4096, 4097), (1500, 1023),
                                   (1500, 1500)])
def test_L10_nohit_lru_large_pool(epp, orc, E, lru):
    """Decode (no scorer) follows the prefix; the prefill profile (queue + no-hit-lru) has no holder among its
    candidates, so every request is cold for it and Adds its decode pick and its prefill pick: hundreds of distinct
    Adds per call fill and trim the LRU over 1024-slot chunks, and most members sit outside the prefill candidates.
    Decisions against tools/nohit_lru_model.py, the LRU after every call, and the prefill profile's cold column
    (epp_score) against the model's."""
    import torch
    rng = np.random.default_rng(E + lru)
    batches = 3
    role = np.where(np.arange(E) % 8 == 5, 2, 1).astype(np.uint8)
    R = min(512, int((role == 1).sum()) // batches)
    kv = rng.choice([0.0, 0.5], E)
    waiting = np.zeros(E, np.int32)
    running = np.zeros(E, np.int32)
    dslots = np.flatnonzero(role == 1)
    prim = [(KV, 1.0, 0.0), (PREFIX, 4.0, 0.0)]
    pref = [(QUEUE, 1.0, 0.0), (M.NO_HIT_LRU, 1.0, float(lru))]
    owners = rng.permutation(dslots)[: R * batches]
    fam = [rng.integers(0, 256, 2 * BB, dtype=np.uint8).tobytes() for _ in owners]
    hs, es = [], []
    for f, e in zip(fam, owners):
        h = _hash(f)
        hs += h
        es += [int(e)] * len(h)
    pool = orc.PoolState(role, kv, waiting, running)
    model = M.Model(orc, pool, E, [(F_DECODE, prim), (F_PREFILL, pref)], lru, always=True, block_size_tokens=BST)
    pcand = list(np.flatnonzero(role == 2))
    with epp.Engine(E, _spec(epp, (F_DECODE, prim)), _spec(epp, (F_PREFILL, pref)), block_size_tokens=BST,
                    max_prefix_blocks=B, always_disagg=True) as eng:
        eng.register_model(MODEL)
        eng.pool_set(np.arange(E), role, kv, waiting, running)
        eng.index_load_snapshot(np.array(hs, np.uint64), np.array(es, np.uint32))
        seen = {}
        for b in range(batches):
            # mostly new owners, a quarter of them repeated from the previous call (moved to the LRU's end)
            pick = list(range(b * R, (b + 1) * R))
            if b:
                pick[: R // 4] = list(range((b - 1) * R, (b - 1) * R + R // 4))
            prompts = [fam[i] + rng.integers(0, 256, int(rng.integers(0, BB)), dtype=np.uint8).tobytes() for i in pick]
            d, o = _pack(prompts)
            match, total = eng.prefix_match(d, offsets=o)
            want = model.schedule(match, total, np.array([len(p) for p in prompts], np.int64))
            assert all(x[5] for x in want)
            dd, do = torch.from_numpy(d).cuda(), torch.from_numpy(o.view(np.int64)).cuda()
            (dec, _), names = kernels_launched(lambda: eng.schedule(dd, offsets=do), repeatable=False)
            for n, c in names.items():
                seen[n] = seen.get(n, 0) + c
            dec = epp.decisions_from_torch(dec)
            st = np.array([x[0] for x in want])
            assert (dec["status"] == st).all()
            np.testing.assert_array_equal(dec["pick"], np.array([x[1] for x in want], np.uint32), err_msg=f"batch {b}")
            np.testing.assert_array_equal(dec["score"].view(np.uint64), np.array([x[2] for x in want]).view(np.uint64))
            np.testing.assert_array_equal(dec["prefill_pick"], np.array([x[3] for x in want], np.uint32),
                                          err_msg=f"L10 E={E} lru={lru} batch {b} prefill pick")
            keys = model.lru.keys()
            assert eng.nohit_lru_get() == keys, f"L10 E={E} lru={lru}: LRU after batch {b}"
            # the cold column the next call scores with (epp_score, scorer 1 of the prefill profile)
            col = eng.score(match[:2], total[:2], 1, 1)
            want_col = M.cold_column(pcand, keys, E)
            np.testing.assert_array_equal(col[0][pcand], want_col[pcand], err_msg=f"L10 E={E} lru={lru} column {b}")
        if helpers.trace_complete(seen):
            for k in ("k_match_pick_sparse_nohit<6, false, 2>", "k_nohit_touch", "k_nohit_trim", "k_nohit_column"):
                assert_ran(seen, k, where=f"L10 E={E} lru={lru}")
        if lru in (1, 1023, 1025):
            assert len(keys) == lru, (len(keys), lru)             # trimmed
        else:
            assert len(keys) > 1024, len(keys)                    # members in more than one 1024-slot chunk
