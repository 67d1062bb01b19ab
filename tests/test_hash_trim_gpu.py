"""Schedule batches whose hash rows are stored only up to the read table's reach (EPP_HASH_TRIM, DESIGN.md section 4.1):
k_hash_fused stops storing a row at the first block the presence bitmap proves absent, and the match kernels never read
past it.  Decisions must equal the oracle's and those of whole rows (EPP_HASH_TRIM=0), bit for bit, for holes in a
cached prefix, stops on the trailing partial block, cold prompts and an empty index, several models, the P/D + encode
handler, both tie rules, a saturated bitmap, a patched commit that adds keys or strips a key's last endpoint, and a
trimmed batch that runs over the stale rows of a deep one.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import assert_ran, assert_decisions_equal, kernels_launched, ran

pytestmark = pytest.mark.gpu

ALL1 = 0xFFFFFFFFFFFFFFFF
E, BST, B = 96, 16, 40            # 64-byte blocks: the k_hash_fused path
BB = 4 * BST
PRIM, PREF, ENC = [(2, 1.0, 0), (1, 1.0, 0), (0, 2.0, 0)], [(2, 1.0, 0), (0, 1.0, 0)], [(1, 1.0, 0)]


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _spec(epp, filt, scorers):
    return epp.ProfileSpec(filt, [epp.ScorerSpec(k, w, p) for k, w, p in scorers])


def _device_batch(prompts):
    """Rows at multiples of 64 bytes with exact lengths (k_hash_fused needs 16-byte aligned rows) -> device tensors."""
    import torch
    starts = np.zeros(len(prompts) + 1, np.uint64)
    np.cumsum([(len(p) + 63) // 64 * 64 + 64 for p in prompts], out=starts[1:])
    data = np.zeros(int(starts[-1]) + 64, np.uint8)
    for s, p in zip(starts, prompts):
        data[int(s): int(s) + len(p)] = np.frombuffer(p, np.uint8)
    lens = np.array([len(p) for p in prompts], np.uint64)
    return (torch.from_numpy(data).cuda(), torch.from_numpy(starts.view(np.int64)).cuda(),
            torch.from_numpy(lens.view(np.int64)).cuda())


def _packed(prompts):
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    return np.frombuffer(b"".join(prompts) + b"\0" * 16, dtype=np.uint8).copy(), offs


class World:
    """Families of cached prefixes per model, an index over them with a hole and a partial-block stop, and a batch that
    walks into every kind of stop."""

    def __init__(self, orc, seed, models=(b"m",), R=301):
        rng = np.random.default_rng(seed)
        self.models = models
        self.fam = {m: [rng.integers(0, 256, BB * (B + 2), dtype=np.uint8).tobytes() for _ in range(6)] for m in models}
        hs, es = [], []
        for m in models:
            for g, f in enumerate(self.fam[m]):
                h = orc.hash_prompt(f, m, BST, B)
                for e in rng.choice(E, size=[1, 3, 6, 12, 30, 2][g], replace=False):
                    depth = B if g == 5 else int(rng.integers(1, B + 1))
                    hs += h[:depth]
                    es += [int(e)] * depth
        m0 = models[0]
        h = orc.hash_prompt(self.fam[m0][0], m0, BST, B)
        hs += h[:8] + h[10:20]                    # present, absent (blocks 8, 9), present again
        es += [1] * 18
        self.partial = self.fam[m0][3][: 12 * BB + 20]
        hp = orc.hash_prompt(self.partial, m0, BST, B)
        hs += hp[:12]                             # the 13th (partial) block is absent: the stop falls on it
        es += [5] * 12
        self.partial_held = self.fam[m0][4][: 7 * BB + 33]
        hs += orc.hash_prompt(self.partial_held, m0, BST, B)
        es += [6] * 8                             # every block held, the partial one included
        hs.append(ALL1)
        es.append(2)
        self.hs, self.es = np.array(hs, np.uint64), np.array(es, np.uint32)
        self.role = rng.choice([1, 2, 3, 5, 7, 0], size=E).astype(np.uint8)
        self.kv = rng.integers(0, 3, E) / 3.0
        self.waiting = rng.integers(0, 3, E).astype(np.int32)
        self.rng = rng
        self.prompts, self.model_idx = self.batch(R)

    def prompt(self, m):
        rng = self.rng
        kind = int(rng.integers(0, 8))
        if kind == 0:
            return rng.integers(0, 256, int(rng.integers(0, BB * (B + 2))), dtype=np.uint8).tobytes()   # cold
        if kind == 1 and m == self.models[0]:
            return self.partial if rng.random() < 0.5 else self.partial_held
        f = self.fam[m][int(rng.integers(0, 6))]
        keep = int(rng.integers(0, len(f) + 1))
        tail = int(rng.integers(0, 3 * BB))
        return f[:keep] + rng.integers(0, 256, tail, dtype=np.uint8).tobytes()

    def batch(self, R):
        mi = self.rng.integers(0, len(self.models), R)
        return [self.prompt(self.models[i]) for i in mi], mi

    def oracle(self, orc, prompts, model_idx, profiles, nct=0, tie_seed=0, mm=None, enc=None, ix=None):
        """One oracle run per request (cycle_batch hashes with one model); tie_base = the request's ordinal in the batch.
        One profile: every endpoint a candidate (the engines of _engine)."""
        if ix is None:
            ix = orc.Indexer()
            ix.load_pairs(self.hs, self.es)
        role = self.role if profiles[1] is not None else np.zeros(E, np.uint8)
        pool = orc.PoolState(role, self.kv, self.waiting)
        odec = np.zeros(len(prompts), dtype=orc.DECISION_DTYPE)
        ototal = np.zeros(len(prompts), np.int64)
        for r, i in enumerate(model_idx):
            d, o = _packed([prompts[r]])
            kw = dict(tie_seed=tie_seed, tie_base=int(r))
            if enc is not None:
                kw.update(encode=enc, multimodal=mm[r: r + 1])
            od, ot = orc.cycle_batch(self.models[i], BST, B, nct, False, ix, profiles[0], profiles[1], pool, d, o, 1, **kw)
            odec[r], ototal[r] = od[0], ot[0]
        return odec, ototal


def _engine(epp, world, stages=1, tie_seed=0, **extra):
    kw = dict(block_size_tokens=BST, max_prefix_blocks=B, tie_seed=tie_seed, **extra)
    if stages == 1:
        specs = (_spec(epp, 0, PRIM),)
    else:
        specs = (_spec(epp, 1, PRIM), _spec(epp, 2, PREF))
        kw["non_cached_tokens"] = 4
    if stages == 3:
        kw["encode"] = _spec(epp, 3, ENC)
    eng = epp.Engine(E, *specs, **kw)
    mids = [eng.register_model(m) for m in world.models]
    role = world.role if stages > 1 else np.zeros(E, np.uint8)
    eng.pool_set(np.arange(E), role, world.kv, world.waiting)
    return eng, mids


def _oracle_profiles(orc, stages):
    if stages == 1:
        return orc.make_profile(0, PRIM), None
    return orc.make_profile(1, PRIM), orc.make_profile(2, PREF)


def _run(epp, eng, mids, prompts, model_idx, mm=None, asynchronous=False):
    import torch
    d, o, ln = _device_batch(prompts)
    mid = torch.from_numpy(np.array(mids, np.int32)[model_idx]).cuda()
    mm = None if mm is None else torch.from_numpy(mm).cuda()
    ddec, ddet = eng.schedule(d, offsets=o, lengths=ln, model_ids=mid, multimodal=mm, asynchronous=asynchronous)
    if asynchronous:
        eng.synchronize()
    torch.cuda.synchronize()
    return epp.decisions_from_torch(ddec), ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)


def _traced(fn, kernels, where):
    """fn() under the profiler -> fn's first result, once a trace has shown every kernel of `kernels`.  fn is an engine
    batch that may be repeated (same rows, same byte count); a trace now and then lacks device records of the engine's
    streams although it kept those of torch's, so up to three traces are taken."""
    first = None
    for attempt in range(3):
        out, names = kernels_launched(fn)
        if attempt == 0:
            first = out
        if all(ran(names, k) for k in kernels):
            break
    for k in kernels:
        assert_ran(names, k, where=where)
    return first


def _both(epp, monkeypatch, world, stages, tie_seed, prompts, model_idx, mm=None, index=True, log2bits=None):
    """(trimmed decisions, details, bytes stored), then the same with whole rows."""
    out = []
    for trim in ("1", "0"):
        monkeypatch.setenv("EPP_HASH_TRIM", trim)
        if log2bits:
            monkeypatch.setenv("EPP_PRESENCE_LOG2BITS", log2bits)
        eng, mids = _engine(epp, world, stages, tie_seed)
        with eng:
            if index:
                eng.index_load_snapshot(world.hs, world.es)
            dec, det = _traced(lambda: _run(epp, eng, mids, prompts, model_idx, mm),
                               ("k_hash_fused(", "k_match_pick_sparse<"), f"EPP_HASH_TRIM={trim}")
            out.append((dec, det, int(eng.stats()["last_hash_bytes_stored"])))
    return out


def _assert_same(a, b, where):
    np.testing.assert_array_equal(a[0], b[0], err_msg=where)
    np.testing.assert_array_equal(a[1], b[1], err_msg=where)


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("stages", [1, 3])
@pytest.mark.parametrize("log2bits", [None, "6"])
def test_trimmed_rows_vs_oracle_and_whole_rows(epp, orc, monkeypatch, stages, tie_seed, log2bits):
    """Two models, 301 requests (not a multiple of 32): holes, partial-block stops, cold prompts, the sentinel hash in
    the index; one profile or the P/D + encode handler; both tie rules; the sized bitmap or a saturated 2^6-bit one."""
    world = World(orc, stages * 7 + (tie_seed != 0) + 100 * (log2bits is not None), models=(b"m", b"other"))
    mm = (world.rng.random(len(world.prompts)) < 0.5).astype(np.uint8) if stages == 3 else None
    trimmed, whole = _both(epp, monkeypatch, world, stages, tie_seed, world.prompts, world.model_idx, mm, log2bits=log2bits)
    _assert_same(trimmed, whole, "trimmed vs whole rows")
    dec, det, stored = trimmed
    odec, ototal = world.oracle(orc, world.prompts, world.model_idx, _oracle_profiles(orc, stages), 4 if stages > 1 else 0,
                                tie_seed, mm, orc.make_profile(3, ENC) if stages == 3 else None)
    assert_decisions_equal(dec, det, odec, ototal, where=f"stages {stages} tie {tie_seed:#x} log2bits {log2bits}")
    nb = dec["total_blocks"].astype(np.int64)
    assert whole[2] == 8 * nb.sum()                                    # whole rows: 256 x 8 B for a full-length request
    assert 8 * np.minimum(dec["match_blocks"].astype(np.int64), nb).sum() <= stored <= whole[2]
    if log2bits is None:
        assert stored < whole[2]                                       # the trimming ran
    assert (dec["match_blocks"] > 0).sum() > 50 and ((dec["match_blocks"] > 0) & (dec["match_blocks"] < nb)).any()
    held = [i for i, p in enumerate(world.prompts) if p is world.partial_held]
    cut = [i for i, p in enumerate(world.prompts) if p is world.partial]
    assert held and cut


def test_cold_batch_and_empty_index(epp, orc, monkeypatch):
    """Nothing indexed: every bound is 0, so no row runs past its first window of 8 hashes (stored before the lookup
    that proves block 0 absent has landed), and the decisions are those of an empty index."""
    world = World(orc, 3)
    trimmed, whole = _both(epp, monkeypatch, world, 1, 0, world.prompts, world.model_idx, index=False)
    _assert_same(trimmed, whole, "empty index")
    nb = trimmed[0]["total_blocks"].astype(np.int64)
    assert trimmed[2] <= 8 * np.minimum(nb, 8).sum() < whole[2]
    odec, ototal = world.oracle(orc, world.prompts, world.model_idx, _oracle_profiles(orc, 1), ix=orc.Indexer())
    assert_decisions_equal(trimmed[0], trimmed[1], odec, ototal, where="empty index")
    assert (trimmed[0]["match_blocks"] == 0).all()


def test_patched_commits_add_keys_and_keep_stale_bits(epp, orc, monkeypatch):
    """An incrementally built index: a patched commit that indexes a new prefix (its bits must be set) and one that
    removes the only endpoint of another (its bits stay, a false positive).  Decisions after each commit vs the oracle
    indexer."""
    world = World(orc, 11)
    monkeypatch.setenv("EPP_HASH_TRIM", "1")
    eng, mids = _engine(epp, world)
    ix = orc.Indexer()
    m = world.models[0]
    new_fam = world.rng.integers(0, 256, BB * (B + 2), dtype=np.uint8).tobytes()
    new_h = orc.hash_prompt(new_fam, m, BST, B)
    by_ep = {}
    for h, e in zip(world.hs, world.es):
        by_ep.setdefault(int(e), []).append(int(h))
    with eng:
        for e, hs in by_ep.items():
            eng.index_add(e, hs)
            ix.add(hs, e)
        extra = [new_fam[: k * BB + 7] for k in (5, 20, B)]
        prompts = world.prompts + extra
        mi = np.concatenate([world.model_idx, np.zeros(len(extra), np.int64)])
        for step in range(3):
            if step == 1:
                eng.index_add(40, new_h[:25])
                ix.add(new_h[:25], 40)
            if step == 2:
                eng.index_remove_endpoint(1)                  # the only holder of the holed prefix
                ix.remove_pod(1)
            dec, det = _run(epp, eng, mids, prompts, mi)
            if step:
                assert eng.stats()["last_index_patched"] == 1, step
            odec, ototal = world.oracle(orc, prompts, mi, _oracle_profiles(orc, 1), ix=ix)
            assert_decisions_equal(dec, det, odec, ototal, where=f"commit {step}")
        assert (dec["match_blocks"][-3:] == [5, 20, 25]).all()


@pytest.mark.parametrize("asynchronous", [False, True])
def test_trimmed_batch_after_deep_batch_and_keep_hashes(epp, orc, monkeypatch, asynchronous):
    """8192 requests (the chunk-pipelined path when asynchronous): a batch of fully cached prompts leaves whole rows,
    then a shallow batch stores short rows over them -- the stale hashes behind each bound must never be read.  Then a
    keep_hashes batch keeps whole rows for epp_index_add_picked, checked against the oracle indexer."""
    world = World(orc, 21, R=8)
    monkeypatch.setenv("EPP_HASH_TRIM", "1")
    R = 8192
    deep = [world.fam[b"m"][5][: B * BB]] * R
    shallow, mi = world.batch(R)
    eng, mids = _engine(epp, world)
    with eng:
        eng.index_load_snapshot(world.hs, world.es)
        dec, _ = _run(epp, eng, mids, deep, np.zeros(R, np.int64), asynchronous=asynchronous)
        assert (dec["match_blocks"] == B).all()
        dec, det = _run(epp, eng, mids, shallow, mi, asynchronous=asynchronous)
        odec, ototal = world.oracle(orc, shallow, mi, _oracle_profiles(orc, 1))
        assert_decisions_equal(dec, det, odec, ototal, where="after the deep batch")
        assert ((dec["match_blocks"] > 0) & (dec["match_blocks"] < B)).sum() > R // 4
        # keep_hashes: whole rows for the picks (the snapshot index cannot take adds: a fresh incremental engine)
    eng, mids = _engine(epp, world)
    ix = orc.Indexer()
    with eng:
        for e in np.unique(world.es):
            hs = world.hs[world.es == e]
            eng.index_add(int(e), hs)
            ix.add(hs, int(e))
        _run(epp, eng, mids, deep[:1000], np.zeros(1000, np.int64))
        import torch
        d, o, ln = _device_batch(shallow[:1000])
        ddec, _ = eng.schedule(d, offsets=o, lengths=ln, keep_hashes=True)
        torch.cuda.synchronize()
        dec = epp.decisions_from_torch(ddec)
        eng.index_add_picked()
        eng.index_commit()
        universe = set()
        for r in range(1000):
            hs = orc.hash_prompt(shallow[r], b"m", BST, B)
            ix.add(hs, int(dec["pick"][r]))
            universe.update(hs)
        for h in sorted(universe):
            assert eng.index_get(h) == ix.get(h), hex(h)
