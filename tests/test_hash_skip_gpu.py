"""Schedule batches that stop reading each prompt where the index stops matching it (EPP_HASH_SKIP, DESIGN.md section
4.1): a block hash depends on blocks 0..b alone, so k_hash_fused loads no window past the first one the presence bitmap
proves absent (plus the ring's lookahead) and no trailing partial block of a closed request.  Decisions must equal the
oracle's and those of an engine that reads every byte (EPP_HASH_SKIP=0), bit for bit, and the bytes the kernel reports
having read (epp_stats.last_prompt_bytes_read) must lie between what the bounds need and that plus the lookahead.  The
bounds are restated on the host from the index keys with a bitmap of known size.  Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

from helpers import assert_ran, assert_decisions_equal, kernels_launched, ran

pytestmark = pytest.mark.gpu

ALL1 = 0xFFFFFFFFFFFFFFFF
E, BST, B = 96, 16, 160           # 64-byte blocks (the k_hash_fused path), 20 windows: well past the lookahead
BB = 4 * BST
W = 8                             # blocks per lookup window of k_hash_fused
LOOKAHEAD = 2                     # windows a closed request may read past its closing one: the ring's stages
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
    """Rows at multiples of 64 bytes plus a gap, exact lengths (ragged offsets / lengths) -> device tensors."""
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
    """Families of cached prefixes per model, an index over them with a hole at a window start and a partial-block stop,
    and a batch that walks into every kind of stop, with prompts shorter than a block and longer than the block cap."""

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
        hs += h[:16] + h[18:60]                   # present, absent (blocks 16, 17: a window start), present again
        es += [1] * 58
        self.partial = self.fam[m0][3][: 72 * BB + 20]
        hp = orc.hash_prompt(self.partial, m0, BST, B)
        hs += hp[:72]                             # the 73rd (partial) block is absent: the stop falls on it
        es += [5] * 72
        self.partial_held = self.fam[m0][4][: 47 * BB + 33]
        hs += orc.hash_prompt(self.partial_held, m0, BST, B)
        es += [6] * 48                            # every block held, the partial one included
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
        kind = int(rng.integers(0, 10))
        if kind == 0:
            return rng.integers(0, 256, int(rng.integers(0, BB * (B + 2))), dtype=np.uint8).tobytes()   # cold
        if kind == 1:
            return rng.integers(0, 256, int(rng.integers(0, BB)), dtype=np.uint8).tobytes()             # no full block
        if kind == 2 and m == self.models[0]:
            return self.partial if rng.random() < 0.5 else self.partial_held
        f = self.fam[m][int(rng.integers(0, 6))]
        keep = int(rng.integers(0, len(f) + 1))
        tail = int(rng.integers(0, 3 * BB)) if kind != 3 else BB * 8 + 5                 # kind 3: past the block cap
        return f[:keep] + rng.integers(0, 256, tail, dtype=np.uint8).tobytes()

    def batch(self, R):
        mi = self.rng.integers(0, len(self.models), R)
        return [self.prompt(self.models[i]) for i in mi], mi

    def oracle(self, orc, prompts, model_idx, profiles, nct=0, tie_seed=0, mm=None, enc=None, ix=None):
        """One oracle run per request; tie_base = the request's ordinal in the batch."""
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

    def read_window(self, orc, prompts, model_idx, keys, log2bits):
        """Host restatement of k_hash_fused's bound with a bitmap of 2^log2bits bits over `keys` -> per request the bytes
        every read must cover and the most a skipping read may take (lookahead included)."""
        shift = 64 - log2bits
        bits = {int(k) >> shift for k in keys if int(k) != ALL1}

        def absent(h):
            return h != ALL1 and (h >> shift) not in bits

        lo = np.zeros(len(prompts), np.int64)
        hi = np.zeros(len(prompts), np.int64)
        for r, (p, i) in enumerate(zip(prompts, model_idx)):
            eff = 0 if len(p) < BB else min(len(p), BB * B)
            nfull = eff // BB
            lo[r] = hi[r] = eff
            if nfull == 0:
                continue
            h = orc.hash_prompt(p, self.models[i], BST, B)
            stop = next((b for b in range(0, nfull, W) if absent(h[b])), None)
            if stop is not None:                  # closed on a full block: no tail, windows past the closing one skipped
                c = stop // W
                lo[r] = min(nfull, (c + 1) * W) * BB
                hi[r] = min(nfull, (c + 1 + LOOKAHEAD) * W) * BB
        return lo, hi


def _eff_bytes(prompts):
    return sum(0 if len(p) < BB else min(len(p), BB * B) for p in prompts)


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


def _run(epp, eng, mids, prompts, model_idx, mm=None, asynchronous=False, keep_hashes=False):
    import torch
    d, o, ln = _device_batch(prompts)
    mid = torch.from_numpy(np.array(mids, np.int32)[model_idx]).cuda()
    mm = None if mm is None else torch.from_numpy(mm).cuda()
    ddec, ddet = eng.schedule(d, offsets=o, lengths=ln, model_ids=mid, multimodal=mm, asynchronous=asynchronous,
                              keep_hashes=keep_hashes)
    if asynchronous:
        eng.synchronize()
    torch.cuda.synchronize()
    return epp.decisions_from_torch(ddec), ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)


def _traced(fn, kernels, where):
    """fn() under the profiler -> fn's first result, once a trace has shown every kernel of `kernels`."""
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


def _both(epp, monkeypatch, world, stages, tie_seed, prompts, model_idx, log2bits, mm=None, index=True):
    """[(decisions, details, bytes stored, bytes read)] with EPP_HASH_SKIP=1, then 0; bitmap of 2^log2bits bits."""
    out = []
    monkeypatch.setenv("EPP_PRESENCE_LOG2BITS", str(log2bits))
    for skip in ("1", "0"):
        monkeypatch.setenv("EPP_HASH_SKIP", skip)
        eng, mids = _engine(epp, world, stages, tie_seed)
        with eng:
            if index:
                eng.index_load_snapshot(world.hs, world.es)
            dec, det = _traced(lambda: _run(epp, eng, mids, prompts, model_idx, mm),
                               ("k_hash_fused(", "k_match_pick_sparse<"), f"EPP_HASH_SKIP={skip}")
            st = eng.stats()
            out.append((dec, det, int(st["last_hash_bytes_stored"]), int(st["last_prompt_bytes_read"])))
    return out


def _assert_same(a, b, where):
    np.testing.assert_array_equal(a[0], b[0], err_msg=where)
    np.testing.assert_array_equal(a[1], b[1], err_msg=where)
    assert a[2] == b[2], where                    # the stored rows are a function of the bounds alone


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("stages", [1, 3])
@pytest.mark.parametrize("log2bits", [20, 6])
def test_skip_vs_oracle_and_full_reads(epp, orc, monkeypatch, stages, tie_seed, log2bits):
    """Two models, 301 requests (not a multiple of 32): holes, partial-block stops, cold prompts, prompts without a full
    block and past the block cap, the sentinel hash in the index; one profile or the P/D + encode handler; both tie
    rules; a sized bitmap or a saturated 2^6-bit one."""
    world = World(orc, stages * 7 + (tie_seed != 0) + 100 * (log2bits == 6), models=(b"m", b"other"))
    mm = (world.rng.random(len(world.prompts)) < 0.5).astype(np.uint8) if stages == 3 else None
    skip, full = _both(epp, monkeypatch, world, stages, tie_seed, world.prompts, world.model_idx, log2bits, mm)
    _assert_same(skip, full, "skip vs full reads")
    dec, det = skip[0], skip[1]
    odec, ototal = world.oracle(orc, world.prompts, world.model_idx, _oracle_profiles(orc, stages), 4 if stages > 1 else 0,
                                tie_seed, mm, orc.make_profile(3, ENC) if stages == 3 else None)
    assert_decisions_equal(dec, det, odec, ototal, where=f"stages {stages} tie {tie_seed:#x} log2bits {log2bits}")
    assert full[3] == _eff_bytes(world.prompts)
    lo, hi = world.read_window(orc, world.prompts, world.model_idx, world.hs, log2bits)
    assert lo.sum() <= skip[3] <= hi.sum(), (lo.sum(), skip[3], hi.sum())
    if log2bits == 20:
        assert skip[3] < full[3]                                        # the skipping ran
    assert (dec["match_blocks"] > 0).sum() > 50 and ((dec["match_blocks"] > W * LOOKAHEAD) & (dec["match_blocks"] < B)).any()


@pytest.mark.parametrize("R", [5, 301])
def test_cold_batch_and_empty_index(epp, orc, monkeypatch, R):
    """Nothing indexed: every bound is 0, so a prompt is read through window 0 and at most the lookahead past it; one
    tile that is not full, or a ragged last tile."""
    world = World(orc, 3 + R, R=R)
    skip, full = _both(epp, monkeypatch, world, 1, 0, world.prompts, world.model_idx, 20, index=False)
    _assert_same(skip, full, "empty index")
    lo, hi = world.read_window(orc, world.prompts, world.model_idx, [], 20)
    assert lo.sum() <= skip[3] <= hi.sum() and full[3] == _eff_bytes(world.prompts)
    odec, ototal = world.oracle(orc, world.prompts, world.model_idx, _oracle_profiles(orc, 1), ix=orc.Indexer())
    assert_decisions_equal(skip[0], skip[1], odec, ototal, where="empty index")
    assert (skip[0]["match_blocks"] == 0).all()


def test_patched_commits(epp, orc, monkeypatch):
    """An incrementally built index: a patched commit that indexes a new prefix (its bits must be set before reads stop
    there) and one that removes the only endpoint of another (its bits stay).  Decisions after each commit vs the oracle."""
    world = World(orc, 11)
    monkeypatch.setenv("EPP_HASH_SKIP", "1")
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
        extra = [new_fam[: k * BB + 7] for k in (5, 100, B)]
        prompts = world.prompts + extra
        mi = np.concatenate([world.model_idx, np.zeros(len(extra), np.int64)])
        for step in range(3):
            if step == 1:
                eng.index_add(40, new_h[:125])
                ix.add(new_h[:125], 40)
            if step == 2:
                eng.index_remove_endpoint(1)                  # the only holder of the holed prefix
                ix.remove_pod(1)
            dec, det = _run(epp, eng, mids, prompts, mi)
            if step:
                assert eng.stats()["last_index_patched"] == 1, step
            odec, ototal = world.oracle(orc, prompts, mi, _oracle_profiles(orc, 1), ix=ix)
            assert_decisions_equal(dec, det, odec, ototal, where=f"commit {step}")
        assert (dec["match_blocks"][-3:] == [5, 100, 125]).all()


@pytest.mark.parametrize("asynchronous", [False, True])
def test_skipping_batch_after_deep_batch(epp, orc, monkeypatch, asynchronous):
    """8192 requests (the chunk-pipelined path when asynchronous): a batch of fully cached prompts fills every ring
    slot and row, then a shallow batch skips most of its bytes over that state; then keep_hashes and epp_hash_prompts
    batches, which must read every byte."""
    world = World(orc, 21, R=8)
    monkeypatch.setenv("EPP_HASH_SKIP", "1")
    monkeypatch.setenv("EPP_PRESENCE_LOG2BITS", "20")
    R = 8192
    deep = [world.fam[b"m"][5][: B * BB]] * R
    shallow, mi = world.batch(R)
    eng, mids = _engine(epp, world)
    with eng:
        eng.index_load_snapshot(world.hs, world.es)
        dec, _ = _run(epp, eng, mids, deep, np.zeros(R, np.int64), asynchronous=asynchronous)
        assert (dec["match_blocks"] == B).all()
        if not asynchronous:
            assert eng.stats()["last_prompt_bytes_read"] == _eff_bytes(deep)
        dec, det = _run(epp, eng, mids, shallow, mi, asynchronous=asynchronous)
        odec, ototal = world.oracle(orc, shallow, mi, _oracle_profiles(orc, 1))
        assert_decisions_equal(dec, det, odec, ototal, where="after the deep batch")
        assert ((dec["match_blocks"] > 0) & (dec["match_blocks"] < B)).sum() > R // 4
        if not asynchronous:
            lo, hi = world.read_window(orc, shallow, mi, world.hs, 20)
            got = eng.stats()["last_prompt_bytes_read"]
            assert lo.sum() <= got <= hi.sum() and got < _eff_bytes(shallow)
        n = 1000
        dec_k, det_k = _run(epp, eng, mids, shallow[:n], mi[:n], keep_hashes=True)
        assert eng.stats()["last_prompt_bytes_read"] == _eff_bytes(shallow[:n])
        assert_decisions_equal(dec_k, det_k, odec[:n], ototal[:n], where="keep_hashes")
        import torch
        d, o, ln = _device_batch(shallow[:n])
        mid = torch.from_numpy(np.array(mids, np.int32)[mi[:n]]).cuda()
        hh, nb = eng.hash_prompts(d, offsets=o, lengths=ln, model_ids=mid)
        torch.cuda.synchronize()
        assert eng.stats()["last_prompt_bytes_read"] == _eff_bytes(shallow[:n])
        hh, nb = hh.cpu().numpy().view(np.uint64), nb.cpu().numpy()
        for r in range(0, n, 37):
            h = orc.hash_prompt(shallow[r], world.models[mi[r]], BST, B)
            assert nb[r] == len(h) and list(hh[r, : nb[r]]) == h, r


def test_scaled_config3(epp, orc, monkeypatch):
    """A scaled config-3 batch of the trace generator (8192 requests of 4096 tokens): every decision equals the oracle's,
    and the kernel reads fewer bytes than the prompts hold."""
    from tools import tracegen as tg
    from tools import workload_setup as helpers
    import torch
    monkeypatch.setenv("EPP_HASH_SKIP", "1")
    w = tg.baseline_configs()["config3"].scaled(E=512, R=8192, T=4096)
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests()
    pool, ix, primary, prefill, _ = helpers.setup_oracle(orc, w, trace)
    odec, ototal = helpers.oracle_decisions(orc, w, pool, ix, primary, prefill, tokens)
    with helpers.make_engine(w) as eng:
        helpers.setup_engine(eng, w, trace)
        ddec, ddet = eng.schedule(torch.from_numpy(tokens.view(np.int32)).cuda(), uniform_len=w.prompt_bytes)
        torch.cuda.synchronize()
        helpers.assert_decisions_equal(epp.decisions_from_torch(ddec), ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1),
                                       odec, ototal, where="scaled config 3")
        assert 0 < eng.stats()["last_prompt_bytes_read"] < w.R * w.prompt_bytes
