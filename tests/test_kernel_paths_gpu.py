"""Every hash, match and probe path the engine can dispatch to, against the CPU oracle (and the python-xxhash golden
vectors): batch layouts, block sizes, prefix caps, the A/B switches of DESIGN.md section 12, and read tables whose probe
chains are long, wrap past the last slot or run through tombstones.  Each test first proves, from a torch.profiler
trace, that the kernel it is about actually ran -- a test that quietly fell back to the default kernel would prove
nothing.  Run on an H100: pytest -m gpu."""
import json
import os
from collections import defaultdict

import numpy as np
import pytest

from helpers import assert_ran, kernels_launched, ran

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "xxh64_vectors.json")
ALL1 = 0xFFFFFFFFFFFFFFFF
FUSED, GENERIC = "k_hash_fused(", "k_hash_generic("
SPARSE, DENSE = "k_match_pick_sparse<", "k_match_pick("


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _pack(prompts, first=0):
    """Tightly packed rows starting at byte `first` -> (data, offsets)."""
    offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in prompts], out=offs[1:])
    offs += np.uint64(first)
    data = np.frombuffer(b"\0" * first + b"".join(prompts) + b"\0" * 16, dtype=np.uint8).copy()
    return data, offs


def _rows(prompts, mod32, pad=0, rng=None):
    """Rows starting at `mod32` (0 or 16) modulo 32, `lengths` shorter than the rows by up to `pad` extra 32-byte units
    -> (starts, end, lengths)."""
    starts, pos = [], mod32
    for p in prompts:
        starts.append(pos)
        extra = 32 * int(rng.integers(0, pad + 1)) if pad else 0
        pos += max(32, (len(p) + 31) // 32 * 32) + extra
    return starts, pos, np.array([len(p) for p in prompts], dtype=np.uint64)


def _aligned(prompts, mod32, pad=0, rng=None):
    """Host layout of _rows -> (data, offsets, lengths)."""
    starts, end, lens = _rows(prompts, mod32, pad, rng)
    data = np.zeros(end + 64, np.uint8)
    for st, p in zip(starts, prompts):
        data[st: st + len(p)] = np.frombuffer(p, np.uint8)
    return data, np.array(starts + [end], dtype=np.uint64), lens


def _to_dev(*arrays):
    import torch
    out = []
    for a in arrays:
        if a is None:
            out.append(None)
        elif a.dtype == np.uint64:
            out.append(torch.from_numpy(a.view(np.int64)).cuda())
        elif a.dtype == np.uint32:
            out.append(torch.from_numpy(a.view(np.int32)).cuda())
        else:
            out.append(torch.from_numpy(a).cuda())
    return out


def _host_hashes(hs, nb):
    if not isinstance(hs, np.ndarray):
        hs, nb = hs.cpu().numpy().view(np.uint64), nb.cpu().numpy()
    return hs, nb


def _assert_hashes(hs, nb, want, where):
    hs, nb = _host_hashes(hs, nb)
    for i, w in enumerate(want):
        assert nb[i] == len(w), (where, i, int(nb[i]), len(w))
        assert [int(x) for x in hs[i, : nb[i]]] == w, (where, i)


def _hash_in_layouts(eng, prompts, model_ids, block_bytes, want, where, profile=True):
    """Hashes one batch as 32-byte-aligned rows, rows at 16 mod 32, a tightly packed blob (odd start: the generic
    kernels) and device pointers; each result against `want`, each launch against the kernel its layout selects."""
    rng = np.random.default_rng(len(prompts))
    vector = block_bytes % 32 == 0
    layouts = []
    for mod in (0, 16):
        d, o, ln = _aligned(prompts, mod, 2, rng)
        layouts.append((f"rows at {mod} mod 32", (d, o, ln), vector))
    d, o = _pack(prompts, first=1)
    layouts.append(("packed", (d, o, None), False))
    d, o, ln = _aligned(prompts, 16, 1, rng)
    layouts.append(("device", tuple(_to_dev(d, o, ln)), vector))
    mids = model_ids if model_ids is None else np.asarray(model_ids, np.uint32)
    for name, (d, o, ln), fused in layouts:
        m = mids
        if name == "device" and mids is not None:
            (m,) = _to_dev(mids)
        call = lambda: eng.hash_prompts(d, offsets=o, lengths=ln, model_ids=m)
        if profile:
            (hs, nb), names = kernels_launched(call)
            if fused:
                assert_ran(names, FUSED, (GENERIC,), where=f"{where} {name}")
            else:
                assert_ran(names, GENERIC, (FUSED,), where=f"{where} {name}")
        else:
            hs, nb = call()
        _assert_hashes(hs, nb, want, f"{where} {name}")


# ------------------------------------------------------------------------------------------------
# 1. hash layout matrix: k_hash_fused / k_hash_generic
# ------------------------------------------------------------------------------------------------
def test_golden_vectors_as_batches(epp):
    """Every prompt vector of tests/golden/xxh64_vectors.json (python-xxhash), hashed as one batch per
    (block size, prefix cap) with per-request models, in every layout."""
    with open(GOLD) as f:
        gold = json.load(f)
    groups = defaultdict(list)
    for v in gold["prompts"]:
        groups[v["block_size_tokens"], v["max_blocks"]].append(v)
    for (bst, maxb), vs in sorted(groups.items()):
        with epp.Engine(8, block_size_tokens=bst, max_prefix_blocks=maxb) as eng:
            mids = {}
            for v in vs:
                key = (v["model"].encode(), v["salt"].encode())
                if key not in mids:
                    mids[key] = eng.register_model(*key)
            model_ids = [mids[v["model"].encode(), v["salt"].encode()] for v in vs]
            prompts = [bytes.fromhex(v["data_hex"]) for v in vs]
            want = [[int(h, 16) for h in v["hashes"]] for v in vs]
            _hash_in_layouts(eng, prompts, model_ids, 4 * bst, want, f"golden bst={bst} max_blocks={maxb}")


def _ragged_prompts(rng, R, bb, maxb):
    """Shorter than a block, exact full blocks, a trailing partial block and truncated at the cap, with full-block counts
    on both sides of the fused kernel's window (8), ring-stage (16) and ring-wrap (64) boundaries."""
    counts = sorted({c for c in (1, 7, 8, 9, 15, 16, 17, 63, 64, 65, maxb - 1, maxb) if 1 <= c <= maxb})
    out = []
    for i in range(R):
        kind = int(rng.integers(0, 4)) if R == 1 else i % 4
        nf = int(counts[int(rng.integers(0, len(counts)))])
        if kind == 0:
            n = int(rng.integers(0, bb))
        elif kind == 1:
            n = nf * bb
        elif kind == 2:
            n = nf * bb + int(rng.integers(1, bb))
        else:
            n = maxb * bb + int(rng.integers(1, 3 * bb))
        out.append(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
    return out


@pytest.mark.parametrize("maxb", [1, 7, 63, 64, 65, 129])
@pytest.mark.parametrize("bst", [8, 16, 24, 64, 256])
def test_ragged_batches_every_layout_vs_oracle(epp, orc, bst, maxb):
    """Random ragged batches, 1 to 32 stripes per block, odd and even prefix caps (the odd ones take the scalar-store
    branch of the chain warp), R = 1, 31, 32, 33, 97 (a partial last tile), two models."""
    rng = np.random.default_rng(bst * 1000 + maxb)
    bb = 4 * bst
    with epp.Engine(8, block_size_tokens=bst, max_prefix_blocks=maxb) as eng:
        models = [b"mdl", b"other-model"]
        for m in models:
            eng.register_model(m)
        for R in (1, 31, 32, 33, 97):
            prompts = _ragged_prompts(rng, R, bb, maxb)
            mids = rng.integers(0, 2, R).astype(np.uint32)
            want = [orc.hash_prompt(p, models[m], bst, maxb) for p, m in zip(prompts, mids)]
            _hash_in_layouts(eng, prompts, mids, bb, want, f"bst={bst} max_blocks={maxb} R={R}", profile=R in (1, 97))


# ------------------------------------------------------------------------------------------------
# shared workload pieces: prompt families, an index over their prefixes, a P/D + encode pool
# ------------------------------------------------------------------------------------------------
def _families(rng, n, nbytes):
    return [rng.integers(0, 256, nbytes, dtype=np.uint8).tobytes() for _ in range(n)]


def _family_pairs(orc, rng, fam, model, bst, maxb, E, holders):
    hs, es = [], []
    for g, p in enumerate(fam):
        h = orc.hash_prompt(p, model, bst, maxb)
        for e in rng.choice(E, size=holders[g], replace=False):
            depth = int(rng.integers(1, len(h) + 1))
            hs += h[:depth]
            es += [int(e)] * depth
    return hs, es


def _prompt_of_len(rng, fam, n):
    """n bytes: a prefix of a random family (or nothing) + random bytes."""
    g = int(rng.integers(0, len(fam) + 1))
    keep = 0 if g == len(fam) else min(n, len(fam[g]), int(rng.integers(0, len(fam[g]) + 1)))
    head = fam[g][:keep] if keep else b""
    return head + rng.integers(0, 256, n - keep, dtype=np.uint8).tobytes()


PRIM, PREF, ENC = [(2, 1.0, 0), (1, 1.0, 0), (0, 2.0, 0)], [(2, 1.0, 0), (0, 1.0, 0)], [(1, 1.0, 0)]


def _spec(epp, filt, scorers):
    return epp.ProfileSpec(filt, [epp.ScorerSpec(k, w, p) for k, w, p in scorers])


# ------------------------------------------------------------------------------------------------
# 2. k_hash_fused: rows at 16 mod 32, one odd-length request per batch
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [1, 1634, 3244])
def test_fused_hash_rows_at_16_vs_oracle(epp, orc, seed):
    """64-byte blocks, rows at 16 mod 32 with `lengths` shorter than the rows: one short request among long ones and one
    long request among short ones, R not a multiple of 16 or 32.  Hashes and decisions against the oracle."""
    import torch
    import helpers
    E, bst, maxb = 48, 16, 77
    bb = 4 * bst
    rng = np.random.default_rng(seed)
    fam = _families(rng, 4, bb * (maxb + 2))
    hs_pairs, es_pairs = _family_pairs(orc, rng, fam, b"m", bst, maxb, E, [2, 5, 9, 40])
    kv = rng.integers(0, 3, E) / 3.0
    waiting = rng.integers(0, 3, E).astype(np.int32)
    ix = orc.Indexer()
    ix.load_pairs(hs_pairs, es_pairs)
    pool = orc.PoolState(np.zeros(E, np.uint8), kv, waiting)
    long_n = lambda: int(rng.integers(40 * bb, (maxb + 2) * bb))
    short_n = lambda: int(rng.integers(0, 3 * bb))
    batches = []
    for R, odd_one, odd_len, usual_len in ((45, 20, short_n, long_n), (77, 50, long_n, short_n), (100, 99, short_n, long_n)):
        batches.append([_prompt_of_len(rng, fam, odd_len() if r == odd_one else usual_len()) for r in range(R)])

    with epp.Engine(E, _spec(epp, 0, PRIM), block_size_tokens=bst, max_prefix_blocks=maxb) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E), np.zeros(E, np.uint8), kv, waiting)
        eng.index_load_snapshot(hs_pairs, es_pairs)
        for bi, prompts in enumerate(batches):
            where = f"seed {seed} batch {bi}"
            d, o, ln = _aligned(prompts, 16, 3, rng=np.random.default_rng(bi))
            (hs, nb), names = kernels_launched(lambda: eng.hash_prompts(d, offsets=o, lengths=ln))
            assert_ran(names, FUSED, (GENERIC,), where=where)
            _assert_hashes(hs, nb, [orc.hash_prompt(p, b"m", bst, maxb) for p in prompts], where)
            dd, do, dl = _to_dev(d, o, ln)
            (ddec, ddet), names = kernels_launched(lambda: eng.schedule(dd, offsets=do, lengths=dl))
            assert_ran(names, FUSED, (GENERIC,), where=f"{where} schedule")
            torch.cuda.synchronize()
            dec = epp.decisions_from_torch(ddec)
            det = ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
            pd, po = _pack(prompts)
            odec, ototal = orc.cycle_batch(b"m", bst, maxb, 0, False, ix, orc.make_profile(0, PRIM), None, pool, pd, po, 4)
            helpers.assert_decisions_equal(dec, det, odec, ototal, where=where)
            assert (dec["match_blocks"] > 0).any()


# ------------------------------------------------------------------------------------------------
# 3. k_cycle_small: prompts staged by one bulk copy, or read by the digest threads themselves
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("bst,B,staged", [(16, 2274, True), (16, 2275, False), (256, 200, False)])
def test_cycle_small_staging_boundary_vs_oracle(epp, orc, monkeypatch, bst, B, staged, tie_seed):
    """2274 blocks of 64 bytes are the last prompt size the single-launch kernel stages into shared memory (exactly
    160 KiB with the stripe states), 2275 the first one it does not; 200 blocks of 1 KiB do not fit either.  Zero-copy
    (3 requests) and DMA (20) batches, rows at 0 and 16 mod 32, EPP_SMALL_PIPELINE on and off, P/D + encode stages, both
    tie rules: equal to the oracle and to the chunked path (EPP_SMALL_BATCH=0)."""
    import helpers
    E = 48
    bb = 4 * bst
    cap = bb * B
    rng = np.random.default_rng(B + tie_seed)
    kv = rng.integers(0, 3, E) / 3.0
    waiting = rng.integers(0, 3, E).astype(np.int32)
    role = rng.choice([1, 2, 3, 5, 7, 0], size=E).astype(np.uint8)
    fam = _families(rng, 4, cap + bb)
    hs_pairs, es_pairs = _family_pairs(orc, rng, fam, b"m", bst, B, E, [2, 6, 12, 40])   # the last overflows the sparse map
    # prompts whose cached prefix ends in a partial block: its hash (the kernel's last, from the parked tail bytes) matches
    tails = [fam[g][: int(rng.integers(1, B)) * bb + int(rng.integers(1, bb))] for g in (0, 1)]
    for p in tails:
        h = orc.hash_prompt(p, b"m", bst, B)
        for e in rng.choice(E, size=3, replace=False):
            hs_pairs += h
            es_pairs += [int(e)] * len(h)
    ix = orc.Indexer()
    ix.load_pairs(hs_pairs, es_pairs)
    pool = orc.PoolState(role, kv, waiting)

    def length():
        kind = int(rng.integers(0, 4))
        if kind == 0:
            return int(rng.integers(0, bb))                          # no hash at all
        if kind == 1:
            return cap + int(rng.integers(1, bb))                     # truncated at the cap
        return int(rng.integers(1, B)) * bb + (int(rng.integers(1, bb)) if kind == 2 else 0)   # partial trailing block

    batches = []
    for mod in (0, 16):
        for n in (3, 20):
            prompts = [tails[len(batches) % 2]] + [_prompt_of_len(rng, fam, length()) for _ in range(n - 1)]
            batches.append((mod, prompts, (rng.random(n) < 0.5).astype(np.uint8)))
    small_kernel = f"k_cycle_small<{'true' if staged else 'false'}>"
    other_kernel = f"k_cycle_small<{'false' if staged else 'true'}>"
    results = {}
    for small, pipe in (("1024", "1"), ("1024", "0"), ("0", "1")):
        monkeypatch.setenv("EPP_SMALL_BATCH", small)
        monkeypatch.setenv("EPP_SMALL_PIPELINE", pipe)
        with epp.Engine(E, _spec(epp, 1, PRIM), _spec(epp, 2, PREF), block_size_tokens=bst, max_prefix_blocks=B,
                        non_cached_tokens=8, encode=_spec(epp, 3, ENC), tie_seed=tie_seed) as eng:
            eng.register_model(b"m")
            eng.pool_set(np.arange(E), role, kv, waiting)
            eng.index_load_snapshot(hs_pairs, es_pairs)
            got = []
            for mod, prompts, mm in batches:
                n = len(prompts)
                starts, end, lens = _rows(prompts, mod)
                buf = epp.PinnedBuffer(end + 64)
                for st, p in zip(starts, prompts):
                    buf.array[st: st + len(p)] = np.frombuffer(p, np.uint8)
                offs = np.array(starts + [end], dtype=np.uint64)
                base = eng.stats()["n_decisions"]
                call = lambda: eng.schedule(buf.array, offsets=offs, lengths=lens, multimodal=mm, n_requests=n)
                where = f"small={small} pipeline={pipe} rows at {mod} mod 32 n={n}"
                if pipe == "0" or small == "0" or not staged:    # (the profiler stays out of the copy / kernel overlap)
                    (dec, det), names = kernels_launched(call)
                    if small == "0":
                        assert_ran(names, FUSED, ("k_cycle_small",), where=where)
                    else:
                        assert_ran(names, small_kernel, (other_kernel, FUSED), where=where)
                else:
                    dec, det = call()
                if small != "0":
                    assert eng.stats()["last_kernel_launches"] in (1, 2), where
                pd, po = _pack(prompts)
                odec, ototal = orc.cycle_batch(b"m", bst, B, 8, False, ix, orc.make_profile(1, PRIM), orc.make_profile(2, PREF),
                                               pool, pd, po, 4, tie_seed=tie_seed, tie_base=base,
                                               encode=orc.make_profile(3, ENC), multimodal=mm)
                helpers.assert_decisions_equal(dec, det, odec, ototal, where=where)
                got.append((base, dec.copy(), det.copy()))
                buf.close()
            results[small, pipe] = got
    for other in (("1024", "0"), ("0", "1")):
        for (ba, a, ad), (bb_, b, bd) in zip(results["1024", "1"], results[other]):
            if ba == bb_:                                # (the random tie rule depends on the decision ordinal)
                np.testing.assert_array_equal(a, b)
                np.testing.assert_array_equal(ad, bd)
    assert any((d["match_blocks"] > 0).any() for _, d, _ in results["1024", "1"])


# ------------------------------------------------------------------------------------------------
# 4. adversarial read tables: long chains, wrap past the last slot, long misses, mid-chain tombstones
# ------------------------------------------------------------------------------------------------
K_FILL = 33                     # same-home keys per targeted hash: every such chain is longer than one 32-lane step
D_INITIAL = 9000                # distinct hashes of the first build (padded up to this): fixes the table size per load


def _fillers(h, k0=1):
    """Keys sharing h's home slot under any mask below 2^40."""
    return [(int(h) ^ (k << 40)) & ALL1 for k in range(k0, k0 + K_FILL)]


@pytest.mark.parametrize("patch", ["0", "1"])
def test_adversarial_read_tables_vs_oracle(epp, orc, monkeypatch, patch):
    """Index contents random keys never produce, under EPP_INDEX_LOAD 2 and 4: more than 32 keys sharing the home slot
    of every cached block (held by other endpoints), absent blocks whose chain is full of same-home keys, runs that wrap
    from the last slot to slot 0 with held and absent prompt blocks homed inside them, and -- through indexer.Add, LRU
    eviction and a commit -- tombstones (hashes whose last endpoint left) in the middle of chains whose later keys are
    still held.  Checked through the sparse kernel (schedule), the dense-counter kernel (prefix_match, and requests with
    more than 32 holders) and the single-launch kernel's follow mode (small pinned batches)."""
    import helpers
    E, bst, B = 40, 8, 40
    bb = 4 * bst
    X, Y = E - 1, E - 2                 # X: small LRU, evicts in the second phase; Y: holds the blocks added then
    monkeypatch.setenv("EPP_INDEX_PATCH", patch)
    monkeypatch.setenv("EPP_SMALL_PIPELINE", "0")    # the profiler stays out of the copy / kernel overlap
    slots_by_load = {}
    for load in (2, 4):
        monkeypatch.setenv("EPP_INDEX_LOAD", str(load))
        rng = np.random.default_rng(700 + load)
        H = lambda p: orc.hash_prompt(p, b"m", bst, B)
        rand = lambda n: rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        with epp.Engine(E) as probe:                                 # the table size this many distinct hashes get
            probe.index_load_snapshot(rng.integers(1, 2**62, D_INITIAL, dtype=np.int64).astype(np.uint64), np.zeros(D_INITIAL, np.uint32))
            slots = int(probe.stats()["index_slots"])
        mask = slots - 1
        adds = []                                                    # (endpoint, hashes, lru capacity) in call order

        # families: cached prefixes, the last one held by more than 32 endpoints (overflow -> dense-counter pass)
        fam = _families(rng, 5, B * bb)
        fam_h = [H(p) for p in fam]
        for g, h in enumerate(fam_h):
            for e in rng.choice(E - 2, size=[3, 8, 20, 36, 5][g], replace=False):
                adds.append((int(e), h[: int(rng.integers(1, B + 1))], 0))
        # long chains: K_FILL same-home keys for every family block, held by other endpoints
        for h in {x for hh in fam_h for x in hh}:
            for k, f in enumerate(_fillers(h)):
                adds.append((k % (E - 2), [f], 0))
        # queries: family prefixes with random tails (and partial trailing blocks), cold prompts
        queries = [p for p in fam]
        for _ in range(30):
            g = int(rng.integers(0, len(fam)))
            keep = int(rng.integers(1, B)) * bb
            queries.append(fam[g][:keep] + rand(int(rng.integers(1, 4)) * bb + int(rng.integers(0, bb))))
        queries += [rand(int(rng.integers(1, B + 1)) * bb) for _ in range(5)]
        # tombstones: X holds 3 same-home keys of every block of T and the first blocks of P2 -- its whole LRU
        T, P2 = rand(10 * bb + 5), rand(18 * bb)
        g_h, p2_h = H(T), H(P2)
        x_initial = [f for h in g_h[:10] for f in _fillers(h)[:3]] + p2_h
        adds.append((X, x_initial, len(x_initial)))
        queries += [T, P2]
        held = {x for _, hs, _ in adds for x in hs}
        # long misses: the first absent block of every query heads a chain full of same-home keys
        for p in queries:
            h = H(p)
            miss = next((x for x in h if x not in held and x not in g_h), None)
            if miss is not None:
                for k, f in enumerate(_fillers(miss, k0=100)):
                    adds.append((k % (E - 2), [f], 0))
        # wrap: a run of same-home keys from the last slots into slot 0 .., and prompts whose first block is homed inside it
        wrap_fill = []
        for s in range(mask - 7, mask + 1):
            n = K_FILL if s == mask else 3
            wrap_fill += [(int(rng.integers(1, 2**20)) << 40) | s for _ in range(n)]
        for k, f in enumerate(wrap_fill):
            adds.append((k % (E - 2), [f], 0))
        window = set(range(mask - 7, mask + 1)) | set(range(0, 8))
        wrap_prompts = []
        while len(wrap_prompts) < 10:
            b0 = rand(bb)
            if H(b0)[0] & mask in window:
                wrap_prompts.append(b0 + rand(int(rng.integers(1, 3)) * bb + int(rng.integers(0, bb))))
        for i, p in enumerate(wrap_prompts):
            if i < 6:                                                # held; the other four are absent
                adds.append((int(rng.integers(0, E - 2)), H(p)[:2], 0))
        queries += wrap_prompts
        # pad to D_INITIAL distinct hashes
        held = {x for _, hs, _ in adds for x in hs}
        assert len(held) <= D_INITIAL
        pad = rng.integers(1, 2**62, D_INITIAL - len(held) + 64, dtype=np.int64).astype(np.uint64)
        pad = [int(x) for x in pad if int(x) not in held][: D_INITIAL - len(held)]
        adds.append((0, pad, 0))

        prof_spec = _spec(epp, 0, [(0, 3.0, 0), (2, 2.0, 0), (1, 2.0, 0)])
        prof = orc.make_profile(0, [(0, 3.0, 0), (2, 2.0, 0), (1, 2.0, 0)])
        kv = rng.integers(0, 4, E) / 4.0
        waiting = rng.integers(0, 3, E).astype(np.int32)
        pool = orc.PoolState(np.zeros(E, np.uint8), kv, waiting)
        ix = orc.Indexer()
        with epp.Engine(E, prof_spec, block_size_tokens=bst, max_prefix_blocks=B) as eng:
            eng.register_model(b"m")
            eng.pool_set(np.arange(E), np.zeros(E, np.uint8), kv, waiting)
            for e, hs, c in adds:
                eng.index_add(e, hs, c)
                ix.add(hs, e, c)
            eng.index_commit()
            st = eng.stats()
            assert st["index_slots"] == slots and st["index_hashes"] == D_INITIAL, (load, st["index_slots"], st["index_hashes"])
            slots_by_load[load] = slots

            def check(phase):
                where = f"load={load} patch={patch} {phase}"
                d, o = _pack(queries)
                odec, ototal = orc.cycle_batch(b"m", bst, B, 0, False, ix, prof, None, pool, d, o, 4)
                # sparse kernel (+ the dense-counter pass for the requests with > 32 holders)
                dd, do = _to_dev(d, o)
                (ddec, ddet), names = kernels_launched(lambda: eng.schedule(dd, offsets=do))
                assert_ran(names, SPARSE, where=where)
                assert_ran(names, DENSE, where=where)
                sdec = epp.decisions_from_torch(ddec)
                helpers.assert_decisions_equal(sdec, ddet.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1), odec, ototal,
                                               where=where + " schedule")
                # dense-counter kernel: Produce rows
                (match, total), names = kernels_launched(lambda: eng.prefix_match(d, offsets=o))
                assert_ran(names, DENSE, (SPARSE,), where=where)
                for r, p in enumerate(queries):
                    h = H(p)
                    want, _ = ix.match_longest_prefix(h, E)
                    np.testing.assert_array_equal(match[r], want, err_msg=f"{where} prefix_match row {r}")
                    assert total[r] == len(h)
                # single-launch kernel, follow mode: small pinned batches (zero-copy and DMA)
                for sel in (np.arange(6), np.arange(len(queries) - 20, len(queries))):
                    sub = [queries[i] for i in sel]
                    starts, end, lens = _rows(sub, 0)
                    buf = epp.PinnedBuffer(end + 64)
                    for s0, p in zip(starts, sub):
                        buf.array[s0: s0 + len(p)] = np.frombuffer(p, np.uint8)
                    offs = np.array(starts + [end], dtype=np.uint64)
                    (dec, det), names = kernels_launched(lambda: eng.schedule(buf.array, offsets=offs, lengths=lens, n_requests=len(sub)))
                    assert_ran(names, "k_cycle_small<", where=where)
                    helpers.assert_decisions_equal(dec, det, odec[sel], ototal[sel], where=where + " small batch")
                    buf.close()
                assert (sdec["match_blocks"] > 0).sum() > 20

            check("first build")
            # second phase: Y adds T's blocks (their slots are claimed behind the same-home keys), X adds 40 new hashes and
            # evicts its 30 same-home keys and the first 10 blocks of P2 -> hashes nobody holds any more
            eng.index_add(Y, g_h)
            ix.add(g_h, Y)
            new = [int(x) for x in rng.integers(1, 2**62, 40, dtype=np.int64)]
            eng.index_add(X, new)
            ix.add(new, X)
            eng.index_commit()
            st = eng.stats()
            assert st["last_index_patched"] == (1 if patch == "1" else 0), st["last_index_patched"]
            assert st["index_slots"] == slots
            assert eng.index_get(int(p2_h[0])) == set() and eng.index_get(int(g_h[0])) == {Y}
            check("after evictions")
    assert slots_by_load[2] != slots_by_load[4]


# ------------------------------------------------------------------------------------------------
# 5. every non-sharded instantiation of k_match_pick_sparse
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("stages", [1, 2, 3])
def test_match_kernel_instantiations_vs_oracle(epp, orc, stages, tie_seed):
    """1 / 2 / 3 handler stages x lowest-slot / random tie rule, with requests whose holders overflow the sparse map:
    decisions equal to the oracle's, through the instantiation launch_match_pick_sparse picks."""
    import helpers
    E, bst, B = 96, 2, 16
    rng = np.random.default_rng(stages * 10 + (tie_seed != 0))
    kv = rng.integers(0, 2, E) / 2.0
    waiting = rng.integers(0, 2, E).astype(np.int32)
    role = rng.choice([1, 2, 3, 5, 7, 0], size=E).astype(np.uint8) if stages > 1 else np.zeros(E, np.uint8)
    fam = _families(rng, 6, 8 * B)
    hs_pairs, es_pairs = _family_pairs(orc, rng, fam, b"m", bst, B, E, [2, 5, 9, 20, 40, 70])
    ix = orc.Indexer()
    ix.load_pairs(hs_pairs, es_pairs)
    pool = orc.PoolState(role, kv, waiting)
    prompts = [_prompt_of_len(rng, fam, 8 * B) for _ in range(300)]
    d, o = _pack(prompts)
    mm = (rng.random(300) < 0.5).astype(np.uint8) if stages == 3 else None
    prim = PRIM
    kw = dict(block_size_tokens=bst, max_prefix_blocks=B, tie_seed=tie_seed)
    if stages == 1:
        specs, oprofs = (_spec(epp, 0, prim),), (orc.make_profile(0, prim), None)
    else:
        specs, oprofs = (_spec(epp, 1, prim), _spec(epp, 2, PREF)), (orc.make_profile(1, prim), orc.make_profile(2, PREF))
        kw["non_cached_tokens"] = 4
    if stages == 3:
        kw["encode"] = _spec(epp, 3, ENC)
    mincta = 8 if stages == 1 and not tie_seed else 6
    kernel = f"k_match_pick_sparse<{mincta}, false, {'true' if tie_seed else 'false'}, {stages}>"
    with epp.Engine(E, *specs, **kw) as eng:
        eng.register_model(b"m")
        eng.pool_set(np.arange(E), role, kv, waiting)
        eng.index_load_snapshot(hs_pairs, es_pairs)
        (dec, det), names = kernels_launched(lambda: eng.schedule(d, offsets=o, multimodal=mm))
        assert_ran(names, kernel, where=kernel)
        assert_ran(names, DENSE, where=kernel)                     # the overflowing requests
    enc = orc.make_profile(3, ENC) if stages == 3 else None
    odec, ototal = orc.cycle_batch(b"m", bst, B, kw.get("non_cached_tokens", 0), False, ix, oprofs[0], oprofs[1], pool, d, o,
                                   4, tie_seed=tie_seed, tie_base=0, encode=enc, multimodal=mm)
    helpers.assert_decisions_equal(dec, det, odec, ototal, where=kernel)
    assert (dec["match_blocks"] > 0).sum() > 50 and (dec["tie_count"] > 1).any()
