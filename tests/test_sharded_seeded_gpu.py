"""Seeded ties in the endpoint-sharded mode (include/epp_engine.h, "Seeded ties"; DESIGN §7) on one GPU, against the CPU
oracle run unsharded on the whole pool with the same tie_seed and ordinal, bit for bit: status, pick, score bits, tie
count, match_blocks, total_blocks, and for the disagg handler the prefill and encode stages and prefill_ran.

Every rank is its own engine on the one GPU (epp_shard_set_seeded, the full pool, the rank's own postings), driven
through the host exchanges (probe -> OR -> pick -> stack of the records -> select on every rank -> stack of the entries
-> finish on every rank), the peer-memory exchange stepped through phases 0..3, or one rank's own
epp_shard_schedule_p2p.  Every rank's decisions must agree.  The cases:
  A  tie groups spanning 2-5 shards with the ranges in descending slot order; ragged, empty and one-slot shards
  B  cold requests on a pool that ties whole; matched candidates inside the equal-base group (prefix weight 0); +inf on
     several shards and -inf on every candidate; more than 32 in-shard holders of one tie group (the dense select)
  C  lora-affinity adapters; consecutive batches (the ordinal advances by R)
  D  P/D: the seeded decode member's match_blocks flips the decider against the lowest slot's; a prefill owner without
     a decode candidate; seeded encode picks
  E  the peer-memory exchange stepped over 2-4 ranks, and one rank's own exchange at R >= 8192 (the split halves)
  F  the refusals, and the spread: a tie group across the shards gets picks on every shard
Every protocol call proves from its profiler trace that its kernels ran.  test_sharded_seeded_cpu.py checks from the
builders and the oracle alone that each case reaches the edge it names.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import test_sharded_disagg_gpu as D
import test_sharded_landscapes_gpu as L

pytestmark = pytest.mark.gpu

SEED = 0x5EED
NO = 0xFFFFFFFF
BST, BB = L.BST, L.BB
(PREFIX, KV, QUEUE) = (0, 1, 2)
PROBE, RESOLVE, SSEL, DSEL, FINISH, MERGE = (L.PROBE, "k_shard_resolve", "k_match_pick_sparse_select", "k_match_pick_select",
                                             "k_shard_finish", L.MERGE)


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


# ------------------------------------------------------------------------------------------------
# scenes (no GPU needed)
# ------------------------------------------------------------------------------------------------
def scene_cold(world, seed=0):
    """Every candidate has the same base and no prompt matches: every request ties the whole pool."""
    rng = np.random.default_rng(L.seed_of("seeded-cold", world, seed))
    E, B = 70, 8
    S = L.Scene(E, B, np.zeros(E, np.uint8), np.zeros(E), np.zeros(E, np.int32),
                (D.F_NONE, [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 2.0, 0.0)]))
    S.prompts = [L.tail(rng, BB * int(rng.integers(1, B + 1)) + int(rng.integers(0, BB))) for _ in range(64)]
    return S


def scene_dense(seed=0):
    """40 slots of the first of two shards and 6 of the second hold family 0 in full at the same base: a 46-way tie whose
    members on the first shard overflow its lane map (the dense select)."""
    rng = np.random.default_rng(L.seed_of("seeded-dense", seed))
    E, B = 96, 10
    cut = L.sharded().shard_range(0, 2, E)[1]
    kv = rng.choice([0.25, 0.5], E)
    waiting = rng.integers(1, 3, E).astype(np.int32)
    group = list(rng.choice(cut, 40, replace=False)) + list(cut + rng.choice(E - cut, 6, replace=False))
    kv[group], waiting[group] = 0.0, 0
    S = L.Scene(E, B, np.zeros(E, np.uint8), kv, waiting, (D.F_NONE, [(KV, 1.0, 0.0), (QUEUE, 1.0, 0.0), (PREFIX, 2.0, 0.0)]))
    fams = [L.fam_bytes(rng, B) for _ in range(2)]
    for e in group:
        S.hold(fams[0], e, range(B))
    for e in rng.choice(E, 5, replace=False):
        S.hold(fams[1], e, range(int(rng.integers(1, B + 1))))
    S.prompts = [fams[0] + L.tail(rng, int(rng.integers(0, BB))) for _ in range(40)] + \
        L.family_prompts(rng, fams, 24, B, cold_share=0.2)
    S.group = sorted(int(e) for e in group)
    return S


def scene_pd_flip(seed=0):
    """Decode slots [0, 24) at one base with the prefix weighted 0, holding family f to random depths: the tied decode
    members differ in match_blocks, so the P/D decider (non_cached_tokens 5) depends on which member the tie rule takes.
    Prefill slots [24, 48) tie in groups too."""
    rng = np.random.default_rng(L.seed_of("seeded-pd-flip", seed))
    E, B = 48, 8
    role = np.where(np.arange(E) < 24, D.R_DECODE, D.R_PREFILL)
    kv = np.where(np.arange(E) < 24, 0.0, rng.choice([0.0, 0.5], E))
    waiting = np.where(np.arange(E) < 24, 0, rng.integers(0, 2, E)).astype(np.int32)
    S = D.PDScene(E, B, role, kv, waiting, (D.F_DECODE, [(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0), (PREFIX, 0.0, 0.0)]), nct=5)
    fams = [L.fam_bytes(rng, B) for _ in range(2)]
    for f in fams:
        for e in rng.choice(24, 10, replace=False):
            S.hold(f, e, range(int(rng.integers(1, B + 1))))
        for e in 24 + rng.choice(24, 6, replace=False):
            S.hold(f, e, range(int(rng.integers(1, B + 1))))
    S.prompts = []
    for r in range(96):
        d = int(rng.integers(1, B + 1))
        S.prompts.append(fams[r % 2][: d * BB] + L.tail(rng, 4 * int(rng.integers(0, 8))))
    return S


# ------------------------------------------------------------------------------------------------
# oracle side
# ------------------------------------------------------------------------------------------------
def expected(orc, S, prompts, base, tie_seed=SEED):
    """orc.cycle_batch on the whole pool and index with tie_seed, request r at ordinal base + r (runs of one adapter
    each take their own call, starting at their own ordinal)."""
    from oracle import pyoracle
    ix = S.oracle_index(orc)
    R = len(prompts)
    out = np.zeros(R, pyoracle.DECISION_DTYPE)
    tot = np.zeros(R, np.int32)
    mb = np.zeros(R, np.int64)
    mo = S.adapters(R)
    prof = lambda p: None if p is None else orc.make_profile(p[0], list(p[1]))
    enc, mm = getattr(S, "encode", None), getattr(S, "mm", None)
    bst = getattr(S, "bst", BST)
    r0 = 0
    while r0 < R:
        r1 = r0
        while r1 < R and mo[r1] == mo[r0]:
            r1 += 1
        a = int(mo[r0])
        ps = prompts[r0:r1]
        d, offs = L.PP._pack(ps)
        kw = dict(tie_seed=tie_seed, tie_base=base + r0)
        if enc is not None:
            kw.update(encode=prof(enc), multimodal=None if mm is None else mm[r0:r1])
        od, ot = orc.cycle_batch(S.models[a], bst, S.B, getattr(S, "nct", 0), getattr(S, "always", False), ix, prof(S.prof),
                                 prof(getattr(S, "prefill", None)), S.oracle_pool(orc, a), d, offs, 4, **kw)
        out[r0:r1], tot[r0:r1] = od, ot
        for j in range(r1 - r0):
            if od["status"][j] == 0:
                m, _ = ix.match_longest_prefix(orc.hash_prompt(ps[j], S.models[a], bst, S.B), S.E)
                mb[r0 + j] = m[od["pick"][j]]
        r0 = r1
    return out, tot, mb


def stages_of(S):
    return S.stages if isinstance(S, D.PDScene) else 1


# ------------------------------------------------------------------------------------------------
# engine side
# ------------------------------------------------------------------------------------------------
def seeded_engine(epp, S, lo, hi, tie_seed=SEED):
    pd = isinstance(S, D.PDScene)
    eng = epp.Engine(S.E, D.spec(epp, S.prof), D.spec(epp, S.prefill) if pd else None,
                     encode=D.spec(epp, S.encode) if pd else None, block_size_tokens=BST, max_prefix_blocks=S.B,
                     non_cached_tokens=S.nct if pd else 0, always_disagg=S.always if pd else False, n_ext_cols=S.n_ext(),
                     tie_seed=tie_seed)
    for m in S.models:
        eng.register_model(m)
    assert eng.shard_set_seeded(lo, hi) == stages_of(S)
    eng.pool_set(*S.pool_arrays())
    if S.lora is not None:
        mx, loaded, state = S.lora
        eng.pool_set_lora(np.arange(S.E), mx, loaded,
                          [(e, a, int(state[a, e])) for a in range(len(S.models)) for e in range(S.E) if state[a, e]])
    hs, es = np.array(S.hs, np.uint64), np.array(S.es, np.uint32)
    k = (es >= lo) & (es < hi)
    if k.any():
        eng.index_load_snapshot(hs[k], es[k])
    return eng


def batch(S, prompts, layout, where):
    rng = np.random.default_rng(L.seed_of("seeded-layout", where))
    if isinstance(S, D.PDScene):
        return D.batch_of(S, prompts, layout, rng)
    ps, buf, offs, lens, T = L.layout_batch(prompts, layout, rng)
    data, kw = L.device_kw(buf, offs, lens, T, None if S.model_of is None else S.adapters(len(ps)))
    return ps, data, kw


def check(epp, decs, dets, exp, where):
    for d, t in zip(decs[1:], dets[1:]):
        np.testing.assert_array_equal(d, decs[0], err_msg=f"{where}: ranks disagree")
        np.testing.assert_array_equal(t, dets[0], err_msg=f"{where}: ranks disagree (detail)")
    D.check(decs[0], dets[0], exp, where)


def run_host(epp, orc, S, ranges, *, batches=1, layout="offsets0", where=""):
    """The host exchanges over one engine per range (stacked in the given order), `batches` consecutive batches of the
    scene's prompts -> (decisions of the last batch, per-batch per-rank records [R, S], per-batch per-rank entries)."""
    import torch
    ps, data, kw = batch(S, S.prompts, layout, where)
    R, St = len(ps), stages_of(S)
    W = (S.B + 31) // 32
    over = (D.dense_ranks if isinstance(S, D.PDScene) else L.overflow_ranks)(orc, S, ps, ranges)
    engines = [seeded_engine(epp, S, lo, hi) for lo, hi in ranges]
    all_recs, all_sels = [], []
    try:
        for k in range(batches):
            at = f"{where} batch {k}"
            masks = []
            for g, eng in enumerate(engines):
                m = torch.zeros((R, W), dtype=torch.int32, device="cuda")
                L.traced(lambda: eng.shard_probe(data, m, **kw), (PROBE,), where=f"{at} probe rank {g}")
                masks.append(m)
            gm = masks[0].clone()
            for m in masks[1:]:
                gm |= m
            torch.cuda.synchronize()
            bests = []
            for g, eng in enumerate(engines):
                b = torch.zeros((R, 24 * St), dtype=torch.uint8, device="cuda")
                L.traced(lambda: eng.shard_pick(R, gm, b), (D.SPARSE_OF[St],), where=f"{at} pick rank {g}")
                bests.append(b)
            allb = torch.stack(bests)
            sels = []
            for g, eng in enumerate(engines):
                s = torch.zeros((R, 8 * St), dtype=torch.uint8, device="cuda")
                L.traced(lambda: eng.shard_select(R, len(engines), allb, s), (RESOLVE, SSEL, DSEL), where=f"{at} select rank {g}")
                sels.append(s)
            alls = torch.stack(sels)
            decs, dets = [], []
            for g, eng in enumerate(engines):
                dec = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
                det = torch.zeros((R, 40), dtype=torch.uint8, device="cuda")
                n0 = eng.stats()["n_decisions"]
                L.traced(lambda: eng.shard_finish(R, len(engines), allb, alls, dec, out_detail=det), (FINISH,),
                         absent=(MERGE,), where=f"{at} finish rank {g}", repeatable=False)
                assert eng.stats()["n_decisions"] == n0 + R, f"{at}: the ordinal advances by R"
                torch.cuda.synchronize()
                decs.append(epp.decisions_from_torch(dec))
                dets.append(det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1))
            check(epp, decs, dets, expected(orc, S, ps, k * R), at)
            all_recs.append([b.cpu().numpy().view(epp.SHARD_BEST_DTYPE).reshape(R, St) for b in bests])
            all_sels.append([s.cpu().numpy().view(L.sharded().SHARD_SEL_DTYPE).reshape(R, St) for s in sels])
    finally:
        for e in engines:
            e.close()
    return decs[0], dets[0], all_recs, all_sels, over


def p2p_engines(epp, S, ranges, R_max):
    engines, ptrs = [], []
    for lo, hi in ranges:
        eng = seeded_engine(epp, S, lo, hi)
        _, ptr = eng.shard_p2p_export(R_max)
        engines.append(eng)
        ptrs.append(ptr)
    for g, eng in enumerate(engines):
        eng.shard_p2p_connect(len(engines), g, np.array(ptrs, dtype=np.uint64), ipc_handles=False)
    return engines


def run_p2p_stepped(epp, orc, S, ranges, *, batches=2, layout="offsets0", where=""):
    """Batches of the scene's prompts (batch k: the first R - 7k of them) through epp_shard_p2p_phase: every rank through
    phase 0, then 1, 2 and 3."""
    import torch
    engines = p2p_engines(epp, S, ranges, len(S.prompts))
    base = 0
    try:
        for k in range(batches):
            at = f"{where} batch {k}"
            ps, data, kw = batch(S, S.prompts[: len(S.prompts) - 7 * k], layout, at)
            R = len(ps)
            outs = [torch.zeros((R, 32), dtype=torch.uint8, device="cuda") for _ in engines]
            dts = [torch.zeros((R, 40), dtype=torch.uint8, device="cuda") for _ in engines]
            torch.cuda.synchronize()

            def phases():
                for phase in range(4):
                    for g, eng in enumerate(engines):
                        eng.shard_p2p_phase(data, outs[g], phase, out_detail=dts[g], **kw)
            L.traced(phases, (PROBE, D.SPARSE_OF[stages_of(S)], RESOLVE, SSEL, DSEL, FINISH) + L.P2P, absent=(MERGE,),
                     where=at, repeatable=False)
            torch.cuda.synchronize()
            check(epp, [epp.decisions_from_torch(o) for o in outs],
                  [d.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1) for d in dts], expected(orc, S, ps, base), at)
            base += R
    finally:
        for e in engines:
            e.close()


def even(world, E):
    return [L.sharded().shard_range(g, world, E) for g in range(world)]


# ------------------------------------------------------------------------------------------------
# A: shard layouts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("kind", ["tie-prefix", "lone"])
def test_A_tie_groups_descending_ranges(epp, orc, kind, world):
    S = L.scene_cross(kind, world)
    dec, _, recs, sels, _ = run_host(epp, orc, S, S.ranges[::-1], where=f"A {kind} x{world}")
    assert (dec["tie_count"] > 1).any()


@pytest.mark.parametrize("layout,world", [("ragged", 3), ("empty", 3), ("single", 5), ("ragged", 5)])
def test_A_ragged_empty_single(epp, orc, layout, world):
    S = L.scene_layout()
    run_host(epp, orc, S, L.layout_ranges(layout, world), where=f"A {layout} x{world}")


# ------------------------------------------------------------------------------------------------
# B: landscapes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
def test_B_cold_whole_pool_ties(epp, orc, world):
    S = scene_cold(world)
    dec, _, _, sels, _ = run_host(epp, orc, S, even(world, S.E), where=f"B cold x{world}")
    assert (dec["tie_count"] == S.E).all()


@pytest.mark.parametrize("kind", ["tie-zero", "inf", "neg-inf"])
def test_B_cross_shard_values(epp, orc, kind):
    S = L.scene_cross(kind, 4)
    run_host(epp, orc, S, S.ranges, layout="odd", where=f"B {kind}")


def test_B_dense_select(epp, orc):
    S = scene_dense()
    ranges = even(2, S.E)
    _, _, _, sels, over = run_host(epp, orc, S, ranges, where="B dense")
    assert over == {0}


# ------------------------------------------------------------------------------------------------
# C: adapters, consecutive batches
# ------------------------------------------------------------------------------------------------
def test_C_lora_adapters(epp, orc):
    S = L.scene_lora()
    run_host(epp, orc, S, even(3, S.E), layout="lengths", where="C lora")


def test_C_lora_adapters_pd(epp, orc):
    S = D.scene_lora()
    run_host(epp, orc, S, even(2, S.E), where="C lora pd")


def test_C_consecutive_batches(epp, orc):
    S = L.scene_cross("tie-prefix", 3)
    run_host(epp, orc, S, S.ranges, batches=3, where="C batches")


# ------------------------------------------------------------------------------------------------
# D: the disagg handler
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
def test_D_decider_flips(epp, orc, world):
    S = scene_pd_flip()
    run_host(epp, orc, S, even(world, S.E)[::-1], where=f"D flip x{world}")


@pytest.mark.parametrize("world", [2, 3])
def test_D_prefill_owner_without_decode(epp, orc, world):
    S = D.scene_roles("split")
    run_host(epp, orc, S, even(world, S.E), where=f"D split x{world}")


@pytest.mark.parametrize("kind", ["all", "some"])
def test_D_encode(epp, orc, kind):
    S = D.scene_encode(kind, 2)
    run_host(epp, orc, S, even(2, S.E), where=f"D encode {kind}")


# ------------------------------------------------------------------------------------------------
# E: the peer-memory exchange
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 4])
def test_E_p2p_stepped(epp, orc, world):
    S = L.scene_cross("tie-prefix", world)
    run_p2p_stepped(epp, orc, S, S.ranges[::-1], where=f"E p2p x{world}")


def test_E_p2p_stepped_pd_encode(epp, orc):
    S = D.scene_encode("all", 3)
    run_p2p_stepped(epp, orc, S, even(3, S.E), where="E p2p encode")


def test_E_p2p_stepped_dense(epp, orc):
    S = scene_dense()
    run_p2p_stepped(epp, orc, S, even(2, S.E), batches=1, where="E p2p dense")


def test_E_p2p_world_one_large_batch(epp, orc):
    """R = 8 257 on one rank's own exchange: the two halves, the second keyed from its own first row."""
    import torch
    S = L.scene_cross("tie-prefix", 2)
    rng = np.random.default_rng(L.seed_of("seeded-large"))
    prompts = [S.prompts[int(i)] for i in rng.integers(0, len(S.prompts), 8257)]
    ps, data, kw = batch(S, prompts, "offsets0", "E large")
    R = len(ps)
    eng = p2p_engines(epp, S, [(0, S.E)], R)[0]
    try:
        out = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
        det = torch.zeros((R, 40), dtype=torch.uint8, device="cuda")
        L.traced(lambda: eng.shard_schedule_p2p(data, out, out_detail=det, **kw), (RESOLVE, SSEL, FINISH), absent=(MERGE,),
                 where="E large", repeatable=False)
        torch.cuda.synchronize()
        assert eng.stats()["n_decisions"] == R
        dec = epp.decisions_from_torch(out)
    finally:
        eng.close()
    D.check(dec, det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1), expected(orc, S, ps, 0), "E large")


# ------------------------------------------------------------------------------------------------
# F: refusals and the spread
# ------------------------------------------------------------------------------------------------
def _code(epp, fn):
    with pytest.raises(epp.EngineError) as ei:
        fn()
    return ei.value.code


def test_F_refusals(epp):
    import torch
    c = epp.capi
    S = L.scene_cross("tie-prefix", 2)
    plain = L.shard_engine(epp, S, 0, 75, tie_seed=SEED)
    unseeded = epp.Engine(S.E, D.spec(epp, S.prof), tie_seed=0)
    topk = epp.Engine(S.E, D.spec(epp, S.prof), tie_seed=SEED, pick_k=2)
    x = torch.zeros(64, dtype=torch.uint8, device="cuda")
    try:
        assert _code(epp, lambda: unseeded.shard_set_seeded(0, 75)) == c.EPP_ERR_INVALID
        assert _code(epp, lambda: topk.shard_set_seeded(0, 75)) == c.EPP_ERR_INVALID
        # a lowest-slot engine has no select / finish and no phase 3
        assert _code(epp, lambda: plain.shard_select(0, 1, x, x)) == c.EPP_ERR_STATE
        assert _code(epp, lambda: plain.shard_finish(0, 1, x, x, x)) == c.EPP_ERR_STATE
        _, ptr = plain.shard_p2p_export(16)
        plain.shard_p2p_connect(1, 0, np.array([ptr], np.uint64), ipc_handles=False)
        assert _code(epp, lambda: plain.shard_p2p_phase(x, x, 3, uniform_len=4)) == c.EPP_ERR_INVALID
        # the buffer was exported for the lowest-slot rule
        assert _code(epp, lambda: plain.shard_set_seeded(0, 75)) == c.EPP_ERR_STATE
    finally:
        for e in (plain, unseeded, topk):
            e.close()
    seeded = seeded_engine(epp, S, 0, 75)
    try:
        assert _code(epp, lambda: seeded.shard_merge(0, 1, x, x)) == c.EPP_ERR_STATE
        seeded.shard_p2p_export(16)
        assert _code(epp, lambda: seeded.shard_set_staged(0, 75)) == c.EPP_ERR_STATE
        assert _code(epp, lambda: seeded.shard_set(0, 75)) == c.EPP_ERR_STATE
    finally:
        seeded.close()
    # a later shard_set_staged returns the engine to the lowest-slot rule: merge is accepted again
    again = seeded_engine(epp, S, 0, 75)
    try:
        assert again.shard_set_staged(0, 75) == 1 and not again.shard_seeded
        again.shard_merge(0, 1, x, x)
    finally:
        again.close()


def test_F_spread(epp, orc):
    """A tie group across four shards: the seeded picks of its requests land on every shard (the lowest-slot rule sends
    them all to the first)."""
    S = L.scene_cross("tie-prefix", 4)
    dec, _, _, _, _ = run_host(epp, orc, S, S.ranges, where="F spread")
    grp = dec["tie_count"] >= 20
    assert grp.sum() >= 20
    shards = {g for g, (lo, hi) in enumerate(S.ranges) for p in dec["pick"][grp] if lo <= p < hi}
    assert shards == set(range(4)), shards
