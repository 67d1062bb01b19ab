"""The disagg profile handler in the endpoint-sharded mode (include/epp_engine.h, "Staged records"; DESIGN §7) on one GPU,
against the CPU oracle run unsharded on the whole pool with the decode, prefill and encode profiles, bit for bit:
status, pick, score bits, tie count, match_blocks, total_blocks, prefill_pick / prefill_ran / prefill score bits and ties,
and the encode fields.

Every rank is its own engine on the one GPU (epp_shard_set_staged, the full pool, the rank's own postings), driven
through the host protocol (probe -> OR of the masks in torch -> pick of S records per request -> stack -> merge with
detail), the peer-memory exchange stepped phase by phase, or one rank's own epp_shard_schedule_p2p_detail.  The cases:
  A  role layouts: decode and prefill interleaved, decode only on the low ranks and prefill only on the high ones, no
     prefill candidate anywhere, no decode candidate anywhere; worlds of 1, 2, 3 and 5; ranges in descending slot order
  B  the P/D decider: prompts whose non-cached tail is exactly non_cached_tokens (prefill runs) or one token less (it
     does not), with the merged decode pick on another rank than the prefill best; always_disagg; non_cached_tokens 0;
     prompts shorter than the threshold; lengths beyond the rows, so that the decider reads the true length
  C  encode: E/P/D with mixed multimodal flags, encode candidates on some ranks or on none
  D  more than 32 in-shard holders (the dense-counter pass), lora-affinity adapters 0 / 1 / 2, config 4 of tools/tracegen
  E  the exchanges: host protocol, peer memory stepped, one rank's own exchange at R = 8 257 (EPP_DEV_CHUNKS 1 and 2)
  F  the contract: a single-profile engine decides the same bytes through shard_set_staged as through shard_set; the
     refusals of shard_set stay; shard_set_staged after an export for another S; out_detail NULL with multimodal requests
Every protocol call proves from its profiler trace that the staged kernels ran.  The builders are plain functions of the
oracle: test_sharded_disagg_cpu.py checks from them alone that each case reaches the edge it names.
Run on an H100: pytest -m gpu."""
import numpy as np
import pytest

import helpers
import test_sharded_landscapes_gpu as L

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
MODEL, BST, BB = L.MODEL, L.BST, L.BB
(PREFIX, KV, QUEUE) = (0, 1, 2)
LORA = 8
F_NONE, F_DECODE, F_PREFILL, F_ENCODE = range(4)
R_DECODE, R_PREFILL, R_BOTH, R_ENCODE, R_EPD = 1, 2, 4, 5, 7
PROBE, MERGE, DENSE = L.PROBE, L.MERGE, L.DENSE
SPARSE_OF = {1: "k_match_pick_sparse<6, true, false, 1>", 2: "k_match_pick_sparse<6, true, false, 2>",
             3: "k_match_pick_sparse<6, true, false, 3>"}
DECODE_SC = [(PREFIX, 2.0, 0.0), (QUEUE, 1.0, 0.0)]
PREFILL_SC = [(PREFIX, 2.0, 0.0), (QUEUE, 1.0, 0.0), (KV, 0.5, 0.0)]
ENCODE_SC = [(QUEUE, 1.0, 0.0), (KV, 1.0, 0.0)]


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
class PDScene(L.Scene):
    """L.Scene with the disagg handler: prefill / encode profiles (None: absent), the P/D decider's settings, the
    multimodal flag of each prompt, and `long` prompts whose rows hold only the bytes the hash reads."""

    def __init__(self, *a, prefill=(F_PREFILL, PREFILL_SC), encode=None, nct=0, always=False, **kw):
        super().__init__(*a, **kw)
        self.prefill, self.encode, self.nct, self.always = prefill, encode, nct, always
        self.mm = None
        self.bst = BST

    @property
    def stages(self):
        return 3 if self.encode is not None else (2 if self.prefill is not None else 1)


def holders(S, rng, fams, slots, per_fam=6):
    for f in fams:
        for e in rng.choice(slots, min(per_fam, len(slots)), replace=False):
            S.hold(f, e, range(int(rng.integers(1, S.B + 1))))


def scene_roles(kind, seed=0, E=60, B=12):
    """interleaved: decode / prefill / both slots alternate; split: decode on the lower half, prefill on the upper;
    no-prefill: decode only; no-decode: prefill and encode only (role 0 counts as decode, so none has it)."""
    rng = np.random.default_rng(L.seed_of("pd-roles", kind, seed))
    role = {"interleaved": np.array([(R_DECODE, R_PREFILL, R_BOTH)[e % 3] for e in range(E)]),
            "split": np.where(np.arange(E) < E // 2, R_DECODE, R_PREFILL),
            "no-prefill": np.full(E, R_DECODE),
            "no-decode": np.array([(R_PREFILL, R_ENCODE)[e % 2] for e in range(E)])}[kind]
    S = PDScene(E, B, role, rng.choice([0.0, 0.25, 0.5], E), rng.integers(0, 4, E), (F_DECODE, DECODE_SC), nct=8)
    fams = [L.fam_bytes(rng, B) for _ in range(4)]
    holders(S, rng, fams, np.arange(E), per_fam=10)
    S.prompts = L.family_prompts(rng, fams, 120, B, cold_share=0.1)
    return S


def scene_decider(kind, seed=0):
    """Decode slots on [0, 20), prefill slots on [20, 40).  Each family is held in full by decode slots (the decode pick's
    match_blocks = the prompt's prefix depth d) and partly by prefill slots.  A prompt is d blocks of a family plus a
    tail of t tokens, so tokens - match_blocks * BST = t:
      boundary  t = nct (prefill runs) or nct - 1 (it does not), nct = 5
      always    always_disagg, the same prompts
      nct0      non_cached_tokens 0: prefill never runs
      short     prompts of fewer than nct tokens, nct = 3 * BST + 1
      long      the boundary prompts with 0-3 blocks of extra bytes behind the hashed cap: the rows carry only the hashed
                bytes, lengths the true length (the decider reads it)"""
    rng = np.random.default_rng(L.seed_of("pd-decider", kind, seed))
    E, B = 40, 8
    role = np.where(np.arange(E) < 20, R_DECODE, R_PREFILL)
    nct = {"boundary": 5, "always": 5, "nct0": 0, "short": 3 * BST + 1, "long": 5}[kind]
    S = PDScene(E, B, role, rng.choice([0.0, 0.5], E), rng.integers(0, 3, E), (F_DECODE, DECODE_SC), nct=nct,
                always=kind == "always")
    fams = [L.fam_bytes(rng, B) for _ in range(3)]
    for f in fams:
        for e in rng.choice(20, 3, replace=False):
            S.hold(f, e, range(B))
        for e in 20 + rng.choice(20, 4, replace=False):
            S.hold(f, e, range(int(rng.integers(1, B + 1))))
    S.prompts = []
    for r in range(96):
        f = fams[r % 3]
        if kind == "short":
            n = int(rng.integers(1, 4 * nct + 8))
            S.prompts.append(f[:n])
            continue
        d = int(rng.integers(1, B - 1))
        t = nct - (r // 3) % 2 if nct else int(rng.integers(0, 8))
        if kind == "long":
            d = B                                         # the cap: bytes past it are never hashed
        S.prompts.append(f[: d * BB] + L.tail(rng, 4 * t))
        if kind == "long":
            S.prompts[-1] += L.tail(rng, BB * int(rng.integers(0, 4)))
    return S


def scene_encode(kind, world, seed=0):
    """E/P/D: decode, prefill and encode slots; multimodal flags mixed.  some: encode slots only on the first rank's
    range; none: no encode slot at all (encode runs and finds nobody)."""
    rng = np.random.default_rng(L.seed_of("pd-encode", kind, world, seed))
    E, B = 48, 10
    cut = L.sharded().shard_range(0, world, E)[1]
    role = np.array([(R_DECODE, R_PREFILL, R_ENCODE, R_EPD)[e % 4] for e in range(E)])
    if kind == "some":
        role = np.where((role == R_ENCODE) & (np.arange(E) >= cut), R_DECODE, role)
    if kind == "none":
        role = np.where((role == R_ENCODE) | (role == R_EPD), R_PREFILL, role)
    S = PDScene(E, B, role, rng.choice([0.0, 0.25, 0.75], E), rng.integers(0, 5, E), (F_DECODE, DECODE_SC),
                encode=(F_ENCODE, ENCODE_SC), nct=6)
    fams = [L.fam_bytes(rng, B) for _ in range(3)]
    holders(S, rng, fams, np.arange(E), per_fam=8)
    S.prompts = L.family_prompts(rng, fams, 100, B, cold_share=0.1)
    S.mm = (rng.random(len(S.prompts)) < 0.5).astype(np.uint8)
    return S


def scene_overflow(seed=0):
    """40 decode holders of one family on the first of two shards (its sparse map overflows: the dense pass) and prefill
    holders on the second."""
    rng = np.random.default_rng(L.seed_of("pd-overflow", seed))
    E, B = 96, 12
    role = np.where(np.arange(E) < 48, R_DECODE, R_PREFILL)
    S = PDScene(E, B, role, rng.choice([0.0, 0.25, 0.5], E), rng.integers(0, 2, E), (F_DECODE, DECODE_SC), nct=4)
    fams = [L.fam_bytes(rng, B) for _ in range(3)]
    for e in rng.choice(48, 40, replace=False):
        S.hold(fams[0], e, range(int(rng.integers(1, B + 1))))
    holders(S, rng, fams, np.arange(48, E), per_fam=10)
    S.prompts = L.family_prompts(rng, fams[:2], 64, B, cold_share=0.1)
    S.holders = 40
    return S


def scene_lora(seed=0):
    """L.scene_lora's adapters and holders under P/D: slots alternate decode / prefill."""
    S0 = L.scene_lora(seed)
    S = PDScene(S0.E, S0.B, np.array([(R_DECODE, R_PREFILL)[e % 2] for e in range(S0.E)]), S0.kv, S0.waiting,
                (F_DECODE, S0.prof[1]), prefill=(F_PREFILL, S0.prof[1]), nct=6, models=S0.models, lora=S0.lora)
    S.hs, S.es, S.prompts, S.model_of = S0.hs, S0.es, S0.prompts, S0.model_of
    return S


def single_of(S):
    """The same scene with the prefill profile removed (the single-profile handler)."""
    T = PDScene(S.E, S.B, S.role, S.kv, S.waiting, S.prof, prefill=None, models=S.models, lora=S.lora)
    T.hs, T.es, T.prompts, T.model_of = S.hs, S.es, S.prompts, S.model_of
    return T


# ------------------------------------------------------------------------------------------------
# oracle side
# ------------------------------------------------------------------------------------------------
def expected(orc, S, prompts):
    """orc.cycle_batch on the whole pool and index (tie_seed 0) with the scene's profiles, per adapter; the prompts are
    the true ones (their length is the decider's input)."""
    from oracle import pyoracle
    ix = S.oracle_index(orc)
    R = len(prompts)
    out = np.zeros(R, pyoracle.DECISION_DTYPE)
    tot = np.zeros(R, np.int32)
    mb = np.zeros(R, np.int64)
    mo = S.adapters(R)
    prof = lambda p: None if p is None else orc.make_profile(p[0], list(p[1]))
    for a in sorted(set(mo.tolist())):
        sel = np.flatnonzero(mo == a)
        ps = [prompts[i] for i in sel]
        d, offs = L.PP._pack(ps)
        kw = {}
        if S.encode is not None:
            kw = dict(encode=prof(S.encode), multimodal=None if S.mm is None else S.mm[sel])
        od, ot = orc.cycle_batch(S.models[a], S.bst, S.B, S.nct, S.always, ix, prof(S.prof), prof(S.prefill),
                                 S.oracle_pool(orc, a), d, offs, 4, **kw)
        out[sel], tot[sel] = od, ot
        for j, i in enumerate(sel):
            if od["status"][j] == 0:
                m, _ = ix.match_longest_prefix(orc.hash_prompt(ps[j], S.models[a], S.bst, S.B), S.E)
                mb[i] = m[od["pick"][j]]
    return out, tot, mb


def check(dec, det, exp, where):
    odec, ototal, mb = exp
    helpers.assert_decisions_equal(dec, det, odec, ototal, where=where)
    ok = odec["status"] == 0
    np.testing.assert_array_equal(dec["match_blocks"][ok].astype(np.int64), mb[ok], err_msg=f"{where}: match_blocks")
    # a request without a decode pick runs no other stage
    assert (dec["prefill_pick"][~ok] == NO).all() and (det["prefill_ran"][~ok] == 0).all(), where
    assert (det["encode_pick"][~ok] == NO).all() and (det["encode_ran"][~ok] == 0).all(), where


# ------------------------------------------------------------------------------------------------
# engine side
# ------------------------------------------------------------------------------------------------
def traced(fn, want, where, repeatable=True):
    return L.traced(fn, want, where=where, repeatable=repeatable)


def spec(epp, p):
    return None if p is None else epp.ProfileSpec(p[0], [epp.ScorerSpec(*s) for s in p[1]])


def pd_engine(epp, S, lo, hi, *, tie_seed=0, staged=True):
    eng = epp.Engine(S.E, spec(epp, S.prof), spec(epp, S.prefill), encode=spec(epp, S.encode), block_size_tokens=S.bst,
                     max_prefix_blocks=S.B, non_cached_tokens=S.nct, always_disagg=S.always, tie_seed=tie_seed)
    for m in S.models:
        eng.register_model(m)
    if staged:
        assert eng.shard_set_staged(lo, hi) == S.stages
    else:
        eng.shard_set(lo, hi)
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


def batch_of(S, prompts, layout, rng):
    """-> (the true prompts, device data, kwargs).  layout "long": rows hold the hashed bytes only, lengths the true
    length."""
    import torch
    if layout == "long":
        cap = S.B * 4 * S.bst
        rows = [p[:cap] for p in prompts]
        offs = np.cumsum([0] + [(len(p) + 31) // 32 * 32 for p in rows]).astype(np.uint64)
        buf = bytearray(int(offs[-1]) + 64)
        for o, p in zip(offs, rows):
            buf[int(o): int(o) + len(p)] = p
        data, kw = L.device_kw(bytes(buf), offs, np.array([len(p) for p in prompts], np.uint64), None)
        ps = list(prompts)
    else:
        ps, buf, offs, lens, T = L.layout_batch(prompts, layout, rng)
        data, kw = L.device_kw(buf, offs, lens, T)
    R = len(ps)
    if S.model_of is not None:
        kw["model_ids"] = torch.from_numpy(np.asarray(S.adapters(R), np.uint32).view(np.int32)).cuda()
    if S.mm is not None:
        kw["multimodal"] = torch.from_numpy(np.asarray(S.mm[:R], np.uint8)).cuda()
    return ps, data, kw


def dense_ranks(orc, S, prompts, ranges):
    """Ranks whose sparse lane map overflows on some request (> 32 in-shard slots hold a block before the global stop,
    or carry the request's adapter)."""
    ix = S.oracle_index(orc)
    mo = S.adapters(len(prompts))
    over = set()
    for r, p in enumerate(prompts):
        eps = set()
        for x in orc.hash_prompt(p, S.models[int(mo[r])], S.bst, S.B):
            got = ix.get(x)
            if not got:
                break
            eps |= got
        if S.lora is not None:
            eps |= set(np.flatnonzero(S.lora[2][int(mo[r])]).tolist())
        for g, (lo, hi) in enumerate(ranges):
            if sum(lo <= e < min(hi, S.E) for e in eps) > 32:
                over.add(g)
    return over


def run_protocol(epp, orc, S, ranges, *, layout="offsets0", tie_seed=0, where=""):
    """The host protocol over one engine per range -> (decisions, details, per-rank records [R, S])."""
    import torch
    rng = np.random.default_rng(L.seed_of("pd-layout", where))
    ps, data, kw = batch_of(S, S.prompts, layout, rng)
    R, St = len(ps), S.stages
    W = (S.B + 31) // 32
    over = dense_ranks(orc, S, ps, ranges)
    engines = [pd_engine(epp, S, lo, hi, tie_seed=tie_seed) for lo, hi in ranges]
    try:
        masks, bests = [], []
        for g, eng in enumerate(engines):
            m = torch.zeros((R, W), dtype=torch.int32, device="cuda")
            traced(lambda: eng.shard_probe(data, m, **kw), (PROBE,), f"{where} probe rank {g}")
            masks.append(m)
        gm = masks[0].clone()
        for m in masks[1:]:
            gm |= m
        torch.cuda.synchronize()
        for g, eng in enumerate(engines):
            b = torch.zeros((R, 24 * St), dtype=torch.uint8, device="cuda")
            traced(lambda: eng.shard_pick(R, gm, b), (SPARSE_OF[St], DENSE) if g in over else (SPARSE_OF[St],),
                   f"{where} pick rank {g} {ranges[g]}")
            bests.append(b)
        allb = torch.stack(bests)
        dec = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
        det = torch.zeros((R, 40), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        traced(lambda: engines[0].shard_merge(R, len(engines), allb, dec, out_detail=det), (MERGE,), f"{where} merge")
        torch.cuda.synchronize()
        out = epp.decisions_from_torch(dec)
        dout = det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
    finally:
        for e in engines:
            e.close()
    check(out, dout, expected(orc, S, ps), where)
    recs = [b.cpu().numpy().view(epp.SHARD_BEST_DTYPE).reshape(R, St) for b in bests]
    return out, dout, recs


def p2p_engines(epp, S, ranges, R_max, tie_seed=0):
    engines, ptrs = [], []
    for lo, hi in ranges:
        eng = pd_engine(epp, S, lo, hi, tie_seed=tie_seed)
        _, ptr = eng.shard_p2p_export(R_max)
        engines.append(eng)
        ptrs.append(ptr)
    for g, eng in enumerate(engines):
        eng.shard_p2p_connect(len(engines), g, np.array(ptrs, dtype=np.uint64), ipc_handles=False)
    return engines


def run_p2p_stepped(epp, orc, S, ranges, layout, where):
    import torch
    rng = np.random.default_rng(L.seed_of("pd-p2p", where))
    ps, data, kw = batch_of(S, S.prompts, layout, rng)
    R = len(ps)
    engines = p2p_engines(epp, S, ranges, R)
    try:
        outs = [torch.zeros((R, 32), dtype=torch.uint8, device="cuda") for _ in engines]
        dets = [torch.zeros((R, 40), dtype=torch.uint8, device="cuda") for _ in engines]
        torch.cuda.synchronize()

        def phases():
            for phase in range(3):
                for g, eng in enumerate(engines):
                    eng.shard_p2p_phase(data, outs[g], phase, out_detail=dets[g], **kw)
        traced(phases, (PROBE, SPARSE_OF[S.stages], MERGE) + L.P2P, where, repeatable=False)
        torch.cuda.synchronize()
        decs = [epp.decisions_from_torch(o) for o in outs]
        dts = [d.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1) for d in dets]
    finally:
        for e in engines:
            e.close()
    for d, t in zip(decs[1:], dts[1:]):
        np.testing.assert_array_equal(d, decs[0], err_msg=f"{where}: ranks disagree")
        np.testing.assert_array_equal(t, dts[0], err_msg=f"{where}: ranks disagree (detail)")
    check(decs[0], dts[0], expected(orc, S, ps), where)
    return decs[0], dts[0]


def even(world, E):
    return [L.sharded().shard_range(g, world, E) for g in range(world)]


# ------------------------------------------------------------------------------------------------
# A: role layouts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [1, 2, 3, 5])
@pytest.mark.parametrize("kind", ["interleaved", "split", "no-prefill", "no-decode"])
def test_A_role_layouts(epp, orc, kind, world):
    S = scene_roles(kind)
    ranges = even(world, S.E)
    dec, det, recs = run_protocol(epp, orc, S, ranges, tie_seed=0x5EED if world == 3 else 0, where=f"A {kind} x{world}")
    ok = dec["status"] == 0
    if kind == "no-decode":
        assert not ok.any()
        assert any((r[:, 1]["status"] == 0).any() for r in recs), "prefill records are published without a decode pick"
    elif kind == "no-prefill":
        assert ok.all() and (det["prefill_ran"] == 1).any() and (dec["prefill_pick"] == NO).all()
    else:
        assert (dec["prefill_pick"][ok] != NO).any() and (det["prefill_ran"][ok] == 0).any()
    if kind == "split" and world == 2:
        # rank 1 has no decode candidate and still publishes its prefill best
        assert (recs[1][:, 0]["status"] == -1).all() and (recs[1][:, 1]["status"] == 0).any()
        assert ((dec["prefill_pick"] >= S.E // 2) & (dec["prefill_pick"] != NO)).any()


@pytest.mark.parametrize("kind", ["interleaved", "split"])
def test_A_descending_ranges(epp, orc, kind):
    S = scene_roles(kind, seed=1)
    run_protocol(epp, orc, S, even(3, S.E)[::-1], where=f"A {kind} descending")


# ------------------------------------------------------------------------------------------------
# B: the P/D decider
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("kind", ["boundary", "always", "nct0", "short", "long"])
def test_B_decider(epp, orc, kind, tie_seed):
    S = scene_decider(kind)
    ranges = even(2, S.E)
    # packed rows ("odd"): a padded layout would add its padding to the prompts' tails
    dec, det, _ = run_protocol(epp, orc, S, ranges, layout="long" if kind == "long" else "odd", tie_seed=tie_seed,
                               where=f"B {kind} seed={tie_seed}")
    ok = dec["status"] == 0
    ran = det["prefill_ran"] == 1
    if kind in ("boundary", "long"):
        assert (ok & ran).any() and (ok & ~ran).any()
    if kind == "always":
        assert ran[ok].all()
    if kind == "nct0":
        assert not ran.any()


@pytest.mark.parametrize("layout", ["lengths", "odd"])
def test_B_decider_p2p(epp, orc, layout):
    S = scene_decider("boundary", seed=1)
    run_p2p_stepped(epp, orc, S, even(2, S.E), layout, f"B p2p {layout}")


# ------------------------------------------------------------------------------------------------
# C: encode
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("kind", ["all", "some", "none"])
def test_C_encode(epp, orc, kind, world):
    S = scene_encode(kind, world)
    dec, det, _ = run_protocol(epp, orc, S, even(world, S.E), where=f"C {kind} x{world}")
    ok = dec["status"] == 0
    mm = S.mm.astype(bool)
    assert (det["encode_ran"][ok] == mm[ok]).all()
    if kind == "none":
        assert (det["encode_pick"] == NO).all() and (det["encode_ran"] == 1).any()
    else:
        assert (det["encode_pick"][ok & mm] != NO).all()


def test_C_encode_p2p(epp, orc):
    S = scene_encode("some", 3, seed=1)
    run_p2p_stepped(epp, orc, S, even(3, S.E), "offsets16", "C p2p")


def test_C_detail_required(epp):
    """With an encode profile and multimodal requests, out_detail NULL is refused by the merge and the peer-memory calls."""
    import torch
    S = scene_encode("all", 1)
    ps, data, kw = batch_of(S, S.prompts[:16], "offsets0", np.random.default_rng(0))
    with pd_engine(epp, S, 0, S.E) as eng:
        m = torch.zeros((16, 1), dtype=torch.int32, device="cuda")
        eng.shard_probe(data, m, **kw)
        b = torch.zeros((16, 72), dtype=torch.uint8, device="cuda")
        eng.shard_pick(16, m, b)
        dec = torch.zeros((16, 32), dtype=torch.uint8, device="cuda")
        with pytest.raises(epp.EngineError, match="out_detail") as e:
            eng.shard_merge(16, 1, b.unsqueeze(0), dec)
        assert e.value.code == -1
        _, ptr = eng.shard_p2p_export(16)
        eng.shard_p2p_connect(1, 0, np.array([ptr], np.uint64), ipc_handles=False)
        for call in (lambda: eng.shard_schedule_p2p(data, dec, **kw), lambda: eng.shard_p2p_phase(data, dec, 0, **kw)):
            with pytest.raises(epp.EngineError, match="out_detail"):
                call()
        det = torch.zeros((16, 40), dtype=torch.uint8, device="cuda")
        eng.shard_schedule_p2p(data, dec, out_detail=det, **kw)          # the same batch with a detail goes through


# ------------------------------------------------------------------------------------------------
# D: the dense pass, LoRA, config 4
# ------------------------------------------------------------------------------------------------
def test_D_dense_pass(epp, orc):
    S = scene_overflow()
    ranges = even(2, S.E)
    assert dense_ranks(orc, S, S.prompts, ranges) == {0}
    dec, det, _ = run_protocol(epp, orc, S, ranges, where="D dense")
    assert (dec["match_blocks"] > 0).any() and (dec["prefill_pick"] != NO).any()


@pytest.mark.parametrize("exchange", ["protocol", "p2p"])
def test_D_lora_adapters(epp, orc, exchange):
    S = scene_lora()
    ranges = even(3, S.E)
    if exchange == "protocol":
        dec, _, _ = run_protocol(epp, orc, S, ranges, layout="odd", where="D lora")
    else:
        dec, _ = run_p2p_stepped(epp, orc, S, ranges, "lengths", "D lora p2p")
    assert len(set(S.adapters(len(S.prompts)).tolist())) == 3 and (dec["prefill_pick"] != NO).any()


def config4_scene(R=512, E=320):
    """Config 4 of tools/tracegen at a reduced size as a PDScene (its pool, index, prompts and profiles)."""
    from oracle import pyoracle as orc
    from tools import tracegen as tg
    w = tg.baseline_configs()["config4"].scaled(E=E, R=R, T=1024)
    trace = tg.Trace(w)
    role, kv, waiting, running = trace.pool()
    S = PDScene(w.E, w.max_prefix_blocks, role, kv, waiting, (w.primary_filter, list(w.primary_scorers)), running=running,
                prefill=(tg.FILTER_PREFILL, list(w.prefill_scorers)), nct=w.non_cached_tokens, models=(tg.MODEL,))
    pool, ix, primary, prefill, (hs, es) = helpers.setup_oracle(orc, w, trace)
    S.hs, S.es, S.bst = hs.tolist(), es.tolist(), w.block_size_tokens
    tokens, _, _ = trace.requests()
    S.prompts = [tokens[r].tobytes() for r in range(tokens.shape[0])]
    return S, w


def test_D_config4(epp, orc):
    S, w = config4_scene()
    dec, det, _ = run_protocol(epp, orc, S, even(4, S.E), layout="uniform", where="D config4")
    ok = dec["status"] == 0
    assert ok.all() and (det["prefill_ran"] == 1).any() and (dec["prefill_pick"] != NO).any()


# ------------------------------------------------------------------------------------------------
# E: one rank's own exchange over a large batch
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunks", ["2", "1"])
def test_E_p2p_world_one_large_batch(epp, orc, monkeypatch, chunks):
    import torch
    monkeypatch.setenv("EPP_DEV_CHUNKS", chunks)
    S0 = scene_encode("all", 1, seed=2)
    R = 8257
    rng = np.random.default_rng(int(chunks))
    idx = rng.integers(0, len(S0.prompts), R)
    S0.prompts = [S0.prompts[int(i)] for i in idx]
    S0.mm = S0.mm[idx]
    ps, data, kw = batch_of(S0, S0.prompts, "offsets0", rng)
    eng = pd_engine(epp, S0, 0, S0.E)
    try:
        _, ptr = eng.shard_p2p_export(R)
        eng.shard_p2p_connect(1, 0, np.array([ptr], np.uint64), ipc_handles=False)
        out = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
        det = torch.zeros((R, 40), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        _, names = traced(lambda: eng.shard_schedule_p2p(data, out, out_detail=det, **kw), (PROBE, SPARSE_OF[3], MERGE) + L.P2P,
                          f"E world 1 chunks={chunks}", repeatable=False)
        torch.cuda.synchronize()
        if helpers.trace_complete(names):
            n = sum(c for k, c in names.items() if SPARSE_OF[3] in k)
            assert n == (2 if chunks == "2" else 1), sorted(names.items())
        check(epp.decisions_from_torch(out), det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1), expected(orc, S0, ps),
              f"E world 1 chunks={chunks}")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------
# F: the contract
# ------------------------------------------------------------------------------------------------
def test_F_single_handler_staged_is_unchanged(epp, orc):
    """A single-profile engine: shard_set_staged returns 1 and every record and decision byte equals shard_set's."""
    import torch
    S = single_of(scene_roles("interleaved", seed=2))
    ranges = even(3, S.E)
    ps, data, kw = batch_of(S, S.prompts, "offsets0", np.random.default_rng(5))
    R = len(ps)
    outs = {}
    for staged in (False, True):
        engines = [pd_engine(epp, S, lo, hi, staged=staged) for lo, hi in ranges]
        try:
            masks = []
            for eng in engines:
                m = torch.zeros((R, 1), dtype=torch.int32, device="cuda")
                eng.shard_probe(data, m, **kw)
                masks.append(m)
            gm = masks[0] | masks[1] | masks[2]
            torch.cuda.synchronize()
            bests = []
            for eng in engines:
                b = torch.zeros((R, 24), dtype=torch.uint8, device="cuda")
                traced(lambda: eng.shard_pick(R, gm, b), (SPARSE_OF[1],), f"F staged={staged}")
                bests.append(b)
            allb = torch.stack(bests)
            dec = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            engines[0].shard_merge(R, 3, allb, dec)
            outs[staged] = (allb.cpu().numpy(), dec.cpu().numpy())
        finally:
            for e in engines:
                e.close()
    np.testing.assert_array_equal(outs[True][0], outs[False][0])
    np.testing.assert_array_equal(outs[True][1], outs[False][1])
    odec, ototal, mb = expected(orc, S, ps)
    helpers.assert_decisions_equal(outs[True][1].view(epp.DECISION_DTYPE).reshape(-1), None, odec, ototal, where="F single")


def test_F_refusals(epp):
    """shard_set_staged refuses what shard_set refuses, other than the disagg handler, with the same messages."""
    P, Sp, capi = epp.ProfileSpec, epp.ScorerSpec, epp.capi
    from tools import nohit_lru_model as NH
    base = [Sp(QUEUE, 1.0, 0.0), Sp(PREFIX, 1.0, 0.0)]
    pf = P(F_PREFILL, base)
    cases = {
        "no-hit-lru": dict(primary=P(1, base + [Sp(NH.NO_HIT_LRU, 1.0, 4.0)])),
        "random picker": dict(primary=P(1, base, picker=capi.PICKER_RANDOM)),
        "weighted random picker": dict(primary=P(1, base, picker=capi.PICKER_WEIGHTED_RANDOM)),
        "inflight producer": dict(primary=P(1, base), inflight_load=True),
        "pick_k > 1": dict(primary=P(1, base), pick_k=2),
        "affinity filter": dict(primary=P(1, base, affinity=epp.AffinityFilterSpec())),
    }
    for name, kw in cases.items():
        with epp.Engine(16, max_prefix_blocks=8, block_size_tokens=BST, **kw) as eng:       # single profile
            with pytest.raises(epp.EngineError, match="endpoint-sharded") as a:
                eng.shard_set(0, 8)
            with pytest.raises(epp.EngineError, match="endpoint-sharded") as b:
                eng.shard_set_staged(0, 8)
            assert a.value.message == b.value.message, name
        with epp.Engine(16, prefill=pf, max_prefix_blocks=8, block_size_tokens=BST, **kw) as eng:   # P/D
            with pytest.raises(epp.EngineError, match="endpoint-sharded") as b:
                eng.shard_set_staged(0, 8)
            assert b.value.message == a.value.message, name
    with epp.Engine(16, P(1, base), pf, max_prefix_blocks=8, block_size_tokens=BST) as eng:
        with pytest.raises(epp.EngineError, match="single-profile handler only"):
            eng.shard_set(0, 8)
        assert eng.shard_set_staged(0, 8) == 2
    with epp.Engine(16, P(1, base), pf, encode=P(F_ENCODE, base), max_prefix_blocks=8, block_size_tokens=BST) as eng:
        assert eng.shard_set_staged(0, 8) == 3


def test_F_staged_after_export(epp):
    """The exchange buffer's record region is sized at export: shard_set_staged for another S after it is EPP_ERR_STATE;
    before it (or for the same S) it is fine."""
    P, Sp = epp.ProfileSpec, epp.ScorerSpec
    base = [Sp(QUEUE, 1.0, 0.0), Sp(PREFIX, 1.0, 0.0)]
    with epp.Engine(16, P(1, base), P(2, base), max_prefix_blocks=8, block_size_tokens=BST) as eng:
        eng.register_model(MODEL)
        eng.shard_p2p_export(64)                       # sized for one record per request
        with pytest.raises(epp.EngineError, match="epp_shard_set_staged before epp_shard_p2p_export") as e:
            eng.shard_set_staged(0, 8)
        assert e.value.code == -5
    with epp.Engine(16, P(1, base), P(2, base), max_prefix_blocks=8, block_size_tokens=BST) as eng:
        assert eng.shard_set_staged(0, 8) == 2
        eng.shard_p2p_export(64)
        assert eng.shard_set_staged(8, 16) == 2
    with epp.Engine(16, P(0, base), max_prefix_blocks=8, block_size_tokens=BST) as eng:
        eng.shard_p2p_export(64)
        assert eng.shard_set_staged(0, 8) == 1


def _nccl_worker(rank, world, port, q):
    import os
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        import epp_b200 as epp
        sh = L.sharded()
        S = scene_encode("some", world, seed=3)
        lo, hi = sh.shard_range(rank, world, S.E)
        ps, data, kw = batch_of(S, S.prompts, "uniform", np.random.default_rng(9))
        eng = epp.Engine(S.E, spec(epp, S.prof), spec(epp, S.prefill), encode=spec(epp, S.encode), device=rank,
                         block_size_tokens=BST, max_prefix_blocks=S.B, non_cached_tokens=S.nct)
        eng.register_model(MODEL)
        eng.shard_set_staged(lo, hi)
        eng.pool_set(*S.pool_arrays())
        hs, es = np.array(S.hs, np.uint64), np.array(S.es, np.uint32)
        k = (es >= lo) & (es < hi)
        eng.index_load_snapshot(hs[k], es[k])
        det = torch.zeros((len(ps), 40), dtype=torch.uint8, device=f"cuda:{rank}")
        T = kw["uniform_len"]
        dec = sh.schedule_sharded(eng, data[: len(ps) * T].view(len(ps), T), T, dist, detail=det, multimodal=kw["multimodal"])
        torch.cuda.synchronize()
        q.put((rank, dec.cpu().numpy().tobytes(), det.cpu().numpy().tobytes(), [bytes(p) for p in ps]))
        eng.close()
    finally:
        dist.destroy_process_group()


def test_F_two_gpus_nccl(epp, orc):
    """schedule_sharded over NCCL on two GPUs with the encode stage; skipped on a machine with one GPU."""
    import socket
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        rank, dec, det, ps = q.get(timeout=300)
        res[rank] = (np.frombuffer(dec, epp.DECISION_DTYPE), np.frombuffer(det, epp.DETAIL_DTYPE), ps)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    np.testing.assert_array_equal(res[0][0], res[1][0])
    S = scene_encode("some", 2, seed=3)
    check(res[0][0], res[0][1], expected(orc, S, res[0][2]), "F nccl x2")
