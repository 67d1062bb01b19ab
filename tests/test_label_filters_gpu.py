"""GPU parity of the label filters (include/epp_engine.h "Label filters"; decided in k_pool_candidates / k_pool_aux).

A: an engine whose profiles hold the role filters is compared bit for bit with one whose profiles hold the same sets as
   by-label (and selector In) filters on llm-d.ai/role, on every scheduling path.
B: general selectors against tools/label_model.py: the C oracle run on the pool narrowed by each profile's filters.
C: landscapes in which a dropped endpoint holds every pool-wide extreme, so a mask missing anywhere changes decisions.
D: snapshot behaviour of epp_pool_set_labels.  E: every rejection, each followed by an unchanged decision.
Run on an H100: pytest -m gpu."""
import ctypes as C
import threading

import numpy as np
import pytest

from tools import label_model as lm
from tools import tracegen as tg

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
ROLE_KEY = "llm-d.ai/role"
ROLE_VALUES = [None, "", "decode", "prefill", "prefill-decode", "both", "encode", "encode-prefill",
               "encode-prefill-decode", "garbage"]
ROLE_TABLES = {   # roles.go:46-70: (allowsNoLabel, validValues)
    1: (True, ["decode", "prefill-decode", "both", "encode-prefill-decode"]),
    2: (False, ["prefill", "encode-prefill", "prefill-decode", "both", "encode-prefill-decode"]),
    3: (False, ["encode", "encode-prefill", "encode-prefill-decode"]),
}


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def role_labels(E, seed):
    rng = np.random.default_rng(seed)
    out = []
    for e in range(E):
        v = ROLE_VALUES[rng.integers(len(ROLE_VALUES))]
        lb = {"other.example.com/x": str(e % 3)}
        if v is not None:
            lb[ROLE_KEY] = v
        out.append(lb)
    return out


def role_codes(epp, labels):
    P = epp.plugins
    return np.array([P.NewEndpoint(P.EndpointMetadata("x", lb)).role_code() for lb in labels], dtype=np.uint8)


def as_label_filter(kind, form):
    allows, values = ROLE_TABLES[kind]
    if form == "selector":
        assert not allows
        return [(ROLE_KEY, lm.IN, values)]
    return [(ROLE_KEY, lm.BY_LABEL_OR_ABSENT if allows else lm.BY_LABEL, values)]


class Pair:
    """Two engines on one trace: `a` with the role filters, `b` with filter NONE and the same sets as label filters."""

    def __init__(self, epp, name, form="bylabel", E=192, R=256, seed=7, picker=0, nohit=False, inflight=False,
                 tie_seed=0, encode=True, affinity=None, pick_k=0, active=False):
        w = tg.baseline_configs()[name].scaled(E=E, R=R, T=512)
        self.w, self.trace = w, tg.Trace(w)
        scorers = [epp.ScorerSpec(*s) for s in w.primary_scorers]
        if nohit:
            scorers.append(epp.ScorerSpec(9, 1.0, 8.0))
        if inflight or active:
            scorers.append(epp.ScorerSpec(7, 1.5, 1.0, 0))
        pre = None if w.prefill_scorers is None else [epp.ScorerSpec(*s) for s in w.prefill_scorers]
        aff = None if affinity is None else epp.AffinityFilterSpec(*affinity)
        self.labels = role_labels(E, seed)
        self.role = role_codes(epp, self.labels)
        kw = dict(block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks,
                  non_cached_tokens=w.non_cached_tokens, tie_seed=tie_seed, pick_k=pick_k, inflight_load=inflight)
        if active and not inflight:
            kw["n_ext_cols"] = 1
        self.ext = np.random.default_rng(seed + 1).integers(0, 9, size=(1, E)).astype(np.float64) if "n_ext_cols" in kw else None
        engines = []
        for labelled in (False, True):
            def spec(kind, sc):
                if sc is None:
                    return None
                if not labelled:
                    return epp.ProfileSpec(kind, sc, aff, picker)
                f = form if kind != 1 else "bylabel"
                return epp.ProfileSpec(0, sc, aff, picker, as_label_filter(kind, f))
            primary_kind = 1 if pre is not None else w.primary_filter or 1
            enc = spec(3, scorers) if (encode and pre is not None) else None
            eng = epp.Engine(w.E, spec(primary_kind, scorers), spec(2, pre), encode=enc, **kw)
            eng.register_model(tg.MODEL)
            fh, _ = eng.hash_prompts(self.trace.family_tokens(), uniform_len=w.prompt_bytes)
            eng.index_load_snapshot(*self.trace.index_pairs(fh))
            _, kv, waiting, running = self.trace.pool()
            eng.pool_set(np.arange(E, dtype=np.uint32), self.role, kv, waiting, running, self.ext)
            if labelled:
                eng.pool_set_labels(np.arange(E, dtype=np.uint32), self.labels)
            engines.append(eng)
        self.a, self.b = engines
        self.tokens, _, _ = self.trace.requests()
        self.mm = (np.arange(R) % 3 == 0).astype(np.uint8)

    def close(self):
        self.a.close()
        self.b.close()


def same(x, y, where):
    x, y = np.ascontiguousarray(x), np.ascontiguousarray(y)
    assert x.dtype == y.dtype and x.shape == y.shape, where
    np.testing.assert_array_equal(x.view(np.uint8), y.view(np.uint8), err_msg=where)


def run_paths(epp, pr, topk=False):
    """Every scheduling path on both engines; returns nothing, asserts equality."""
    import torch
    w, toks = pr.w, pr.tokens
    outs = []
    for eng in (pr.a, pr.b):
        o = {}
        r = eng.schedule(toks, uniform_len=w.prompt_bytes, multimodal=pr.mm, topk=topk)
        o["host"] = r
        r = eng.schedule(toks[:8], uniform_len=w.prompt_bytes, multimodal=pr.mm[:8], topk=topk)
        o["host_small"] = r
        pin = epp.PinnedBuffer(toks[:4].nbytes)
        pin.array[:] = toks[:4].view(np.uint8).reshape(-1)
        o["zero_copy"] = eng.schedule(pin.array, uniform_len=w.prompt_bytes, multimodal=pr.mm[:4], topk=topk)
        dt = torch.from_numpy(toks.view(np.int32)).cuda()
        mm = torch.from_numpy(pr.mm).cuda()
        d = eng.schedule(dt, uniform_len=w.prompt_bytes, multimodal=mm, topk=topk)
        torch.cuda.synchronize()
        o["device"] = [epp.decisions_from_torch(d[0]), d[1].cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)] + \
            ([{k: v.cpu().numpy() for k, v in d[2].items()}] if topk else [])
        d = eng.schedule(dt, uniform_len=w.prompt_bytes, multimodal=mm, asynchronous=True)
        eng.synchronize()
        o["async"] = [epp.decisions_from_torch(d[0]), d[1].cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)]
        subsets = [None if r % 2 else list(range(r % 17, w.E, 3)) for r in range(64)]
        o["subset"] = eng.schedule(toks[:64], uniform_len=w.prompt_bytes, multimodal=pr.mm[:64], subsets=subsets, topk=topk)
        match, total = eng.prefix_match(toks[:64], uniform_len=w.prompt_bytes)
        o["with_match"] = eng.schedule_with_match(match, total, np.full(64, w.prompt_bytes), topk=topk)
        o["score"] = eng.score(match, total, 0, -1)
        if eng.cfg.handler:
            o["score1"] = eng.score(match, total, 1, -1)
        outs.append(o)
        pin.close()
    for k in outs[0]:
        xa, xb = outs[0][k], outs[1][k]
        if isinstance(xa, np.ndarray):
            same(xa, xb, k)
            continue
        for i, (ya, yb) in enumerate(zip(xa, xb)):
            if isinstance(ya, dict):
                for n in ya:
                    same(ya[n], yb[n], f"{k} topk {n}")
            elif ya is not None:
                same(ya, yb, f"{k}[{i}]")
    dec = outs[0]["host"][0]
    return dec


# ---- A: role equivalence --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,form,tie_seed", [("config4", "bylabel", 0), ("config4", "selector", 0),
                                               ("config4", "bylabel", 0x5EED), ("config3", "bylabel", 0),
                                               ("config1", "bylabel", 0x5EED)])
def test_role_equivalence_every_path(epp, name, form, tie_seed):
    pr = Pair(epp, name, form=form, tie_seed=tie_seed)
    try:
        dec = run_paths(epp, pr)
        assert (dec["status"] == 0).any()
    finally:
        pr.close()


@pytest.mark.parametrize("picker", [1, 2])
def test_role_equivalence_random_pickers(epp, picker):
    pr = Pair(epp, "config4", picker=picker, tie_seed=0xABC)
    try:
        run_paths(epp, pr)
    finally:
        pr.close()


def test_role_equivalence_nohit_lru(epp):
    pr = Pair(epp, "config4", nohit=True)
    try:
        for b in range(3):
            toks, _, _ = pr.trace.requests(b * 64, 64)
            da = pr.a.schedule(toks, uniform_len=pr.w.prompt_bytes)
            db = pr.b.schedule(toks, uniform_len=pr.w.prompt_bytes)
            same(da[0], db[0], f"batch {b}")
            assert pr.a.nohit_lru_get() == pr.b.nohit_lru_get()
        run_paths(epp, pr)
        assert pr.a.nohit_lru_get() == pr.b.nohit_lru_get()
    finally:
        pr.close()


def test_role_equivalence_inflight(epp):
    pr = Pair(epp, "config4", inflight=True)
    try:
        run_paths(epp, pr)
        ra, ta = pr.a.inflight_get()
        rb, tb = pr.b.inflight_get()
        np.testing.assert_array_equal(ra, rb)
        np.testing.assert_array_equal(ta, tb)
    finally:
        pr.close()


def test_role_equivalence_affinity_topk(epp):
    pr = Pair(epp, "config4", affinity=(0.5, 0.0, 5000.0, -1), pick_k=4, active=True)
    try:
        run_paths(epp, pr, topk=True)
    finally:
        pr.close()


def test_role_equivalence_batcher(epp):
    pr = Pair(epp, "config4", encode=False)
    try:
        toks = pr.tokens[:256]
        res = {}
        for tag, eng in (("a", pr.a), ("b", pr.b)):
            out = [None] * 256
            with epp.Batcher(eng, max_batch=32, max_delay_us=100) as bt:
                def worker(t):
                    for r in range(t, 256, 64):
                        out[r] = bt.schedule(toks[r])
                ths = [threading.Thread(target=worker, args=(t,)) for t in range(64)]
                for t in ths:
                    t.start()
                for t in ths:
                    t.join()
            res[tag] = out
        for r in range(256):   # the batches differ between the runs; each decision is request-local (no index adds)
            assert bytes(res["a"][r][0]) == bytes(res["b"][r][0]), r
    finally:
        pr.close()


@pytest.mark.parametrize("exchange", ["protocol", "p2p"])
def test_role_equivalence_sharded_one_gpu(epp, exchange):
    """The endpoint-sharded mode over two ranks on one GPU, through epp_shard_probe / pick / merge or stepped through
    epp_shard_p2p_phase: every rank gets the whole pool's labels."""
    import torch
    pr = Pair(epp, "config3", encode=False)
    w = pr.w
    try:
        toks = torch.from_numpy(pr.tokens[:64].view(np.int32)).cuda()
        nw = (w.max_prefix_blocks + 31) // 32
        res = {}
        for tag, labelled in (("a", False), ("b", True)):
            ranks = []
            for lo, hi in ((0, w.E // 3), (w.E // 3, w.E)):
                sc = [epp.ScorerSpec(*s) for s in w.primary_scorers]
                pri = epp.ProfileSpec(0, sc, labels=as_label_filter(1, "bylabel")) if labelled else epp.ProfileSpec(1, sc)
                eng = epp.Engine(w.E, pri, block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks)
                eng.register_model(tg.MODEL)
                fh, _ = eng.hash_prompts(pr.trace.family_tokens(), uniform_len=w.prompt_bytes)
                hs, es = pr.trace.index_pairs(fh)
                keep = (es >= lo) & (es < hi)
                eng.index_load_snapshot(hs[keep], es[keep])
                eng.shard_set(lo, hi)
                _, kv, waiting, running = pr.trace.pool()
                eng.pool_set(np.arange(w.E, dtype=np.uint32), pr.role, kv, waiting, running)
                if labelled:
                    eng.pool_set_labels(np.arange(w.E, dtype=np.uint32), pr.labels)
                ranks.append(eng)
            if exchange == "p2p":
                ptrs = [eng.shard_p2p_export(64)[1] for eng in ranks]
                for i, eng in enumerate(ranks):
                    eng.shard_p2p_connect(len(ranks), i, np.array(ptrs, dtype=np.uint64), ipc_handles=False)
                outs = [torch.zeros((64, 32), dtype=torch.uint8, device="cuda") for _ in ranks]
                torch.cuda.synchronize()
                for phase in range(3):          # every rank through one phase before the next: they share the GPU
                    for eng, o in zip(ranks, outs):
                        eng.shard_p2p_phase(toks, o, phase, uniform_len=w.prompt_bytes)
                torch.cuda.synchronize()
                same(epp.decisions_from_torch(outs[1]), epp.decisions_from_torch(outs[0]), "ranks agree")
                out = outs[0]
            else:
                masks = [torch.zeros((64, nw), dtype=torch.int32, device="cuda") for _ in ranks]
                for eng, m in zip(ranks, masks):
                    eng.shard_probe(toks, m, uniform_len=w.prompt_bytes)
                g = masks[0] | masks[1]
                best = torch.zeros((2, 64, 24), dtype=torch.uint8, device="cuda")
                for i, eng in enumerate(ranks):
                    eng.shard_pick(64, g, best[i])
                out = torch.zeros((64, 32), dtype=torch.uint8, device="cuda")
                ranks[0].shard_merge(64, 2, best, out)
                torch.cuda.synchronize()
            res[tag] = epp.decisions_from_torch(out)
            assert (res[tag]["status"] == 0).any()
            for eng in ranks:
                eng.close()
        same(res["a"], res["b"], f"sharded {exchange}")
    finally:
        pr.close()


# ---- B / C: model parity -------------------------------------------------------------------------------------------
def model_case(epp, orc, E, labels, role, reqs, scorers, pre_reqs=None, pre_scorers=None, R=24, seed=3, nct=0,
               waiting=None, running=None, kv=None, ext=None, hits=None, affinity=None, primary_filter=0, pre_filter=0):
    """Engine (schedule_with_match) against label_model.pd_schedule / orc.schedule on the narrowed pools."""
    rng = np.random.default_rng(seed)
    waiting = rng.integers(0, 50, E).astype(np.int32) if waiting is None else np.asarray(waiting, np.int32)
    running = rng.integers(0, 50, E).astype(np.int32) if running is None else np.asarray(running, np.int32)
    kv = rng.random(E) if kv is None else np.asarray(kv, np.float64)
    total = np.full(R, 16, dtype=np.int32)
    match = np.zeros((R, E), dtype=np.int32)
    for r in range(R):
        hs = hits if hits is not None else rng.choice(E, size=min(E, 3), replace=False)
        for e in hs:
            match[r, e] = rng.integers(1, 17)
    in_len = rng.integers(1, 4096, R).astype(np.int64)
    n_ext = 0 if ext is None else np.asarray(ext).reshape(-1, E).shape[0]
    aff = None if affinity is None else epp.AffinityFilterSpec(*affinity)
    pspec = epp.ProfileSpec(primary_filter, [epp.ScorerSpec(*s) for s in scorers], aff, labels=reqs)
    fspec = None if pre_scorers is None else epp.ProfileSpec(pre_filter, [epp.ScorerSpec(*s) for s in pre_scorers],
                                                            labels=pre_reqs or [])
    with epp.Engine(E, pspec, fspec, non_cached_tokens=nct, n_ext_cols=n_ext) as eng:
        eng.pool_set(np.arange(E, dtype=np.uint32), role, kv, waiting, running, ext)
        eng.pool_set_labels(np.arange(E, dtype=np.uint32), labels)
        dec, det = eng.schedule_with_match(match, total, in_len, 16)
    keys, codes, comp = lm.compile_masks([reqs, pre_reqs or []])
    lc = lm.label_codes(keys, codes, labels)
    pd = lm.narrowed(orc, role, kv, waiting, running, ext, lm.keep_vector(comp[0], lc))
    pp = lm.narrowed(orc, role, kv, waiting, running, ext, lm.keep_vector(comp[1], lc))
    prim = orc.make_profile(primary_filter, list(scorers), affinity)
    pref = None if pre_scorers is None else orc.make_profile(pre_filter, list(pre_scorers))
    for r in range(R):
        m = lm.pd_schedule(orc, prim, pref, pd, pp, match[r], int(total[r]), 16, int(in_len[r]), nct)
        where = f"request {r}"
        assert dec["status"][r] == m["status"], where
        if m["status"] != 0:
            continue
        assert (int(dec["pick"][r]), int(dec["tie_count"][r]), int(dec["prefill_pick"][r])) == \
            (m["pick"], m["tie_count"], m["prefill_pick"]), where
        assert dec["score"][r].view(np.uint64) == np.float64(m["score"]).view(np.uint64), where
        assert int(det["prefill_ran"][r]) == m["prefill_ran"], where
        if m["prefill_pick"] != NO:
            assert det["prefill_score"][r].view(np.uint64) == np.float64(m["prefill_score"]).view(np.uint64), where
            assert int(det["prefill_tie_count"][r]) == m["prefill_tie_count"], where
    return dec, det


SC = [(2, 1.0, 0.0), (1, 1.0, 0.0), (0, 2.0, 0.0)]     # queue, kv, prefix


def test_custom_key_pd(epp, orc):
    """docs/disaggregation.md: P/D on labels the operator chooses, not llm-d.ai/role."""
    E = 97
    k = "example.com/stage"
    rng = np.random.default_rng(11)
    labels = [{k: v} if v else {} for v in rng.choice(["decode", "prefill", "", "other", None], E)]
    role = np.zeros(E, np.uint8)
    dec, det = model_case(epp, orc, E, labels, role, [(k, lm.IN, ["decode"])], SC, [(k, lm.IN, ["prefill"])], SC, nct=16)
    assert (det["prefill_ran"] == 1).any()


def test_lws_configuration(epp, orc):
    E = 64
    k = "leaderworkerset.sigs.k8s.io/worker-index"
    labels = [{k: str(e % 4)} if e % 5 else {} for e in range(E)]
    model_case(epp, orc, E, labels, np.zeros(E, np.uint8), [(k, lm.IN, ["0"])], SC, [(k, lm.DOES_NOT_EXIST, [])], SC, nct=8)
    model_case(epp, orc, E, labels, np.zeros(E, np.uint8), [(k, lm.NOT_IN, ["0"])], SC)


def test_multi_requirement_selectors_with_role(epp, orc):
    E = 150
    rng = np.random.default_rng(5)
    labels = [{kk: str(rng.integers(3)) for kk in ("a", "b", "c") if rng.random() < 0.6} for _ in range(E)]
    role = rng.choice([0, 1, 2, 3, 8], E).astype(np.uint8)
    reqs = [("a", lm.NOT_IN, ["1"]), ("b", lm.DOES_NOT_EXIST, []), ("c", lm.BY_LABEL, ["", "2"])]
    model_case(epp, orc, E, labels, role, reqs, SC, primary_filter=0)
    model_case(epp, orc, E, labels, role, reqs, SC, [("a", lm.EXISTS, []), ("c", lm.BY_LABEL_OR_ABSENT, ["0"])], SC,
               primary_filter=1, pre_filter=2, nct=4)


def test_zero_and_one_candidate(epp, orc):
    E = 40
    labels = [{"k": "one"} if e == 17 else {"k": "x"} for e in range(E)]
    role = np.zeros(E, np.uint8)
    dec, _ = model_case(epp, orc, E, labels, role, [("k", lm.IN, ["none"])], SC)
    assert (dec["status"] == -1).all()
    dec, _ = model_case(epp, orc, E, labels, role, [("k", lm.IN, ["one"])], SC, affinity=(0.3, 0.0, 5000.0, -1))
    assert (dec["pick"] == 17).all() and (dec["tie_count"] == 1).all()
    dec, det = model_case(epp, orc, E, labels, role, [("k", lm.IN, ["x"])], SC, [("k", lm.IN, ["none"])], SC, nct=1)
    assert (det["prefill_ran"] == 1).any() and (dec["prefill_pick"] == NO).all()


@pytest.mark.parametrize("E", [1, 1023, 131073])
def test_pool_sizes(epp, orc, E):
    labels = [{"z": str(e % 7)} if e % 11 else {} for e in range(E)]
    model_case(epp, orc, E, labels, np.zeros(E, np.uint8), [("z", lm.NOT_IN, ["3", "4"])], SC, R=8)


def leak_pool(E=48):
    """Slots 5 and 9 are dropped by every leak filter; they hold the pool's waiting / running extremes, the largest
    active count and the requests' only prefix hits.  Slots 20-29 have no label at all."""
    waiting = np.full(E, 10, np.int32)
    running = np.full(E, 10, np.int32)
    waiting[5], running[5], waiting[9], running[9] = 0, 1000, 1000, 0
    waiting[12], running[12] = 3, 17
    ext = np.full((1, E), 2.0)
    ext[0, 9] = 500.0
    ext[0, 12] = 7.0
    kv = np.linspace(0.1, 0.9, E)
    return waiting, running, ext, kv


LEAK_SCORERS = [(2, 1.0, 0.0), (5, 1.0, 0.0), (7, 1.0, 1.0, 0), (0, 1.0, 0.0)]


@pytest.mark.parametrize("form", ["notin", "bylabel_empty", "selector_in"])
def test_dropped_endpoint_holds_every_extreme(epp, orc, form):
    E = 48
    waiting, running, ext, kv = leak_pool(E)
    labels = []
    for e in range(E):
        if e in (5, 9):
            labels.append({"zone": "bad", "tier": "bad"})
        elif 20 <= e < 30:
            labels.append({})
        else:
            labels.append({"zone": "ok", "tier": "gold"})
    reqs = {"notin": [("zone", lm.NOT_IN, ["bad"])], "bylabel_empty": [("tier", lm.BY_LABEL, ["", "gold"])],
            "selector_in": [("zone", lm.IN, ["ok"])]}[form]
    dec, _ = model_case(epp, orc, E, labels, np.zeros(E, np.uint8), reqs, LEAK_SCORERS, waiting=waiting, running=running,
                        kv=kv, ext=ext, hits=[5, 9])
    assert not np.isin(dec["pick"], [5, 9]).any()
    if form != "selector_in":         # the unlabelled slots stay candidates
        assert dec["tie_count"].min() >= 1


def test_dropped_endpoint_with_inf_score(epp, orc):
    E = 32
    ext = np.zeros((1, E))
    ext[0, 3] = np.inf
    labels = [{"k": "drop"} if e == 3 else {"k": "keep"} for e in range(E)]
    dec, _ = model_case(epp, orc, E, labels, np.zeros(E, np.uint8), [("k", lm.IN, ["keep"])],
                        [(4, 1.0, 0.0), (0, 1.0, 0.0)], ext=ext)
    assert (dec["pick"] != 3).all()


def test_score_marks_dropped_slots(epp):
    E = 16
    labels = [{"k": "a"} if e % 2 else {} for e in range(E)]
    with epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(2, 1.0)], labels=[("k", lm.EXISTS, [])])) as eng:
        eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), np.zeros(E), np.arange(E), np.zeros(E))
        eng.pool_set_labels(np.arange(E, dtype=np.uint32), labels)
        s = eng.score(np.zeros((1, E), np.int32), np.zeros(1, np.int32))
    assert (s[0, ::2] == -1.0).all() and (s[0, 1::2] >= 0.0).all()


def test_nohit_lru_cold_slot_dropped(epp):
    """The least-recently-used no-hit-lru slot is dropped by the label filter: it never gets picked, and the LRU of a
    labelled engine equals the LRU of an engine whose pool lacks the dropped slots."""
    E = 24
    labels = [{"k": "drop"} if e in (0, 1) else {"k": "keep"} for e in range(E)]
    sc = [epp.ScorerSpec(9, 1.0, 6.0), epp.ScorerSpec(2, 1.0)]
    rng = np.random.default_rng(1)
    toks = rng.integers(0, 1000, (32, 64)).astype(np.uint32)
    with epp.Engine(E, epp.ProfileSpec(0, sc, labels=[("k", lm.IN, ["keep"])])) as a, epp.Engine(E, epp.ProfileSpec(0, sc)) as b:
        a.register_model(tg.MODEL)
        b.register_model(tg.MODEL)
        a.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), np.zeros(E), np.zeros(E), np.zeros(E))
        a.pool_set_labels(np.arange(E, dtype=np.uint32), labels)
        ids = np.arange(2, E, dtype=np.uint32)
        b.pool_set(ids, np.zeros(E - 2, np.uint8), np.zeros(E - 2), np.zeros(E - 2), np.zeros(E - 2))
        for i in range(4):
            da, _ = a.schedule(toks[i * 8:(i + 1) * 8], uniform_len=256)
            db, _ = b.schedule(toks[i * 8:(i + 1) * 8], uniform_len=256)
            same(da, db, f"call {i}")
            assert a.nohit_lru_get() == b.nohit_lru_get()
            assert not np.isin(da["pick"], [0, 1]).any()


# ---- D: snapshots ----------------------------------------------------------------------------------------------------
def test_snapshot_behaviour(epp):
    import torch
    E, w_len = 64, 256
    rng = np.random.default_rng(2)
    toks = rng.integers(0, 1000, (128, 64)).astype(np.uint32)
    v1 = [{"g": "a" if e < 32 else "b"} for e in range(E)]
    v2 = [{"g": "b" if e < 32 else "a"} for e in range(E)]
    sc = [epp.ScorerSpec(2, 1.0), epp.ScorerSpec(1, 1.0)]
    spec = epp.ProfileSpec(0, sc, labels=[("g", lm.IN, ["a"])])
    waiting = rng.integers(0, 9, E)
    kv = rng.random(E)

    def make(labels):
        eng = epp.Engine(E, spec)
        eng.register_model(tg.MODEL)
        eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), kv, waiting, np.zeros(E))
        eng.pool_set_labels(np.arange(E, dtype=np.uint32), labels)
        return eng

    e1, e2, x = make(v1), make(v2), make(v1)
    try:
        ref1, _ = e1.schedule(toks, uniform_len=w_len)
        ref2, _ = e2.schedule(toks, uniform_len=w_len)
        assert (ref1["pick"] < 32).all() and (ref2["pick"] >= 32).all()
        dt = torch.from_numpy(toks.view(np.int32)).cuda()
        d, _ = x.schedule(dt, uniform_len=w_len, asynchronous=True)
        x.pool_set_labels(np.arange(E, dtype=np.uint32), v2)          # after the enqueue: the batch keeps v1
        x.synchronize()
        same(epp.decisions_from_torch(d)["pick"], ref1["pick"], "async batch enqueued before the change")
        got, _ = x.schedule(toks, uniform_len=w_len)
        same(got["pick"], ref2["pick"], "after the change")
        x.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), kv, waiting, np.zeros(E))   # keeps v2
        got, _ = x.schedule(toks, uniform_len=w_len)
        same(got, e2.schedule(toks, uniform_len=w_len)[0], "pool_set alone keeps the labels")
    finally:
        for e in (e1, e2, x):
            e.close()


def test_no_requirement_engine_accepts_labels_unchanged(epp):
    E = 32
    rng = np.random.default_rng(4)
    toks = rng.integers(0, 1000, (16, 64)).astype(np.uint32)
    with epp.Engine(E) as a, epp.Engine(E) as b:
        for eng in (a, b):
            eng.register_model(tg.MODEL)
            eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), rng.random(E) * 0 + 0.5, np.arange(E), np.zeros(E))
        a.pool_set_labels(np.arange(E, dtype=np.uint32), [{"x": "y"}] * E)
        same(a.schedule(toks, uniform_len=256)[0], b.schedule(toks, uniform_len=256)[0], "no requirement")


# ---- E: rejections ---------------------------------------------------------------------------------------------------
def raw_labels(eng, ids, text_parts):
    ids = np.ascontiguousarray(ids, dtype=np.uint32)
    offs = np.zeros(len(text_parts) + 1, dtype=np.uint64)
    np.cumsum([len(p) for p in text_parts], out=offs[1:])
    text = np.frombuffer(b"".join(text_parts) + b"\0", dtype=np.uint8)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    return eng._lib.epp_pool_set_labels(eng._h, len(text_parts), p(ids), p(offs), p(text))


def test_every_rejection_leaves_state_unchanged(epp):
    E = 32
    rng = np.random.default_rng(9)
    toks = rng.integers(0, 1000, (16, 64)).astype(np.uint32)
    INV, ST = epp.capi.EPP_ERR_INVALID, epp.capi.EPP_ERR_STATE
    sc = [epp.ScorerSpec(2, 1.0)]
    eng = epp.Engine(E, epp.ProfileSpec(0, sc))
    eng.register_model(tg.MODEL)
    try:
        bad_sets = [
            (1, [("k", lm.IN, ["a"])]),                               # profile 1 is not configured
            (0, [("k", 6, [])]), (0, [("k", -1, [])]),                # unknown op
            (0, [("k", lm.IN, [])]), (0, [("k", lm.NOT_IN, [])]), (0, [("k", lm.BY_LABEL, [])]),
            (0, [("k", lm.EXISTS, ["a"])]), (0, [("k", lm.DOES_NOT_EXIST, ["a"])]),
            (0, [("", lm.EXISTS, [])]), (0, [("a=b", lm.EXISTS, [])]), (0, [("a\nb", lm.EXISTS, [])]),
            (0, [("k", lm.IN, ["a\nb"])]),
            (0, [("k", lm.EXISTS, [])] * 33),                        # over 32 requirements
            (0, [(f"k{i}", lm.EXISTS, []) for i in range(17)]),       # over 16 keys
            (0, [("k", lm.IN, [str(i) for i in range(63)])]),        # over 62 values
        ]
        for profile, reqs in bad_sets:
            with pytest.raises(epp.EngineError) as ei:
                eng.label_filters_set(profile, reqs)
            assert ei.value.code == INV, (profile, reqs[:1])
        eng.label_filters_set(0, [("k", lm.IN, ["a"])])
        eng.label_filters_set(0, [("k", lm.IN, ["b"])])               # replaces: only the last set counts
        eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), np.zeros(E), np.arange(E), np.zeros(E))
        eng.pool_set_labels(np.arange(E, dtype=np.uint32), [{"k": "b" if e % 2 else "a"} for e in range(E)])
        good, _ = eng.schedule(toks, uniform_len=256)
        assert (good["pick"] % 2 == 1).all()
        with pytest.raises(epp.EngineError) as ei:
            eng.label_filters_set(0, [("k", lm.IN, ["a"])])
        assert ei.value.code == ST
        ok = [b"k=a\n"] * 2
        for ids, parts in [([0, E], ok), ([3, 3], ok), ([0], [b"k\n"]), ([0], [b"k=a"]), ([0], [b"=a\n"]),
                           ([0], [b"k=a\nk=b\n"]), ([0], [b"x=1\nx=2\n"])]:
            assert raw_labels(eng, ids, parts) == INV, (ids, parts)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        ids = np.zeros(1, np.uint32)
        assert eng._lib.epp_pool_set_labels(eng._h, 1, p(ids), None, None) == INV
        assert eng._lib.epp_pool_set_labels(eng._h, -1, None, None, None) == INV
        offs = np.array([4, 0], np.uint64)
        txt = np.frombuffer(b"k=a\n", np.uint8)
        assert eng._lib.epp_pool_set_labels(eng._h, 1, p(ids), p(offs), p(txt)) == INV
        after, _ = eng.schedule(toks, uniform_len=256)
        same(after, good, "decisions after the rejected calls")
        assert raw_labels(eng, [0, 1], [b"k=b\nother=1\n", b""]) == 0       # valid: labels replaced
        got, _ = eng.schedule(toks, uniform_len=256)
        assert (got["pick"] == 0).all()
    finally:
        eng.close()
