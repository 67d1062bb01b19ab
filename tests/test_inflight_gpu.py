"""GPU parity of the inflight-load producer (csrc/inflight.cu and its update behind every scheduling call).  Before each
call the counters of tools/inflight_model.py go into a C-oracle run as ordinary ext columns (tokens = column 0, requests =
column 1); the call's decisions must equal the oracle's bit for bit, and epp_inflight_get must equal the model after it.
Releases and resets are made between the calls.  Paths the oracle does not restate (random pickers, no-hit-lru) are
compared against a twin engine without the producer whose ext columns are set to the model's counters before each call.
Run on an H100: pytest -m gpu."""
import dataclasses
import threading

import numpy as np
import pytest

import helpers
from tools import inflight_model as M

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
TL = (M.TOKEN_LOAD, 1.0, 65536.0, M.TOKEN_COL, 0.0)          # queueThresholdTokens 65536
AR = (M.ACTIVE_REQUEST, 2.0, 1.0, M.REQUEST_COL, 0.0)         # maxBusyScore 1, idleThreshold 0


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _workload(name, E, R, scorers=(TL, AR)):
    from tools import tracegen as tg
    w = tg.baseline_configs()[name].scaled(E=E, R=R, T=512)
    w = dataclasses.replace(w, primary_scorers=tuple(w.primary_scorers) + tuple(scorers))
    if w.prefill_scorers is not None:
        w = dataclasses.replace(w, prefill_scorers=tuple(w.prefill_scorers) + tuple(scorers))
    return w


def _ran(names, frag):
    return sum(c for n, c in names.items() if frag in n)


class Rig:
    """An engine with the producer, the oracle's index and profiles for the same workload, and the counters' model."""

    def __init__(self, epp, orc, w, *, tie_seed=0, pick_k=0, affinity=None, encode=None, role=None, pickers=(0, 0),
                 twin=False, inflight=True):
        from tools import tracegen as tg
        self.epp, self.orc, self.w = epp, orc, w
        self.tie_seed, self.pick_k, self.encode = tie_seed, pick_k, encode
        self.trace = tg.Trace(w)
        role0, kv, waiting, running = self.trace.pool()
        self.pool = [role0 if role is None else np.asarray(role, np.uint8), kv, waiting, running]
        aff = epp.AffinityFilterSpec(*affinity) if affinity else None
        primary = epp.ProfileSpec(w.primary_filter, [epp.ScorerSpec(*s) for s in w.primary_scorers], aff, pickers[0])
        prefill = None
        if w.prefill_scorers is not None:
            prefill = epp.ProfileSpec(tg.FILTER_PREFILL, [epp.ScorerSpec(*s) for s in w.prefill_scorers], None, pickers[1])
        enc = epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in encode]) if encode else None
        kw = dict(block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks,
                  non_cached_tokens=w.non_cached_tokens, tie_seed=tie_seed, pick_k=pick_k, encode=enc)
        self.eng = epp.Engine(w.E, primary, prefill, inflight_load=inflight, **kw)
        self.twin = epp.Engine(w.E, primary, prefill, n_ext_cols=2, **kw) if twin else None
        fam = self.trace.family_tokens()
        for e, ext in ((self.eng, None), (self.twin, np.zeros((2, w.E)))):
            if e is None:
                continue
            e.register_model(tg.MODEL)
            e.pool_set(np.arange(w.E, dtype=np.uint32), *self.pool, ext=ext)
            fh, _ = e.hash_prompts(fam, uniform_len=w.prompt_bytes)
            e.index_load_snapshot(*self.trace.index_pairs(fh))
        _, self.ix, _, _, _ = helpers.setup_oracle(orc, w, self.trace)
        self.prim = orc.make_profile(w.primary_filter, list(w.primary_scorers), affinity)
        self.pref = orc.make_profile(tg.FILTER_PREFILL, list(w.prefill_scorers)) if prefill is not None else None
        self.enc = orc.make_profile(0, list(encode)) if encode else None
        self.model = M.Counters(w.E)
        self.n_dec = 0
        self.rng = np.random.default_rng(0x1F1)

    def close(self):
        self.eng.close()
        if self.twin is not None:
            self.twin.close()

    def tokens(self, b, R=None):
        return self.trace.requests(b * self.w.R, R or self.w.R)[0]

    def expect(self, tokens, mm=None):
        """The oracle's decisions for the next call, against the model's counters as they stand now."""
        R = tokens.shape[0]
        pool = self.orc.PoolState(*self.pool, ext=self.model.ext())
        kw = dict(tie_seed=self.tie_seed, tie_base=self.n_dec)
        if self.enc is not None:
            kw.update(encode=self.enc, multimodal=mm)
        if self.pick_k > 1:
            kw["topk"] = self.pick_k
        self.n_dec += R
        return helpers.oracle_decisions(self.orc, self.w, pool, self.ix, self.prim, self.pref, tokens, **kw)

    def expect_twin(self, tokens):
        """The twin engine's decisions (host batch) with the model's counters as its ext columns."""
        self.twin.pool_set(np.arange(self.w.E, dtype=np.uint32), *self.pool, ext=self.model.ext())
        return self.twin.schedule(tokens, uniform_len=self.w.prompt_bytes)

    def add(self, dec, det, lengths=None):
        L = lengths if lengths is not None else [self.w.prompt_bytes] * len(dec)
        self.model.pre_request(dec, L, det if self.encode else None)

    def check_counters(self, where):
        req, tok = self.eng.inflight_get()
        np.testing.assert_array_equal(req, self.model.req, err_msg=where + " requests")
        np.testing.assert_array_equal(tok, self.model.tok, err_msg=where + " tokens")

    def churn(self, dec, det):
        """ResponseBody for a random half of the call's requests (every target released), a reset of one slot, and a
        release on that slot after it (the count goes negative)."""
        eps, lens = [], []
        for r in np.flatnonzero(self.rng.random(len(dec)) < 0.5):
            for e in self.model.targets(dec, det if self.encode else None, r):
                eps.append(e)
                lens.append(self.w.prompt_bytes)
        eps.append(NO)
        lens.append(7)
        self.eng.inflight_release(eps, lens)
        self.model.release(eps, lens)
        busy = int(np.argmax(self.model.req))
        self.eng.inflight_reset([busy])
        self.model.reset([busy])
        self.eng.inflight_release([busy], [13])
        self.model.release([busy], [13])


def _torch_out(epp, dec, det):
    import torch
    torch.cuda.synchronize()
    d = epp.decisions_from_torch(dec)
    dd = None if det is None else det.cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
    return d, dd


def _check(dec, det, want, where):
    helpers.assert_decisions_equal(dec, det, want[0], want[1], where=where)


# ---- the main parity check on every path the engine dispatches to ---------------------------------------------------
@pytest.mark.parametrize("path", ["device", "host_small", "host_chunked", "with_match"])
@pytest.mark.parametrize("name", ["config3", "config4"])
def test_parity_paths(epp, orc, name, path):
    import torch
    R = 2048 if path == "host_chunked" else 256              # > 1024 requests: the chunked host path
    w = _workload(name, 64, R)
    rig = Rig(epp, orc, w)
    kern = {"device": "k_match_pick_sparse", "host_small": "k_cycle_small", "host_chunked": "k_match_pick_sparse",
            "with_match": "k_dense_pick"}[path]
    try:
        for b in range(4):
            tokens = rig.tokens(b)
            if path == "with_match":
                match, total = rig.eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
            want = rig.expect(tokens)
            if path == "device":
                dt = torch.from_numpy(tokens.view(np.int32)).cuda()
                fn = lambda: rig.eng.schedule(dt, uniform_len=w.prompt_bytes)
            elif path == "with_match":
                fn = lambda: rig.eng.schedule_with_match(match, total, np.full(R, w.prompt_bytes, np.int64),
                                                         w.block_size_tokens)
            else:
                fn = lambda: rig.eng.schedule(tokens, uniform_len=w.prompt_bytes)
            (dec, det), names = helpers.kernels_launched(fn, repeatable=False)
            if path == "device":
                dec, det = _torch_out(epp, dec, det)
            _check(dec, det, want, f"{name} {path} batch {b}")
            if helpers.trace_complete(names):
                assert _ran(names, "k_inflight_add") == 1 and _ran(names, kern) > 0, sorted(names)
                if path == "host_chunked":
                    assert _ran(names, "k_cycle_small") == 0
            rig.add(dec, det)
            rig.check_counters(f"{name} {path} after batch {b}")
            if b % 2 == 0:                   # the call after an odd batch sees only that batch's adds
                rig.churn(dec, det)
        rig.check_counters(f"{name} {path} after the releases")
        if path == "device":
            assert rig.eng.stats()["last_kernel_ms"][5] > 0
    finally:
        rig.close()


def test_parity_zero_copy_small_batches(epp, orc):
    w = _workload("config3", 64, 8)
    rig = Rig(epp, orc, w)
    try:
        for b in range(6):
            tokens = rig.tokens(b)
            buf = epp.PinnedBuffer(tokens.nbytes + 64)
            buf.array[: tokens.nbytes] = tokens.reshape(-1).view(np.uint8)
            want = rig.expect(tokens)
            (dec, det), names = helpers.kernels_launched(
                lambda: rig.eng.schedule(buf.array, uniform_len=w.prompt_bytes, n_requests=w.R), repeatable=False)
            _check(dec, det, want, f"zero-copy batch {b}")
            if helpers.trace_complete(names):
                assert _ran(names, "k_cycle_small") == 1 and _ran(names, "k_inflight_add") == 1
            rig.add(dec, det)
            rig.check_counters(f"zero-copy batch {b}")
            rig.churn(dec, det)
            buf.close()
    finally:
        rig.close()


def test_pipelined_async_batches(epp, orc):
    """Three two-chunk pipelined batches with releases between the enqueues and one epp_synchronize: each batch sees the
    adds of the ones before it and the releases made before it was called.  The first chunk's prompts are one block long
    and the second chunk's are whole, so the second chunk (stream 1) finishes well after the first (stream 0): an update
    that did not wait for stream 1 would miss its decisions, and a next batch whose stream-1 chunk did not wait for the
    update would score against stale counters."""
    import torch
    from tools import tracegen as tg
    w = _workload("config3", 64, 8192)
    rig = Rig(epp, orc, w)
    R, L = w.R, w.prompt_bytes
    lens = np.where(np.arange(R) < R // 2, 4 * w.block_size_tokens, L).astype(np.uint64)
    offs = np.zeros(R + 1, np.uint64)
    np.cumsum(lens, out=offs[1:])
    try:
        datas, wants, rels = [], [], []
        for b in range(3):
            rows = rig.tokens(b).view(np.uint8)
            data = np.concatenate([rows[r, : int(lens[r])] for r in range(R)])
            datas.append(data)
            pool = orc.PoolState(*rig.pool, ext=rig.model.ext())
            want = orc.cycle_batch(tg.MODEL, w.block_size_tokens, w.max_prefix_blocks, w.non_cached_tokens, False, rig.ix,
                                   rig.prim, rig.pref, pool, data, offs, 4, tie_seed=0, tie_base=rig.n_dec)
            rig.n_dec += R
            wants.append(want)
            rig.add(want[0], None, lengths=lens)
            eps = [int(e) & NO for e in want[0]["pick"][::3]]
            rels.append(eps)
            rig.model.release(eps, [L] * len(eps))
        dts = [torch.from_numpy(d).cuda() for d in datas]
        d_offs = torch.from_numpy(offs.view(np.int64)).cuda()
        torch.cuda.synchronize()

        def run():
            outs = []
            for dt, eps in zip(dts, rels):
                outs.append(rig.eng.schedule(dt, offsets=d_offs, asynchronous=True, detail=False))
                rig.eng.inflight_release(eps, [L] * len(eps))
            rig.eng.synchronize()
            return outs
        outs, names = helpers.kernels_launched(run, repeatable=False)
        for b, (dec, _) in enumerate(outs):
            _check(epp.decisions_from_torch(dec), None, wants[b], f"pipelined batch {b}")
        rig.check_counters("after the pipelined batches")
        if helpers.trace_complete(names):
            assert _ran(names, "k_hash_fused") == 6 and _ran(names, "k_inflight_add") == 3
    finally:
        rig.close()


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
def test_pd_encode(epp, orc, tie_seed):
    """P/D + encode.  Half the pool is prefill-decode, so a request's decode and prefill pick can be the same slot (it
    counts twice)."""
    from tools import tracegen as tg
    w = _workload("config4", 64, 256)
    role = tg.Trace(w).pool()[0].copy()
    role[: w.E // 2] = 3                              # EPP_ROLE_PREFILL_DECODE
    rig = Rig(epp, orc, w, tie_seed=tie_seed, encode=[(2, 1.0, 0.0), (0, 2.0, 0.0), TL, AR], role=role)
    same = 0
    try:
        for b in range(4):
            tokens = rig.tokens(b)
            mm = (rig.rng.random(w.R) < 0.5).astype(np.uint8)
            want = rig.expect(tokens, mm)
            dec, det = rig.eng.schedule(tokens, uniform_len=w.prompt_bytes, multimodal=mm)
            _check(dec, det, want, f"P/D + encode batch {b}")
            same += int(((dec["pick"] == dec["prefill_pick"]) & (dec["status"] == 0)).sum())
            assert (det["encode_pick"] != NO).any()
            rig.add(dec, det)
            rig.check_counters(f"P/D + encode after batch {b}")
            rig.churn(dec, det)
        assert same > 0
        rig.check_counters("P/D + encode after the releases")
    finally:
        rig.close()


def test_topk_and_affinity_filter(epp, orc):
    """pick_k = 4 (only entry 0 of each list counts) with a prefix-cache-affinity-filter (the active-request max is taken
    over the narrowed set)."""
    import torch
    w = _workload("config3", 64, 256)
    rig = Rig(epp, orc, w, pick_k=4, affinity=(0.5, 0.0, 0.0))
    try:
        for b in range(4):
            tokens = rig.tokens(b)
            odec, ototal, olists = rig.expect(tokens)
            dt = torch.from_numpy(tokens.view(np.int32)).cuda()
            (dec, det, lists), names = helpers.kernels_launched(
                lambda: rig.eng.schedule(dt, uniform_len=w.prompt_bytes, topk=True), repeatable=False)
            dec, det = _torch_out(epp, dec, det)
            _check(dec, det, (odec, ototal), f"top-k batch {b}")
            np.testing.assert_array_equal(lists["primary"].cpu().numpy(), olists["primary"], err_msg=f"top-k lists batch {b}")
            if helpers.trace_complete(names):
                assert _ran(names, "k_match_pick(") > 0 and _ran(names, "k_inflight_add") == 1
            rig.add(dec, det)
            rig.check_counters(f"top-k after batch {b}")
            rig.churn(dec, det)
    finally:
        rig.close()


def test_status_minus_one_adds_nothing(epp, orc):
    """A pool with no decode candidate: every request is a Schedule error and the counters stay as they are."""
    from tools import tracegen as tg
    w = dataclasses.replace(_workload("config3", 32, 64), primary_filter=tg.FILTER_DECODE)
    rig = Rig(epp, orc, w, role=np.full(32, 2, np.uint8))         # every endpoint prefill-only
    try:
        rig.eng.inflight_release([3, 5], [16, 16])
        rig.model.release([3, 5], [16, 16])
        tokens = rig.tokens(0)
        want = rig.expect(tokens)
        dec, det = rig.eng.schedule(tokens, uniform_len=w.prompt_bytes)
        assert (dec["status"] == -1).all()
        _check(dec, det, want, "status -1")
        rig.check_counters("status -1")
    finally:
        rig.close()


# ---- paths the oracle does not restate: the twin engine is the yardstick ---------------------------------------------
def _twin_compare(dec, det, tdec, tdet, where):
    for f in ("status", "pick", "prefill_pick", "tie_count", "match_blocks"):
        np.testing.assert_array_equal(dec[f], tdec[f], err_msg=f"{where} {f}")
    np.testing.assert_array_equal(dec["score"].view(np.uint64), tdec["score"].view(np.uint64), err_msg=where + " score")
    np.testing.assert_array_equal(det["encode_pick"], tdet["encode_pick"], err_msg=where + " encode")


@pytest.mark.parametrize("kind", ["random_pickers", "nohit_lru"])
def test_twin_engine_paths(epp, orc, kind):
    import torch
    if kind == "random_pickers":
        w = _workload("config4", 64, 256)
        rig = Rig(epp, orc, w, tie_seed=0x77, pickers=(2, 1), twin=True)      # weighted-random decode, random prefill
        kern = "_rand"
    else:
        w = _workload("config3", 64, 256, scorers=(TL, AR, (9, 1.0, 0.0)))
        rig = Rig(epp, orc, w, twin=True)
        kern = "_nohit"
    try:
        for b in range(4):
            tokens = rig.tokens(b)
            tdec, tdet = rig.expect_twin(tokens)
            dt = torch.from_numpy(tokens.view(np.int32)).cuda()
            (dec, det), names = helpers.kernels_launched(lambda: rig.eng.schedule(dt, uniform_len=w.prompt_bytes),
                                                         repeatable=False)
            dec, det = _torch_out(epp, dec, det)
            _twin_compare(dec, det, tdec, tdet, f"{kind} batch {b}")
            if helpers.trace_complete(names):
                assert _ran(names, kern) > 0 and _ran(names, "k_inflight_add") == 1
            rig.add(dec, det)
            rig.check_counters(f"{kind} after batch {b}")
            if b % 2 == 0:
                rig.churn(dec, det)
        if kind == "nohit_lru":
            assert rig.eng.nohit_lru_get() == rig.twin.nohit_lru_get()
    finally:
        rig.close()


def test_counters_alone_change_no_decision(epp, orc):
    """Switch on, no token-load / active-request scorer: the same decisions as with the switch off, the add kernel alone."""
    import torch
    w = _workload("config3", 64, 256, scorers=())
    on, off = Rig(epp, orc, w), Rig(epp, orc, w, inflight=False)
    try:
        for b in range(3):
            dt = torch.from_numpy(on.tokens(b).view(np.int32)).cuda()
            (d1, t1), names = helpers.kernels_launched(lambda: on.eng.schedule(dt, uniform_len=w.prompt_bytes),
                                                       repeatable=False)
            d2, t2 = off.eng.schedule(dt, uniform_len=w.prompt_bytes)
            d1, t1 = _torch_out(epp, d1, t1)
            d2, t2 = _torch_out(epp, d2, t2)
            _twin_compare(d1, t1, d2, t2, f"counters alone batch {b}")
            if helpers.trace_complete(names):
                assert _ran(names, "k_inflight_add") == 1 and _ran(names, "k_inflight_columns") == 0
            on.add(d1, t1)
            on.check_counters(f"counters alone batch {b}")
        assert off.eng.stats()["last_kernel_ms"][5] == 0
    finally:
        on.close()
        off.close()


# ---- the batcher ------------------------------------------------------------------------------------------------------
def test_batcher_threads(epp, orc):
    w = _workload("config3", 64, 64)
    rig = Rig(epp, orc, w)
    rng = np.random.default_rng(5)
    toks = rig.tokens(0, 64 * 4)
    lens = rng.integers(1, w.prompt_bytes // 4 + 1, size=toks.shape[0]) * 4 - rng.integers(0, 4, size=toks.shape[0])
    got = [None] * toks.shape[0]
    try:
        with epp.Batcher(rig.eng, max_batch=48, max_delay_us=100) as bt:
            def worker(t):
                for i in range(t, toks.shape[0], 64):
                    got[i] = bt.schedule(toks[i].view(np.uint8)[: lens[i]].tobytes())
            th = [threading.Thread(target=worker, args=(t,)) for t in range(64)]
            for x in th:
                x.start()
            for x in th:
                x.join()
        dec = np.array([g[0] for g in got], dtype=epp.DECISION_DTYPE)
        det = np.array([g[1] for g in got], dtype=epp.DETAIL_DTYPE)
        assert (dec["status"] == 0).all()
        rig.add(dec, det, lengths=lens)
        rig.check_counters("after the batcher")
    finally:
        rig.close()


# ---- calls that never update, errors, scale ---------------------------------------------------------------------------
def test_score_match_and_hash_never_update(epp, orc):
    w = _workload("config3", 64, 128)
    rig = Rig(epp, orc, w)
    try:
        tokens = rig.tokens(0)
        dec, det = rig.eng.schedule(tokens, uniform_len=w.prompt_bytes)
        rig.add(dec, det)
        rig.check_counters("after schedule")
        match, total = rig.eng.prefix_match(tokens, uniform_len=w.prompt_bytes)
        rig.eng.score(match, total, 0, -1)
        rig.eng.hash_prompts(tokens, uniform_len=w.prompt_bytes)
        rig.check_counters("after score / prefix_match / hash_prompts")
    finally:
        rig.close()


def test_errors(epp, orc):
    w = _workload("config3", 16, 8)
    rig = Rig(epp, orc, w)
    w_plain = _workload("config3", 16, 8, scorers=())
    try:
        with pytest.raises(epp.EngineError) as ei:
            rig.eng.inflight_release([16], [4])
        assert ei.value.code == epp.capi.EPP_ERR_INVALID
        with pytest.raises(epp.EngineError) as ei:
            rig.eng.inflight_reset([1 << 20])
        assert ei.value.code == epp.capi.EPP_ERR_INVALID
        rig.check_counters("a rejected call changes nothing")
        with pytest.raises(epp.EngineError) as ei:
            rig.eng.shard_set(0, 8)
        assert ei.value.code == epp.capi.EPP_ERR_INVALID
    finally:
        rig.close()
    off = Rig(epp, orc, w_plain, inflight=False)
    try:
        for fn in (lambda: off.eng.inflight_release([1], [4]), lambda: off.eng.inflight_reset([1]), off.eng.inflight_get):
            with pytest.raises(epp.EngineError) as ei:
                fn()
            assert ei.value.code == epp.capi.EPP_ERR_STATE
    finally:
        off.close()
    with pytest.raises(epp.EngineError):        # the columns are validated when the switch is off
        epp.Engine(16, epp.ProfileSpec(0, [epp.ScorerSpec(*TL)]))
    epp.Engine(16, epp.ProfileSpec(0, [epp.ScorerSpec(*TL)]), inflight_load=True).close()


def test_scale_every_pick_on_one_slot(epp, orc):
    """A cold config-3 batch of 8192 requests on a uniform pool under the lowest-slot rule: every pick lands on one slot,
    which the add kernel's aggregated atomics must count exactly."""
    import torch
    w = _workload("config3", 256, 8192)
    E = w.E
    rig = Rig(epp, orc, w)
    try:
        rig.eng.pool_set(np.arange(E, dtype=np.uint32), np.zeros(E, np.uint8), np.zeros(E), np.zeros(E, np.int32),
                         np.zeros(E, np.int32))
        tokens = np.random.default_rng(9).integers(1 << 20, 1 << 30, size=rig.tokens(0).shape).astype(np.uint32)  # cold
        dt = torch.from_numpy(tokens.view(np.int32)).cuda()
        dec, det = _torch_out(epp, *rig.eng.schedule(dt, uniform_len=w.prompt_bytes))
        assert (dec["status"] == 0).all() and len(set(dec["pick"].tolist())) == 1
        rig.add(dec, det)
        rig.check_counters("one slot")
        assert rig.model.req.max() == 8192
    finally:
        rig.close()


def test_plugins_producer(epp):
    """plugins.InFlightLoadProducer over plugins.Scheduler: a pick raises the target's load, ResponseBody at the end of
    the stream takes it off again, DeleteEndpoint clears it."""
    from epp_b200 import plugins as P
    eps = [P.NewEndpoint(P.EndpointMetadata(n)) for n in ("a", "b", "c")]
    prof = P.NewSchedulerProfile().WithScorers(P.NewWeightedScorer(P.TokenLoadScorer(), 1.0),
                                               P.NewWeightedScorer(P.NewActiveRequest(), 1.0))
    sched = P.Scheduler(P.SingleProfileHandler(), {"default": prof}, max_endpoints=3, inflight_load=True)
    prod = P.InFlightLoadProducer(sched)
    reqs = [P.InferenceRequest(Prompt=b"x" * 16) for _ in range(3)]
    names = []
    for r in reqs:                                   # one at a time: each pick sees the ones before it
        r.SchedulingResult = sched.Schedule(r, eps)
        names.append(r.SchedulingResult.ProfileResults["default"].TargetEndpoints[0].GetMetadata().Name)
    assert names == ["a", "b", "c"]
    assert prod.Get(0) == (1, 10)
    prod.ResponseBody(reqs[0], start_of_stream=True)             # no prefill profile: nothing released yet
    assert prod.Get(0) == (1, 10)
    prod.ResponseBody(reqs[0], end_of_stream=True)
    assert prod.Get(0) == (0, 0)
    prod.DeleteEndpoint(1)
    assert prod.Get(1) == (0, 0)
    prod.ResponseBody(reqs[1], end_of_stream=True)
    assert prod.Get(1) == (-1, -10)
    sched.engine.close()
