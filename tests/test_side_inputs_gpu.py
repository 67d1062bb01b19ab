"""Scheduling calls that carry every side input at once -- endpoint subsets, latency predictions, context lengths and
admission rows -- on the GPU, against tools/context_length_model.py (over tools/latency_model.py) and
tools/admission_model.py, bit for bit: status, pick, score bits, tie count, match_blocks, the prefill fields, the first-k
lists with their scores, and the in-flight counters after the calls.  An expected row is the context-length model's
decision (latency chain, the row's predictions, its subset as `keep`) with the admission model's result applied at the
call's ordinal base.

The calls go through the one staged upload of a call's side inputs (engine.cu check_inputs / stage_inputs): every path,
the section layouts of tests/test_side_inputs_cpu.py, calls that change the input set and size on one engine (also
enqueued back to back as async device batches, two chunk-pipelined ones among them), a refused call between two good
ones, and batcher flushes whose rows mix every kind.  Large calls are compared byte for byte with a twin engine and
model-checked on a sample: every rejected row, every subset row, the rows around each chunk boundary and 200 random
rows."""
from __future__ import annotations

import ctypes as C
import importlib

import numpy as np
import pytest

import test_side_inputs_cpu as c
from tools import context_length_model as cm

pytestmark = pytest.mark.gpu

E, PB = c.E, c.PB
PIPE_R = 8192 + 544


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


def _mod():
    return importlib.import_module("llm-d-inference-scheduler_b200.engine")


def _specs(epp):
    p, q = c.PRIMARY, c.PREFILL
    prim = epp.ProfileSpec(0, [epp.ScorerSpec(k, w, pa) for k, w, pa in p["scorers"]], epp.AffinityFilterSpec(*p["a2"]),
                           0, latency=dict(p["lcfg"]), context_length=dict(label=None, enable_filtering=True))
    pre = epp.ProfileSpec(0, [epp.ScorerSpec(k, w, pa) for k, w, pa in q["scorers"]], None, 0,
                          context_length=dict(label=None, enable_filtering=False))
    return prim, pre


def set_pool(eng, w):
    role, kv, waiting, running = w.pool
    ids = np.flatnonzero(role != 0xFF).astype(np.uint32)
    eng.pool_set(ids, role[ids], kv[ids], waiting[ids], running[ids])
    eng.pool_set_labels(np.arange(E, dtype=np.uint32), w.labels)


def chain_engine(epp, w):
    """Context-length filter and scorer, latency scorer behind the tier filter, both admitters, the inflight-load
    producer, pick_k = 4 and a P/D prefill profile."""
    prim, pre = _specs(epp)
    eng = epp.Engine(E, prim, pre, tie_seed=c.SEED, pick_k=c.K, block_size_tokens=16, max_prefix_blocks=16,
                     non_cached_tokens=c.NCT, inflight_load=True)
    eng.register_model(b"m")
    eng.admission_set(**c.ACFG)
    set_pool(eng, w)
    return eng


def load(eng, w, data, offsets=None, uniform_len=None):
    """The snapshot that gives the prompts the world's match counts; checked through prefix_match."""
    h, nb = eng.hash_prompts(data, offsets=offsets, uniform_len=uniform_len)
    R = nb.shape[0]
    match = w.match[:R]
    rs, es = np.nonzero(match)
    hs = np.concatenate([h[r, :match[r, e]] for r, e in zip(rs, es)])
    eps = np.repeat(es.astype(np.uint32), match[rs, es])
    eng.index_load_snapshot(hs, eps)
    got, total = eng.prefix_match(data, offsets=offsets, uniform_len=uniform_len)
    assert np.array_equal(got, match) and np.array_equal(total, w.total[:R])


def prompts_of(R, seed):
    return np.random.default_rng(seed).integers(0, 256, (R, PB)).astype(np.uint8)


def host_out(epp, out):
    dec = epp.decisions_from_torch(out[0])
    det = out[1].cpu().numpy().view(epp.DETAIL_DTYPE).reshape(-1)
    lists = {n: v.cpu().numpy().view(np.uint32 if n != "primary_scores" else np.float64) for n, v in out[2].items()}
    return dec, det, lists


def same(a, b, what):
    assert a[0].tobytes() == b[0].tobytes(), f"{what}: decisions"
    assert a[1].tobytes() == b[1].tobytes(), f"{what}: details"
    for n in ("primary", "primary_scores", "prefill", "encode"):
        assert a[2][n].tobytes() == b[2][n].tobytes(), f"{what}: {n}"


def check_call(orc, w, inp, out, base, rows=None, row0=0, in_len=None, with_subsets=True):
    """-> the model's rejected rows of the call."""
    dec, det, lists = out
    rej = c.rejected(w, inp, base, with_subsets=with_subsets)
    for r in (range(inp.R) if rows is None else rows):
        m = c.decide_row(orc, w, inp, r, base, row=row0 + r, in_len=None if in_len is None else in_len[r])
        c.check_row(m, bool(rej[r]), r, w.match[row0 + r], dec, det, lists)
    return rej


def check_counters(eng, calls):
    req, tok = eng.inflight_get()
    want = c.counters_after(E, calls)
    assert np.array_equal(req, want.req) and np.array_equal(tok, want.tok)


def structs(epp, inp, R):
    """The C records of a call's side inputs (None when absent) and the arrays they point to."""
    m = _mod()
    sub = pr = ct = ad = None
    hold = []
    if inp.subsets is not None:
        sp = epp.pack_subsets(inp.subsets)
        sub = epp.capi.Subset()
        sub.struct_size = C.sizeof(epp.capi.Subset)
        sub.counts, sub.offsets, sub.slots = (m._ptr(a) for a in sp)
        hold.append(sp)
    if inp.preds is not None:
        pp = epp.pack_predictions(inp.preds)
        pr = m._predictions_struct(pp)
        hold.append(pp)
    if inp.ctx is not None:
        ct, a = m._context_struct(inp.ctx, R)
        hold.append(a)
    if inp.adm:
        ad, a = m._admission_struct(inp.admission(), R, inp.preds)
        hold.append(a)
    return (sub, pr, ct, ad), hold


def ref(x):
    return None if x is None else C.byref(x)


def direct(epp, eng, data, inp, offsets=None, uniform_len=None, lengths=None, flags=0, bad_adm=False):
    """epp_schedule_admit on a host or (synchronous) device batch with each input passed only when present ->
    (rc, (dec, det, lists)) on the host."""
    m = _mod()
    b, R, dev, keep = eng._batch(data, offsets, uniform_len, None, None, lengths, None)
    b.flags |= flags
    if dev:
        import torch
        dec = torch.zeros((R, 32), dtype=torch.uint8, device=data.device)
        det = torch.zeros((R, 40), dtype=torch.uint8, device=data.device)
        torch.cuda.synchronize()
    else:
        dec = np.zeros(R, epp.DECISION_DTYPE)
        det = np.zeros(R, epp.DETAIL_DTYPE)
    lists, tk = eng._topk_out(R, data.device if dev else None)
    (sub, pr, ct, ad), hold = structs(epp, inp, R)
    if bad_adm:
        ad.struct_size += 8
    rc = eng._lib.epp_schedule_admit(eng._h, C.byref(b), ref(sub), ref(pr), ref(ct), ref(ad), m._ptr(dec), m._ptr(det), 0,
                                     C.byref(tk))
    if dev:
        torch.cuda.synchronize()
        return rc, host_out(epp, (dec, det, lists))
    return rc, (dec, det, lists)


def with_match_device(epp, eng, w, inp):
    """epp_schedule_with_match_admit with EPP_BATCH_DEVICE_PTRS: match, totals, lengths and outputs are CUDA tensors."""
    import torch
    m = _mod()
    R = inp.R
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    match, total, il = cuda(w.match[:R]), cuda(w.total[:R]), cuda(w.in_len[:R])
    dec = torch.zeros((R, 32), dtype=torch.uint8, device="cuda")
    det = torch.zeros((R, 40), dtype=torch.uint8, device="cuda")
    lists, tk = eng._topk_out(R, match.device)
    (_, pr, ct, ad), hold = structs(epp, inp, R)
    torch.cuda.synchronize()
    eng._check(eng._lib.epp_schedule_with_match_admit(eng._h, R, m._ptr(match), m._ptr(total), None, m._ptr(il), 0,
                                                      m._ptr(dec), m._ptr(det), epp.capi.EPP_BATCH_DEVICE_PTRS,
                                                      C.byref(tk), ref(pr), ref(ct), ref(ad)))
    torch.cuda.synchronize()
    return host_out(epp, (dec, det, lists))


def no_subsets(inp):
    return c.Inputs(inp.R, None, inp.preds, inp.valid, inp.ctx, inp.prio, inp.ttft, inp.tpot)


# ---- 1. all four inputs in one call, every path -----------------------------------------------------------------
@pytest.mark.parametrize("path", ["host", "device", "async", "with_match", "with_match_device"])
def test_all_four_every_path(epp, orc, path):
    import torch
    R = 203
    w = c.World(3, R)
    inp = c.full_inputs(R, 21, w.pool)
    with chain_engine(epp, w) as eng:
        prompts = prompts_of(R, 4)
        load(eng, w, prompts, uniform_len=PB)
        if path == "host":
            out = eng.schedule(prompts, uniform_len=PB, topk=True, **inp.kwargs())
        elif path in ("device", "async"):
            data = torch.from_numpy(prompts).cuda()
            res = eng.schedule(data, uniform_len=PB, topk=True, asynchronous=path == "async", **inp.kwargs())
            eng.synchronize()
            torch.cuda.synchronize()
            out = host_out(epp, res)
        elif path == "with_match":
            inp = no_subsets(inp)
            out = eng.schedule_with_match(w.match[:R], w.total[:R], input_len_bytes=w.in_len[:R], topk=True,
                                          predictions=inp.preds, context_tokens=inp.ctx, admission=inp.admission())
        else:
            inp = no_subsets(inp)
            out = with_match_device(epp, eng, w, inp)
        rej = check_call(orc, w, inp, out, 0)
        assert rej.any() and (~rej[inp.prio < 0]).any()
        assert eng.stats()["n_decisions"] == R
        check_counters(eng, [(out[0], out[1], w.in_len[:R])])


def plain_decide(orc, w, inp, r, base):
    role, kv, waiting, running = w.pool
    m = cm.profile_decide(orc, 0, PLAIN_SCORERS, 0, role, kv, waiting, running, w.match[r], int(w.total[r]),
                          [None] * E, c.ctx_of(inp, r, PB), False, {}, None, None, c.SEED, 4 * (base + r), 1)
    return dict(primary=m, prefill=None, go=False)


PLAIN_SCORERS = [(c.QUEUE, 2.0, 0.0), (c.KV, 2.0, 0.0), (c.PREFIX, 3.0, 0.0)]


@pytest.mark.parametrize("R", [1, 8, 9])
def test_plain_engine_small_batches(epp, orc, R):
    """Admitters only: sheddable rows send a small batch to the chunked host path, rows without any (context lengths
    accepted and ignored) keep the single-launch path -- from pinned and from pageable memory, on both sides of the
    zero-copy limit (8 requests)."""
    w = c.World(5, 9)
    mk = lambda: epp.Engine(E, epp.ProfileSpec(0, [epp.ScorerSpec(k, wt, pa) for k, wt, pa in PLAIN_SCORERS]),  # noqa: E731
                            tie_seed=c.SEED, block_size_tokens=16, max_prefix_blocks=16)
    base, eng = mk(), mk()
    eng.admission_set(**c.ACFG)
    prompts = prompts_of(R, 6)
    pinned = epp.PinnedBuffer(R * PB)
    pinned.array[:] = prompts.reshape(-1)
    with base, eng:
        for e in (base, eng):
            e.register_model(b"m")
            set_pool(e, w)
            load(e, w, prompts, uniform_len=PB)
        for mem, data in (("pinned", pinned.array.reshape(R, PB)), ("pageable", prompts)):
            for shed in (True, False):
                inp = c.side_inputs(R, 40 + R + shed, w.pool, pred=list(range(R)), ctx=True,
                                    shed=list(range(0, R, 2)) if shed else [])
                if not shed:
                    inp.preds = inp.valid = None
                b0 = eng.stats()["n_decisions"]
                base.schedule(data, uniform_len=PB)
                got = eng.schedule(data, uniform_len=PB, **inp.kwargs())
                small = eng.stats()["last_kernel_launches"] == base.stats()["last_kernel_launches"]
                assert small != shed, (mem, shed)
                rej = c.rejected(w, inp, b0, with_subsets=False)
                for r in range(R):
                    c.check_row(plain_decide(orc, w, inp, r, b0), bool(rej[r]), r, w.match[r], got[0], got[1], None)
    pinned.close()


# ---- 2. section packing --------------------------------------------------------------------------------------------
def test_section_packing(epp, orc):
    import torch
    w = c.World(3, 37)
    prompts = prompts_of(37, 8)
    data = torch.from_numpy(prompts).cuda()
    with chain_engine(epp, w) as eng:
        load(eng, w, prompts, uniform_len=PB)
        calls, base = [], 0
        for name, inp, pat in c.packing_calls(w.pool):
            assert c.pattern(c.layout(inp)[0]) == pat
            for batch in (prompts, data):              # a host batch, then a device batch
                rc, out = direct(epp, eng, batch, inp, uniform_len=PB)
                assert rc == 0, (name, eng._lib.epp_last_error())
                check_call(orc, w, inp, out, base)
                calls.append((out[0], out[1], w.in_len[:37]))
                base += 37
        check_counters(eng, calls)


# ---- 3. consecutive calls on one engine -----------------------------------------------------------------------------
def test_consecutive_host_calls(epp, orc):
    seq = c.sequence_calls(c.make_pool(3))
    R = max(inp.R for _, inp in seq)
    w = c.World(3, R)
    prompts = prompts_of(R, 9)
    with chain_engine(epp, w) as eng:
        load(eng, w, prompts, uniform_len=PB)
        base, calls = 0, []
        for name, inp in seq:
            out = eng.schedule(prompts[:inp.R], uniform_len=PB, topk=True, **inp.kwargs())
            check_call(orc, w, inp, out, base)
            base += inp.R
            calls.append((out[0], out[1], w.in_len[:inp.R]))
            check_counters(eng, calls)


def pipelined_calls(pool):
    R = PIPE_R
    return [("pipelined, all four", c.full_inputs(R, 31, pool)),
            ("pipelined, subsets and context lengths", c.side_inputs(R, 32, pool, sub=c.every(R, 3, 1), ctx=True))]


def test_back_to_back_async_calls(epp, orc):
    """The sequence, then two chunk-pipelined calls with different inputs, enqueued as async device batches without a
    synchronisation in between (the staging is refilled and regrown while the call before is in flight), against a
    twin engine making the same calls on the host path."""
    import torch
    w = c.World(3, PIPE_R)
    seq = c.sequence_calls(w.pool) + pipelined_calls(w.pool)
    prompts = prompts_of(PIPE_R, 10)
    data = torch.from_numpy(prompts).cuda()
    with chain_engine(epp, w) as eng, chain_engine(epp, w) as twin:
        for e in (eng, twin):
            load(e, w, prompts, uniform_len=PB)
        outs = [eng.schedule(data[:inp.R], uniform_len=PB, topk=True, asynchronous=True, **inp.kwargs()) for _, inp in seq]
        want = [twin.schedule(prompts[:inp.R], uniform_len=PB, topk=True, **inp.kwargs()) for _, inp in seq]
        eng.synchronize()
        torch.cuda.synchronize()
        base, calls = 0, []
        for (name, inp), o, h in zip(seq, outs, want):
            got = host_out(epp, o)
            same(got, h, name)
            rows = None
            if inp.R == PIPE_R:
                rows = c.pipelined_sample(inp, c.rejected(w, inp, base))
            check_call(orc, w, inp, got, base, rows=rows)
            base += inp.R
            calls.append((got[0], got[1], w.in_len[:inp.R]))
        check_counters(eng, calls)
        check_counters(twin, calls)


# ---- 4. a refused call between two good ones ------------------------------------------------------------------------
def test_refused_call_between_good_ones(epp, orc):
    w = c.World(3, 160)
    prompts = prompts_of(160, 11)
    first = c.full_inputs(160, 41, w.pool)
    second = c.full_inputs(97, 42, w.pool)
    with chain_engine(epp, w) as eng:
        load(eng, w, prompts, uniform_len=PB)
        out = eng.schedule(prompts, uniform_len=PB, topk=True, **first.kwargs())
        check_call(orc, w, first, out, 0)
        calls = [(out[0], out[1], w.in_len[:160])]
        before = eng.inflight_get()
        # the admission record is checked last: everything else of this call was validated
        rc, _ = direct(epp, eng, prompts[:97], c.full_inputs(97, 43, w.pool), uniform_len=PB, bad_adm=True)
        assert rc != 0
        # without admission rows the context lengths are checked last
        bad = c.full_inputs(97, 44, w.pool)
        bad.prio = None
        bad.ctx[96] = -2
        with pytest.raises(epp.EngineError):
            eng.schedule(prompts[:97], uniform_len=PB, topk=True, **bad.kwargs())
        assert eng.stats()["n_decisions"] == 160
        after = eng.inflight_get()
        assert all(np.array_equal(a, b) for a, b in zip(before, after))
        out = eng.schedule(prompts[:97], uniform_len=PB, topk=True, **second.kwargs())
        check_call(orc, w, second, out, 160)
        calls.append((out[0], out[1], w.in_len[:97]))
        check_counters(eng, calls)


# ---- 5. batcher flushes with mixed rows -----------------------------------------------------------------------------
SPECIAL = [
    [c.ADM_NO_PRED, c.PLAIN, c.ADM_NO_PRED, c.CTX_ONLY, c.ADM_NO_PRED, c.PLAIN, c.ADM_NO_PRED, c.ADM_NO_PRED],  # no pred_valid
    [c.PLAIN, c.PRED_ONLY, c.PLAIN, c.CTX_ONLY, c.ADM_NO_PRED, c.PLAIN, c.PRED_ONLY, c.PLAIN],   # one context length
]


def flush_kinds(f):
    if f < len(SPECIAL):
        return SPECIAL[f]
    lap = f // 4
    return [c.row_kind(i, lap) for i in range(c.M)]


def row_inputs(rng, kind, pool):
    """(subset, predictions, valid, ctx, admission) of one submitted row of this kind."""
    one = c.side_inputs(1, int(rng.integers(1 << 30)), pool, sub=[0] if kind in (c.SUB_EMPTY_PRED, c.EVERYTHING) else None,
                        pred=[0] if kind in (c.PRED_ONLY, c.EVERYTHING) else None,
                        ctx=kind in (c.CTX_ONLY, c.EVERYTHING), shed=[0] if rng.random() < 0.8 else [])
    sub = one.subsets[0] if one.subsets is not None else None
    pred = one.preds[0] if one.preds is not None else ([] if kind == c.SUB_EMPTY_PRED else None)
    valid = one.valid[0] if one.valid is not None else None
    ctx = int(rng.choice(c.EDGES + [375, 256, 0, 5000])) if one.ctx is not None else None
    adm = None
    if kind in (c.ADM_NO_PRED, c.EVERYTHING):
        adm = dict(priority=int(one.prio[0]), ttft_slo=float(one.ttft[0]), tpot_slo=float(one.tpot[0]))
        if kind == c.EVERYTHING:
            adm["pred_valid"] = valid
    return sub, pred, valid, ctx, adm


def flush_inputs(rows):
    """The twin call of one flush: each input present exactly when some row carries it."""
    n = len(rows)
    subs = [r[0] for r in rows]
    preds = [r[1] if r[1] else None for r in rows]
    ctx = [r[3] for r in rows]
    adms = [r[4] for r in rows]
    inp = c.Inputs(n)
    if any(s is not None for s in subs):
        inp.subsets = subs
    if any(p is not None for p in preds):
        inp.preds = preds
        inp.valid = [None if p is None else (r[2] if r[4] is not None else [0] * len(p)) for p, r in zip(preds, rows)]
    if any(x is not None for x in ctx):
        inp.ctx = np.array([-1 if x is None else x for x in ctx], np.int64)
    if any(a is not None for a in adms):
        inp.prio = np.array([0 if a is None else a["priority"] for a in adms], np.int32)
        inp.ttft = np.array([0.0 if a is None else a["ttft_slo"] for a in adms])
        inp.tpot = np.array([0.0 if a is None else a["tpot_slo"] for a in adms])
    return inp


def test_batcher_mixed_flushes(epp, orc):
    """One submitting thread and full flushes of M rows, so every flush's rows are known; prompts of 1500 bytes exceed
    the hashed row (1024 bytes) and take the default context length from their true length (375 tokens)."""
    n_flush = 4 * (c.LAPS + 1)
    N = n_flush * c.M
    lens = np.where(np.arange(N) % 5 == 2, 1500, PB).astype(np.int64)
    w = c.World(3, N)
    w.in_len = lens
    w.total = np.where(lens > 1024, 16, 10).astype(np.int32)
    rng = np.random.default_rng(12)
    raw = rng.integers(0, 256, (N, 1500)).astype(np.uint8)
    cap = 1024
    rows_buf = np.zeros((N, cap), np.uint8)
    for r in range(N):
        rows_buf[r, :min(lens[r], cap)] = raw[r, :min(lens[r], cap)]
    offs = (np.arange(N + 1) * cap).astype(np.uint64)
    kinds = [k for f in range(n_flush) for k in flush_kinds(f)]
    rows = [row_inputs(rng, k, w.pool) for k in kinds]
    hashed = np.minimum(lens, cap)                       # the bytes of each prompt the engine hashes
    packed = np.concatenate([raw[r, :hashed[r]] for r in range(N)])
    poffs = np.concatenate([[0], np.cumsum(hashed)]).astype(np.uint64)
    with chain_engine(epp, w) as eng, chain_engine(epp, w) as twin:
        for e in (eng, twin):
            load(e, w, packed, offsets=poffs)
        got_dec = np.zeros(N, epp.DECISION_DTYPE)
        got_det = np.zeros(N, epp.DETAIL_DTYPE)
        got_lists = []
        with epp.Batcher(eng, max_batch=c.M, max_delay_us=10_000_000) as b:
            tickets = []

            def submit(r0, r1):
                for r in range(r0, r1):
                    sub, pred, _, ctx, adm = rows[r]
                    tickets.append(b.submit(raw[r, :lens[r]], subset=sub, predictions=pred, context_tokens=ctx,
                                            admission=adm))
            # the first flush completes before any row with predictions is submitted: no validity bytes at all
            submit(0, c.M)
            b.wait_topk(tickets[0])
            submit(c.M, N)
            for r, t in enumerate(tickets):
                assert t >> 20 == r // c.M and t & 0xFFFFF == r % c.M
                d, dd, lists = b.wait_topk(t)
                got_dec[r], got_det[r] = d, dd
                got_lists.append(lists)
        calls = []
        seen_default = 0
        for f in range(n_flush):
            r0, r1 = f * c.M, (f + 1) * c.M
            inp = flush_inputs(rows[r0:r1])
            if f == 0:
                assert inp.preds is None and inp.adm and inp.ctx is not None
            if f == 1:
                assert (inp.ctx != -1).sum() == 1
            rc, want = direct(epp, twin, rows_buf[r0:r1], inp, offsets=offs[:c.M + 1], lengths=lens[r0:r1],
                              flags=epp.capi.EPP_BATCH_LENGTHS_EXCEED_ROWS)
            assert rc == 0, eng._lib.epp_last_error()
            assert got_dec[r0:r1].tobytes() == want[0].tobytes(), f"flush {f}: decisions"
            assert got_det[r0:r1].tobytes() == want[1].tobytes(), f"flush {f}: details"
            for i in range(c.M):
                for n in ("primary", "prefill"):
                    assert got_lists[r0 + i][n] == [int(x) for x in want[2][n][i] if int(x) != c.NO], (f, i, n)
            check_call(orc, w, inp, want, r0, row0=r0, in_len=lens[r0:r1])
            seen_default += sum(1 for i in range(c.M) if lens[r0 + i] > cap and (inp.ctx is None or inp.ctx[i] == -1))
            calls.append((want[0], want[1], lens[r0:r1]))
        assert seen_default > 0
        check_counters(eng, calls)
        check_counters(twin, calls)
