"""Landscapes of scheduling calls that carry every side input at once -- endpoint subsets, latency predictions, context
lengths and admission rows -- and the model that decides them, for tests/test_side_inputs_gpu.py.  Here they run through
the models only (tools/context_length_model.py over tools/latency_model.py, then tools/admission_model.py), and each test
asserts that the edge a GPU test is built around is reached:
  - the staged sections of every chosen call (restated from engine.cu stage_inputs: one pinned buffer, each section from
    a 256-byte boundary) end off a 256-byte boundary, with empty sections between non-empty ones and the first or last
    section alone;
  - every call has rejected and admitted rows, rows whose subset empties the candidate set, and context lengths on the
    edges of the endpoints' label ranges;
  - every staging row of the batcher's 4-buffer ring holds every row kind after every other kind."""
from __future__ import annotations

import numpy as np
import pytest

from tools import admission_model as am
from tools import context_length_model as cm
from tools import inflight_model as im
from tools import latency_model as lm

E = 48
NO = 0xFFFFFFFF
PB = 640                       # prompt bytes: 10 blocks of 16 tokens; default context length 160
NCT = 8                        # non_cached_tokens of the P/D decider
K = 4                          # pick_k of the chain engine
SEED = 0x5EED
CL, LAT, QUEUE, KV, PREFIX = 11, 10, 2, 1, 0
KEY = cm.DEFAULT_LABEL
VALUES = ["0-100", "100-200", "150-150", "160-160", "0-2048", "161-5000", "0-159", "10-5", "abc", "200-100000",
          "5000-9000", "375-375", "256-256"]
EDGES = [0, 1, 99, 100, 101, 149, 150, 151, 159, 160, 161, 199, 200, 201, 2047, 2048, 2049, 4999, 5000, 5001, 9000, 9001]

# decode: context-length filter and scorer, the latency scorer behind the tier filter, the affinity filter after it
PRIMARY = dict(scorers=[(CL, 1.0, 0.0), (LAT, 1.0, 0.0), (KV, 0.5, 0.0), (QUEUE, 1.0, 0.0)], picker=0,
               a2=(0.80, 0.2, 100.0), filt=True, lcfg=dict(tier_filter=1, epsilon_explore_neg=0.5))
# prefill: the context-length scorer only among the ordinary ones
PREFILL = dict(scorers=[(QUEUE, 2.0, 0.0), (KV, 2.0, 0.0), (PREFIX, 3.0, 0.0), (CL, 1.5, 0.0)], picker=0, a2=None,
               filt=False, lcfg=None)
# saturation about 0.3-0.5 over the pool below: rejection probabilities away from 0 and 1
ACFG = dict(latency_slo=True, probabilistic=True, queue_depth_threshold=10, kv_cache_util_threshold=1.5, power=2.0, k=1.5)

# the batcher's row kinds
PLAIN, SUB_EMPTY_PRED, PRED_ONLY, CTX_ONLY, ADM_NO_PRED, EVERYTHING = range(6)
M = 8                          # max_batch of the batcher test
LAPS = 37


def de_bruijn_6_2():
    """The cyclic sequence of 36 kinds in which every ordered pair (a, b) of kinds appears once as neighbours."""
    seq, a = [], [0] * 3

    def db(t, p):
        if t > 2:
            if 2 % p == 0:
                seq.extend(a[1:p + 1])
            return
        a[t] = a[t - p]
        db(t + 1, p)
        for j in range(a[t - p] + 1, 6):
            a[t] = j
            db(t + 1, t)
    db(1, 1)
    return seq


DB = de_bruijn_6_2()


def row_kind(row, lap):
    """Kind of row `row` of a flush on lap `lap` of the ring: a window of 37 consecutive laps of one staging row holds
    every ordered pair of kinds."""
    return DB[(row + lap) % len(DB)]


# ---- the world: pool, labels, match landscape ---------------------------------------------------------------------------
def make_pool(seed, absent=4):
    rng = np.random.default_rng(seed)
    role = np.zeros(E, np.uint8)
    role[rng.choice(E, absent, replace=False)] = 0xFF
    kv = rng.choice([0.05, 0.25, 0.5, 0.75], E)
    return role, kv, rng.integers(0, 6, E), rng.integers(1, 6, E)


def adm_pool(pool):
    role, kv, waiting, running = pool
    return dict(present=role != 0xFF, kv=np.asarray(kv, np.float64), waiting=np.asarray(waiting), running=np.asarray(running))


def make_labels(seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(E):
        c = rng.integers(0, 10)
        out.append(None if c == 0 else {"other": "x"} if c == 1 else {KEY: VALUES[rng.integers(0, len(VALUES))]})
    return out


def landscape(R, seed, top=10):
    rng = np.random.default_rng(seed)
    match = np.zeros((R, E), np.int32)
    for r in range(R):
        sticky = rng.choice(E, 6, replace=False)
        match[r, sticky[:3]] = top
        match[r, sticky[3:]] = top - 1
        match[r, rng.choice(E, 6)] = rng.integers(1, top - 2, 6)
    return match


class World:
    def __init__(self, seed, R):
        self.pool = make_pool(seed)
        self.labels = make_labels(seed + 1)
        self.ranges = [cm.endpoint_state(lb, KEY) for lb in self.labels]
        self.match = landscape(R, seed + 2)
        self.total = np.full(R, 10, np.int32)
        self.in_len = np.full(R, PB, np.int64)


# ---- one call's side inputs ---------------------------------------------------------------------------------------
class Inputs:
    """The side inputs of one call over R rows; an absent input is None.  subsets[r]: None or sorted slots; preds[r]:
    None or (slot, ttft, ttft_headroom, tpot_headroom, dispatched) tuples, slots ascending; valid[r]: their validity
    bytes; prio / ttft / tpot: the admission rows."""

    def __init__(self, R, subsets=None, preds=None, valid=None, ctx=None, prio=None, ttft=None, tpot=None):
        self.R, self.subsets, self.preds, self.valid, self.ctx = R, subsets, preds, valid, ctx
        self.prio, self.ttft, self.tpot = prio, ttft, tpot

    @property
    def adm(self):
        return self.prio is not None

    def admission(self):
        if not self.adm:
            return None
        a = dict(priority=self.prio, ttft_slo=self.ttft, tpot_slo=self.tpot)
        if self.preds is not None:
            a["pred_valid"] = self.valid
        return a

    def kwargs(self):
        return dict(subsets=self.subsets, predictions=self.preds, context_tokens=self.ctx, admission=self.admission())

    def part(self, r0, r1):
        cut = lambda x: None if x is None else x[r0:r1]   # noqa: E731
        return Inputs(r1 - r0, cut(self.subsets), cut(self.preds), cut(self.valid), cut(self.ctx), cut(self.prio),
                      cut(self.ttft), cut(self.tpot))


def side_inputs(R, seed, pool, sub=None, pred=None, ctx=True, shed=None, sub_sizes=None, pred_sizes=None):
    """sub / pred / shed: the rows that carry a subset / predictions / a sheddable priority (None: the input is absent).
    sub_sizes / pred_sizes: per listed row its slot / entry count (default random); a subset size of -1 lists absent
    slots only, so the row has no candidate."""
    rng = np.random.default_rng(seed)
    role = pool[0]
    absent = np.flatnonzero(role == 0xFF)
    subsets = preds = valid = prio = ttft = tpot = None
    if sub is not None:
        subsets = [None] * R
        for i, r in enumerate(sub):
            n = int(sub_sizes[i]) if sub_sizes is not None else int(rng.integers(-1, 21))
            subsets[r] = sorted(absent[:2].tolist()) if n < 0 else sorted(rng.choice(E, n, replace=False).tolist())
    if pred is not None:
        preds, valid = [None] * R, [None] * R
        for i, r in enumerate(pred):
            n = int(pred_sizes[i]) if pred_sizes is not None else int(rng.integers(1, 25))
            slots = np.sort(rng.choice(E, n, replace=False))
            preds[r] = [(int(s), float(rng.integers(1, 400)), float(rng.integers(-50, 150)), float(rng.integers(-5, 20)), 0)
                        for s in slots]
            valid[r] = [int(b) for b in rng.choice([0, 1, 2, 3, 3], n)]
    if shed is not None:
        prio = rng.choice([0, 1, 2], R).astype(np.int32)
        prio[list(shed)] = -1
        ttft = rng.choice([0.0, 80.0, 80.0], R)
        tpot = rng.choice([0.0, 0.0, 20.0], R)
    c = None
    if ctx:
        c = np.array([-1 if r % 7 == 0 else EDGES[(r * 5) % len(EDGES)] if r % 3 else int(rng.integers(0, 12000))
                      for r in range(R)], np.int64)
    return Inputs(R, subsets, preds, valid, c, prio, ttft, tpot)


def every(R, step, first=0):
    return list(range(first, R, step))


def full_inputs(R, seed, pool):
    """All four inputs: a subset on every 5th row, predictions on about 7 rows in 10, 2 in 5 rows sheddable."""
    rng = np.random.default_rng(seed + 100)
    pred = [r for r in range(R) if rng.random() < 0.7]
    shed = [r for r in range(R) if rng.random() < 0.4]
    return side_inputs(R, seed, pool, sub=every(R, 5, 2), pred=pred, ctx=True, shed=shed)


# ---- engine.cu check_admission and stage_inputs, restated ---------------------------------------------------------
def admit_rows(inp, latency_slo=True, probabilistic=True, lat_engine=True):
    """(rows, entries) the admission section lists for a call (check_admission)."""
    if not inp.adm:
        return 0, 0
    with_pred = latency_slo and inp.preds is not None and inp.R > 0
    rows = ents = 0
    for r in range(inp.R):
        if inp.prio[r] >= 0:
            continue
        if inp.subsets is not None and inp.subsets[r] is not None and len(inp.subsets[r]) == 0:
            continue
        n = 0 if inp.preds is None or inp.preds[r] is None else len(inp.preds[r])
        lat = with_pred and n > 0 and (inp.ttft[r] > 0 or inp.tpot[r] > 0)
        if probabilistic or lat:
            rows += 1
            ents += n if lat else 0
    return rows, ents


SECTIONS = ("rows", "slots", "cnt", "off", "ent", "ctx", "adm", "adm_ent")


def layout(inp, lat_engine=True, cl_engine=True, **adm):
    """stage_inputs' sections of a call: {name: (offset, bytes)} and the total; None when nothing is staged."""
    R = inp.R
    sub_rows = 0 if inp.subsets is None else sum(s is not None for s in inp.subsets)
    n_slots = 0 if inp.subsets is None else sum(len(s) for s in inp.subsets if s is not None)
    use_pred = inp.preds is not None and R > 0 and lat_engine
    use_ctx = inp.ctx is not None and R > 0 and cl_engine
    n_ent = 0 if inp.preds is None else sum(len(p) for p in inp.preds if p is not None)
    n_adm, n_adm_ent = admit_rows(inp, **adm)
    sizes = [16 * sub_rows, 4 * n_slots, 4 * R if use_pred else 0, 8 * R if use_pred else 0, 32 * n_ent if use_pred else 0,
             8 * R if use_ctx else 0, 32 * n_adm, 4 * n_adm_ent]
    if not (sub_rows or use_pred or use_ctx or n_adm):
        return None, 0
    total, out = 0, {}
    for name, b in zip(SECTIONS, sizes):
        at = (total + 255) & ~255
        total = at + b
        out[name] = (at, b)
    return out, total


def pattern(lay):
    return "".join("x" if lay[n][1] else "." for n in SECTIONS)


# The calls of the packing test: every non-empty section ends off a 256-byte boundary.  R = 37: 148-byte counts,
# 296-byte offsets and context lengths.  "x" marks a staged section in SECTIONS order.
def packing_calls(pool):
    R = 37
    one = dict(sub=[4], sub_sizes=[7], pred=[1, 4, 9, 20], pred_sizes=[3, 5, 1, 2], shed=[4])
    many = dict(sub=[0, 3, 5, 8, 11, 14, 17, 21, 26, 29, 31, 33, 36], sub_sizes=[1, 0, 3, 5, -1, 2, 7, 9, 1, 4, 6, 11, 12],
                pred=every(R, 2, 1), pred_sizes=[(3 * i) % 7 + 1 for i in range(18)], shed=every(R, 3))
    calls = [
        ("all, one row each", side_inputs(R, 1, pool, ctx=True, **one), "xxxxxxxx"),
        ("all, odd totals", side_inputs(R, 2, pool, ctx=True, **many), "xxxxxxxx"),
        ("no predictions", side_inputs(R, 3, pool, sub=many["sub"], sub_sizes=many["sub_sizes"], ctx=True,
                                       shed=many["shed"]), "xx...xx."),
        ("no context lengths", side_inputs(R, 4, pool, ctx=False, **many), "xxxxx.xx"),
        ("no subsets", side_inputs(R, 5, pool, pred=one["pred"], pred_sizes=one["pred_sizes"], ctx=True, shed=[4]),
         "..xxxxxx"),
        ("only admission", side_inputs(R, 6, pool, ctx=False, shed=[11]), "......x."),
        ("only subset rows", side_inputs(R, 7, pool, sub=[30], sub_sizes=[5], ctx=False), "xx......"),
    ]
    for _, inp, _ in calls:                   # row 4's SLO makes it a latency-slo-admitter row with its 5 entries
        if inp.adm:
            inp.ttft[4] = 80.0
    return calls


# The consecutive calls of one engine: the input set and the size change from call to call.
def sequence_calls(pool):
    return [
        ("all four", full_inputs(301, 11, pool)),
        ("context lengths only", side_inputs(77, 12, pool, ctx=True)),
        ("nothing", side_inputs(40, 13, pool, ctx=False)),
        ("subsets and admission", side_inputs(150, 14, pool, sub=every(150, 3), ctx=False, shed=every(150, 2))),
        ("all four, larger", full_inputs(517, 15, pool)),
    ]


# ---- the model of one row -----------------------------------------------------------------------------------------
def model_cfg(acfg):
    c = dict(am.DEFAULTS)
    c.update({k: v for k, v in acfg.items() if k in am.DEFAULTS})
    c.update(latency_slo=acfg["latency_slo"], probabilistic=acfg["probabilistic"])
    return c


def info_of(p):
    return {} if p is None else {int(s): lm.Info(t, th, tp, d) for s, t, th, tp, d in p}


def keep_of(inp, r):
    if inp.subsets is None or inp.subsets[r] is None:
        return None
    return np.isin(np.arange(E), inp.subsets[r])


def ctx_of(inp, r, in_len):
    c = -1 if inp.ctx is None else int(inp.ctx[r])
    return c if c >= 0 else cm.default_ctx(int(in_len))


def decide_row(orc, w, inp, r, base, row=None, in_len=None):
    """The chain engine's row r of a call whose first ordinal is base (row: the world's row it was built from):
    dict(primary=..., prefill=... or None, go=bool)."""
    row = r if row is None else row
    L = int(w.in_len[row] if in_len is None else in_len)
    role, kv, waiting, running = w.pool
    info, keep, ctx = info_of(None if inp.preds is None else inp.preds[r]), keep_of(inp, r), ctx_of(inp, r, L)
    key = 4 * (base + r)
    match, total = w.match[row], int(w.total[row])
    m = cm.profile_decide(orc, 0, PRIMARY["scorers"], 0, role, kv, waiting, running, match, total, w.ranges, ctx, True,
                          info, PRIMARY["lcfg"], PRIMARY["a2"], SEED, key, K, keep=keep)
    out = dict(primary=m, prefill=None, go=False)
    if m["picks"]:
        t = L // 4
        out["go"] = t >= NCT and t - int(match[m["picks"][0]]) * 16 >= NCT
        if out["go"]:
            out["prefill"] = cm.profile_decide(orc, 0, PREFILL["scorers"], 0, role, kv, waiting, running, match, total,
                                               w.ranges, ctx, False, info, None, None, SEED, key + 1, 1, keep=keep)
    return out


def rejected(w, inp, base, acfg=ACFG, with_subsets=True):
    if not inp.adm:
        return np.zeros(inp.R, bool)
    slots = None if inp.preds is None else [None if p is None else [e[0] for e in p] for p in inp.preds]
    return am.rejects(model_cfg(acfg), adm_pool(w.pool), inp.prio, inp.ttft, inp.tpot, slots, inp.valid,
                      inp.subsets if with_subsets else None, SEED, base)


def check_row(m, rej, r, match_r, dec, det, lists):
    """Row r of the engine's outputs against the model's decision m and admission result rej, bit for bit."""
    d = dec[r]
    if rej:
        assert (int(d["status"]), int(d["pick"]), int(d["prefill_pick"]), int(d["tie_count"]), int(d["match_blocks"])) == \
            (am.STATUS_REJECTED, NO, NO, 0, 0), r
        assert np.float64(d["score"]).tobytes() == bytes(8), r
        if det is not None:
            for f in det.dtype.names:
                assert det[r][f] == (NO if f == "encode_pick" else 0), (r, f)
        if lists is not None:
            for n in ("primary", "prefill", "encode"):
                assert all(int(x) == NO for x in lists[n][r]), (r, n)
            assert lists["primary_scores"][r].tobytes() == bytes(8 * K), r
        return
    p = m["primary"]
    ok = bool(p["picks"])
    assert int(d["status"]) == (0 if ok else -1), r
    assert int(d["tie_count"]) == (p["ties"] if ok else 0), r
    if lists is not None:
        n = len(p["picks"])
        assert [int(x) for x in lists["primary"][r, :n]] == p["picks"], r
        assert lists["primary_scores"][r, :n].tobytes() == np.asarray(p["scores"], np.float64).tobytes(), r
        assert all(int(x) == NO for x in lists["primary"][r, n:]), r
    if not ok:
        return
    assert int(d["pick"]) == p["picks"][0], r
    assert np.float64(d["score"]).tobytes() == np.float64(p["scores"][0]).tobytes(), r
    assert int(d["match_blocks"]) == int(match_r[p["picks"][0]]), r
    if det is not None:
        assert int(det[r]["prefill_ran"]) == int(m["go"]), r
    q = m["prefill"]
    if not m["go"]:
        return
    assert int(d["prefill_pick"]) == (q["picks"][0] if q["picks"] else NO), r
    if q["picks"] and det is not None:
        assert np.float64(det[r]["prefill_score"]).tobytes() == np.float64(q["scores"][0]).tobytes(), r
        assert int(det[r]["prefill_tie_count"]) == q["ties"], r


def counters_after(E_, calls):
    """The in-flight counters after calls [(decisions, details, prompt lengths)]."""
    c = im.Counters(E_)
    for dec, det, lengths in calls:
        c.pre_request(dec, lengths, det)
    return c


# ---- the edges, through the models ----------------------------------------------------------------------------------
def test_packing_sections_off_256():
    pool = make_pool(3)
    seen = set()
    for name, inp, want in packing_calls(pool):
        lay, total = layout(inp)
        assert pattern(lay) == want, name
        for s in SECTIONS:
            at, b = lay[s]
            assert at % 256 == 0
            if b:
                assert b % 256, (name, s, b)
        seen.add(want)
        if name == "all, one row each":
            assert admit_rows(inp) == (1, 5) and lay["rows"][1] == 16 and lay["slots"][1] == 28
            # the offsets the GPU test exercises for this call
            assert {s: lay[s][0] for s in SECTIONS} == dict(rows=0, slots=256, cnt=512, off=768, ent=1280, ctx=1792,
                                                             adm=2304, adm_ent=2560)
            assert total == 2580
    # an empty section between two staged ones (no predictions, no context lengths), the first and the last alone
    assert {"xx...xx.", "xxxxx.xx", "......x.", "xx......"} <= seen


def test_sequence_changes_every_input(orc):
    pool = make_pool(3)
    pats = [pattern(layout(inp)[0]) if layout(inp)[0] else "" for _, inp in sequence_calls(pool)]
    assert pats == ["xxxxxxxx", ".....x..", "", "xx....x.", "xxxxxxxx"]
    totals = [layout(inp)[1] for _, inp in sequence_calls(pool)]
    assert totals[-1] > totals[0] > totals[1] and totals[3] > totals[1]   # the staging grows on the last call


@pytest.mark.parametrize("which", ["full", "sequence", "packing"])
def test_model_edges_reached(orc, which):
    w = World(3, 8192 + 544)
    if which == "full":
        calls = [("full", full_inputs(203, 21, w.pool))]
    elif which == "sequence":
        calls = [c for c in sequence_calls(w.pool) if c[1].adm]
    else:
        calls = [(n, i) for n, i, _ in packing_calls(w.pool)][1:2]   # odd totals: many sheddable rows
    for name, inp in calls:
        rej = rejected(w, inp, 0)
        shed = inp.prio < 0
        assert rej.any() and (shed & ~rej).any(), name
        if inp.subsets is not None:
            empty = [r for r in range(inp.R) if inp.subsets[r] is not None and
                     not decide_row(orc, w, inp, r, 0)["primary"]["picks"] and
                     all(w.pool[0][s] == 0xFF for s in inp.subsets[r])]
            assert empty, name
        if inp.ctx is not None:
            hit = set()
            for r in range(inp.R):
                for st in w.ranges:
                    if isinstance(st, tuple) and int(inp.ctx[r]) in (st[0], st[1], st[0] - 1, st[1] + 1):
                        hit.add(int(inp.ctx[r]))
            assert len(hit) >= 8, name


def test_pipelined_sample_rows():
    """The rows the pipelined call is model-checked on: every rejected, subset and chunk-edge row among 500 or more."""
    w = World(3, 8192 + 544)
    inp = full_inputs(8192 + 544, 31, w.pool)
    rows = pipelined_sample(inp, rejected(w, inp, 0))
    assert len(rows) >= 500
    per = ((inp.R + 1) // 2 + 31) & ~31                  # two chunks of engine.cu run_device
    assert {per - 1, per, 0, inp.R - 1} <= set(rows)


def pipelined_sample(inp, rej):
    R = inp.R
    per = ((R + 1) // 2 + 31) & ~31
    rows = set(np.flatnonzero(rej).tolist())
    rows |= {r for r in range(R) if inp.subsets[r] is not None}
    rows |= set(range(0, 16)) | set(range(per - 16, per + 16)) | set(range(R - 16, R))
    rows |= set(np.random.default_rng(7).choice(R, 200, replace=False).tolist())
    return sorted(rows)


def test_batcher_kinds_cover_every_pair():
    assert sorted(DB) == sorted(list(range(6)) * 6)
    for idx in range(M):
        seq = [row_kind(idx, lap) for lap in range(LAPS)]
        assert {(a, b) for a, b in zip(seq, seq[1:])} == {(a, b) for a in range(6) for b in range(6)}, idx
    for lap in range(LAPS):
        assert len({row_kind(i, lap) for i in range(M)}) >= 3            # every flush mixes the kinds
