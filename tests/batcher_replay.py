"""Replaying the flushes a micro-batcher (csrc/batcher.cu) actually ran.

A ticket is (seq << 20) | idx: the flush `seq` it went into and its row in that flush.  A submit the batcher refuses
reserves no row, so once every ticket has been waited for, the tickets grouped by seq are exactly the flushes that ran, in
order, each flush's rows in idx order.  Every flush is one scheduling call of the engine: it takes the ordinals
[base, base + n) (the key of the seeded tie rule, the random draws and the probabilistic admitter), where base is the
engine's decision count before the batcher plus the sizes of the earlier successful flushes (a failed call decides
nothing and takes no ordinal).  A test replays those calls one by one with its models and compares bit for bit; it also
replays the same rows as one call in request order, which must NOT match, so that the test can fail at all."""
from __future__ import annotations

import threading

import numpy as np

SEQ_SHIFT = 20
IDX_MASK = (1 << SEQ_SHIFT) - 1


def split(ticket: int) -> tuple[int, int]:
    return int(ticket) >> SEQ_SHIFT, int(ticket) & IDX_MASK


def flushes(tickets, contiguous: bool = True):
    """tickets: {row: ticket} or a sequence whose entry r is row r's ticket (None: a refused submit, no row) ->
    [(seq, [row, ...])] in flush order, each flush's rows in idx order.  Every flush must hold the rows idx 0 .. n-1 (a
    gap is a row that was reserved but whose ticket is missing); with contiguous, the seqs must also follow each other."""
    items = tickets.items() if isinstance(tickets, dict) else enumerate(tickets)
    by = {}
    for r, t in items:
        if t is None:
            continue
        s, i = split(t)
        rows = by.setdefault(s, {})
        assert i not in rows, f"ticket {t:#x} given to rows {rows[i]} and {r}"
        rows[i] = r
    out = []
    for s in sorted(by):
        rows = by[s]
        assert sorted(rows) == list(range(len(rows))), f"flush {s}: rows {sorted(rows)} are not 0 .. {len(rows) - 1}"
        out.append((s, [rows[i] for i in range(len(rows))]))
    if contiguous and out:
        seqs = [s for s, _ in out]
        assert seqs == list(range(seqs[0], seqs[0] + len(seqs))), f"flushes missing between {seqs[0]} and {seqs[-1]}"
    return out


def with_bases(fl, base0: int, failed=()):
    """[(seq, rows)] -> [(seq, rows, ordinal base)]: a flush in `failed` (seqs) takes no ordinals."""
    out, b = [], int(base0)
    for s, rows in fl:
        out.append((s, rows, b))
        if s not in failed:
            b += len(rows)
    return out


def single(rows, base0: int):
    """The wrong replay of the sensitivity guard: every row in request order as one call at the first ordinal."""
    return [(0, sorted(rows), int(base0))]


def sizes(fl):
    return [len(rows) for _, rows in fl]


def run_threads(n_threads: int, rows, fn):
    """fn(row) on n_threads threads (row i on thread i % n_threads, each thread in row order) -> {row: fn's result}.
    Raises the first exception a thread met."""
    rows = list(rows)
    out, errors = {}, []

    def worker(t):
        try:
            for r in rows[t::n_threads]:
                out[r] = fn(r)
        except Exception as e:      # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    if errors:
        raise errors[0]
    return out


# ---- landscapes and their replays on the models (shared by the GPU tests and the CPU guard tests) --------------------
SEED = 0x5EED


def flat_pool(E: int, seed: int):
    """kv and waiting drawn from two values each, nothing running: large arg-max sets, so the seeded tie rule (and
    with it the ordinal) decides many picks."""
    rng = np.random.default_rng(seed)
    kv = rng.choice([0.25, 0.5], E)
    waiting = rng.choice([0, 0, 3], E).astype(np.int32)
    return kv, waiting, np.zeros(E, np.int32)


def pd_landscape(tg, E=96, R=64 * 24, seed=7):
    """Scaled config 4 (P/D, prefix w2 + queue w1 in both profiles) over a flat pool, starting from an empty index:
    prompts of the trace's families, so that a request matches what earlier requests of its family indexed."""
    w = tg.baseline_configs()["config4"].scaled(E=E, R=R, T=256, name="config4")
    w.non_cached_tokens = 32
    trace = tg.Trace(w)
    tokens, _, _ = trace.requests()
    role = trace.pool()[0]
    kv, waiting, running = flat_pool(E, seed)
    return w, tokens, (role, kv, waiting, running)


def pd_replay(orc, tg, w, tokens, pool, plan, tie_seed=SEED, index_picks=True, ix=None):
    """plan: [(seq, rows, base)] -> ({row: (oracle decision, total, match_blocks)}, the oracle's indexer afterwards).
    One oracle call per flush at its ordinal base; with index_picks, PreRequest after it (each decided row's hashes
    for its pick and its prefill pick)."""
    import helpers
    ix = orc.Indexer() if ix is None else ix
    opool = orc.PoolState(*pool)
    prim = orc.make_profile(w.primary_filter, list(w.primary_scorers))
    pref = orc.make_profile(tg.FILTER_PREFILL, list(w.prefill_scorers)) if w.prefill_scorers is not None else None
    out = {}
    for _, rows, base in plan:
        toks = tokens[rows]
        odec, ototal = helpers.oracle_decisions(orc, w, opool, ix, prim, pref, toks, 2, tie_seed=tie_seed, tie_base=base)
        hs = [orc.hash_prompt(toks[i].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks) for i in range(len(rows))]
        for i, r in enumerate(rows):
            mb = 0
            if odec["status"][i] == 0:
                mb = int(ix.match_longest_prefix(hs[i], w.E)[0][int(odec["pick"][i])])
            out[r] = (odec[i], int(ototal[i]), mb)
        if index_picks:
            for i in range(len(rows)):
                if odec["status"][i] != 0:
                    continue
                ix.add(hs[i], int(odec["pick"][i]))
                if odec["prefill_ran"][i] and odec["prefill_pick"][i] >= 0:
                    ix.add(hs[i], int(odec["prefill_pick"][i]))
    return out, ix


class PickerWorld:
    """E endpoints (every eleventh outside the pool), six prompt families with hand-placed holders (family 0 held by 40
    endpoints, so the sparse map overflows), a share of cold prompts; 32-byte blocks, 12 per prompt."""
    BST, B = 8, 12
    L = 4 * 8 * 12
    MODEL = b"m"

    def __init__(self, orc, E=70, R=1600, seed=1):
        rng = np.random.default_rng(seed)
        self.orc, self.E, self.R = orc, E, R
        self.ids = np.array([e for e in range(E) if e % 11 != 5], np.uint32)
        self.role = np.full(E, 0xFF, np.uint8)
        self.role[self.ids] = 0
        self.kv = rng.choice([0.1, 0.4, 0.7], E)
        self.waiting = rng.integers(0, 3, E).astype(np.int32)
        self.running = np.zeros(E, np.int32)
        BB = 4 * self.BST
        fams = [rng.integers(0, 256, self.L, dtype=np.uint8) for _ in range(6)]
        holders = [[(e, 2) for e in range(0, 40)], [(0, 12), (69, 5)], [(33, 3), (34, 3), (35, 8)], [(64, 1)], [(1, 12)],
                   [(68, 6), (2, 6)]]
        toks = rng.integers(0, 256, (R, self.L), dtype=np.uint8)
        kind = rng.integers(-1, len(fams), R)
        for r in range(R):
            if kind[r] >= 0:
                n = int(rng.integers(1, self.B + 1)) * BB
                toks[r, :n] = fams[kind[r]][:n]
        self.tokens = toks
        hs, es = [], []
        for g, hl in enumerate(holders):
            h = orc.hash_prompt(fams[g].tobytes(), self.MODEL, self.BST, self.B)
            for e, depth in hl:
                hs += h[:depth]
                es += [e] * depth
        self.pairs = (np.array(hs, np.uint64), np.array(es, np.uint32))
        ix = orc.Indexer()
        ix.load_pairs(*self.pairs)
        self.match = np.zeros((R, E), np.int32)
        self.total = np.zeros(R, np.int32)
        for r in range(R):
            h = orc.hash_prompt(toks[r].tobytes(), self.MODEL, self.BST, self.B)
            self.match[r] = ix.match_longest_prefix(h, E)[0]
            self.total[r] = len(h)
        self.opool = orc.PoolState(self.role, self.kv, self.waiting, self.running)

    def load(self, eng):
        eng.register_model(self.MODEL)
        eng.pool_set(self.ids, self.role[self.ids], self.kv[self.ids], self.waiting[self.ids], self.running[self.ids])
        eng.index_load_snapshot(*self.pairs)

    def draw(self, picker, sc, r, key):
        """One profile of row r with tools/picker_model.py's draw -> (pick, score, candidates)."""
        from tools import picker_model as PM
        orc = self.orc
        prof = orc.make_profile(0, sc)
        scores, _, _, _ = orc.profile_run(prof, self.opool, self.match[r], int(self.total[r]))
        base, _, _, _ = orc.profile_run(prof, self.opool, np.zeros(self.E, np.int32), int(self.total[r]))
        cands = [int(e) for e in self.ids]
        explicit = {e for e in cands if self.match[r][e] > 0}
        return PM.draw(picker, cands, base, scores, explicit, SEED, key, [s[1] for s in sc])


PICKER_DECODE = [(2, 2.0, 0.0), (1, 2.0, 0.0), (0, 3.0, 0.0)]      # queue, kv, prefix
PICKER_PREFILL = [(2, 0.5, 0.0), (1, 1.0, 0.0), (0, 1.0, 0.0)]


def picker_replay(world, picker, plan):
    """P/D with the same picker in both profiles, always disaggregated: decode draws with key 4 * ordinal, prefill with
    4 * ordinal + 1 -> {row: (pick, score, ties, match_blocks, prefill pick, prefill score, prefill ties)}."""
    out = {}
    for _, rows, base in plan:
        for i, r in enumerate(rows):
            o = base + i
            p, s, n = world.draw(picker, PICKER_DECODE, r, 4 * o)
            p1, s1, n1 = world.draw(picker, PICKER_PREFILL, r, 4 * o + 1)
            out[r] = (p, s, n, int(world.match[r][p]), p1, s1, n1)
    return out


def inflight_landscape(tg, E=64, R=640):
    """Scaled config 3 with a token-load and an active-request scorer read from the in-flight counters."""
    import dataclasses

    from tools import inflight_model as M
    TL = (M.TOKEN_LOAD, 1.0, 65536.0, M.TOKEN_COL, 0.0)
    AR = (M.ACTIVE_REQUEST, 2.0, 1.0, M.REQUEST_COL, 0.0)
    w = tg.baseline_configs()["config3"].scaled(E=E, R=R, T=512)
    w = dataclasses.replace(w, primary_scorers=tuple(w.primary_scorers) + (TL, AR))
    trace = tg.Trace(w)
    return w, trace


def inflight_replay(orc, tg, w, trace, ix, counters, plan, tokens):
    """One oracle call per flush with the counters as they stand as ext columns, then PreRequest of the producer ->
    {row: (oracle decision, total, match_blocks)}; counters is updated in place."""
    import helpers
    role, kv, waiting, running = trace.pool()
    prim = orc.make_profile(w.primary_filter, list(w.primary_scorers))
    out = {}
    for _, rows, base in plan:
        pool = orc.PoolState(role, kv, waiting, running, ext=counters.ext())
        toks = tokens[rows]
        odec, ototal = helpers.oracle_decisions(orc, w, pool, ix, prim, None, toks, 2, tie_base=base)
        counters.pre_request(odec, [w.prompt_bytes] * len(rows))
        for i, r in enumerate(rows):
            mb = 0
            if odec["status"][i] == 0:
                h = orc.hash_prompt(toks[i].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks)
                mb = int(ix.match_longest_prefix(h, w.E)[0][int(odec["pick"][i])])
            out[r] = (odec[i], int(ototal[i]), mb)
    return out


# ---- no-hit-lru: the LRU of cold picks that every flush updates ------------------------------------------------------
NOHIT_LRU = 20
NOHIT_SCORERS = PICKER_DECODE + [(9, 2.0, float(NOHIT_LRU))]           # + no-hit-lru w2 over an LRU of 20


def nohit_model(orc, world, picker):
    """tools/nohit_lru_model.Model over the world's pool, one profile with NOHIT_SCORERS; with a random picker the
    profile's draw of tools/picker_model.py replaces max-score over the same warm or cold scores."""
    from tools import nohit_lru_model as M
    from tools import picker_model as PM

    class PickerModel(M.Model):
        def run_profile(self, pi, match_row, total, key, lru_keys):
            filt, scs = self.profiles[pi]
            cand = self.candidates(filt)
            if not cand:
                return M.NO, 0.0, 0, None
            cold = M.is_cold(cand, match_row)
            mask = np.zeros(self.E, dtype=np.uint8)
            mask[cand] = 1
            idx = np.asarray(cand)

            def fold(mrow):
                acc = np.zeros(self.E, np.float64)
                for s, sc in enumerate(scs):
                    if sc[0] == M.NO_HIT_LRU:
                        col = M.cold_column(cand, lru_keys, self.E) if cold else np.full(self.E, 0.5)
                    elif sc[0] == 0:
                        col = (np.asarray(mrow, np.float64) / float(total)) if total else np.zeros(self.E)
                        col = np.minimum(np.maximum(col, 0.0), 1.0)
                    else:
                        col = self.column(pi, s, mask)
                    acc[idx] = acc[idx] + col[idx] * sc[1]
                return acc

            pick, s, n = PM.draw(picker, cand, fold(np.zeros(self.E, np.int32)), fold(match_row),
                                 {e for e in cand if match_row[e] > 0}, self.tie_seed, key, [sc[1] for sc in scs])
            return pick, s, n, cold

    cls = M.Model if picker == PM.MAX_SCORE else PickerModel
    return cls(orc, world.opool, world.E, [(0, NOHIT_SCORERS)], NOHIT_LRU, block_size_tokens=world.BST, tie_seed=SEED)


def nohit_replay(model, world, plan):
    """One Model.schedule per flush at its ordinal base -> {row: (status, pick, score, prefill pick, match_blocks,
    cold)}; the model's LRU ends as the engine's should."""
    out = {}
    for _, rows, base in plan:
        model.n_decisions = base
        for r, o in zip(rows, model.schedule(world.match[rows], world.total[rows])):
            out[r] = o
    return out


# ---- admitters: the probabilistic draw keyed by the ordinal, rejected rows leaving no trace -------------------------
ADMIT_POWER = 2.0


def admit_landscape(tg, orc, E=48, R=16 * 30, seed=5):
    """Scaled config 3 (no role filter) over a busy, warm pool -- nothing idle or cold, so the latency-slo-admitter can
    reject -- with an empty index; per row a priority (two thirds sheddable), SLOs and, for every third row,
    predictions.  The probabilistic-admitter's k puts its rejection probability at about one half."""
    import dataclasses

    from tools import admission_model as am
    w = tg.baseline_configs()["config3"].scaled(E=E, R=R, T=256, name="config3")
    w = dataclasses.replace(w, primary_filter=tg.FILTER_NONE)
    tokens = tg.Trace(w).requests()[0]
    rng = np.random.default_rng(seed)
    pool = dict(present=np.ones(E, bool), kv=rng.choice([0.3, 0.6, 0.9], E),
                waiting=rng.choice([2, 5, 9], E).astype(np.int32), running=rng.integers(1, 5, E).astype(np.int32))
    cfg = dict(am.DEFAULTS, latency_slo=True, probabilistic=True, power=ADMIT_POWER)
    eps = [am.Endpoint(int(pool["waiting"][s]), float(pool["kv"][s]), int(pool["running"][s])) for s in range(E)]
    cfg["k"] = 0.5 / am.go_pow(am.saturation(eps, cfg), ADMIT_POWER)
    prio = rng.choice([-1, -1, 0], R).astype(np.int32)
    ttft = rng.choice([0.0, 50.0], R)
    tpot = rng.choice([0.0, 20.0], R)
    preds, valid = [], []
    for r in range(R):
        if r % 3:
            preds.append(None)
            valid.append(None)
            continue
        slots = sorted(int(s) for s in rng.choice(E, int(rng.integers(1, 6)), replace=False))
        bits = [int(rng.choice([0, 1, 2, 3, 0])) for _ in slots]
        preds.append([(s, 10.0, 1.0 - (b & 1), 1.0 - (b >> 1), 0) for s, b in zip(slots, bits)])
        valid.append(bits)
    rows = dict(priority=prio, ttft=ttft, tpot=tpot, preds=preds, valid=valid)
    return w, tokens, pool, cfg, rows


def admit_replay(orc, tg, am, w, tokens, pool, cfg, rows, plan, ix=None, counters=None):
    """Per flush: the oracle's decisions at its ordinal base, the admitters' rejections (tools/admission_model.py at
    the same base), then PreRequest and the in-flight adds of the admitted, decided rows only -> ({row: (oracle
    decision with rejected rows at status EPP_STATUS_REJECTED, total, match_blocks)}, indexer, counters)."""
    import helpers
    from tools import inflight_model as IM
    ix = orc.Indexer() if ix is None else ix
    counters = IM.Counters(w.E) if counters is None else counters
    opool = orc.PoolState(np.zeros(w.E, np.uint8), pool["kv"], pool["waiting"], pool["running"])
    prim = orc.make_profile(w.primary_filter, list(w.primary_scorers))
    out = {}
    for _, rr, base in plan:
        toks = tokens[rr]
        odec, ototal = helpers.oracle_decisions(orc, w, opool, ix, prim, None, toks, 2, tie_seed=SEED, tie_base=base)
        preds = [None if rows["preds"][r] is None else [e[0] for e in rows["preds"][r]] for r in rr]
        rej = am.rejects(cfg, pool, rows["priority"][rr], rows["ttft"][rr], rows["tpot"][rr], preds,
                         [rows["valid"][r] for r in rr], None, tie_seed=SEED, ord_base=base)
        odec = odec.copy()
        odec["status"][rej] = am.STATUS_REJECTED
        hs = [orc.hash_prompt(toks[i].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks) for i in range(len(rr))]
        for i, r in enumerate(rr):
            mb = int(ix.match_longest_prefix(hs[i], w.E)[0][int(odec["pick"][i])]) if odec["status"][i] == 0 else 0
            out[r] = (odec[i], int(ototal[i]), mb)
        for i in range(len(rr)):
            if odec["status"][i] == 0:
                ix.add(hs[i], int(odec["pick"][i]))
        counters.pre_request(odec, [w.prompt_bytes] * len(rr))
    return out, ix, counters
