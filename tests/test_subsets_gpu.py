"""GPU parity of per-request endpoint subsets (epp_schedule_subset, epp_submit_subset; csrc/subset_pick.cu) against the C
oracle.  A restricted request's expected decision is orc_cycle_batch run on that request alone, on the pool with every
slot outside its subset absent (role 0xFF), with tie_base = the request's ordinal: Schedule called with the subset's
endpoints.  No-hit-lru cold columns come from tools/nohit_lru_model.py over the restricted candidates (fed to the oracle
as an external column), random picks from tools/picker_model.py with every candidate explicit.  Run on an H100:
pytest -m gpu."""
import dataclasses
import threading

import numpy as np
import pytest

import helpers
from tools import nohit_lru_model as NH
from tools import picker_model as PM
from tools import tracegen as tg

pytestmark = pytest.mark.gpu

NO = 0xFFFFFFFF
ABSENT = 0xFF


@pytest.fixture(scope="module")
def epp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import epp_b200
    epp_b200.build.build()
    return epp_b200


class Rig:
    """A trace workload on the engine and on the oracle.  absent: slots left out of the engine's pool (stale subset
    entries)."""

    def __init__(self, epp, orc, name, E=64, R=256, T=512, tie_seed=0, absent=(), primary=None, engine_kw=None,
                 oracle_primary=None, encode=None, affinity=None, ext=None):
        self.epp, self.orc = epp, orc
        w = tg.baseline_configs()[name].scaled(E=E, R=R, T=T)
        if primary is not None:
            w = dataclasses.replace(w, primary_scorers=tuple(primary))
        self.w, self.trace, self.tie_seed = w, tg.Trace(w), tie_seed
        kw = dict(engine_kw or {})
        self.ext = None if ext is None else np.asarray(ext, np.float64).reshape(-1, w.E)
        if self.ext is not None:
            kw["n_ext_cols"] = self.ext.shape[0]
        if encode is not None:
            kw["encode"] = epp.ProfileSpec(0, [epp.ScorerSpec(*s) for s in encode])
        if affinity is not None:
            prefill = None if w.prefill_scorers is None else \
                epp.ProfileSpec(tg.FILTER_PREFILL, [epp.ScorerSpec(*s) for s in w.prefill_scorers])
            spec = epp.ProfileSpec(w.primary_filter, [epp.ScorerSpec(*s) for s in w.primary_scorers],
                                   affinity=epp.AffinityFilterSpec(*affinity))
            self.eng = epp.Engine(w.E, spec, prefill, block_size_tokens=w.block_size_tokens,
                                  max_prefix_blocks=w.max_prefix_blocks, non_cached_tokens=w.non_cached_tokens,
                                  tie_seed=tie_seed, **kw)
        else:
            self.eng = helpers.make_engine(w, tie_seed=tie_seed, **kw)
        self.eng.register_model(tg.MODEL)                 # helpers.setup_engine without its ext-less pool_set
        fh, _ = self.eng.hash_prompts(self.trace.family_tokens(), uniform_len=w.prompt_bytes)
        self.eng.index_load_snapshot(*self.trace.index_pairs(fh))
        self.role, self.kv, self.waiting, self.running = self.trace.pool()
        self.role = self.role.copy()
        self.role[list(absent)] = ABSENT
        present = np.array([e for e in range(w.E) if e not in set(absent)], dtype=np.uint32)
        self.present = present
        self.set_pool()
        _, self.ix, self.primary, self.prefill, _ = helpers.setup_oracle(orc, w, self.trace)
        if oracle_primary is not None:
            self.primary = oracle_primary
        elif affinity is not None:
            self.primary = orc.make_profile(w.primary_filter, list(w.primary_scorers), affinity=affinity)
        self.encode = orc.make_profile(0, list(encode)) if encode is not None else None
        self.ordinal = 0

    def set_pool(self, ext=None):
        """(Re)sends the pool snapshot; ext replaces the ext columns."""
        if ext is not None:
            self.ext = np.asarray(ext, np.float64).reshape(-1, self.w.E)
        p = self.present
        x = None if self.ext is None else np.ascontiguousarray(self.ext[:, p])
        self.eng.pool_set(p, self.role[p], self.kv[p], self.waiting[p], self.running[p], x)

    def close(self):
        self.eng.close()

    def tokens(self, b=0, R=None):
        return self.trace.requests(b * self.w.R, R or self.w.R)[0]

    def match(self, row):
        h = self.orc.hash_prompt(row.tobytes(), tg.MODEL, self.w.block_size_tokens, self.w.max_prefix_blocks)
        m, _ = self.ix.match_longest_prefix(h, self.w.E)
        return m, len(h)

    def expect(self, row, subset, ordinal, ext=None, multimodal=0, topk=0, primary=None):
        """orc_cycle_batch of one request on the pool narrowed to `subset` (None: the whole pool)."""
        role = self.role.copy()
        if subset is not None:
            keep = np.zeros(self.w.E, bool)
            keep[list(subset)] = True
            role[~keep] = ABSENT
        pool = self.orc.PoolState(role, self.kv, self.waiting, self.running, ext=self.ext if ext is None else ext)
        w = self.w
        kw = dict(tie_seed=self.tie_seed, tie_base=ordinal)
        if self.encode is not None:
            kw.update(encode=self.encode, multimodal=np.array([multimodal], np.uint8))
        if topk > 1:
            kw["topk"] = topk
        return self.orc.cycle_batch(tg.MODEL, w.block_size_tokens, w.max_prefix_blocks, w.non_cached_tokens, False, self.ix,
                                    primary or self.primary, self.prefill, pool, row[None],
                                    np.array([0, w.prompt_bytes], np.uint64), 1, **kw)

    def check(self, dec, det, tokens, subsets, ordinal0, where, **kw):
        dec = np.asarray(dec)
        for r, s in enumerate(subsets):
            if s is None and not kw.get("all_rows"):
                continue
            out = self.expect(tokens[r], s, ordinal0 + r, multimodal=int(kw["mm"][r]) if "mm" in kw else 0)
            odec, ototal = out[0], out[1]
            helpers.assert_decisions_equal(dec[r:r + 1], None if det is None else np.asarray(det)[r:r + 1], odec, ototal,
                                           where=f"{where} request {r} subset {None if s is None else len(s)}")
            if odec["status"][0] == 0:                     # the whole index's matchBlocks of the pick
                m, _ = self.match(tokens[r])
                assert int(dec["match_blocks"][r]) == int(m[int(odec["pick"][0])]), f"{where} request {r} match_blocks"


def _subsets(rng, E, R, sizes, every=2, absent=()):
    """Every `every`-th request whole-pool, the others restricted to random subsets of the given sizes (in turn)."""
    out = []
    for r in range(R):
        if r % every == 0:
            out.append(None)
            continue
        n = sizes[(r // every) % len(sizes)]
        s = set(rng.choice(E, size=min(n, E), replace=False).tolist())
        if absent and r % 3 == 1:
            s |= set(absent)
        out.append(sorted(s))
    return out


def _decs(epp, dec, det):
    import torch
    if isinstance(dec, torch.Tensor):
        torch.cuda.synchronize()
        return epp.decisions_from_torch(dec), np.frombuffer(det.cpu().numpy().tobytes(), dtype=epp.DETAIL_DTYPE)
    return dec, det


# ---- the batch shapes and paths -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
@pytest.mark.parametrize("path", ["device", "host"])
@pytest.mark.parametrize("name", ["config3", "config4"])
def test_parity_mixed_batches(epp, orc, name, path, tie_seed):
    """Mixed EPP_SUBSET_ALL / restricted rows of sizes 0 (empty), 1, 5, 33 and E, with stale slots, on the synchronous
    device path and the chunked host path."""
    import torch
    E = 64
    rig = Rig(epp, orc, name, E=E, R=192, tie_seed=tie_seed, absent=(61, 62, 63))
    rng = np.random.default_rng(17)
    try:
        for b in range(2):
            tokens = rig.tokens(b)
            subsets = _subsets(rng, E, rig.w.R, [1, 5, 33, E, 0], absent=(61, 62, 63))
            n0 = rig.eng.stats()["n_decisions"]
            data = torch.from_numpy(tokens.view(np.int32)).cuda() if path == "device" else tokens
            (dec, det), names = helpers.kernels_launched(
                lambda: rig.eng.schedule(data, uniform_len=rig.w.prompt_bytes, subsets=subsets), repeatable=False)
            dec, det = _decs(epp, dec, det)
            rig.check(dec, det, tokens, subsets, n0, f"{name} {path} batch {b}", all_rows=(b == 0))
            assert (dec["status"][[r for r, s in enumerate(subsets) if s == []]] == -1).all()
            if helpers.trace_complete(names):
                helpers.assert_ran(names, "k_subset_pick", absent=("k_cycle_small",), where=f"{name} {path}")
    finally:
        rig.close()


def test_role_filter_empties_the_subset(epp, orc):
    """config4: subsets of prefill-only endpoints leave the decode profile nothing (status -1); subsets of decode-only
    endpoints leave the prefill stage nobody (no prefill pick)."""
    rig = Rig(epp, orc, "config4", E=64, R=64)
    try:
        dec_ok = [e for e in range(64) if rig.role[e] in (0, 1, 3, 4, 7)]          # decode-filter (roles.go:46-48)
        pre_only = [e for e in range(64) if e not in dec_ok]
        assert pre_only and dec_ok
        tokens = rig.tokens()
        subsets = [pre_only if r % 2 else dec_ok[:8] for r in range(rig.w.R)]
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
        rig.check(dec, det, tokens, subsets, n0, "role-emptied")
        assert (dec["status"][1::2] == -1).all()
        assert (dec["prefill_pick"][0::2] == NO).all()
    finally:
        rig.close()


def test_pipelined_async_restricted_rows_in_both_chunks(epp, orc):
    import torch
    rig = Rig(epp, orc, "config3", E=64, R=8192, tie_seed=0x77)
    rng = np.random.default_rng(5)
    try:
        tokens = rig.tokens()
        rows = sorted(set(rng.choice(rig.w.R, size=96, replace=False).tolist()) | {0, 4095, 4096, 8191})
        subsets = [None] * rig.w.R
        for i, r in enumerate(rows):
            subsets[r] = sorted(rng.choice(64, size=[1, 5, 33, 64][i % 4], replace=False).tolist())
        dt = torch.from_numpy(tokens.view(np.int32)).cuda()
        dec0, _ = rig.eng.schedule(dt, uniform_len=rig.w.prompt_bytes)          # the same rows without subsets
        torch.cuda.synchronize()
        dec0 = epp.decisions_from_torch(dec0)
        n0 = rig.eng.stats()["n_decisions"]

        def run():
            r = rig.eng.schedule(dt, uniform_len=rig.w.prompt_bytes, subsets=subsets, asynchronous=True)
            rig.eng.synchronize()
            return r
        (dec, det), names = helpers.kernels_launched(run, repeatable=False)
        dec, det = _decs(epp, dec, det)
        sub = [r for r in rows]
        for r in sub:
            out = rig.expect(tokens[r], subsets[r], n0 + r)
            helpers.assert_decisions_equal(dec[r:r + 1], det[r:r + 1], out[0], out[1], where=f"pipelined request {r}")
        rest = np.ones(rig.w.R, bool)
        rest[sub] = False
        # whole-pool rows: only the tie ranks depend on the ordinal; the arg-max records do not
        for f in ("status", "score", "tie_count", "total_blocks"):
            np.testing.assert_array_equal(dec[f][rest], dec0[f][rest], err_msg=f)
        assert rig.eng.stats()["last_kernel_ms"][6] > 0
        if helpers.trace_complete(names):
            assert sum(c for n, c in names.items() if "k_hash_fused" in n) == 2          # two chunks: pipelined
            assert sum(c for n, c in names.items() if "k_subset_pick" in n) == 2
    finally:
        rig.close()


def test_subsets_past_1024_slots(epp, orc):
    E = 1536
    rig = Rig(epp, orc, "config3", E=E, R=24, tie_seed=3)
    rng = np.random.default_rng(9)
    try:
        tokens = rig.tokens()
        subsets = [sorted(rng.choice(E, size=[1100, 1400, E][r % 3], replace=False).tolist()) for r in range(rig.w.R)]
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
        rig.check(dec, det, tokens, subsets, n0, "past 1024")
    finally:
        rig.close()


# ---- configurations ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 4, 64])
@pytest.mark.parametrize("tie_seed", [0, 0xABC])
def test_topk_and_affinity_filter(epp, orc, k, tie_seed):
    """pick_k 1 / 4 / 64 and the prefix-cache-affinity-filter, whose len(endpoints) <= 1 gate and sticky sets are
    taken over the subset's candidates."""
    import torch
    aff = (0.5, 0.25, 0.0)
    E = 64
    rig = Rig(epp, orc, "config3", E=E, R=160, tie_seed=tie_seed, engine_kw=dict(pick_k=k), affinity=aff)
    try:
        w = rig.w
        rng = np.random.default_rng(k)
        tokens = rig.tokens()
        subsets = []
        for r in range(w.R):
            m, _ = rig.match(tokens[r])
            holders = [e for e in range(E) if m[e] > 0]
            if r % 4 == 0:
                subsets.append(None)
            elif r % 4 == 1 and holders:                    # one candidate: the gate keeps the filter off
                subsets.append([holders[0]])
            elif r % 4 == 2 and holders:                    # holders + others: sticky sets inside the subset
                subsets.append(sorted(set(holders[:2]) | set(rng.choice(E, size=6, replace=False).tolist())))
            else:
                subsets.append(sorted(rng.choice(E, size=12, replace=False).tolist()))
        n0 = rig.eng.stats()["n_decisions"]
        dt = torch.from_numpy(tokens.view(np.int32)).cuda()
        if k > 1:
            dec, det, lists = rig.eng.schedule(dt, uniform_len=w.prompt_bytes, subsets=subsets, topk=True)
            lists = {n: v.cpu().numpy() for n, v in lists.items()}
        else:
            dec, det = rig.eng.schedule(dt, uniform_len=w.prompt_bytes, subsets=subsets)
        dec, det = _decs(epp, dec, det)
        for r, s in enumerate(subsets):
            out = rig.expect(tokens[r], s, n0 + r, topk=k)
            helpers.assert_decisions_equal(dec[r:r + 1], det[r:r + 1], out[0], out[1], where=f"k={k} request {r}")
            if k > 1:
                want = [int(x) for x in out[2]["primary"][0] if x >= 0]
                got = [int(x) for x in lists["primary"][r].astype(np.int64) & 0xFFFFFFFF if int(x) != NO]
                assert got == want, f"k={k} request {r}"
                np.testing.assert_array_equal(lists["primary_scores"][r][: len(want)].view(np.uint64),
                                              out[2]["primary_scores"][0][: len(want)].view(np.uint64))
    finally:
        rig.close()


@pytest.mark.parametrize("kinds", [
    ((tg.QUEUE, 2.0, 0.0), (tg.PREFIX, 1.0, 0.0)),
    ((5, 3.0, 0.0), (tg.KV_UTIL, 1.0, 0.0)),                 # running-requests-size
    ((3, 1.0, 4.0), (tg.PREFIX, 2.0, 0.0)),                  # load-aware
])
def test_every_scorer_normalises_over_the_subset(epp, orc, kinds):
    """Queue / running min-max over the subset's candidates: landscapes where pool-wide and subset normalisation
    disagree (the subset omits the pool's extremes)."""
    E = 64
    rig = Rig(epp, orc, "config3", E=E, R=96, primary=kinds)
    rng = np.random.default_rng(21)
    try:
        rig.waiting[:] = rng.integers(0, 40, E)
        rig.running[:] = rng.integers(0, 40, E)
        rig.waiting[0], rig.running[0] = 1000, 1000            # pool extremes outside every subset
        rig.waiting[1], rig.running[1] = 0, 0
        rig.eng.pool_set(np.arange(E, dtype=np.uint32), rig.role, rig.kv, rig.waiting, rig.running)
        tokens = rig.tokens()
        subsets = [sorted(rng.choice(np.arange(2, E), size=[3, 9, 20][r % 3], replace=False).tolist()) for r in range(rig.w.R)]
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
        rig.check(dec, det, tokens, subsets, n0, f"scorers {kinds}")
    finally:
        rig.close()


ACTIVE, TOKEN, EXTERNAL = 7, 6, 4
LOAD_SCORERS = ((ACTIVE, 2.0, 1.0, 1, 0.0),                 # active-request: ext column 1, maxBusyScore 1, idle 0
                (TOKEN, 1.0, 65536.0, 0, 0.0),              # token-load: ext column 0, queueThresholdTokens 65536
                (EXTERNAL, 1.0, 2.0),                       # external: ext column 2
                (tg.PREFIX, 2.0, 0.0))


@pytest.mark.parametrize("affinity", [None, (0.5, 0.0, 0.0)])
def test_active_request_token_load_and_external_over_the_subset(epp, orc, affinity):
    """The active-request max is taken over the subset's candidates (and over the sticky set when the affinity filter
    narrows): the pool's busiest endpoints lie outside every subset, and listed slots that are no candidates -- stale
    slots and slots the decode filter drops -- are busier still."""
    E = 64
    rng = np.random.default_rng(33)
    ext = np.zeros((3, E))
    ext[0] = rng.integers(0, 200000, E)                     # tokens in flight
    ext[1] = rng.integers(0, 20, E)                         # requests in flight
    ext[2] = rng.random(E)
    ext[1, [0, 1]] = 1000                                   # the pool's maximum: never listed
    ext[1, [58, 59, 60]] = 3000                             # listed, dropped by the decode filter
    ext[1, [61, 62, 63]] = 5000                             # listed, not in the pool
    rig = Rig(epp, orc, "config3", E=E, R=128, primary=LOAD_SCORERS, absent=(61, 62, 63), ext=ext, affinity=affinity)
    try:
        rig.role[[58, 59, 60]] = 2                          # prefill: not a decode candidate
        rig.set_pool()
        tokens = rig.tokens()
        subsets = []
        for r in range(rig.w.R):
            m, _ = rig.match(tokens[r])
            holders = [e for e in range(2, 58) if m[e] > 0][:3]
            s = set(rng.choice(np.arange(2, 58), size=[2, 6, 20][r % 3], replace=False).tolist()) | set(holders)
            if r % 2:
                s |= {58, 59, 60, 61, 62, 63}
            subsets.append(sorted(s))
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
        rig.check(dec, det, tokens, subsets, n0, f"load scorers affinity={affinity}")
    finally:
        rig.close()


def test_inflight_counters_fed_to_the_oracle(epp, orc):
    """inflight_load = 1: token-load and active-request read the engine's counters.  Expected: the oracle with the
    counters of tools/inflight_model.py (the adds of every earlier call's picks, and releases) as ext columns."""
    from tools import inflight_model as IM
    prim = tuple(tg.baseline_configs()["config4"].primary_scorers) + (
        (IM.TOKEN_LOAD, 1.0, 4096.0, IM.TOKEN_COL, 0.0), (IM.ACTIVE_REQUEST, 2.0, 1.0, IM.REQUEST_COL, 0.0))
    rig = Rig(epp, orc, "config4", E=64, R=128, primary=prim, engine_kw=dict(inflight_load=True), tie_seed=0x1F)
    rng = np.random.default_rng(2)
    cnt = IM.Counters(64)
    try:
        for b in range(3):
            tokens = rig.tokens(b)
            subsets = _subsets(rng, 64, rig.w.R, [1, 5, 33, 64])
            n0 = rig.eng.stats()["n_decisions"]
            ext = cnt.ext()
            dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
            for r, s in enumerate(subsets):
                out = rig.expect(tokens[r], s, n0 + r, ext=ext)
                helpers.assert_decisions_equal(dec[r:r + 1], det[r:r + 1], out[0], out[1], where=f"inflight batch {b} request {r}")
            cnt.pre_request(dec, np.full(rig.w.R, rig.w.prompt_bytes))
            rel = [int(dec["pick"][r]) for r in range(0, rig.w.R, 3) if dec["status"][r] == 0]
            rig.eng.inflight_release(np.array(rel, np.uint32), np.full(len(rel), rig.w.prompt_bytes, np.uint64))
            cnt.release(rel, [rig.w.prompt_bytes] * len(rel))
            got_req, got_tok = rig.eng.inflight_get()
            np.testing.assert_array_equal(got_req[:64], cnt.req, err_msg=f"requests after batch {b}")
            np.testing.assert_array_equal(got_tok[:64], cnt.tok, err_msg=f"tokens after batch {b}")
        assert cnt.req.max() > 1
    finally:
        rig.close()


def test_affinity_filter_ttft_gate_over_the_subset(epp, orc):
    """The filter's TTFT gate compares the best predicted TTFT of the subset's sticky candidates with the best of its
    other candidates (plugin.go:137-146): a TTFT column and a penalty > 0."""
    E = 64
    rng = np.random.default_rng(41)
    ttft = rng.uniform(0.0, 200.0, (1, E))
    aff = (0.5, 0.0, 40.0, 0)
    rig = Rig(epp, orc, "config3", E=E, R=160, tie_seed=0x2A, ext=ttft, affinity=aff)
    try:
        tokens = rig.tokens()
        subsets = []
        for r in range(rig.w.R):
            m, _ = rig.match(tokens[r])
            holders = [e for e in range(E) if m[e] > 0]
            s = set(rng.choice(E, size=[3, 8, 16][r % 3], replace=False).tolist()) | set(holders[:2])
            subsets.append(sorted(s))
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
        rig.check(dec, det, tokens, subsets, n0, "ttft gate")
        # the gate decides something here: without the penalty some decisions change
        free = orc.make_profile(rig.w.primary_filter, list(rig.w.primary_scorers), affinity=aff[:2] + (0.0, 0))
        changed = sum(int(rig.expect(tokens[r], s, n0 + r, primary=free)[0]["pick"][0]) != int(dec["pick"][r])
                      for r, s in enumerate(subsets))
        assert changed > 0
    finally:
        rig.close()


def test_chunked_host_batch_with_restricted_rows_in_every_chunk(epp, orc):
    """64 KiB prompts: a host batch of 1600 requests runs as several chunks of the chunked host path, each with its own
    restricted rows."""
    E = 64
    rig = Rig(epp, orc, "config3", E=E, R=1600, T=16384, tie_seed=0)
    rng = np.random.default_rng(55)
    try:
        tokens = rig.tokens()
        assert tokens.nbytes > 2 * (48 << 20)               # more than two 48 MiB chunks
        rows = sorted(set(rng.choice(rig.w.R, size=60, replace=False).tolist()) | {0, 767, 768, 1535, 1536, 1599})
        subsets = [None] * rig.w.R
        for i, r in enumerate(rows):
            subsets[r] = sorted(rng.choice(E, size=[1, 5, 33, 64][i % 4], replace=False).tolist())
        dec0, _ = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes)
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets)
        for r in rows:
            out = rig.expect(tokens[r], subsets[r], n0 + r)
            helpers.assert_decisions_equal(dec[r:r + 1], det[r:r + 1], out[0], out[1], where=f"chunked host request {r}")
        rest = np.ones(rig.w.R, bool)
        rest[rows] = False
        np.testing.assert_array_equal(dec[rest], dec0[rest])   # lowest-slot rule: whole-pool rows do not move
        assert rig.eng.stats()["last_kernel_ms"][6] == 0.0     # host batches do not time the subset kernel
    finally:
        rig.close()


def test_disagg_with_decider_and_encode_stage(epp, orc):
    enc = [(tg.QUEUE, 1.0, 0.0), (tg.PREFIX, 2.0, 0.0)]
    rig = Rig(epp, orc, "config4", E=64, R=128, tie_seed=0x99, encode=enc)
    rng = np.random.default_rng(8)
    try:
        tokens = rig.tokens()
        mm = (rng.random(rig.w.R) < 0.5).astype(np.uint8)
        subsets = _subsets(rng, 64, rig.w.R, [5, 33, 64, 1])
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=subsets, multimodal=mm)
        rig.check(dec, det, tokens, subsets, n0, "encode", mm=mm, all_rows=True)
        assert det["encode_ran"].any() and det["prefill_ran"].any()
    finally:
        rig.close()


def test_lora_affinity(epp, orc):
    E, n_models = 32, 3
    prim = ((tg.PREFIX, 2.0, 0.0), (8, 1.0, 0.0))
    rig = Rig(epp, orc, "config3", E=E, R=64, primary=prim)
    rng = np.random.default_rng(4)
    try:
        for m in range(1, n_models):
            rig.eng.register_model(b"adapter-%d" % m)
        max_active = rng.integers(1, 3, E).astype(np.int32)
        members = [(int(e), int(m), int(rng.integers(1, 3))) for m in range(n_models) for e in rng.choice(E, 6, replace=False)]
        loaded = np.zeros(E, np.int32)
        for e, _, _ in members:
            loaded[e] += 1
        rig.eng.pool_set_lora(np.arange(E, dtype=np.uint32), max_active, loaded, members)
        tokens = rig.tokens()
        mids = rng.integers(0, n_models, rig.w.R).astype(np.uint32)
        mids[:] = 0                                            # the trace's prompts hash with model 0
        subsets = [sorted(rng.choice(E, size=[4, 11][r % 2], replace=False).tolist()) for r in range(rig.w.R)]
        n0 = rig.eng.stats()["n_decisions"]
        dec, det = rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, model_ids=mids, subsets=subsets)
        for r, s in enumerate(subsets):
            st = np.zeros(E, np.uint8)
            for e, m, x in members:
                if m == mids[r] and (st[e] == 0 or x == 1):
                    st[e] = x
            role = rig.role.copy()
            keep = np.zeros(E, bool)
            keep[s] = True
            role[~keep] = ABSENT
            pool = orc.PoolState(role, rig.kv, rig.waiting, rig.running).set_lora(st, max_active, loaded)
            out = orc.cycle_batch(tg.MODEL, rig.w.block_size_tokens, rig.w.max_prefix_blocks, 0, False, rig.ix, rig.primary,
                                  None, pool, tokens[r][None], np.array([0, rig.w.prompt_bytes], np.uint64), 1,
                                  tie_base=n0 + r)
            helpers.assert_decisions_equal(dec[r:r + 1], det[r:r + 1], out[0], out[1], where=f"lora request {r}")
    finally:
        rig.close()


def test_nohit_lru_cold_for_the_subset(epp, orc):
    """Requests warm for the pool but cold for their subset (no listed candidate holds a block) are scored with the
    LRU's cold ranks over the subset's candidates, and their picks are Added to the LRU."""
    E, w_nh = 64, 2.0
    prim = tuple(tg.baseline_configs()["config3"].primary_scorers) + ((NH.NO_HIT_LRU, w_nh, 0.0),)
    ext_prim = orc.make_profile(tg.FILTER_DECODE, list(prim[:-1]) + [(4, w_nh, 0.0)])
    rig = Rig(epp, orc, "config3", E=E, R=96, primary=prim, oracle_primary=ext_prim)
    w = rig.w
    lru = NH.GoLRU(0)
    rng = np.random.default_rng(12)
    cand_all = [e for e in range(E) if rig.role[e] in (0, 1, 3, 4, 7)]
    try:
        n_warm_cold = 0
        for b in range(3):
            tokens = rig.tokens(b)
            subsets, cold = [], []
            for r in range(w.R):
                m, _ = rig.match(tokens[r])
                holders = [e for e in cand_all if m[e] > 0]
                if r % 5 == 0:
                    s = None
                elif holders and r % 2:                 # warm for the pool, cold for the subset
                    s = sorted(rng.choice([e for e in range(E) if m[e] == 0], size=7, replace=False).tolist())
                    n_warm_cold += 1
                else:
                    s = sorted(rng.choice(E, size=9, replace=False).tolist())
                subsets.append(s)
            keys = lru.keys()
            n0 = rig.eng.stats()["n_decisions"]
            dec, det = rig.eng.schedule(tokens, uniform_len=w.prompt_bytes, subsets=subsets)
            for r, s in enumerate(subsets):
                m, _ = rig.match(tokens[r])
                cands = [e for e in cand_all if s is None or e in s]
                c = NH.is_cold(cands, m)
                col = NH.cold_column(cands, keys, E) if c else np.full(E, 0.5)
                out = rig.expect(tokens[r], s, n0 + r, ext=col.reshape(1, E), primary=ext_prim)
                helpers.assert_decisions_equal(dec[r:r + 1], det[r:r + 1], out[0], out[1], where=f"nohit batch {b} request {r}")
                if c and dec["status"][r] == 0:
                    lru.add(int(dec["pick"][r]))
            assert rig.eng.nohit_lru_get() == lru.keys(), f"LRU after batch {b}"
        assert n_warm_cold > 0
    finally:
        rig.close()


@pytest.mark.parametrize("picker", [PM.RANDOM, PM.WEIGHTED_RANDOM])
@pytest.mark.parametrize("k", [1, 4])
def test_random_pickers_all_explicit(epp, orc, picker, k):
    E, tie_seed = 64, 0x1234
    w = tg.baseline_configs()["config3"].scaled(E=E, R=128, T=512)
    trace = tg.Trace(w)
    spec = epp.ProfileSpec(w.primary_filter, [epp.ScorerSpec(*s) for s in w.primary_scorers], picker=picker)
    rng = np.random.default_rng(picker * 10 + k)
    with epp.Engine(E, spec, block_size_tokens=w.block_size_tokens, max_prefix_blocks=w.max_prefix_blocks,
                    tie_seed=tie_seed, pick_k=k) as eng:
        helpers.setup_engine(eng, w, trace)
        _, ix, prim, _, _ = helpers.setup_oracle(orc, w, trace)
        role, kv, waiting, running = trace.pool()
        tokens = trace.requests(0, w.R)[0]
        subsets = [sorted(rng.choice(E, size=[1, 5, 33, E][r % 4], replace=False).tolist()) for r in range(w.R)]
        n0 = eng.stats()["n_decisions"]
        if k > 1:
            dec, _, lists = eng.schedule(tokens, uniform_len=w.prompt_bytes, subsets=subsets, topk=True)
        else:
            dec, _ = eng.schedule(tokens, uniform_len=w.prompt_bytes, subsets=subsets)
        weights = [s[1] for s in w.primary_scorers]
        for r, s in enumerate(subsets):
            h = orc.hash_prompt(tokens[r].tobytes(), tg.MODEL, w.block_size_tokens, w.max_prefix_blocks)
            m, _ = ix.match_longest_prefix(h, E)
            r_role = role.copy()
            keep = np.zeros(E, bool)
            keep[s] = True
            r_role[~keep] = ABSENT
            scores, _, _, _ = orc.profile_run(prim, orc.PoolState(r_role, kv, waiting, running), m, len(h))
            cands = [e for e in s if scores[e] != -1.0]
            picks = PM.draw_k(picker, cands, None, {e: float(scores[e]) for e in cands}, set(), tie_seed, 4 * (n0 + r),
                              weights, k, gaps=False)
            assert int(dec["pick"][r]) == picks[0][0] and dec["score"][r] == picks[0][1], f"request {r}"
            assert int(dec["tie_count"][r]) == len(cands)
            if k > 1:
                got = [int(x) for x in lists["primary"][r] if int(x) != NO]
                assert got == [p for p, _ in picks], f"request {r}"


# ---- indexing, equivalences, launches ----------------------------------------------------------------------------------
def test_keep_hashes_indexes_the_subset_picks(epp):
    """PreRequest (epp_index_add_picked) indexes every request's prefix on its pick, subset picks included."""
    w = tg.baseline_configs()["config3"].scaled(E=64, R=32, T=512)
    trace = tg.Trace(w)
    with helpers.make_engine(w) as eng:                    # an incrementally built (empty) index
        eng.register_model(tg.MODEL)
        role, kv, waiting, running = trace.pool()
        eng.pool_set(np.arange(w.E, dtype=np.uint32), role, kv, waiting, running)
        tokens = trace.requests(0, w.R)[0]
        cand = [e for e in range(w.E) if role[e] in (0, 1, 3, 4, 7)]
        subsets = [[cand[(3 * r) % len(cand)]] if r % 2 else None for r in range(w.R)]
        dec, _ = eng.schedule(tokens, uniform_len=w.prompt_bytes, subsets=subsets, keep_hashes=True)
        eng.index_add_picked()
        hashes, _ = eng.hash_prompts(tokens, uniform_len=w.prompt_bytes)
        for r in range(w.R):
            assert dec["status"][r] == 0
            if subsets[r] is not None:
                assert int(dec["pick"][r]) == subsets[r][0]
            assert int(dec["pick"][r]) in eng.index_get(int(hashes[r, 0])), f"request {r}"


@pytest.mark.parametrize("tie_seed", [0, 0x5EED])
def test_all_whole_pool_equals_schedule_and_full_subset_equals_it(epp, orc, tie_seed):
    import torch
    E = 64
    rig = Rig(epp, orc, "config4", E=E, R=256, tie_seed=tie_seed)
    rig2 = Rig(epp, orc, "config4", E=E, R=256, tie_seed=tie_seed)
    try:
        tokens = rig.tokens()
        dt = torch.from_numpy(tokens.view(np.int32)).cuda()
        (d1, t1), n1 = helpers.kernels_launched(lambda: rig.eng.schedule(dt, uniform_len=rig.w.prompt_bytes), repeatable=False)
        (d2, t2), n2 = helpers.kernels_launched(
            lambda: rig2.eng.schedule(dt, uniform_len=rig.w.prompt_bytes, subsets=[None] * rig.w.R), repeatable=False)
        torch.cuda.synchronize()
        assert torch.equal(d1, d2) and torch.equal(t1, t2)
        if helpers.trace_complete(n2):
            assert not helpers.ran(n2, "k_subset_pick")
        # a full explicit subset: the max-score decisions of no subset
        d3, t3 = rig.eng.schedule(dt, uniform_len=rig.w.prompt_bytes, subsets=[list(range(E))] * rig.w.R)
        d4, t4 = rig2.eng.schedule(dt, uniform_len=rig.w.prompt_bytes)
        torch.cuda.synchronize()
        assert torch.equal(d3, d4) and torch.equal(t3, t4)
    finally:
        rig.close()
        rig2.close()


# ---- rejections ---------------------------------------------------------------------------------------------------------
def test_invalid_subsets_change_nothing(epp, orc):
    E = 32
    prim = tuple(tg.baseline_configs()["config3"].primary_scorers) + ((NH.NO_HIT_LRU, 1.0, 0.0),)
    rig = Rig(epp, orc, "config3", E=E, R=8, primary=prim, engine_kw=dict(inflight_load=True))
    try:
        tokens = rig.tokens()
        rig.eng.schedule(tokens, uniform_len=rig.w.prompt_bytes, subsets=[[1, 2]] * rig.w.R)
        before = (rig.eng.stats()["n_decisions"], rig.eng.nohit_lru_get(), [a.tolist() for a in rig.eng.inflight_get()])
        import ctypes
        C = epp.capi
        lib = C.load()
        b, R, _, _ = rig.eng._batch(tokens, uniform_len=rig.w.prompt_bytes)
        dec = np.zeros(R, dtype=epp.DECISION_DTYPE)
        size = ctypes.sizeof(C.Subset)
        bad = [
            (np.full(R, 2, np.uint32), np.array([3, 3], np.uint32), size),        # duplicated slot
            (np.full(R, 2, np.uint32), np.array([5, 4], np.uint32), size),        # unsorted
            (np.full(R, 1, np.uint32), np.array([E], np.uint32), size),           # slot >= max_endpoints
            (np.full(R, 1, np.uint32), np.array([1], np.uint32), size - 8),       # struct_size
        ]
        offsets = np.zeros(R, np.uint64)
        for counts, slots, sz in bad:
            s = C.Subset()
            s.struct_size = sz
            s.counts, s.offsets, s.slots = counts.ctypes.data, offsets.ctypes.data, slots.ctypes.data
            rc = lib.epp_schedule_subset(rig.eng._h, ctypes.byref(b), ctypes.byref(s), dec.ctypes.data, None, 0, None)
            assert rc == C.EPP_ERR_INVALID
        after = (rig.eng.stats()["n_decisions"], rig.eng.nohit_lru_get(), [a.tolist() for a in rig.eng.inflight_get()])
        assert after == before
    finally:
        rig.close()


def test_sharded_engine_rejects_subsets(epp, orc):
    import torch
    rig = Rig(epp, orc, "config3", E=32, R=8)
    try:
        rig.eng.shard_set(0, 16)
        role, kv, waiting, running = rig.trace.pool()
        rig.eng.pool_set(np.arange(32, dtype=np.uint32), role, kv, waiting, running)
        n0 = rig.eng.stats()["n_decisions"]
        dt = torch.from_numpy(rig.tokens().view(np.int32)).cuda()
        with pytest.raises(epp.EngineError) as ei:
            rig.eng.schedule(dt, uniform_len=rig.w.prompt_bytes, subsets=[[1]] * rig.w.R)
        assert ei.value.code == epp.capi.EPP_ERR_INVALID
        assert rig.eng.stats()["n_decisions"] == n0
    finally:
        rig.close()


# ---- the micro-batcher -------------------------------------------------------------------------------------------------
def test_batcher_mixes_subset_and_plain_submits(epp, orc):
    E = 64
    rig = Rig(epp, orc, "config3", E=E, R=256)
    rng = np.random.default_rng(31)
    try:
        tokens = rig.tokens()
        subsets = _subsets(rng, E, rig.w.R, [1, 5, 33, E], every=3)
        results = [None] * rig.w.R
        with epp.Batcher(rig.eng, max_batch=32, max_delay_us=200) as bt:
            def worker(t):
                for r in range(t, rig.w.R, 8):
                    tk = bt.submit(tokens[r].tobytes(), subset=subsets[r])
                    results[r] = bt.wait(tk)[0]
            th = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
            for x in th:
                x.start()
            for x in th:
                x.join()
            with pytest.raises(epp.EngineError) as ei:
                bt.submit(tokens[0].tobytes(), subset=list(range(1025)))
            assert ei.value.code == epp.capi.EPP_ERR_CAPACITY
        for r, s in enumerate(subsets):
            d = results[r]
            # flush ordinals depend on the threads' interleaving: the engine runs the lowest-slot tie rule (tie_seed 0),
            # under which no decision depends on its ordinal
            out = rig.expect(tokens[r], s, 0)
            helpers.assert_decisions_equal(np.array([d]), None, out[0], out[1], where=f"batcher request {r}")
    finally:
        rig.close()
