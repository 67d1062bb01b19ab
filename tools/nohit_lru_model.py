"""CPU restatement of the no-hit-lru scorer (scorer/nohitlru/no_hit_lru.go) and of the engine's batch semantics for it:
golang-lru's Add / Keys, the cold and warm score columns, and a scheduling model that evaluates every request of a call
against the LRU as it stood when the call started and then Adds the cold requests' picks in request order.  The other
scorers' columns come from the C oracle (oracle/pyoracle.py score_column), so the engine's tests compare against code that
shares nothing with it.  Also the device update's algorithm (sequence numbers, atomicMax, trim to lruSize) on the CPU."""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

NO_HIT_LRU = 9
NO = 0xFFFFFFFF


class GoLRU:
    """hashicorp/golang-lru/v2 Cache: Add moves an existing key to most-recent or inserts it and evicts the oldest beyond
    the size; Keys() lists oldest first."""

    def __init__(self, size: int):
        self.size = size if size > 0 else 1024           # no_hit_lru.go:93-95
        self.d = OrderedDict()

    def add(self, k):
        if k in self.d:
            self.d.move_to_end(k)
        else:
            self.d[k] = None
            if len(self.d) > self.size:
                self.d.popitem(last=False)

    def keys(self):
        return list(self.d)


def cold_column(cand, lru_keys, E):
    """scoreColdRequestByLRU (no_hit_lru.go:198-242) over the candidate slots in ascending order -> [E] (0 elsewhere)."""
    cand = sorted(cand)
    n = len(cand)
    col = np.zeros(E, dtype=np.float64)
    if n == 1:
        col[cand[0]] = 1.0
        return col
    pos = {k: i for i, k in enumerate(lru_keys)}
    never = [e for e in cand if e not in pos]
    for i, e in enumerate(never):
        col[e] = 1.0 - float(i) / float(n - 1)
    for e in cand:
        if e in pos:
            s = 1.0 - float(len(never) + pos[e]) / float(n - 1)
            col[e] = 0.0 if s < 0 else s
    return col


def is_cold(cand, match_row):
    """isColdRequest (no_hit_lru.go:140-155): no candidate has MatchBlocks() > 0."""
    return not any(int(match_row[e]) > 0 for e in cand)


class Model:
    """Scheduler.Schedule for the single / disagg handler with the lowest-slot or the reproducible tie rule, over
    injected match rows.  profiles: [(filter, [(kind, weight, param[, column[, param2]]), ...])] for decode / prefill;
    encode: the same for the encode profile (disagg_profile_handler.go:284-295, run for multimodal requests)."""

    def __init__(self, orc, pool, E, profiles, lru_size, *, nct=0, always=False, block_size_tokens=16, tie_seed=0,
                 encode=None):
        self.orc, self.pool, self.E = orc, pool, E
        self.profiles = list(profiles) + ([None] * (2 - len(profiles)) + [encode] if encode else [])
        self.n_stages = len(profiles)
        self.lru = GoLRU(lru_size)
        self.nct, self.always, self.bst, self.tie_seed = nct, always, block_size_tokens, tie_seed
        self.n_decisions = 0
        self._cand, self._cols = {}, {}

    def candidates(self, filt):
        if filt not in self._cand:
            orc = self.orc
            scores, _, _, _ = orc.profile_run(orc.make_profile(filt, [(1, 0.0, 0.0)]), self.pool,
                                              np.zeros(self.E, dtype=np.int32), 0)
            self._cand[filt] = [e for e in range(self.E) if scores[e] != -1.0]
        return self._cand[filt]

    def column(self, pi, s, mask):
        """Clamped raw column of the request-independent scorer s of profile pi (C oracle), cached per pool."""
        if (pi, s) not in self._cols:
            sc = tuple(self.profiles[pi][1][s])
            col = self.orc.score_column(sc, self.pool, mask, np.zeros(self.E, dtype=np.int32), 0)
            self._cols[(pi, s)] = np.minimum(np.maximum(col, 0.0), 1.0)
        return self._cols[(pi, s)]

    def run_profile(self, pi, match_row, total, key, lru_keys):
        """-> (pick, max, ties, cold or None when the profile lacks the scorer / has no candidates)."""
        filt, scorers = self.profiles[pi]
        cand = self.candidates(filt)
        if not cand:
            return NO, 0.0, 0, None
        has = any(sc[0] == NO_HIT_LRU for sc in scorers)
        cold = is_cold(cand, match_row) if has else None
        mask = np.zeros(self.E, dtype=np.uint8)
        mask[cand] = 1
        idx = np.asarray(cand)
        acc = np.zeros(len(cand), dtype=np.float64)
        for s, sc in enumerate(scorers):
            if sc[0] == NO_HIT_LRU:
                col = cold_column(cand, lru_keys, self.E) if cold else np.full(self.E, 0.5)
            elif sc[0] == 0:                              # prefix-cache-scorer, scorer/prefix/plugin.go:100-111
                col = (np.asarray(match_row, dtype=np.float64) / float(total)) if total else np.zeros(self.E)
                col = np.minimum(np.maximum(col, 0.0), 1.0)
            else:
                col = self.column(pi, s, mask)
            acc = acc + col[idx] * sc[1]                  # clamp(score) * weight, in scorer order, never fused
        mx = acc.max()
        ties = [int(e) for e in idx[acc == mx]]
        pick = ties[0]
        if self.tie_seed and len(ties) > 1:
            pick = ties[self.orc.tie_rank(self.tie_seed, key, len(ties))]
        return pick, float(mx), len(ties), cold

    def set_pool(self, pool):
        self.pool = pool
        self._cand, self._cols = {}, {}

    def schedule(self, match, total, in_len=None, multimodal=None):
        """One scheduling call: decisions against the LRU at the call's start, then PreRequest in request order.
        -> list of (status, pick, score, prefill_pick, match_blocks, cold)."""
        keys = self.lru.keys()
        out = []
        for r in range(match.shape[0]):
            key = 4 * (self.n_decisions + r)
            pick, mx, ties, cold = self.run_profile(0, match[r], int(total[r]), key, keys)
            last_cold = bool(cold)
            if ties == 0:
                out.append((-1, NO, 0.0, NO, 0, False))
                continue
            mb = int(match[r][pick])
            ppick = NO
            if len(self.profiles) > 2 and multimodal is not None and multimodal[r]:    # encode stage, key + 2
                _, _, _, c2 = self.run_profile(2, match[r], int(total[r]), key + 2, keys)
                if c2 is not None:
                    last_cold = c2
            if self.n_stages > 1:
                il = 0 if in_len is None else int(in_len[r])
                go = self.always or self.orc.pd_decide(self.nct, il, mb, self.bst)
                if go:
                    p1, _, t1, c1 = self.run_profile(1, match[r], int(total[r]), key + 1, keys)
                    if t1:
                        ppick = p1
                    if c1 is not None:
                        last_cold = c1
            out.append((0, pick, mx, ppick, mb, last_cold))
        for st, pick, _, ppick, _, cold in out:          # PreRequest (no_hit_lru.go:279-321), in request order
            if st == 0 and cold:
                self.lru.add(pick)
                if ppick != NO:
                    self.lru.add(ppick)
        self.n_decisions += match.shape[0]
        return out


def device_update(last_seq, adds_per_call, lru_size):
    """The engine's update (csrc/nohit_lru.cu) on the CPU: per call, last_seq[e] = max(last_seq[e], seq0 + 2r + k) for
    every Add (r = request, k = 0 pick / 1 prefill pick), then every member but the lru_size newest is cleared.
    adds_per_call: list of calls, each a list of (r, k, slot).  Returns the LRU oldest first after every call."""
    seq0 = 1
    out = []
    for adds in adds_per_call:
        R = 1 + max([r for r, _, _ in adds], default=-1)
        for r, k, e in adds:
            last_seq[e] = max(last_seq[e], seq0 + 2 * r + k)
        seq0 += 2 * max(R, 1)
        members = sorted((s, e) for e, s in enumerate(last_seq) if s)
        for s, e in members[:max(0, len(members) - lru_size)]:
            last_seq[e] = 0
        out.append([e for s, e in members[max(0, len(members) - lru_size):]])
    return out
