"""CPU restatement of the label filters (include/epp_engine.h "Label filters"): what each requirement keeps, the engine's
interning of keys and values into per-slot codes and per-requirement masks, and a scheduling model built on the C oracle.

The oracle itself knows only role filters.  A profile with label filters is the same profile run on a pool in which the
slots its label filters drop are absent (role 0xFF), so decisions come from orc.profile_run / orc.schedule on that
narrowed pool, and the P/D stages are joined with orc.pd_decide as the disagg handler joins them."""
from __future__ import annotations

import numpy as np

IN, NOT_IN, EXISTS, DOES_NOT_EXIST, BY_LABEL, BY_LABEL_OR_ABSENT = range(6)
OTHER = 63                        # code of a present value that no requirement names
MAX_KEYS, MAX_VALUES = 16, 62
NO = 0xFFFFFFFF


def matches(req, labels) -> bool:
    """One requirement (key, op, values) on a label dict (None = no labels)."""
    key, op, values = req
    labels = labels or {}
    present = key in labels
    v = labels.get(key, "")
    if op == IN:
        return present and v in values
    if op == NOT_IN:
        return not present or v not in values
    if op == EXISTS:
        return present
    if op == DOES_NOT_EXIST:
        return not present
    if op == BY_LABEL:                # filter.go:108-111: an absent key reads ""
        return v in values
    if op == BY_LABEL_OR_ABSENT:
        return not present or v in values
    raise ValueError(op)


def keeps(reqs, labels) -> bool:
    return all(matches(q, labels) for q in reqs)


def compile_masks(profiles):
    """profiles: list of requirement lists.  -> (keys, codes [dict value -> 1..62 per key], per profile [(key, mask)])."""
    keys, codes, out = [], [], []
    for reqs in profiles:
        comp = []
        for key, op, values in reqs:
            if key not in keys:
                if len(keys) == MAX_KEYS:
                    raise ValueError("too many keys")
                keys.append(key)
                codes.append({})
            k = keys.index(key)
            named = 0
            for v in values:
                if v not in codes[k]:
                    if len(codes[k]) == MAX_VALUES:
                        raise ValueError("too many values")
                    codes[k][v] = len(codes[k]) + 1
                named |= 1 << codes[k][v]
            full = (1 << 64) - 1
            mask = {IN: named, NOT_IN: full & ~named, EXISTS: full & ~1, DOES_NOT_EXIST: 1,
                    BY_LABEL: named | (1 if "" in values else 0), BY_LABEL_OR_ABSENT: named | 1}[op]
            comp.append((k, mask))
        out.append(comp)
    return keys, codes, out


def label_codes(keys, codes, labels_per_slot):
    """-> uint8 [len(keys)][E]: 0 absent, the value's code, or OTHER."""
    lc = np.zeros((len(keys), len(labels_per_slot)), dtype=np.uint8)
    for e, lb in enumerate(labels_per_slot):
        for k, key in enumerate(keys):
            if lb and key in lb:
                lc[k, e] = codes[k].get(lb[key], OTHER)
    return lc


def keep_vector(comp, lc):
    """The compiled requirements of one profile over every slot -> bool [E]."""
    keep = np.ones(lc.shape[1], dtype=bool)
    for k, mask in comp:
        keep &= ((np.uint64(mask) >> lc[k].astype(np.uint64)) & np.uint64(1)).astype(bool)
    return keep


def narrowed(orc, role, kv, waiting, running, ext, keep):
    """The oracle pool with every slot the label filters drop marked absent."""
    r = np.where(keep, np.asarray(role, dtype=np.uint8), np.uint8(0xFF))
    return orc.PoolState(r, kv, waiting, running, ext)


def pd_schedule(orc, primary, prefill, pool_dec, pool_pre, match, total, bst, in_len, nct, always=False):
    """The disagg handler with a decode pool and a prefill pool narrowed separately -> dict of the decision fields."""
    d = orc.schedule(primary, None, pool_dec, match, total, bst, in_len, nct)
    out = dict(status=d.status, pick=NO if d.pick < 0 else d.pick, score=d.score, tie_count=d.tie_count,
               prefill_pick=NO, prefill_score=0.0, prefill_tie_count=0, prefill_ran=0)
    if d.status != 0 or prefill is None:
        return out
    go = always or orc.pd_decide(nct, in_len, int(match[d.pick]), bst)
    out["prefill_ran"] = int(go)
    if go:
        _, mx, pick, amax = orc.profile_run(prefill, pool_pre, match, total)
        if amax:
            out.update(prefill_pick=pick, prefill_score=mx, prefill_tie_count=len(amax))
    return out
