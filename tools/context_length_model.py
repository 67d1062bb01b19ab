"""CPU restatement of the context-length-aware plugin (scorer/contextlengthaware/context_length_aware.go, include/
epp_engine.h "Context length"): parseContextRange, calculateRangeScore, the filter, the request's context length, and a
scheduling model built on the C oracle.

The Go functions are restated line by line on Python ints (wrapped to int64 where Go's int arithmetic wraps) and floats
(IEEE doubles, no fused multiply-add).  A profile is decided as tools/latency_model.py decides one: the chain runs here,
the pool handed to the unchanged oracle holds only the final set, and the latency and context-length scorers become
external columns holding this module's scores.
"""
from __future__ import annotations

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import latency_model as lm  # noqa: E402
import picker_model as pm  # noqa: E402

DEFAULT_LABEL = "llm-d.ai/context-length-range"
CHAR_TO_TOKEN = 0.25
SCORER_EXTERNAL, SCORER_LATENCY, SCORER_CONTEXT_LENGTH = 4, 10, 11
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1

# unicode.IsSpace
_SPACES = {0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000} | \
    set(range(0x2000, 0x200B))


def wrap64(x: int) -> int:
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def trim_space(s: str) -> str:
    """strings.TrimSpace on a (valid UTF-8) string."""
    b, e = 0, len(s)
    while b < e and ord(s[b]) in _SPACES:
        b += 1
    while e > b and ord(s[e - 1]) in _SPACES:
        e -= 1
    return s[b:e]


def atoi(s: str) -> int:
    """strconv.Atoi on a 64-bit platform; ValueError like its *NumError."""
    if s == "":
        raise ValueError("invalid syntax")
    i, neg = 0, False
    if s[0] in "+-":
        neg = s[0] == "-"
        i = 1
        if len(s) == 1:
            raise ValueError("invalid syntax")
    digits = s[i:]
    if not all("0" <= c <= "9" for c in digits):
        raise ValueError("invalid syntax")
    v = int(digits)
    v = -v if neg else v
    if not INT64_MIN <= v <= INT64_MAX:
        raise ValueError("value out of range")
    return v


# ---- context_length_aware.go -------------------------------------------------------------------------------------------
def parse_context_range(range_str: str):
    """parseContextRange -> (min, max); ValueError on every error the Go function returns."""
    if range_str == "":
        raise ValueError("empty range string")
    bounds = range_str.split("-")
    if len(bounds) != 2:
        raise ValueError(f"invalid range format: {range_str} (expected 'min-max')")
    lo = atoi(trim_space(bounds[0]))
    hi = atoi(trim_space(bounds[1]))
    if lo > hi:
        raise ValueError(f"min ({lo}) cannot be greater than max ({hi})")
    return lo, hi


def calculate_range_score(ctx: int, r) -> float:
    max_fallback = 0.3
    lo, hi = r
    if lo <= ctx <= hi:
        width = wrap64(hi - lo)
        if width == 0:
            return 1.0
        width_score = 1.0 / (1.0 + float(width) / 10000.0)
        headroom = float(wrap64(hi - ctx))
        position_score = headroom / float(width)
        raw = 0.7 * width_score + 0.3 * position_score
        return max_fallback + raw * 0.7                 # (1.0 - maxFallbackScore) folded to 0.7 by the Go compiler
    distance = wrap64(ctx - hi) if ctx > hi else wrap64(lo - ctx)
    return max_fallback / (1.0 + float(distance) / 1000.0)


def endpoint_state(labels: dict | None, key: str):
    """None: no label; "invalid": the label does not parse; else (min, max)."""
    if labels is None or key not in labels:
        return None
    try:
        return parse_context_range(labels[key])
    except ValueError:
        return "invalid"


def filter_keeps(state, ctx: int) -> bool:
    if state is None:
        return True
    if state == "invalid":
        return False
    return state[0] <= ctx <= state[1]


def score_of(state, ctx: int) -> float:
    if state is None:
        return 0.5
    if state == "invalid":
        return 0.0
    return calculate_range_score(ctx, state)


def context_length(token_ids=None, chat_messages=(), completions_prompt=None) -> int:
    """getContextLength / estimateContextLength: the token count, else int(float64(chars) * 0.25)."""
    if token_ids is not None and len(token_ids) > 0:
        return len(token_ids)
    chars = sum(len(m.encode()) if isinstance(m, str) else len(m) for m in chat_messages)
    if completions_prompt is not None:
        chars += len(completions_prompt.encode()) if isinstance(completions_prompt, str) else len(completions_prompt)
    return lm.go_int(float(chars) * CHAR_TO_TOKEN)


def default_ctx(prompt_len: int) -> int:
    """The engine's default context length of a request whose true prompt length is prompt_len bytes."""
    return lm.go_int(float(prompt_len) * CHAR_TO_TOKEN)


# ---- a profile decision ------------------------------------------------------------------------------------------------
def profile_decide(orc, filter_kind, scorers, picker, role, kv, waiting, running, match, total, ranges, ctx,
                   enable_filtering=False, info=None, lcfg=None, a2=None, seed=0, key=0, k=1, keep=None, lora=None):
    """One chain profile for one request -> dict(ties, picks, scores, final).  ranges: per slot endpoint_state values;
    scorers: oracle tuples with kind SCORER_CONTEXT_LENGTH / SCORER_LATENCY for the chain scorers; the rest as
    latency_model.profile_decide."""
    info = info or {}
    lcfg = dict(lm.DEFAULT_CFG, **(lcfg or {}))
    E = len(role)
    cands = [e for e in range(E) if role[e] != 0xFF and orc.lib().orc_role_filter_keeps(filter_kind, int(role[e]))
             and (keep is None or keep[e]) and (not enable_filtering or filter_keeps(ranges[e], ctx))]
    final = lm.chain(cands, match, total, info, lcfg, a2, seed, key)
    prefix = [(match[e] / total) if total > 0 else 0.0 for e in range(E)]
    col = np.zeros((2, E), dtype=np.float64)
    for e, v in lm.latency_score(lcfg, final, info, waiting, kv, prefix).items():
        col[0, e] = v
    for e in final:
        col[1, e] = score_of(ranges[e], ctx)
    r = np.full(E, 0xFF, dtype=np.uint8)
    for e in final:
        r[e] = role[e]
    pool = orc.PoolState(r, kv, waiting, running, col)
    if lora is not None:
        pool.set_lora(*lora)
    sc = [(SCORER_EXTERNAL, s[1], 0.0) if s[0] == SCORER_LATENCY else
          (SCORER_EXTERNAL, s[1], 1.0) if s[0] == SCORER_CONTEXT_LENGTH else s for s in scorers]
    prof = orc.make_profile(filter_kind, sc)
    picks, pscores, ties, allsc = orc.profile_run_topk(prof, pool, np.asarray(match, dtype=np.int32), total, k, seed, key)
    if picker and final:
        weights = [s[1] for s in scorers]
        score = {e: float(allsc[e]) for e in final}
        # candidates in ascending slot order, as tools/latency_model.py draws them
        drawn = pm.draw_k(picker, sorted(final), None, score, set(final), seed, key, weights, k, gaps=False)
        picks = [p for p, _ in drawn]
        pscores = [s for _, s in drawn]
        ties = len(final)
    return dict(ties=ties, picks=picks, scores=pscores, final=final)
