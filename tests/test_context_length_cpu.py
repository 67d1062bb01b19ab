"""The context-length-aware plugin's model (tools/context_length_model.py) against the reference's own tests, re-encoded,
the exact float bits of calculateRangeScore, parse edge cases against a literal TrimSpace + Atoi restatement, and the
placement rules of plugins.py.  No GPU."""
from __future__ import annotations

import struct

import pytest

from tools import context_length_model as cm

DEF = cm.DEFAULT_LABEL


def bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# ---- context_length_aware_test.go ------------------------------------------------------------------------------------
@pytest.mark.parametrize("raw,ok", [(None, True), ('{"label": "custom", "enableFiltering": true}', True),
                                    ('{"label": ""}', False), ('{"label": "test"', False)])
def test_factory(raw, ok):
    import epp_b200
    if ok:
        assert epp_b200.plugins.ContextLengthAwareFactory("x", raw).kind == 11
    else:
        with pytest.raises(ValueError):
            epp_b200.plugins.ContextLengthAwareFactory("x", raw)


def test_filter():
    labels = {"short-range": {DEF: "0-100"}, "medium-range": {DEF: "100-500"}, "wide-range": {DEF: "0-2000"},
              "no-label": {}}
    ctx = cm.context_length()                              # empty body: 0
    kept = [n for n, lb in labels.items() if cm.filter_keeps(cm.endpoint_state(lb, DEF), ctx)]
    assert sorted(kept) == sorted(["short-range", "wide-range", "no-label"])


def test_score():
    s = {n: cm.score_of(cm.endpoint_state({DEF: v} if v else {}, DEF), 0)
         for n, v in (("tight", "0-20"), ("wide", "0-10000"), ("nomatch", "500-1000"), ("nolabel", None))}
    assert s["tight"] > s["wide"] > 0.3
    assert 0.0 < s["nomatch"] < 0.3 < s["wide"]
    assert s["nolabel"] == 0.5


@pytest.mark.parametrize("v,want", [("0-100", (0, 100)), ("", None), ("0-100-200", None), ("200-100", None),
                                    ("abc-100", None)])
def test_parse_context_range(v, want):
    if want is None:
        with pytest.raises(ValueError):
            cm.parse_context_range(v)
    else:
        assert cm.parse_context_range(v) == want


def test_range_score_fallback():
    small, large = cm.calculate_range_score(9000, (0, 2048)), cm.calculate_range_score(9000, (0, 8192))
    assert 0 < small < large < 0.3
    far, close = cm.calculate_range_score(50, (500, 2048)), cm.calculate_range_score(50, (100, 1024))
    assert 0 < far < close < 0.3
    assert cm.calculate_range_score(14999, (0, 15000)) > 0.3 > cm.calculate_range_score(14999, (15001, 20000))


def test_tokenized_and_fallback():
    ids = list(range(1, 43))
    ctx = cm.context_length(ids, completions_prompt="some prompt text")
    assert ctx == 42
    assert cm.filter_keeps((0, 52), ctx) and not cm.filter_keeps((142, 242), ctx)
    ctx = cm.context_length(None, completions_prompt="Hello, how are you?")
    assert ctx == 4
    assert cm.filter_keeps((0, 50), ctx) and not cm.filter_keeps((100, 200), ctx)
    assert cm.context_length([], chat_messages=["ab", "cdef"], completions_prompt="xy") == 2


# ---- parse edge cases against a literal TrimSpace + Atoi ---------------------------------------------------------------
def literal(v):
    if v == "":
        return None
    parts = v.split("-")
    if len(parts) != 2:
        return None
    out = []
    for p in parts:
        p = p.strip(" \t\n\v\f\r\x85\xa0")
        body = p[1:] if p[:1] in ("+", "-") else p
        if not body or not body.isascii() or not body.isdigit():
            return None
        n = int(p)
        if not -(1 << 63) <= n < (1 << 63):
            return None
        out.append(n)
    return tuple(out) if out[0] <= out[1] else None


@pytest.mark.parametrize("v", ["+0-+10", "007-9", " 0 - 2048 ", "0-9223372036854775807", "0-9223372036854775808",
                               "1-2-3", "", "10-5", "\t5- 6　", "5 - 6x", "+-5", "0x10-20", "1_0-20"])
def test_parse_edges(v):
    try:
        got = cm.parse_context_range(v)
    except ValueError:
        got = None
    assert got == literal(v) or ("　" in v and got == (5, 6))


# ---- exact float bits --------------------------------------------------------------------------------------------------
def test_score_bits():
    assert bits(cm.calculate_range_score(7, (7, 7))) == bits(1.0)
    w = 2048
    at_min = 0.3 + (0.7 * (1.0 / (1.0 + w / 10000.0)) + 0.3 * (w / w)) * 0.7
    at_max = 0.3 + (0.7 * (1.0 / (1.0 + w / 10000.0)) + 0.3 * (0 / w)) * 0.7
    assert bits(cm.calculate_range_score(100, (100, 2148))) == bits(at_min)
    assert bits(cm.calculate_range_score(2148, (100, 2148))) == bits(at_max)
    assert bits(cm.calculate_range_score(99, (100, 2148))) == bits(0.3 / (1.0 + 1 / 1000.0))
    assert bits(cm.calculate_range_score(2149, (100, 2148))) == bits(0.3 / (1.0 + 1 / 1000.0))
    for width in ((1 << 53) - 1, 1 << 53, (1 << 53) + 1, (1 << 62) + 3):
        s = cm.calculate_range_score(5, (0, width))
        assert bits(s) == bits(0.3 + (0.7 * (1.0 / (1.0 + float(width) / 10000.0)) + 0.3 * (float(width - 5) / float(width))) * 0.7)
        assert 0.3 < s <= 1.0


def test_default_ctx():
    for L in (0, 1, 3, 4, 5, 16384, (1 << 53) - 1):
        assert cm.default_ctx(L) == L // 4


# ---- placement in plugins.py -------------------------------------------------------------------------------------------
def test_placement():
    import epp_b200
    p = epp_b200.plugins
    cl = p.NewContextLengthAware("cl", enableFiltering=True)
    prof = p.NewSchedulerProfile()
    prof.AddPlugins(p.NewWeightedScorer(p.QueueScorer(), 1.0), p.NewWeightedScorer(cl, 2.0))
    assert prof.filters == [cl] and prof.spec().context_length == dict(label=DEF, enable_filtering=True)
    with pytest.raises(ValueError):                        # a scorer registered without a weight
        p.NewSchedulerProfile().AddPlugins(cl)
    with pytest.raises(AssertionError):                    # a filtering instance after the affinity filter
        p.NewSchedulerProfile().WithFilters(p.PrefixCacheAffinityFilter(), cl)
    with pytest.raises(AssertionError):                    # two instances in one profile
        p.NewSchedulerProfile().WithFilters(cl, p.NewContextLengthAware("b"))
    ok = p.NewSchedulerProfile().WithFilters(p.PrefixCacheAffinityFilter(), p.NewContextLengthAware("c"))
    spec = ok.spec()                                       # a pass-through filter anywhere; its score weighs 0
    assert spec.context_length["enable_filtering"] is False and spec.scorers[-1].kind == 11 and spec.scorers[-1].weight == 0
