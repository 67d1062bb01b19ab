"""Label filters without a GPU: the reference's own selector / by-label / role test cases re-encoded through the plugin
mirror (plugins.py) and the CPU model (tools/label_model.py), the rules apimachinery decides and the reference does not
pin, and the model's per-profile mask compilation against a literal restatement of Requirement.Matches."""
import json
import random

import numpy as np
import pytest

import epp_b200 as epp
from tools import label_model as lm

P = epp.plugins

# selector_test.go:149-184 / filter_test.go:154-194
PODS = {
    "nginx-1": {"app": "nginx", "version": "v1.0", "tier": "frontend"},
    "nginx-2": {"app": "nginx", "version": "v1.1", "tier": "frontend"},
    "coredns-1": {"app": "coredns", "tier": "system"},
    "redis-1": {"app": "redis", "tier": "backend", "deprecated": "true"},
    "web-1": {"app": "web", "tier": "frontend", "environment": "production"},
}
PODS_BYLABEL = dict(PODS, **{"no-tier-pod": {"app": "unknown"}})


def kept(f, pods):
    """Names the filter keeps, by the literal rule and by the compiled masks (which must agree)."""
    names = list(pods)
    lit = [n for n in names if lm.keeps(f.reqs, pods[n])]
    keys, codes, (comp,) = lm.compile_masks([f.reqs])
    keep = lm.keep_vector(comp, lm.label_codes(keys, codes, [pods[n] for n in names]))
    assert [n for n, k in zip(names, keep) if k] == lit
    return sorted(lit)


SELECTOR_CASES = [   # selector_test.go:186-289
    ({"matchLabels": {"app": "nginx"}}, ["nginx-1", "nginx-2"]),
    ({"matchLabels": {"app": "nginx", "version": "v1.0"}}, ["nginx-1"]),
    ({"matchExpressions": [{"key": "tier", "operator": "In", "values": ["frontend", "backend"]}]},
     ["nginx-1", "nginx-2", "redis-1", "web-1"]),
    ({"matchExpressions": [{"key": "tier", "operator": "NotIn", "values": ["system"]}]},
     ["nginx-1", "nginx-2", "redis-1", "web-1"]),
    ({"matchExpressions": [{"key": "deprecated", "operator": "Exists"}]}, ["redis-1"]),
    ({"matchExpressions": [{"key": "deprecated", "operator": "DoesNotExist"}]}, ["nginx-1", "nginx-2", "coredns-1", "web-1"]),
    ({"matchLabels": {"tier": "frontend"}, "matchExpressions": [{"key": "environment", "operator": "Exists"}]}, ["web-1"]),
    ({}, ["nginx-1", "nginx-2", "coredns-1", "redis-1", "web-1"]),
    ({"matchLabels": {"app": "nonexistent"}}, []),
]


@pytest.mark.parametrize("sel,expected", SELECTOR_CASES, ids=range(len(SELECTOR_CASES)))
def test_selector_filtering(sel, expected):
    f = P.SelectorFactory("test-selector", json.dumps(sel))
    assert f.TypedName() == (P.LabelSelectorFilterType, "test-selector")
    assert kept(f, PODS) == sorted(expected)


def test_selector_factory_accepts_and_rejects():
    ok = [  # selector_test.go:19-91
        '{"matchLabels": {"app": "nginx", "version": "v1.0"}}',
        '{"matchLabels": {"tier": "frontend"}, "matchExpressions": [{"key": "environment", "operator": "In", '
        '"values": ["production", "staging"]}, {"key": "deprecated", "operator": "DoesNotExist"}]}',
        "{}",
        '{"matchExpressions": [{"key": "component", "operator": "NotIn", "values": ["test", "debug"]}]}',
        '{"matchExpressions": [{"key": "release", "operator": "Exists"}]}',
    ]
    for raw in ok:
        assert P.SelectorFactory("s", raw) is not None
    for raw in ['{"matchLabels": {"app": "nginx"}',     # selector_test.go:110-146
                '{"matchExpressions": [{"key": "app", "operator": "InvalidOperator", "values": ["nginx"]}]}']:
        with pytest.raises(ValueError):
            P.SelectorFactory("s", raw)
    with pytest.raises(ValueError, match="missing filter name"):   # selector.go:65-67
        P.NewSelector("", {})
    d = P.DeprecatedSelectorFactory("compat-test", '{"matchLabels": {"app": "nginx"}}')
    assert d.TypedName() == (P.ByLabelSelectorType, "compat-test")
    assert kept(d, {"nginx-1": {"app": "nginx"}, "redis-1": {"app": "redis"}}) == ["nginx-1"]


def test_selector_edge_cases():
    """selector_test.go:318-349: nil and empty label maps never match a matchLabels selector; empty input, empty output."""
    f = P.SelectorFactory("test-selector", '{"matchLabels": {"app": "test"}}')
    assert kept(f, {}) == []
    assert kept(f, {"pod-1": None}) == [] and kept(f, {"pod-1": {}}) == []


def test_lws_example():
    """selector_test.go:351-394: the LWS leader (worker-index 0) is accepted by decode-role only."""
    pod = {"vllm": {"app.kubernetes.io/component": "vllm-worker", "app.kubernetes.io/name": "some-model",
                    "leaderworkerset.sigs.k8s.io/worker-index": "0"}}
    k = "leaderworkerset.sigs.k8s.io/worker-index"
    filters = [P.SelectorFactory("decode-role", json.dumps({"matchLabels": {k: "0"}})),
               P.SelectorFactory("ignore-decode-workers", json.dumps(
                   {"matchExpressions": [{"key": k, "operator": "NotIn", "values": ["0"]}]})),
               P.SelectorFactory("prefill-role", json.dumps({"matchExpressions": [{"key": k, "operator": "DoesNotExist"}]}))]
    accepted = [f.name for f in filters if kept(f, pod)]
    assert accepted == ["decode-role"]


BYLABEL_FACTORY = [  # filter_test.go:17-91
    ({"label": P.RoleLabel, "allowsNoLabel": False, "validValues": [P.RolePrefill]}, True),
    ({"label": P.RoleLabel, "allowsNoLabel": True, "validValues": []}, True),
    ({"label": P.RoleLabel, "allowsNoLabel": True, "validValues": [P.RoleDecode, P.RoleBoth]}, True),
    ({"label": "", "allowsNoLabel": False, "validValues": [P.RolePrefill]}, False),
    ({"allowsNoLabel": False, "validValues": [P.RolePrefill]}, False),
    ({"label": P.RoleLabel, "allowsNoLabel": False, "validValues": []}, False),
    ({"label": P.RoleLabel, "allowsNoLabel": False}, False),
]


@pytest.mark.parametrize("params,ok", BYLABEL_FACTORY, ids=range(len(BYLABEL_FACTORY)))
def test_bylabel_factory(params, ok):
    if ok:
        assert P.ByLabelFactory("f", json.dumps(params)).TypedName() == (P.ByLabelType, "f")
    else:
        with pytest.raises(ValueError, match="invalid configuration"):
            P.ByLabelFactory("f", json.dumps(params))


def test_bylabel_factory_invalid_json():
    for raw in ['{"label": "app", "validValues": ["a"', '{"label": "app", "validValues": "true"}',   # filter_test.go:110-138
                '{"label": "app", "allowsNoLabel": "yes", "validValues": ["true"]}']:
        with pytest.raises(ValueError):
            P.ByLabelFactory("test", raw)
    with pytest.raises(ValueError, match="name cannot be empty"):
        P.ByLabelFactory("", '{"label": "app", "validValues": ["a"]}')


BYLABEL_FILTERING = [  # filter_test.go:196-230
    ("app", ["nginx"], False, ["nginx-1", "nginx-2"]),
    ("version", ["v1.0"], False, ["nginx-1"]),
    ("tier", [], True, ["no-tier-pod"]),
    ("tier", ["frontend", "backend", "system"], False, ["nginx-1", "nginx-2", "coredns-1", "redis-1", "web-1"]),
]


@pytest.mark.parametrize("label,values,allows,expected", BYLABEL_FILTERING, ids=range(len(BYLABEL_FILTERING)))
def test_bylabel_filtering(label, values, allows, expected):
    f = P.ByLabelFactory("test-label", json.dumps({"label": label, "validValues": values, "allowsNoLabel": allows}))
    assert kept(f, PODS_BYLABEL) == sorted(expected)


ROLE_TABLES = {   # roles.go:46-70
    "decode": (True, [P.RoleDecode, P.RolePrefillDecode, P.RoleBoth, P.RoleEncodePrefillDecode]),
    "prefill": (False, [P.RolePrefill, P.RoleEncodePrefill, P.RolePrefillDecode, P.RoleBoth, P.RoleEncodePrefillDecode]),
    "encode": (False, [P.RoleEncode, P.RoleEncodePrefill, P.RoleEncodePrefillDecode]),
}
ROLE_VALUES = [None, "", "decode", "prefill", "prefill-decode", "both", "encode", "encode-prefill",
               "encode-prefill-decode", "garbage"]


@pytest.mark.parametrize("role", sorted(ROLE_TABLES))
def test_role_filters_in_bylabel_form(role):
    """roles_test.go: the role filters are by-label instances on llm-d.ai/role; the engine's role codes agree."""
    allows, values = ROLE_TABLES[role]
    f = P.NewByLabel(role + "-filter", P.RoleLabel, allows, *values)
    kind = {"decode": epp.capi.FILTER_DECODE, "prefill": epp.capi.FILTER_PREFILL, "encode": epp.capi.FILTER_ENCODE}[role]
    table = {  # score.cuh filter_keeps, restated
        epp.capi.FILTER_DECODE: {epp.capi.ROLE_NONE, epp.capi.ROLE_DECODE, epp.capi.ROLE_PREFILL_DECODE, epp.capi.ROLE_BOTH,
                                 epp.capi.ROLE_ENCODE_PREFILL_DECODE},
        epp.capi.FILTER_PREFILL: {epp.capi.ROLE_PREFILL, epp.capi.ROLE_ENCODE_PREFILL, epp.capi.ROLE_PREFILL_DECODE,
                                  epp.capi.ROLE_BOTH, epp.capi.ROLE_ENCODE_PREFILL_DECODE},
        epp.capi.FILTER_ENCODE: {epp.capi.ROLE_ENCODE, epp.capi.ROLE_ENCODE_PREFILL, epp.capi.ROLE_ENCODE_PREFILL_DECODE},
    }[kind]
    for v in ROLE_VALUES:
        labels = {} if v is None else {P.RoleLabel: v}
        ep = P.NewEndpoint(P.EndpointMetadata("x", labels))
        assert lm.keeps(f.reqs, labels) == (ep.role_code() in table), v
    if role != "decode":                      # label required: the same set as a selector In
        s = P.NewSelector(role, {"matchExpressions": [{"key": P.RoleLabel, "operator": "In", "values": values}]})
        for v in ROLE_VALUES:
            labels = {} if v is None else {P.RoleLabel: v}
            assert lm.keeps(s.reqs, labels) == lm.keeps(f.reqs, labels), v


def test_unpinned_rules_and_empty_values():
    """The apimachinery rules the reference does not pin, and a label value "" present versus absent."""
    k = "tier"
    notin = P.NewSelector("n", {"matchExpressions": [{"key": k, "operator": "NotIn", "values": ["a"]}]})
    inn = P.NewSelector("i", {"matchExpressions": [{"key": k, "operator": "In", "values": ["", "a"]}]})
    assert lm.keeps(notin.reqs, {}) and not lm.keeps(notin.reqs, {k: "a"}) and lm.keeps(notin.reqs, {k: ""})
    assert not lm.keeps(inn.reqs, {}) and lm.keeps(inn.reqs, {k: ""}) and lm.keeps(inn.reqs, {k: "a"})
    # by-label: an absent key reads "", so "" admits unlabelled endpoints even with allowsNoLabel = false
    bl = P.NewByLabel("b", k, False, "", "a")
    assert lm.keeps(bl.reqs, {}) and lm.keeps(bl.reqs, {k: ""}) and not lm.keeps(bl.reqs, {k: "b"})
    bl2 = P.NewByLabel("b", k, False, "a")
    assert not lm.keeps(bl2.reqs, {}) and not lm.keeps(bl2.reqs, {k: ""})
    bl3 = P.NewByLabel("b", k, True, "a")
    assert lm.keeps(bl3.reqs, {}) and not lm.keeps(bl3.reqs, {k: ""}) and lm.keeps(bl3.reqs, {k: "a"})
    ex = P.NewSelector("e", {"matchExpressions": [{"key": k, "operator": "Exists"}]})
    assert lm.keeps(ex.reqs, {k: ""}) and not lm.keeps(ex.reqs, {})
    assert kept(P.NewSelector("nothing", None), PODS) == []


def test_selector_syntax_validation():
    bad = [{"matchLabels": {"bad key": "v"}}, {"matchLabels": {"-k": "v"}}, {"matchLabels": {"k": "bad value"}},
           {"matchLabels": {"k": "-v"}}, {"matchLabels": {"k": "v" * 64}}, {"matchLabels": {"Up.Case/k": "v"}},
           {"matchLabels": {"a/b/c": "v"}}, {"matchLabels": {"/k": "v"}}, {"matchLabels": {"": "v"}},
           {"matchExpressions": [{"key": "k", "operator": "In", "values": []}]},
           {"matchExpressions": [{"key": "k", "operator": "NotIn"}]},
           {"matchExpressions": [{"key": "k", "operator": "Exists", "values": ["x"]}]},
           {"matchExpressions": [{"key": "k", "operator": "DoesNotExist", "values": ["x"]}]},
           {"matchExpressions": [{"key": "k", "operator": "in", "values": ["x"]}]}]
    for sel in bad:
        with pytest.raises(ValueError):
            P.NewSelector("s", sel)
    good = [{"matchLabels": {"leaderworkerset.sigs.k8s.io/worker-index": "0"}}, {"matchLabels": {"k": ""}},
            {"matchLabels": {"a.b-c_d": "x.Y-z_9"}}, {"matchLabels": {"k" * 63: "v" * 63}}]
    for sel in good:
        P.NewSelector("s", sel)


def test_filter_chain_rules():
    sel = P.NewSelector("s", {"matchLabels": {"a": "b"}})
    aff = P.PrefixCacheAffinityFilter()
    P.NewSchedulerProfile().WithFilters(sel, P.NewDecodeRole(), P.NewByLabel("b", "x", True), aff)
    P.NewSchedulerProfile().WithFilters(P.NewPrefillRole(), sel, sel)
    for chain in [(sel, aff, sel), (P.NewDecodeRole(), P.NewPrefillRole()), (aff, P.NewDecodeRole()), (aff, aff)]:
        with pytest.raises(AssertionError):
            P.NewSchedulerProfile().WithFilters(*chain)
    p = P.NewSchedulerProfile()
    p.AddPlugins(sel, aff)
    with pytest.raises(AssertionError):
        p.AddPlugins(sel)
    spec = P.NewSchedulerProfile().WithFilters(sel, P.NewDecodeRole()).spec()
    assert spec.filter == epp.capi.FILTER_DECODE and spec.labels == [("a", epp.capi.LABEL_IN, ["b"])]


def literal_matches(op, values, present, value):
    """k8s.io/apimachinery labels.Requirement.Matches and filter.go's ByLabel.Filter, written out case by case."""
    if op == lm.IN:
        return present and value in set(values)
    if op == lm.NOT_IN:
        return (not present) or value not in set(values)
    if op == lm.EXISTS:
        return present
    if op == lm.DOES_NOT_EXIST:
        return not present
    val = value if present else ""
    if op == lm.BY_LABEL:
        return val in set(values)
    return (not present) or val in set(values)


def test_masks_against_literal_matches_randomized():
    rnd = random.Random(20261016)
    vals = ["", "a", "b", "c", "d", "0", "1"]
    keys = ["k0", "k1", "k2", "k3"]
    for trial in range(300):
        profiles = []
        for _ in range(3):
            reqs = []
            for _ in range(rnd.randint(0, 5)):
                op = rnd.randrange(6)
                n = 0 if op in (lm.EXISTS, lm.DOES_NOT_EXIST) else rnd.randint(1 if op != lm.BY_LABEL_OR_ABSENT else 0, 4)
                reqs.append((rnd.choice(keys), op, [rnd.choice(vals) for _ in range(n)]))
            profiles.append(reqs)
        slots = [{k: rnd.choice(vals + ["zz"]) for k in keys if rnd.random() < 0.6} for _ in range(40)]
        kk, codes, comp = lm.compile_masks(profiles)
        lc = lm.label_codes(kk, codes, slots)
        for p, reqs in enumerate(profiles):
            got = lm.keep_vector(comp[p], lc)
            want = [all(literal_matches(op, v, key in s, s.get(key, "")) for key, op, v in reqs) for s in slots]
            np.testing.assert_array_equal(got, np.array(want, dtype=bool), err_msg=f"trial {trial} profile {p}")


def test_compile_caps():
    with pytest.raises(ValueError):
        lm.compile_masks([[(f"k{i}", lm.EXISTS, []) for i in range(17)]])
    with pytest.raises(ValueError):
        lm.compile_masks([[("k", lm.IN, [str(i) for i in range(63)])]])
    lm.compile_masks([[(f"k{i}", lm.EXISTS, []) for i in range(16)], [("k0", lm.IN, [str(i) for i in range(62)])]])


def test_selector_factory_null_and_unknown_fields():
    """json.Unmarshal of null leaves the empty LabelSelector (Everything) and ignores fields it does not know."""
    assert kept(P.SelectorFactory("s", "null"), PODS) == sorted(PODS)
    f = P.SelectorFactory("s", '{"matchLabels": {"app": "nginx"}, "somethingElse": 1}')
    assert kept(f, PODS) == ["nginx-1", "nginx-2"]
    with pytest.raises(ValueError):
        P.SelectorFactory("s", "[]")
