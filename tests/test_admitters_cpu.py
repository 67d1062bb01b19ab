"""The admitters' model (tools/admission_model.py) against the reference's own tests, re-encoded
(latencyslo/plugin_test.go, probabilisticadmitter/plugin_test.go), the math.Pow restatement against exact powers, the
strconv.ParseFloat restatement, the plugin factories and the ctypes layout of the new structs.  No GPU."""
from __future__ import annotations

import ctypes as C
import math
import struct
from fractions import Fraction

import pytest

from tools import admission_model as am

CFG = dict(am.DEFAULTS)


def bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# ---- latencyslo/plugin_test.go TestAdmitRequest: all 7 table rows (+ the nil request, which admits) -------------------
INVALID, VALID = 0, 3
LAT_ROWS = [
    ("non-sheddable request - always admit", 1, "100", "30", [(0.5, 5, INVALID)], False),
    ("no SLO headers - admit", -1, "", "", [(0.5, 5, None)], False),
    ("sheddable, all invalid, all busy, no cold - reject", -1, "100", "30", [(0.5, 5, INVALID), (0.4, 3, INVALID)], True),
    ("sheddable, all invalid, but one pod idle - admit", -1, "100", "30", [(0.5, 5, INVALID), (0.4, 0, INVALID)], False),
    ("sheddable, all invalid, but cold pod exists - admit", -1, "100", "30", [(0.5, 5, INVALID), (0.01, 3, INVALID)], False),
    ("sheddable, one valid endpoint - admit", -1, "100", "30", [(0.5, 5, INVALID), (0.4, 3, VALID)], False),
    ("sheddable, no prediction data on endpoints - admit (fail-open)", -1, "100", "30", [(0.5, 5, None)], False),
]


@pytest.mark.parametrize("name,prio,ttft,tpot,eps,want", LAT_ROWS, ids=[r[0] for r in LAT_ROWS])
def test_latency_slo_table(name, prio, ttft, tpot, eps, want):
    endpoints = [am.Endpoint(kv=kv, running=run, valid=v) for kv, run, v in eps]
    got = am.latency_slo_rejects(prio, am.parse_float_header(ttft), am.parse_float_header(tpot), endpoints)
    assert got == want


def test_latency_slo_one_validity_bit_is_not_valid():
    eps = [am.Endpoint(kv=0.5, running=5, valid=1), am.Endpoint(kv=0.4, running=3, valid=2)]
    assert am.latency_slo_rejects(-1, 100.0, 0.0, eps)
    assert not am.latency_slo_rejects(-1, math.nan, 0.0, eps)        # NaN > 0 is false: no SLO


# ---- probabilisticadmitter/plugin_test.go ----------------------------------------------------------------------------
def test_factory_and_defaults():
    import epp_b200
    P = epp_b200.plugins
    p = P.Factory("test-admitter", '{"queueDepthThreshold":10,"kvCacheUtilThreshold":0.9,"power":3,"k":100}')
    assert (p.name, p.queueDepthThreshold, p.kvCacheUtilThreshold, p.power, p.k) == ("test-admitter", 10, 0.9, 3.0, 100.0)
    d = P.Factory("test", None)
    assert (d.queueDepthThreshold, d.kvCacheUtilThreshold, d.power, d.k) == (5, 0.8, 5.0, 300.0)
    assert P.LatencyAdmissionFactory("x", None).name == "x"
    with pytest.raises(ValueError):
        P.LatencyAdmissionFactory("x", "{invalid}")


@pytest.mark.parametrize("raw,msg", [
    ("{invalid}", "failed to parse parameters"),
    ('{"queueDepthThreshold":0}', "queueDepthThreshold must be > 0, got 0"),
    ('{"kvCacheUtilThreshold":0}', "kvCacheUtilThreshold must be > 0, got 0"),
    ('{"power":-1}', "power must be > 0, got -1"),
    ('{"power":0}', "power must be > 0, got 0"),
    ('{"k":-1}', "k must be > 0, got -1"),
    ('{"k":0}', "k must be > 0, got 0"),
    ('{"queueDepthThreshold":1.5}', "of type int"),
])
def test_factory_rejects(raw, msg):
    import epp_b200
    with pytest.raises(ValueError, match=msg):
        epp_b200.plugins.Factory("test", raw)


def ep(q, kv):
    return am.Endpoint(waiting=q, kv=kv, running=1)


def test_protected_tiers_always_admitted():
    for prio in (0, 100):
        assert not am.probabilistic_rejects(prio, [ep(100, 0)], CFG, 0.0)


def test_high_saturation_rejects_and_zero_admits():
    assert am.probabilistic_rejects(-1, [ep(100, 0)], CFG, 0.0)
    assert not am.probabilistic_rejects(-1, [ep(0, 0)], CFG, 0.0)


def test_nil_metrics_treated_as_saturated():                # model only: a pool slot always has metrics
    assert am.probabilistic_rejects(-1, [am.Endpoint(metrics=False)], CFG, 0.0)


def test_no_pods_admits():
    assert not am.probabilistic_rejects(-1, [], CFG, 0.0)


def test_saturation_averaging():
    eps = [ep(10, 0), ep(0, 0)]
    assert am.saturation(eps, CFG) == 1.0
    assert am.probabilistic_rejects(-1, eps, CFG, 0.0)


def test_quintic_property():
    sat = 0.272 / 0.8
    assert am.go_min(am.go_pow(sat, 5) * 300, 1.0) >= 0.99
    assert am.probabilistic_rejects(-1, [ep(0, 0.272)], CFG, 0.999)


def test_probabilistic_shedding():
    eps = [ep(0, 0.16)]
    assert not am.probabilistic_rejects(-1, eps, CFG, 0.9)
    assert am.probabilistic_rejects(-1, eps, CFG, 0.0)
    assert 0.09 < am.probabilistic_p(eps, CFG) < 0.1


# ---- math.Pow ----------------------------------------------------------------------------------------------------------
def _square_and_multiply(x: float, n: int) -> float:
    """Go's loop without the Frexp / Ldexp split: in the normal range scaling by powers of two is exact, so both round
    every product the same way."""
    a = 1.0
    while n:
        if n & 1:
            a *= x
        x *= x
        n >>= 1
    return a


def test_pow_integer_powers_bit_exact():
    import random
    rnd = random.Random(7)
    xs = [rnd.uniform(0, 4) for _ in range(300)] + [0.34, 0.2, 1.0, 2.0, 0.5, 3.0, 1e-3, 7.25]
    for x in xs:
        for n in (2, 3, 5, 7, 10, 16, 33):
            want = _square_and_multiply(x, n)
            if want == 0 or math.isinf(want) or abs(want) < 2.0 ** -1022:
                continue
            assert bits(am.go_pow(x, n)) == bits(want)
            # Go's product of rounded squares drifts from the exact power by at most about one ulp per multiplication
            assert abs(bits(want) - bits(float(Fraction(x) ** n))) <= 2 * n


def test_pow_matches_python_on_exact_products():
    for x in (0.5, 0.75, 1.5, 2.0, 3.0, 0.125, 1.25):
        for n in (2, 3, 5):
            assert bits(am.go_pow(x, n)) == bits(x ** n)


def test_pow_subnormal_results():
    # the mantissa products are exact here, so the one rounding is Ldexp's into the subnormal range (2^-1074 units)
    tiny = 2.0 ** -1074
    assert am.go_pow(2.0 ** -600, 2) == 0.0                          # 2^-1200
    assert am.go_pow(0.75 * 2.0 ** -537, 2) == tiny                  # 0.5625 units -> 1
    assert am.go_pow(1.25 * 2.0 ** -537, 2) == 2 * tiny              # 1.5625 units -> 2
    assert am.go_pow(1.5 * 2.0 ** -358, 3) == 3 * tiny               # 3.375 units -> 3
    assert am.go_pow(2.0 ** -358, 3) == tiny                         # exactly one unit
    assert am.go_pow(2.0 ** -215, 5) == 0.0                          # 2^-1075: a half unit, ties to even -> 0


def test_pow_special_cases():
    assert am.go_pow(0.0, 5) == 0.0 and am.go_pow(-0.0, 5) == 0.0 and math.copysign(1, am.go_pow(-0.0, 5)) < 0
    assert math.isnan(am.go_pow(math.nan, 5)) and math.isnan(am.go_pow(-2.0, 2.5))
    assert am.go_pow(math.inf, 5) == math.inf and am.go_pow(-math.inf, 5) == -math.inf
    assert am.go_pow(4.0, 0.5) == 2.0 and am.go_pow(1.0, math.nan) == 1.0
    assert am.go_pow(-2.0, 5) == -32.0 and am.go_pow(1e300, 5) == math.inf


# ---- strconv.ParseFloat ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,want", [
    ("100", 100.0), ("", 0.0), ("abc", 0.0), (" 1", 0.0), ("1 ", 0.0), ("1e400", 0.0), ("-1e400", 0.0),
    ("1e-400", 0.0), ("NaN", math.nan), ("nan", math.nan), ("+NaN", 0.0), ("Inf", math.inf), ("+inf", math.inf),
    ("-Infinity", -math.inf), ("infin", 0.0), ("0x1p-2", 0.25), ("0X1.8P1", 3.0), ("0x1", 0.0), ("0x1p", 0.0),
    ("1_000", 1000.0), ("1__0", 0.0), ("_1", 0.0), ("1_", 0.0), ("1_.5", 0.0), ("0x_1p0", 1.0), (".5", 0.5),
    ("5.", 5.0), (".", 0.0), ("1e", 0.0), ("+.5e1", 5.0), ("0x1p2000", 0.0),
])
def test_parse_float_header(s, want):
    got = am.parse_float_header(s)
    assert (math.isnan(got) and math.isnan(want)) or got == want


# ---- the draw and the C structs --------------------------------------------------------------------------------------
def test_draw_is_keyed_on_index_3():
    assert am.draw(0, 0) != am.draw(0, 1)
    assert 0.0 <= am.draw(12345, 77) < 1.0
    assert am.draw(5, 9) == (am.mix64((5 ^ am.ADMIT_DOMAIN) ^ am.mix64(4 * 9 + 3)) >> 11) * 2.0 ** -53


def test_struct_layouts():
    import epp_b200
    capi = epp_b200.capi
    assert C.sizeof(capi.AdmissionCfg) == 40
    assert [getattr(capi.AdmissionCfg, f).offset for f in ("latency_slo", "probabilistic", "queue_depth_threshold",
                                                             "kv_cache_util_threshold", "power", "k")] == [4, 8, 12, 16, 24, 32]
    assert C.sizeof(capi.Admission) == 40
    assert [getattr(capi.Admission, f).offset for f in ("priority", "ttft_slo", "tpot_slo", "pred_valid")] == [8, 16, 24, 32]
    assert capi.EPP_STATUS_REJECTED == -2
    for name in ("epp_admission_cfg_default", "epp_admission_set", "epp_schedule_admit", "epp_schedule_with_match_admit",
                 "epp_submit_admit"):
        assert name in capi.SIGNATURES
