"""Python restatement of the two Admitter plugins (include/epp_engine.h "Admission"): the latency-slo-admitter
(requestcontrol/admitter/latencyslo/plugin.go:99-158) and the probabilistic-admitter
(requestcontrol/admitter/probabilisticadmitter/plugin.go:125-162), with Go's math.Pow, math.Max / math.Min and
strconv.ParseFloat restated rather than approximated.  `rejects` decides an engine call's rows; `apply` rewrites the
rejected rows of the decisions the same call made without admission inputs, which is what the engine returns."""
from __future__ import annotations

import math

import numpy as np

EPP_NO_ENDPOINT = 0xFFFFFFFF
STATUS_REJECTED = -2
ADMIT_DOMAIN = 0x1D8E4E27C47D124F
M64 = (1 << 64) - 1

DEFAULTS = dict(queue_depth_threshold=5, kv_cache_util_threshold=0.8, power=5.0, k=300.0)


# ---- Go's math ------------------------------------------------------------------------------------------------------
def go_max(x: float, y: float) -> float:
    if x == math.inf or y == math.inf:
        return math.inf
    if math.isnan(x) or math.isnan(y):
        return math.nan
    if x == 0 and x == y:
        return y if math.copysign(1.0, x) < 0 else x
    return x if x > y else y


def go_min(x: float, y: float) -> float:
    if x == -math.inf or y == -math.inf:
        return -math.inf
    if math.isnan(x) or math.isnan(y):
        return math.nan
    if x == 0 and x == y:
        return x if math.copysign(1.0, x) < 0 else y
    return x if x < y else y


def _is_odd_int(x: float) -> bool:
    if abs(x) >= 2.0 ** 53:
        return False
    xf, xi = math.modf(x)
    return xf == 0 and int(xi) & 1 == 1


def go_pow(x: float, y: float) -> float:
    """math.Pow (math/pow.go): special cases, x**yf = Exp(yf * Log(x)), x**yi by squaring Frexp's mantissa, Ldexp."""
    if y == 0 or x == 1:
        return 1.0
    if y == 1:
        return x
    if math.isnan(x) or math.isnan(y):
        return math.nan
    if x == 0:
        if y < 0:
            return -math.inf if math.copysign(1.0, x) < 0 and _is_odd_int(y) else math.inf
        if y > 0:
            return x if math.copysign(1.0, x) < 0 and _is_odd_int(y) else 0.0
    if math.isinf(y):
        if x == -1:
            return 1.0
        return 0.0 if (abs(x) < 1) == (y > 0) else math.inf
    if math.isinf(x):
        if x < 0:
            return go_pow(1 / x, -y)
        if y < 0:
            return 0.0
        if y > 0:
            return math.inf
    if y == 0.5:
        return math.sqrt(x)
    if y == -0.5:
        return 1 / math.sqrt(x)
    yf, yi = math.modf(abs(y))
    if yf != 0 and x < 0:
        return math.nan
    if yi >= 2.0 ** 63:
        if x == -1:
            return 1.0
        return 0.0 if (abs(x) < 1) == (y > 0) else math.inf
    a1, ae = 1.0, 0
    if yf != 0:
        if yf > 0.5:
            yf -= 1
            yi += 1
        a1 = math.exp(yf * math.log(x))
    x1, xe = math.frexp(x)
    i = int(yi)
    while i != 0:
        if xe < -(1 << 12) or (1 << 12) < xe:
            ae += xe
            break
        if i & 1:
            a1 *= x1
            ae += xe
        x1 *= x1
        xe <<= 1
        if x1 < 0.5:
            x1 += x1
            xe -= 1
        i >>= 1
    if y < 0:
        a1 = 1 / a1
        ae = -ae
    try:
        return math.ldexp(a1, ae)
    except OverflowError:
        return math.copysign(math.inf, a1)


# ---- strconv.ParseFloat, as parseFloatHeaderValue uses it (restated in plugins.py, which the Scheduler reads) -----
def parse_float(s: str):
    """strconv.ParseFloat(s, 64) -> (value, ok): ok is False for a syntax or range error."""
    from epp_b200 import plugins
    return plugins.ParseFloat(s)


def parse_float_header(s: str) -> float:
    """parseFloatHeaderValue (latencyslo/plugin.go:150-158): 0 when absent, unparsable or out of range."""
    from epp_b200 import plugins
    return plugins.parseFloatHeaderValue(s)


# ---- the plugins --------------------------------------------------------------------------------------------------
def mix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw(tie_seed: int, ordinal: int) -> float:
    """u of the probabilistic-admitter for the request of this ordinal: key = 4 * ordinal + 3."""
    key = (4 * ordinal + 3) & M64
    return (mix64((tie_seed ^ ADMIT_DOMAIN) ^ mix64(key)) >> 11) * 2.0 ** -53


class Endpoint:
    """What the admitters read of an endpoint: its metrics (None = nil) and its LatencyPredictionInfo validity bits (None =
    no attribute)."""

    def __init__(self, waiting=0, kv=0.0, running=0, valid=None, metrics=True):
        self.waiting, self.kv, self.running, self.valid, self.metrics = waiting, kv, running, valid, metrics


def latency_slo_rejects(priority: int, ttft_slo: float, tpot_slo: float, endpoints) -> bool:
    """LatencyAdmission.AdmitRequest: True = rejected."""
    if priority >= 0 or not (ttft_slo > 0 or tpot_slo > 0):
        return False
    has_valid = has_cold = has_idle = has_pred = False
    for e in endpoints:
        if e.kv < 0.02:
            has_cold = True
        if e.running == 0:
            has_idle = True
        if e.valid is not None:
            has_pred = True
            if e.valid & 3 == 3:
                has_valid = True
    return has_pred and not has_valid and not has_idle and not has_cold


def saturation(endpoints, cfg) -> float:
    total = 0.0
    for e in endpoints:
        if not e.metrics:
            total += 1.0
            continue
        total += go_max(float(e.waiting) / float(cfg["queue_depth_threshold"]), e.kv / cfg["kv_cache_util_threshold"])
    return total / float(len(endpoints))


def probabilistic_rejects(priority: int, endpoints, cfg, u: float) -> bool:
    """ProbabilisticAdmitter.AdmitRequest with randFn() = u: True = rejected."""
    if priority >= 0 or not endpoints:
        return False
    sat = saturation(endpoints, cfg)
    return u < go_min(go_pow(sat, cfg["power"]) * cfg["k"], 1.0)


def probabilistic_p(endpoints, cfg) -> float:
    return go_min(go_pow(saturation(endpoints, cfg), cfg["power"]) * cfg["k"], 1.0)


# ---- an engine call -------------------------------------------------------------------------------------------------
def rejects(cfg, pool, priority, ttft_slo, tpot_slo, predictions=None, pred_valid=None, subsets=None, tie_seed=0,
            ord_base=0):
    """Rejected rows of one engine call -> bool [R].  cfg: {"latency_slo", "probabilistic", + DEFAULTS' keys}.  pool:
    dict of slot-indexed arrays "present", "kv", "waiting", "running".  predictions[r]: None or its entries' slots;
    pred_valid[r]: their validity bytes.  subsets[r]: None (the whole pool) or its slots."""
    R = len(priority)
    present = np.asarray(pool["present"], dtype=bool)
    out = np.zeros(R, dtype=bool)
    for r in range(R):
        if priority[r] >= 0:
            continue
        slots = np.flatnonzero(present) if subsets is None or subsets[r] is None else \
            np.array(sorted({int(s) for s in subsets[r] if s < len(present) and present[s]}), dtype=np.int64)
        if slots.size == 0:
            continue                               # no candidate: status -1 stands
        valid = {}
        if predictions is not None and predictions[r] is not None:
            for s, v in zip(predictions[r], pred_valid[r]):
                valid[int(s)] = int(v)
        eps = [Endpoint(int(pool["waiting"][s]), float(pool["kv"][s]), int(pool["running"][s]), valid.get(int(s)))
               for s in slots]
        rej = False
        if cfg.get("probabilistic"):
            rej = probabilistic_rejects(int(priority[r]), eps, cfg, draw(tie_seed, ord_base + r))
        if not rej and cfg.get("latency_slo") and predictions is not None:
            rej = latency_slo_rejects(int(priority[r]), float(ttft_slo[r]), float(tpot_slo[r]), eps)
        out[r] = rej
    return out


def apply(dec, det, rejected, lists=None):
    """The rows of a call made without admission inputs, with the rejected rows rewritten as the engine rewrites them."""
    dec, det = dec.copy(), None if det is None else det.copy()
    idx = np.flatnonzero(rejected)
    dec["status"][idx] = STATUS_REJECTED
    dec["pick"][idx] = EPP_NO_ENDPOINT
    dec["score"][idx] = 0.0
    dec["prefill_pick"][idx] = EPP_NO_ENDPOINT
    dec["tie_count"][idx] = 0
    dec["match_blocks"][idx] = 0
    if det is not None:
        for f in det.dtype.names:
            det[f][idx] = 0
        det["encode_pick"][idx] = EPP_NO_ENDPOINT
    if lists is not None:
        lists = {k: v.copy() for k, v in lists.items()}
        for k in ("primary", "prefill", "encode"):
            lists[k][idx] = EPP_NO_ENDPOINT
        lists["primary_scores"][idx] = 0.0
    return (dec, det, lists) if lists is not None else (dec, det)
