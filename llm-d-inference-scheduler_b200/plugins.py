"""Host-side mirror of the reference's plugin/scheduler interface FOR THIS PATH ONLY (same names, argument meaning
and error behaviour), so that parity tests read like the reference's own Go tests.  It is configuration and
marshalling: every score, match count and pick comes out of the CUDA engine through the C ABI.

Reference interfaces mirrored (paths relative to the reference root):
  fwksched.Endpoint / fwkdl.Metrics / EndpointMetadata   pkg/epp/framework/interface/scheduling/types.go:71-117
  Scorer / Filter / Picker / ProfileHandler               pkg/epp/framework/interface/scheduling/plugins.go:43-78
  NewWeightedScorer                                       pkg/epp/scheduling/weighted_scorer.go:24-40
  SchedulerProfile (WithFilters/WithScorers/WithPicker)   pkg/epp/scheduling/scheduler_profile.go
  Scheduler.Schedule                                      pkg/epp/scheduling/scheduler.go:54-102
  MaxScorePicker (maxNumOfEndpoints)                      .../picker/maxscore/picker.go:58-115
  prefix-cache-affinity-filter                            .../filter/prefixcacheaffinity/plugin.go:45-151
  label-selector-filter / by-label-selector / by-label    .../filter/bylabel/selector.go:34-101, filter.go:34-117
  approximateprefix dataProducer Produce / PreRequest     .../approximateprefix/plugin.go:135-200
  LatencyPredictionInfo (LatencyPredictionInfoKey)        .../datalayer/attribute/latency/data_types.go:23-96
  slo-headroom-tier-filter                                .../filter/sloheadroomtier/plugin.go:43-73
  latency-scorer                                          .../scorer/latency/plugin.go:59-125
  context-length-aware (scorer and filter)                .../scorer/contextlengthaware/context_length_aware.go
"""
from __future__ import annotations

import json
import math
import re
from dataclasses import dataclass, field

import numpy as np

from . import _capi as capi
from .engine import AffinityFilterSpec, Engine, ProfileSpec, ScorerSpec

RoleLabel = "llm-d.ai/role"
_ROLE_BY_LABEL = {
    "decode": capi.ROLE_DECODE, "prefill": capi.ROLE_PREFILL, "prefill-decode": capi.ROLE_PREFILL_DECODE,
    "both": capi.ROLE_BOTH, "encode": capi.ROLE_ENCODE, "encode-prefill": capi.ROLE_ENCODE_PREFILL,
    "encode-prefill-decode": capi.ROLE_ENCODE_PREFILL_DECODE,
}
RoleDecode, RolePrefill, RolePrefillDecode, RoleBoth = "decode", "prefill", "prefill-decode", "both"
RoleEncode, RoleEncodePrefill, RoleEncodePrefillDecode = "encode", "encode-prefill", "encode-prefill-decode"


class SchedulingError(RuntimeError):
    """Schedule returned an error (scheduler_profile.go:119-121 / disagg_profile_handler.go:335-338)."""


@dataclass
class Metrics:                                   # fwkdl.Metrics, framework/interface/datalayer/metrics.go:26-42
    WaitingQueueSize: int = 0
    KVCacheUsagePercent: float = 0.0
    RunningRequestsSize: int = 0
    CacheBlockSize: int = 0
    CacheNumBlocks: int = 0


@dataclass
class EndpointMetadata:
    Name: str
    Labels: dict = field(default_factory=dict)
    Address: str = ""


class Endpoint:
    """fwksched.Endpoint: metadata + metrics + attribute map (PrefixCacheMatchInfo lives under Put/Get)."""

    def __init__(self, metadata: EndpointMetadata, metrics: Metrics | None = None):
        self.metadata = metadata
        self.metrics = metrics or Metrics()
        self.attrs: dict = {}

    def GetMetadata(self):
        return self.metadata

    def GetMetrics(self):
        return self.metrics

    def Put(self, key, value):
        self.attrs[key] = value

    def Get(self, key):
        return self.attrs.get(key), key in self.attrs

    def role_code(self) -> int:
        if RoleLabel not in self.metadata.Labels:
            return capi.ROLE_NONE
        return _ROLE_BY_LABEL.get(self.metadata.Labels[RoleLabel], capi.ROLE_OTHER)


def NewEndpoint(metadata: EndpointMetadata, metrics: Metrics | None = None, attrs=None) -> Endpoint:
    return Endpoint(metadata, metrics)


PrefixCacheMatchInfoKey = "PrefixCacheMatchInfoKey"          # attribute/prefix/data_types.go:24


@dataclass
class PrefixCacheMatchInfo:                      # attribute/prefix/data_types.go:27-54
    matchBlocks: int
    totalBlocks: int
    blockSizeTokens: int

    def MatchBlocks(self):
        return self.matchBlocks

    def TotalBlocks(self):
        return self.totalBlocks

    def BlockSizeTokens(self):
        return self.blockSizeTokens


def NewPrefixCacheMatchInfo(match, total, block_size_tokens):
    return PrefixCacheMatchInfo(match, total, block_size_tokens)


# ---- scorers (configuration objects; the arithmetic is in pick_kernels.cu) ----
@dataclass
class _Scorer:
    kind: int
    param: float = 0.0
    type_name: str = ""
    column: int = 0
    param2: float = 0.0


def PrefixCacheScorer():                         # scorer/prefix "prefix-cache-scorer"
    return _Scorer(capi.SCORER_PREFIX, 0.0, "prefix-cache-scorer")


def KVCacheUtilizationScorer():                  # "kv-cache-utilization-scorer"
    return _Scorer(capi.SCORER_KV_UTIL, 0.0, "kv-cache-utilization-scorer")


def QueueScorer():                               # "queue-scorer"
    return _Scorer(capi.SCORER_QUEUE, 0.0, "queue-scorer")


def RunningRequestsScorer():                     # "running-requests-size-scorer"
    return _Scorer(capi.SCORER_RUNNING, 0.0, "running-requests-size-scorer")


def NewLoadAware(queueThreshold: int = 128):     # loadaware.NewLoadAware, load_aware.go:43-52
    return _Scorer(capi.SCORER_LOAD_AWARE, float(queueThreshold), "load-aware-scorer")


def TokenLoadScorer(column: int = 0, queueThresholdTokens: int = 4194304):
    """ "token-load-scorer" (scorer/tokenload/token_load.go:84-112); `column` = ext column holding InFlightLoad.Tokens,
    not needed (ignored) when the Scheduler runs the InFlightLoadProducer."""
    return _Scorer(capi.SCORER_TOKEN_LOAD, float(queueThresholdTokens), "token-load-scorer", column)


def NewActiveRequest(column: int = 0, idleThreshold: int = 0, maxBusyScore: float = 1.0):
    """ "active-request-scorer" (scorer/activerequest/active_request.go:72-101, 140-173); `column` = ext column holding
    InFlightLoad.Requests, not needed (ignored) when the Scheduler runs the InFlightLoadProducer."""
    return _Scorer(capi.SCORER_ACTIVE_REQUEST, float(maxBusyScore), "active-request-scorer", column, float(idleThreshold))


def LoraAffinityScorer():
    """ "lora-affinity-scorer" (scorer/loraaffinity/lora_affinity.go:76-100); residency via Engine.pool_set_lora."""
    return _Scorer(capi.SCORER_LORA_AFFINITY, 0.0, "lora-affinity-scorer")


def NoHitLRU(lruSize: int = 1024):
    """ "no-hit-lru-scorer" (scorer/nohitlru/no_hit_lru.go:80-110, 259-321): cold requests (no candidate holds a block of
    the prompt) prefer the endpoints that least recently received a cold request; lruSize <= 0 means 1024.  The engine's
    own prefix match decides coldness, and every Schedule call updates the LRU with its cold requests' picks."""
    return _Scorer(capi.SCORER_NO_HIT_LRU, float(lruSize), "no-hit-lru-scorer")


def ExternalScorer(column: int):                 # host-computed column (e.g. lora-affinity)
    return _Scorer(capi.SCORER_EXTERNAL, float(column), "external")


@dataclass
class WeightedScorer:
    scorer: _Scorer
    weight: float


def NewWeightedScorer(scorer: _Scorer, weight: float) -> WeightedScorer:
    return WeightedScorer(scorer, float(weight))


@dataclass
class _RoleFilter:
    kind: int


def NewDecodeRole():
    return _RoleFilter(capi.FILTER_DECODE)


def NewPrefillRole():
    return _RoleFilter(capi.FILTER_PREFILL)


def NewEncodeRole():
    return _RoleFilter(capi.FILTER_ENCODE)


# ---- label filters (filter/bylabel/selector.go, filter.go; decided in the pool kernels, include/epp_engine.h) ----
LabelSelectorFilterType, ByLabelSelectorType, ByLabelType = "label-selector-filter", "by-label-selector", "by-label"
_NAME_RE = re.compile(r"^([A-Za-z0-9]([-A-Za-z0-9_.]*[A-Za-z0-9])?)?$")
_DNS1123_RE = re.compile(r"^[a-z0-9]([-a-z0-9]*[a-z0-9])?(\.[a-z0-9]([-a-z0-9]*[a-z0-9])?)*$")
_OPS = {"In": capi.LABEL_IN, "NotIn": capi.LABEL_NOT_IN, "Exists": capi.LABEL_EXISTS,
        "DoesNotExist": capi.LABEL_DOES_NOT_EXIST}


def _validate_key(k: str):
    """apimachinery validation.IsQualifiedName: [prefix/]name, prefix a DNS-1123 subdomain <= 253, name <= 63."""
    if not isinstance(k, str):
        raise ValueError(f"invalid label key {k!r}")
    parts = k.split("/")
    if len(parts) > 2:
        raise ValueError(f"invalid label key {k!r}: a qualified name must consist of alphanumeric characters, '-', '_' "
                         "or '.', with an optional DNS subdomain prefix and '/'")
    name = parts[-1]
    if len(parts) == 2 and (not parts[0] or len(parts[0]) > 253 or not _DNS1123_RE.match(parts[0])):
        raise ValueError(f"invalid label key {k!r}: prefix part must be a lowercase RFC 1123 subdomain")
    if not name or len(name) > 63 or not _NAME_RE.match(name):
        raise ValueError(f"invalid label key {k!r}: name part must be non-empty, at most 63 characters, alphanumeric, "
                         "'-', '_' or '.', and start and end with an alphanumeric character")


def _validate_value(v: str):
    """apimachinery validation.IsValidLabelValue: empty, or <= 63 characters of the name form."""
    if not isinstance(v, str) or len(v) > 63 or not _NAME_RE.match(v):
        raise ValueError(f"invalid label value: {v!r}: a valid label must be an empty string or consist of alphanumeric "
                         "characters, '-', '_' or '.', and must start and end with an alphanumeric character")


@dataclass
class _LabelFilter:
    """A label filter: its typed name and its requirements (key, capi.LABEL_* op, values), all ANDed."""
    type_name: str
    name: str
    reqs: list

    def TypedName(self):
        return (self.type_name, self.name)


def _requirement(key, op_name, values):
    """labels.NewRequirement: operator, value count, key and value syntax."""
    if op_name not in _OPS:
        raise ValueError(f"{op_name!r} is not a valid label selector operator")
    _validate_key(key)
    values = list(values or [])
    op = _OPS[op_name]
    if op in (capi.LABEL_IN, capi.LABEL_NOT_IN) and not values:
        raise ValueError("for 'in', 'notin' operators, values set can't be empty")
    if op in (capi.LABEL_EXISTS, capi.LABEL_DOES_NOT_EXIST) and values:
        raise ValueError("values set must be empty for exists and does not exist")
    for v in values:
        _validate_value(v)
    return (key, op, values)


def _selector_requirements(selector):
    """metav1.LabelSelectorAsSelector: None = Nothing, {} = Everything, else matchLabels (k In [v]) AND matchExpressions."""
    if selector is None:
        # labels.Nothing(): Exists and DoesNotExist on one key, which no endpoint meets together.  The key counts against
        # the engine's 16 interned keys; llm-d.ai/role is the one a P/D configuration is most likely to name anyway.
        return [(RoleLabel, capi.LABEL_EXISTS, []), (RoleLabel, capi.LABEL_DOES_NOT_EXIST, [])]
    if not isinstance(selector, dict):
        raise ValueError(f"not a label selector: {selector!r}")
    # fields other than matchLabels / matchExpressions are ignored, as json.Unmarshal ignores them
    reqs = [_requirement(k, "In", [v]) for k, v in (selector.get("matchLabels") or {}).items()]
    for ex in selector.get("matchExpressions") or []:
        reqs.append(_requirement(ex.get("key"), ex.get("operator"), ex.get("values")))
    return reqs


def NewSelector(name: str, selector):
    """bylabel.NewSelector (selector.go:62-77): selector is a metav1.LabelSelector as a dict."""
    if name == "":
        raise ValueError("Selector: missing filter name")
    return _LabelFilter(LabelSelectorFilterType, name, _selector_requirements(selector))


def SelectorFactory(name: str, rawParameters):
    """ "label-selector-filter" (selector.go:34-42): rawParameters is JSON text, bytes, a dict or None."""
    params = {}
    if rawParameters is not None:
        try:
            params = json.loads(rawParameters) if isinstance(rawParameters, (str, bytes)) else rawParameters
        except json.JSONDecodeError as e:
            raise ValueError(f"failed to parse the parameters of the '{LabelSelectorFilterType}' filter - {e}") from e
    if params is None:                    # JSON null leaves the empty LabelSelector: Everything, not Nothing
        params = {}
    return NewSelector(name, params)


LabelSelectorFilterFactory = SelectorFactory


def DeprecatedSelectorFactory(name: str, rawParameters):
    """ "by-label-selector" (selector.go:44-60): SelectorFactory reporting the legacy type."""
    f = SelectorFactory(name, rawParameters)
    f.type_name = ByLabelSelectorType
    return f


def NewByLabel(name: str, labelName: str, allowsNoLabel: bool, *validValues):
    """bylabel.NewByLabel (filter.go:64-77): keeps an endpoint whose label is absent and allowsNoLabel holds, or whose
    labels[labelName] is among validValues (an absent label reads as "")."""
    op = capi.LABEL_BY_LABEL_OR_ABSENT if allowsNoLabel else capi.LABEL_BY_LABEL
    if not validValues and not allowsNoLabel:
        return _LabelFilter(ByLabelType, name, _selector_requirements(None))      # keeps nothing, as in Go
    return _LabelFilter(ByLabelType, name, [(labelName, op, list(dict.fromkeys(validValues)))])


def ByLabelFactory(name: str, rawParameters):
    """ "by-label" (filter.go:34-57) with its errors."""
    params = {}
    if rawParameters is not None:
        try:
            params = json.loads(rawParameters) if isinstance(rawParameters, (str, bytes)) else dict(rawParameters)
        except json.JSONDecodeError as e:
            raise ValueError(f"failed to parse the parameters of the '{ByLabelType}' filter - {e}") from e
    label, values, allows = params.get("label", ""), params.get("validValues") or [], params.get("allowsNoLabel", False)
    if not isinstance(label, str) or not isinstance(allows, bool) or not isinstance(values, list) or \
            not all(isinstance(v, str) for v in values):
        raise ValueError(f"failed to parse the parameters of the '{ByLabelType}' filter")
    if name == "":
        raise ValueError(f"invalid configuration for '{ByLabelType}' filter: name cannot be empty")
    if label == "":
        raise ValueError(f"invalid configuration for '{ByLabelType}' filter: 'label' must be specified")
    if not values and not allows:
        raise ValueError(f"invalid configuration for '{ByLabelType}' filter: either 'validValues' must be non-empty or "
                         "'allowsNoLabel' must be true")
    return NewByLabel(name, label, allows, *values)


# ---- latency predictions (include/epp_engine.h "Latency predictions") ----
LatencyPredictionInfoKey = "LatencyPredictionInfoKey"        # attribute/latency/data_types.go:24


class LatencyPredictionInfo:                     # attribute/latency/data_types.go:36-80
    def __init__(self, ttftValid, tpotValid, ttftHeadroom, tpotHeadroom, ttft, tpot, dispatchedRequestCount):
        self._ttft_valid, self._tpot_valid = bool(ttftValid), bool(tpotValid)
        self._ttft_headroom, self._tpot_headroom = float(ttftHeadroom), float(tpotHeadroom)
        self._ttft, self._tpot = float(ttft), float(tpot)
        self._dispatched = int(dispatchedRequestCount)

    def TTFTValid(self): return self._ttft_valid
    def TPOTValid(self): return self._tpot_valid
    def IsValid(self): return self._ttft_valid and self._tpot_valid
    def TTFTHeadroom(self): return self._ttft_headroom
    def TPOTHeadroom(self): return self._tpot_headroom
    def TTFT(self): return self._ttft
    def TPOT(self): return self._tpot
    def DispatchedRequestCount(self): return self._dispatched

    def entry(self, slot: int):
        """The engine's prediction entry (slot, ttft, ttft_headroom, tpot_headroom, dispatched): the four values the
        plugins read."""
        return (slot, self._ttft, self._ttft_headroom, self._tpot_headroom, self._dispatched)


def NewLatencyPredictionInfo(ttftValid, tpotValid, ttftHeadroom, tpotHeadroom, ttft, tpot, dispatchedRequestCount):
    return LatencyPredictionInfo(ttftValid, tpotValid, ttftHeadroom, tpotHeadroom, ttft, tpot, dispatchedRequestCount)


def _unmarshal(raw, fields: dict, type_name: str) -> dict:
    """json.Unmarshal of rawParameters into a Config struct: keys match field names case-insensitively, unknown keys
    are ignored, null leaves the defaults, a value of the wrong JSON type is an error.  fields: json name -> float / str."""
    if raw is None:
        return {}
    if isinstance(raw, (str, bytes, bytearray)):
        if len(raw) == 0:
            return {}
        try:
            raw = json.loads(raw)
        except json.JSONDecodeError as e:
            raise ValueError(f"failed to unmarshal config: {e}") from e
    if raw is None:
        return {}
    if not isinstance(raw, dict):
        raise ValueError(f"failed to unmarshal config: json: cannot unmarshal {type(raw).__name__} into Go value of type "
                         f"{type_name}")
    out = {}
    lower = {k.lower(): k for k in fields}
    for k, v in raw.items():
        name = lower.get(k.lower())
        if name is None or v is None:
            continue
        want = fields[name]
        ok = isinstance(v, str) if want is str else (isinstance(v, (int, float)) and not isinstance(v, bool))
        if not ok:
            raise ValueError(f"failed to unmarshal config: json: cannot unmarshal {type(v).__name__} into Go struct field "
                             f"Config.{name} of type {'string' if want is str else 'float64'}")
        out[name] = want(v)
    return out


SLOHeadroomTierFilterType = "slo-headroom-tier-filter"


@dataclass
class SLOHeadroomTierFilter:                     # filter/sloheadroomtier; DefaultConfig :50-52
    epsilonExploreNeg: float = 0.01
    name: str = SLOHeadroomTierFilterType


def SLOHeadroomTierFilterFactory(name: str, rawParameters=None):
    """ "slo-headroom-tier-filter" (plugin.go:59-73): rawParameters is JSON text, bytes, a dict or None."""
    cfg = _unmarshal(rawParameters, {"epsilonExploreNeg": float}, "sloheadroomtier.Config")
    eps = cfg.get("epsilonExploreNeg", 0.01)
    if eps < 0 or eps > 1.0:
        raise ValueError(f"epsilonExploreNeg must be in [0, 1], got {eps:f}")
    return SLOHeadroomTierFilter(eps, name)


LatencyScorerType = "latency-scorer"


@dataclass
class LatencyScorerConfig:                       # scorer/latency Config; DefaultConfig :83-90
    ttftWeight: float = 0.8
    tpotWeight: float = 0.2
    headroomSelectionStrategy: str = "least"
    compositeKVWeight: float = 1.0
    compositeQueueWeight: float = 1.0
    compositePrefixWeight: float = 1.0


@dataclass
class _LatencyScorer(_Scorer):
    config: LatencyScorerConfig = field(default_factory=LatencyScorerConfig)


def NewLatencyScorer(config: LatencyScorerConfig | None = None, name: str = LatencyScorerType):    # NewPlugin, :107-112
    return _LatencyScorer(capi.SCORER_LATENCY, 0.0, name, config=config or LatencyScorerConfig())


def LatencyScorerFactory(name: str, rawParameters=None):
    """ "latency-scorer" (plugin.go:114-125).  A strategy other than "most" scores as "least" (the switch's default,
    :303-310)."""
    cfg = _unmarshal(rawParameters, {"ttftWeight": float, "tpotWeight": float, "headroomSelectionStrategy": str,
                                     "compositeKVWeight": float, "compositeQueueWeight": float,
                                     "compositePrefixWeight": float}, "latency.Config")
    return NewLatencyScorer(LatencyScorerConfig(**cfg), name)


def _latency_fields(tier, a1, scorer) -> dict:
    """Engine.latency_profile_set fields of a profile's tier filter, first affinity filter and latency scorer."""
    f = {}
    if tier is not None:
        f.update(tier_filter=1, epsilon_explore_neg=tier.epsilonExploreNeg)
    if a1 is not None:
        f.update(a1_affinity_threshold=a1.affinityThreshold, a1_exploration_probability=a1.explorationProbability,
                 a1_max_ttft_penalty_ms=a1.maxTTFTPenaltyMs)
    if scorer is not None:
        c = scorer.config
        f.update(ttft_weight=c.ttftWeight, tpot_weight=c.tpotWeight,
                 strategy=capi.HEADROOM_MOST if c.headroomSelectionStrategy == "most" else capi.HEADROOM_LEAST,
                 composite_kv_weight=c.compositeKVWeight, composite_queue_weight=c.compositeQueueWeight,
                 composite_prefix_weight=c.compositePrefixWeight)
    return f


ContextLengthAwareType = "context-length-aware"
DefaultContextLengthLabel = capi.CONTEXT_LENGTH_LABEL


@dataclass
class _ContextLengthAware(_Scorer):             # both a scorer and a filter (include/epp_engine.h "Context length")
    label: str = DefaultContextLengthLabel
    enableFiltering: bool = False


def NewContextLengthAware(name: str, label: str = DefaultContextLengthLabel, enableFiltering: bool = False):
    return _ContextLengthAware(capi.SCORER_CONTEXT_LENGTH, 0.0, name, label=label, enableFiltering=enableFiltering)


def ContextLengthAwareFactory(name: str, rawParameters=None):
    """ "context-length-aware" Factory: rawParameters is JSON text, bytes, a dict or None; json.Unmarshal into
    {label string, enableFiltering bool} over the defaults, then an empty label is an error."""
    raw = rawParameters
    try:
        if isinstance(raw, (str, bytes, bytearray)):
            raw = json.loads(raw)
        fields = {"label": str, "enablefiltering": bool}
        params = {"label": DefaultContextLengthLabel, "enablefiltering": False}
        if raw is not None:
            if not isinstance(raw, dict):
                raise ValueError(f"json: cannot unmarshal {type(raw).__name__} into Go value of type "
                                 f"contextlengthaware.contextLengthAwareParameters")
            for k, v in raw.items():
                want = fields.get(k.lower())
                if want is None or v is None:
                    continue
                if not isinstance(v, want):
                    raise ValueError(f"json: cannot unmarshal {type(v).__name__} into Go struct field "
                                     f"contextLengthAwareParameters.{k} of type {'string' if want is str else 'bool'}")
                params[k.lower()] = v
    except (ValueError, json.JSONDecodeError) as e:
        raise ValueError(f"failed to parse the parameters of the '{ContextLengthAwareType}' plugin - {e}") from e
    if params["label"] == "":
        raise ValueError(f"invalid configuration for '{ContextLengthAwareType}' plugin: 'label' must be specified")
    return NewContextLengthAware(name, params["label"], params["enablefiltering"])


# ---- strconv.ParseFloat, as parseFloatHeaderValue (latencyslo/plugin.go:150-158) uses it --------------------------------------------------------------
def _underscore_ok(s: str) -> bool:
    saw, i = "^", 0
    if s[:1] in ("+", "-"):
        s = s[1:]
    hexa = False
    if len(s) >= 2 and s[0] == "0" and s[1].lower() in "box":
        i, saw, hexa = 2, "0", s[1].lower() == "x"
    while i < len(s):
        c = s[i]
        if "0" <= c <= "9" or (hexa and "a" <= c.lower() <= "f"):
            saw = "0"
        elif c == "_":
            if saw != "0":
                return False
            saw = "_"
        else:
            if saw == "_":
                return False
            saw = "!"
        i += 1
    return saw != "_"


_DEC = re.compile(r"[+-]?([0-9_]*)(\.[0-9_]*)?([eE][+-]?[0-9_]+)?\Z")
_HEX = re.compile(r"[+-]?0[xX]([0-9a-fA-F_]*)(\.[0-9a-fA-F_]*)?[pP][+-]?[0-9_]+\Z")


def ParseFloat(s: str):
    """strconv.ParseFloat(s, 64) -> (value, ok): ok is False for a syntax or range error."""
    if not s:
        return 0.0, False
    m = re.fullmatch(r"([+-]?)(inf|infinity|nan)", s, flags=re.IGNORECASE)
    if m:
        if m.group(2).lower() == "nan":
            return (math.nan, True) if not m.group(1) else (0.0, False)
        return (-math.inf if m.group(1) == "-" else math.inf), True
    hexa = _HEX.match(s)
    dec = None if hexa else _DEC.match(s)
    mm = hexa or dec
    if not mm:
        return 0.0, False
    mant = (mm.group(1) or "") + (mm.group(2) or "").lstrip(".")
    if not any(c != "_" for c in mant):
        return 0.0, False                          # no mantissa digit
    if "_" in s and not _underscore_ok(s):
        return 0.0, False
    t = s.replace("_", "")
    try:
        v = float.fromhex(t) if hexa else float(t)
    except OverflowError:
        return 0.0, False
    if math.isinf(v):
        return v, False                            # ErrRange
    return v, True


def parseFloatHeaderValue(s: str) -> float:
    """parseFloatHeaderValue (latencyslo/plugin.go:150-158): 0 when absent, unparsable or out of range."""
    v, ok = ParseFloat(s or "")
    return v if ok else 0.0


LatencyAdmissionPluginType = "latency-slo-admitter"
ProbabilisticAdmitterType = "probabilistic-admitter"


class AdmissionError(SchedulingError):
    """A request an admitter rejected (status capi.EPP_STATUS_REJECTED): the director answers it with "request cannot be
    admitted" (requestcontrol/director.go:238-240) and never schedules it."""


@dataclass
class LatencyAdmission:                          # requestcontrol/admitter/latencyslo; LatencyAdmissionConfig has no fields
    name: str = LatencyAdmissionPluginType


def NewLatencyAdmission(name: str = LatencyAdmissionPluginType) -> LatencyAdmission:
    return LatencyAdmission(name)


def LatencyAdmissionFactory(name: str, rawParameters=None) -> LatencyAdmission:
    try:
        _unmarshal(rawParameters, {}, "latencyslo.LatencyAdmissionConfig")
    except ValueError as e:
        raise ValueError(f"failed to unmarshal config for LatencyAdmission: {e}") from e
    return NewLatencyAdmission(name)


@dataclass
class ProbabilisticAdmitter:                     # requestcontrol/admitter/probabilisticadmitter; defaults :37-42
    queueDepthThreshold: int = 5
    kvCacheUtilThreshold: float = 0.8
    power: float = 5.0
    k: float = 300.0
    name: str = ProbabilisticAdmitterType


def ProbabilisticAdmitterFactory(name: str, rawParameters=None) -> ProbabilisticAdmitter:
    """probabilisticadmitter.Factory: json.Unmarshal over the defaults, then the four range checks (plugin.go:71-84)."""
    t = ProbabilisticAdmitterType
    p = ProbabilisticAdmitter(name=name)
    try:
        got = _unmarshal(rawParameters, {"queueDepthThreshold": float, "kvCacheUtilThreshold": float, "power": float,
                                         "k": float}, "probabilisticadmitter.Parameters")
    except ValueError as e:
        raise ValueError(f"failed to parse parameters for '{t}' plugin: {e}") from e
    if "queueDepthThreshold" in got:
        q = got.pop("queueDepthThreshold")
        if q != int(q) or not -2 ** 63 <= q < 2 ** 63:
            raise ValueError(f"failed to parse parameters for '{t}' plugin: json: cannot unmarshal number {q} into Go "
                             f"struct field Parameters.queueDepthThreshold of type int")
        p.queueDepthThreshold = int(q)
    for k, v in got.items():
        setattr(p, k, v)
    if p.queueDepthThreshold <= 0:
        raise ValueError(f"plugin '{t}': queueDepthThreshold must be > 0, got {p.queueDepthThreshold}")
    if p.kvCacheUtilThreshold <= 0.0:
        raise ValueError(f"plugin '{t}': kvCacheUtilThreshold must be > 0, got {p.kvCacheUtilThreshold:g}")
    if p.power <= 0:
        raise ValueError(f"plugin '{t}': power must be > 0, got {p.power:g}")
    if p.k <= 0:
        raise ValueError(f"plugin '{t}': k must be > 0, got {p.k:g}")
    return p


Factory = ProbabilisticAdmitterFactory           # the reference's name for the probabilistic-admitter's factory


def admission_fields(admitters) -> dict:
    """Engine.admission_set keywords for a list of admitter instances."""
    out = dict(latency_slo=False, probabilistic=False)
    for a in admitters:
        if isinstance(a, LatencyAdmission):
            out["latency_slo"] = True
        elif isinstance(a, ProbabilisticAdmitter):
            if out["probabilistic"]:
                raise ValueError("the engine runs one probabilistic-admitter")
            out.update(probabilistic=True, queue_depth_threshold=a.queueDepthThreshold,
                       kv_cache_util_threshold=a.kvCacheUtilThreshold, power=a.power, k=a.k)
        else:
            raise TypeError(f"not an admitter: {a!r}")
    return out


def _context_length_of(plugin):
    """The context-length instance of a filter-list entry or WeightedScorer, or None."""
    inner = plugin.scorer if isinstance(plugin, WeightedScorer) else plugin
    return inner if isinstance(inner, _ContextLengthAware) else None


@dataclass
class PrefixCacheAffinityFilter:                 # filter/prefixcacheaffinity "prefix-cache-affinity-filter"; DefaultConfig :62-66
    affinityThreshold: float = 0.80
    explorationProbability: float = 0.01
    maxTTFTPenaltyMs: float = 5000.0
    ttft_column: int = -1                        # ext column carrying LatencyPredictionInfo.TTFT (-1: attribute absent)


@dataclass
class MaxScorePicker:                            # picker/maxscore; tie rule: include/epp_engine.h "Tie rule" / "Top-k"
    maxNumOfEndpoints: int = 1


def NewMaxScorePicker(maxNumOfEndpoints: int = 1):
    if maxNumOfEndpoints <= 0:                   # picker.go:59-61: invalid value -> DefaultMaxNumOfEndpoints
        maxNumOfEndpoints = 1
    return MaxScorePicker(maxNumOfEndpoints)


@dataclass
class RandomPicker:                              # picker/random; draw: include/epp_engine.h "Random pickers"
    maxNumOfEndpoints: int = 1


def NewRandomPicker(maxNumOfEndpoints: int = 1):
    if maxNumOfEndpoints <= 0:                   # random/picker.go:65-67
        maxNumOfEndpoints = 1
    return RandomPicker(maxNumOfEndpoints)


@dataclass
class WeightedRandomPicker:                      # picker/weightedrandom; P(endpoint) = score+ / sum of scores+
    maxNumOfEndpoints: int = 1


def NewWeightedRandomPicker(maxNumOfEndpoints: int = 1):
    if maxNumOfEndpoints <= 0:                   # weightedrandom/picker.go:67-69
        maxNumOfEndpoints = 1
    return WeightedRandomPicker(maxNumOfEndpoints)


_PICKER_KIND = {MaxScorePicker: capi.PICKER_MAX_SCORE, RandomPicker: capi.PICKER_RANDOM,
                WeightedRandomPicker: capi.PICKER_WEIGHTED_RANDOM}


class SchedulerProfile:
    def __init__(self):
        self.filters: list = []
        self.scorers: list = []
        self.picker = MaxScorePicker()

    def WithFilters(self, *filters):
        filters = [_context_length_of(f) or f for f in filters]
        _check_chain(filters)
        self.filters = list(filters)
        return self

    def WithScorers(self, *scorers):
        self.scorers = list(scorers)
        return self

    def AddPlugins(self, *plugins):
        for p in plugins:
            if isinstance(p, _ContextLengthAware):
                raise ValueError(f"plugin '{p.type_name}' is a scorer: it must be registered with a weight")
            if isinstance(p, WeightedScorer) and isinstance(p.scorer, _ContextLengthAware):
                _check_chain(self.filters + [p.scorer])              # scheduler_profile.go:76-95: also a filter, here
                self.filters.append(p.scorer)
                self.scorers.append(p)
            elif isinstance(p, WeightedScorer):
                self.scorers.append(p)
            elif isinstance(p, (_RoleFilter, _LabelFilter, PrefixCacheAffinityFilter, SLOHeadroomTierFilter)):
                _check_chain(self.filters + [p])
                self.filters.append(p)
            elif isinstance(p, (MaxScorePicker, RandomPicker, WeightedRandomPicker)):
                self.picker = p
        return None

    def WithPicker(self, picker):
        assert type(picker) in _PICKER_KIND, "the pickers are MaxScorePicker, RandomPicker and WeightedRandomPicker"
        self.picker = picker
        return self

    def spec(self) -> ProfileSpec:
        """The engine profile: the affinity filter after the tier filter (or the only one) is the profile's own; one
        before the tier filter, the tier filter and a latency scorer go into ProfileSpec.latency."""
        roles = [f for f in self.filters if isinstance(f, _RoleFilter)]
        tier_at = [i for i, f in enumerate(self.filters) if isinstance(f, SLOHeadroomTierFilter)]
        affs = [(i, f) for i, f in enumerate(self.filters) if isinstance(f, PrefixCacheAffinityFilter)]
        a1 = next((f for i, f in affs if tier_at and i < tier_at[0]), None)
        a2 = [f for i, f in affs if not tier_at or i > tier_at[0]]
        lat_scorers = [ws.scorer for ws in self.scorers if isinstance(ws.scorer, _LatencyScorer)]
        assert len(lat_scorers) <= 1, "at most one latency-scorer per profile"
        tier = self.filters[tier_at[0]] if tier_at else None
        cls = {id(f): f for f in self.filters if isinstance(f, _ContextLengthAware)}
        cls.update({id(ws.scorer): ws.scorer for ws in self.scorers if isinstance(ws.scorer, _ContextLengthAware)})
        assert len(cls) <= 1, "at most one context-length-aware instance per profile"
        cl = next(iter(cls.values()), None)
        scorers = [ScorerSpec(ws.scorer.kind, ws.weight, ws.scorer.param, ws.scorer.column, ws.scorer.param2)
                   for ws in self.scorers]
        context_length = None
        if cl is not None:
            in_filters = any(f is cl for f in self.filters)
            context_length = dict(label=cl.label, enable_filtering=bool(cl.enableFiltering and in_filters))
            if not any(ws.scorer is cl for ws in self.scorers):
                scorers.append(ScorerSpec(capi.SCORER_CONTEXT_LENGTH, 0.0))    # a filter only: its score weighs 0
        latency = None
        if tier is not None or lat_scorers:
            latency = _latency_fields(tier, a1, lat_scorers[0] if lat_scorers else None)
            if a2:
                assert a2[0].ttft_column < 0, "a latency profile reads TTFT from the predictions, not from an ext column"
        if cl is not None and a2:
            assert a2[0].ttft_column < 0, "a context-length profile reads TTFT from the predictions, not from an ext column"
        return ProfileSpec(roles[0].kind if roles else capi.FILTER_NONE, scorers,
                           AffinityFilterSpec(a2[0].affinityThreshold, a2[0].explorationProbability,
                                              a2[0].maxTTFTPenaltyMs, a2[0].ttft_column) if a2 else None,
                           _PICKER_KIND[type(self.picker)],
                           [q for f in self.filters if isinstance(f, _LabelFilter) for q in f.reqs],
                           latency, context_length)


def _check_chain(filters):
    """A profile's filter chain: label filters (any number) and at most one role filter, in any order (pure per-endpoint
    predicates, so their order does not matter), then at most one prefix-cache-affinity-filter, last: it depends on
    the set it receives.  With a slo-headroom-tier-filter the chain is [role + labels] -> [affinity] -> tier ->
    [affinity] (include/epp_engine.h "Latency predictions")."""
    filters = list(filters)
    roles = [f for f in filters if isinstance(f, _RoleFilter)]
    aff = [i for i, f in enumerate(filters) if isinstance(f, PrefixCacheAffinityFilter)]
    tier = [i for i, f in enumerate(filters) if isinstance(f, SLOHeadroomTierFilter)]
    assert all(isinstance(f, (_RoleFilter, _LabelFilter, PrefixCacheAffinityFilter, SLOHeadroomTierFilter,
                              _ContextLengthAware)) for f in filters), \
        "a profile's filters are role filters, label filters, the prefix-cache-affinity-filter, the " \
        "slo-headroom-tier-filter and context-length-aware"
    cls = [i for i, f in enumerate(filters) if isinstance(f, _ContextLengthAware)]
    assert len({id(filters[i]) for i in cls}) <= 1, "at most one context-length-aware instance per profile"
    gates = [i for i, f in enumerate(filters) if isinstance(f, (PrefixCacheAffinityFilter, SLOHeadroomTierFilter))]
    assert not any(filters[i].enableFiltering and gates and i > gates[0] for i in cls), \
        "a filtering context-length-aware comes before the affinity and tier filters (it is a per-endpoint predicate)"
    filters = [f for f in filters if not isinstance(f, _ContextLengthAware)]   # the rest of the chain as without it
    assert len(roles) <= 1, "at most one role filter per profile"
    assert len(tier) <= 1, "at most one slo-headroom-tier-filter per profile"
    if tier:
        t = tier[0]
        before = [i for i in aff if i < t]
        after = [i for i in aff if i > t]
        assert len(before) <= 1 and (not before or before[0] == t - 1), \
            "an affinity filter before the slo-headroom-tier-filter comes right before it"
        assert all(isinstance(f, (_RoleFilter, _LabelFilter)) for f in filters[:t - len(before)]), \
            "role and label filters come before the affinity and tier filters"
        assert len(after) <= 1 and (not after or after[0] == len(filters) - 1) and \
            all(i in after for i in range(t + 1, len(filters))), \
            "only one prefix-cache-affinity-filter may follow the slo-headroom-tier-filter"
    else:
        assert len(aff) <= 1 and (not aff or aff[0] == len(filters) - 1), \
            "the prefix-cache-affinity-filter comes last: no filter may follow it"
    n = sum(len(f.reqs) for f in filters if isinstance(f, _LabelFilter))
    assert n <= capi.EPP_LABEL_MAX_REQS, f"{n} label requirements, at most {capi.EPP_LABEL_MAX_REQS} per profile"


def NewSchedulerProfile():
    return SchedulerProfile()


@dataclass
class PrefixBasedPDDecider:                      # disagg.NewPrefixBasedPDDecider(NonCachedTokens)
    NonCachedTokens: int


@dataclass
class AlwaysDisaggPDDecider:
    pass


@dataclass
class SingleProfileHandler:
    pass


@dataclass
class DisaggProfileHandler:                      # disagg.NewDisaggProfileHandler(decode, prefill, "", decider, nil)
    decodeProfile: str
    prefillProfile: str
    pdDecider: object = None


@dataclass
class ProfileRunResult:
    TargetEndpoints: list
    Score: float = 0.0
    TieCount: int = 1
    TargetSlots: list = field(default_factory=list)   # engine slot ids of TargetEndpoints


@dataclass
class SchedulingResult:
    ProfileResults: dict
    PrimaryProfileName: str


@dataclass
class RequestObjectives:
    Priority: int = 0


@dataclass
class InferenceRequest:
    RequestID: str = ""
    TargetModel: str = ""
    Prompt: bytes = b""                          # Body.Completions.Prompt.Raw as bytes
    CacheSalt: str = ""
    SchedulingResult: object = None              # set by the caller after Schedule (read by ResponseBody processors)
    TokenizedPrompt: list | None = None          # Body.TokenizedPrompt.TokenIDs, or None (no token producer)
    Objectives: "RequestObjectives" = None       # Objectives.Priority (< 0 = sheddable); None = priority 0
    Headers: dict = field(default_factory=dict)  # request headers (the admitters read x-slo-ttft-ms / x-slo-tpot-ms)


class Scheduler:
    """scheduling.NewSchedulerWithConfig(NewSchedulerConfig(profileHandler, profiles)) over the CUDA engine.

    Schedule() takes a LIST of requests (a batch against one frozen snapshot, SURVEY App. A.8) and the candidate
    endpoints; PrefixCacheMatchInfo already Put on the endpoints is honoured exactly like the reference's scheduler
    tests do (disagg/scheduler_test.go:264-268); otherwise pass match info via `produce`."""

    def __init__(self, profileHandler, profiles: dict, *, max_endpoints: int = 64, block_size_tokens: int = 16,
                 max_prefix_blocks: int = 256, ext_columns: int = 0, device: int = 0, tie_seed: int = 0,
                 inflight_load: bool = False, admitters=()):
        """inflight_load: the engine runs the inflight-load producer's counters (InFlightLoadProducer) and the token-load /
        active-request scorers read them.  admitters: LatencyAdmission / ProbabilisticAdmitter instances the engine runs
        before its picks take effect (include/epp_engine.h "Admission"); a rejected request raises AdmissionError."""
        self.handler = profileHandler
        self.profiles = profiles
        if isinstance(profileHandler, DisaggProfileHandler):
            primary = profiles[profileHandler.decodeProfile].spec()
            prefill = profiles[profileHandler.prefillProfile].spec() if profileHandler.prefillProfile in profiles else None
            self.primary_name = profileHandler.decodeProfile
            self.prefill_name = profileHandler.prefillProfile
            dec = profileHandler.pdDecider
            nct = dec.NonCachedTokens if isinstance(dec, PrefixBasedPDDecider) else 0
            always = isinstance(dec, AlwaysDisaggPDDecider)
            if prefill is not None and dec is None:
                prefill = None               # no decider => the prefill stage never runs (disagg_profile_handler.go:298)
        else:
            (self.primary_name, prof), = profiles.items()
            primary, prefill, nct, always = prof.spec(), None, 0, False
            self.prefill_name = None
        ks = {p.picker.maxNumOfEndpoints for p in profiles.values()}
        assert len(ks) == 1, "the engine has one maxNumOfEndpoints for all profiles"
        self.pick_k = ks.pop()
        self.engine = Engine(max_endpoints, primary, prefill, device=device, block_size_tokens=block_size_tokens,
                             max_prefix_blocks=max_prefix_blocks, non_cached_tokens=nct, always_disagg=always,
                             n_ext_cols=ext_columns, tie_seed=tie_seed, pick_k=self.pick_k, inflight_load=inflight_load)
        self.block_size_tokens = block_size_tokens
        self.has_context_length = any(p.spec().context_length is not None for p in profiles.values())
        self.has_labels = any(p.spec().labels for p in profiles.values()) or self.has_context_length
        self.has_latency = any(p.spec().latency is not None for p in profiles.values())
        self.admission = admission_fields(admitters) if admitters else None
        if self.admission:
            self.engine.admission_set(**self.admission)

    def _push_pool(self, endpoints, ext=None):
        n = len(endpoints)
        self.engine.pool_set(np.arange(n, dtype=np.uint32), [e.role_code() for e in endpoints],
                             [e.metrics.KVCacheUsagePercent for e in endpoints],
                             [e.metrics.WaitingQueueSize for e in endpoints],
                             [e.metrics.RunningRequestsSize for e in endpoints], ext)
        if self.has_labels:
            self.engine.pool_set_labels(np.arange(n, dtype=np.uint32), [e.metadata.Labels for e in endpoints])

    def Schedule(self, requests, candidateEndpoints, ext=None, predictions=None):
        """predictions: None (each endpoint's LatencyPredictionInfoKey attribute, the same for every request), or one
        entry per request, each a dict endpoint index -> LatencyPredictionInfo (the producer's per-request output)."""
        single = isinstance(requests, InferenceRequest)
        reqs = [requests] if single else list(requests)
        eps = list(candidateEndpoints)
        if not eps:
            raise SchedulingError("no endpoints available for the given request")
        self._push_pool(eps, ext)
        E = self.engine.E
        match = np.zeros((len(reqs), E), dtype=np.int32)
        total = np.zeros(len(reqs), dtype=np.int32)
        bst = self.block_size_tokens
        for i, ep in enumerate(eps):                     # injected PrefixCacheMatchInfo (same for every request)
            info, ok = ep.Get(PrefixCacheMatchInfoKey)
            if ok and info is not None:
                match[:, i] = info.MatchBlocks()
                total[:] = info.TotalBlocks()
                bst = info.BlockSizeTokens()
        in_len = np.array([len(r.Prompt) for r in reqs], dtype=np.int64)
        preds = None
        if predictions is not None:
            if single:
                predictions = [predictions]
            assert len(predictions) == len(reqs), "one predictions entry per request"
            infos = [None if p is None else sorted(p.items()) for p in predictions]
        elif self.has_latency or (self.admission and self.admission["latency_slo"]):
            attrs = [(i, ep.Get(LatencyPredictionInfoKey)) for i, ep in enumerate(eps)]
            infos = [[(i, info) for i, (info, ok) in attrs if ok and info is not None]] * len(reqs)
        else:
            infos = None
        preds = None if infos is None else [None if p is None else [info.entry(i) for i, info in p] for p in infos]
        if preds is not None and not self.has_latency and not (self.admission and self.admission["latency_slo"]):
            raise SchedulingError("latency predictions need a profile with a latency-scorer or slo-headroom-tier-filter")
        admission = None
        if self.admission:
            admission = dict(priority=[r.Objectives.Priority if r.Objectives else 0 for r in reqs],
                             ttft_slo=[parseFloatHeaderValue(r.Headers.get("x-slo-ttft-ms", "")) for r in reqs],
                             tpot_slo=[parseFloatHeaderValue(r.Headers.get("x-slo-tpot-ms", "")) for r in reqs])
            if infos is not None:
                admission["pred_valid"] = [None if p is None else [int(info.TTFTValid()) | int(info.TPOTValid()) << 1
                                                                   for _, info in p] for p in infos]
        # getContextLength: the token count, else the engine's default int(float64(len(prompt)) * 0.25) (-1)
        ctx = np.array([len(r.TokenizedPrompt) if r.TokenizedPrompt else -1 for r in reqs], dtype=np.int64) \
            if self.has_context_length else None
        if self.pick_k > 1:
            dec, det, lists = self.engine.schedule_with_match(match, total, in_len, bst, topk=True, predictions=preds,
                                                              context_tokens=ctx, admission=admission)
        else:
            dec, det = self.engine.schedule_with_match(match, total, in_len, bst, predictions=preds, context_tokens=ctx,
                                                       admission=admission)
            lists = {"primary": dec["pick"].reshape(-1, 1), "prefill": dec["prefill_pick"].reshape(-1, 1)}
        out = [self._result(dec[i], det[i], eps, lists["primary"][i], lists["prefill"][i]) for i in range(len(reqs))]
        return out[0] if single else out

    def _result(self, d, dd, eps, primary, prefill):
        if d["status"] == capi.EPP_STATUS_REJECTED:
            raise AdmissionError("request cannot be admitted")
        if d["status"] != 0:
            raise SchedulingError("failed to find available decode workers" if self.prefill_name
                                  else "no endpoints available for the given request")
        slots = lambda row: [int(s) for s in row if int(s) != capi.EPP_NO_ENDPOINT]            # picker order, k at most
        res = {self.primary_name: ProfileRunResult([eps[s] for s in slots(primary)], float(d["score"]), int(d["tie_count"]),
                                                   slots(primary))}
        if self.prefill_name and d["prefill_pick"] != capi.EPP_NO_ENDPOINT:
            res[self.prefill_name] = ProfileRunResult([eps[s] for s in slots(prefill)], float(dd["prefill_score"]),
                                                      int(dd["prefill_tie_count"]), slots(prefill))
        return SchedulingResult(res, self.primary_name)


class InFlightLoadProducer:
    """ "inflight-load-producer" (requestcontrol/dataproducer/inflightload/producer.go) on a Scheduler created with
    inflight_load=True.  PreRequest (:110-129) runs on the device inside every Schedule call; this object carries the
    other two hooks.  The token estimate reads the request's prompt length in bytes (include/epp_engine.h "In-flight
    load"), where the reference reads the HTTP body size."""

    def __init__(self, scheduler: Scheduler):
        self.engine = scheduler.engine
        self.prefill_name = scheduler.prefill_name

    def ResponseBody(self, request: InferenceRequest, start_of_stream: bool = False, end_of_stream: bool = False):
        """producer.go:131-168: the prefill target is released at the first chunk, every other target at the end."""
        result = request.SchedulingResult
        if result is None:
            return
        eps = []
        for name, pr in result.ProfileResults.items():
            if not pr.TargetSlots:
                continue
            if (start_of_stream and name == self.prefill_name) or (end_of_stream and name != self.prefill_name):
                eps.append(pr.TargetSlots[0])
        if eps:
            self.engine.inflight_release(eps, [len(request.Prompt)] * len(eps))

    def DeleteEndpoint(self, slot: int):
        """producer.go:189-192 (endpoint-delete event): the slot's counters become 0."""
        self.engine.inflight_reset([slot])

    def Get(self, slot: int):
        """InFlightLoad{Requests, Tokens} of a slot as the scorers see it now."""
        req, tok = self.engine.inflight_get()
        return int(req[slot]), int(tok[slot])


class ApproxPrefixCacheProducer:
    """approximateprefix dataProducer: Produce (plugin.go:135-160) + PreRequest (plugin.go:164-200) on the engine."""

    def __init__(self, engine: Engine, model: bytes):
        self.engine = engine
        self.model_id = engine.register_model(model)
        self._last = None

    def Produce(self, prompts: list, endpoints: list):
        data = np.frombuffer(b"".join(prompts), dtype=np.uint8) if prompts else np.zeros(0, np.uint8)
        offs = np.zeros(len(prompts) + 1, dtype=np.uint64)
        np.cumsum([len(p) for p in prompts], out=offs[1:])
        if data.size == 0:
            data = np.zeros(16, np.uint8)
        match, total = self.engine.prefix_match(data, offsets=offs,
                                                model_ids=np.full(len(prompts), self.model_id, np.uint32))
        hashes, nb = self.engine.hash_prompts(data, offsets=offs,
                                              model_ids=np.full(len(prompts), self.model_id, np.uint32))
        self._last = (hashes, nb)
        bst = self.engine.cfg.block_size_tokens
        if len(prompts) == 1:
            for i, ep in enumerate(endpoints):
                ep.Put(PrefixCacheMatchInfoKey, NewPrefixCacheMatchInfo(int(match[0, i]), int(total[0]), bst))
        return match, total

    def PreRequest(self, request_index: int, target_slots: list):
        hashes, nb = self._last
        for s in target_slots:
            self.engine.index_add(s, hashes[request_index, : nb[request_index]])
