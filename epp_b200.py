"""Import alias: the package directory `llm-d-inference-scheduler_b200/` is not a valid Python identifier.

    import epp_b200 as epp        # epp.Engine, epp.capi, epp.plugins, epp.build
"""
import importlib
import os
import sys

_ROOT = os.path.dirname(os.path.abspath(__file__))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

_pkg = importlib.import_module("llm-d-inference-scheduler_b200")
build = importlib.import_module("llm-d-inference-scheduler_b200.build")
plugins = importlib.import_module("llm-d-inference-scheduler_b200.plugins")
capi = _pkg.capi
Engine = _pkg.Engine
EngineError = _pkg.EngineError
ProfileSpec = _pkg.ProfileSpec
ScorerSpec = _pkg.ScorerSpec
AffinityFilterSpec = _pkg.AffinityFilterSpec
PinnedBuffer = _pkg.PinnedBuffer
DECISION_DTYPE = _pkg.DECISION_DTYPE
DETAIL_DTYPE = _pkg.DETAIL_DTYPE
SHARD_BEST_DTYPE = _pkg.SHARD_BEST_DTYPE
decisions_from_torch = _pkg.decisions_from_torch
pack_subsets = _pkg.pack_subsets
pack_predictions = _pkg.pack_predictions
PREDICTION_DTYPE = _pkg.PREDICTION_DTYPE
Batcher = _pkg.Batcher
