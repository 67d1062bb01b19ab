"""llm-d-inference-scheduler_b200 -- H100-native Endpoint-Picker scoring engine (hot path only).

csrc/        hand-written sm_90a CUDA kernels + the C ABI (include/epp_engine.h) -> libepp_engine.so
_capi.py     ctypes view of the C ABI
engine.py    Engine: marshals numpy / torch-CUDA buffers into the ABI
plugins.py   host-side mirror of the reference's Scorer/Filter/Scheduler/DataProducer interface for this path
build.py     nvcc build (in-tree, sm_90a)

The directory name is not a Python identifier; import it with importlib (see epp_b200.py at the repo root).
"""
from . import _capi as capi
from .engine import (DECISION_DTYPE, DETAIL_DTYPE, PREDICTION_DTYPE, SHARD_BEST_DTYPE, AffinityFilterSpec, Batcher, Engine, EngineError, PinnedBuffer, ProfileSpec,
                     ScorerSpec, decisions_from_torch, pack_predictions, pack_subsets)

__all__ = ["capi", "Engine", "Batcher", "EngineError", "ProfileSpec", "ScorerSpec", "AffinityFilterSpec", "PinnedBuffer", "DECISION_DTYPE", "DETAIL_DTYPE",
           "SHARD_BEST_DTYPE", "PREDICTION_DTYPE", "decisions_from_torch", "pack_predictions", "pack_subsets"]
