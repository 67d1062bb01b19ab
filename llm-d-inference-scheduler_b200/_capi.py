"""ctypes view of include/epp_engine.h (the C ABI of libepp_engine.so).  No torch, no numpy types in the ABI:
plain pointers and sizes.  Loading fails loudly when the library has not been built; creating an engine fails
loudly (EPP_ERR_NO_DEVICE) when there is no CUDA device -- there is no CPU fallback anywhere in this package."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libepp_engine.so")

EPP_MAX_SCORERS = 8
EPP_NO_ENDPOINT = 0xFFFFFFFF
EPP_BATCH_DEVICE_PTRS = 1
EPP_BATCH_ASYNC = 2
EPP_BATCH_LENGTHS_EXCEED_ROWS = 4

EPP_OK, EPP_ERR_INVALID, EPP_ERR_CUDA, EPP_ERR_NO_DEVICE, EPP_ERR_CAPACITY, EPP_ERR_STATE, EPP_ERR_NCCL = \
    0, -1, -2, -3, -4, -5, -6
(SCORER_PREFIX, SCORER_KV_UTIL, SCORER_QUEUE, SCORER_LOAD_AWARE, SCORER_EXTERNAL, SCORER_RUNNING, SCORER_TOKEN_LOAD,
 SCORER_ACTIVE_REQUEST, SCORER_LORA_AFFINITY, SCORER_NO_HIT_LRU, SCORER_LATENCY, SCORER_CONTEXT_LENGTH) = range(12)
(ROLE_NONE, ROLE_DECODE, ROLE_PREFILL, ROLE_PREFILL_DECODE, ROLE_BOTH, ROLE_ENCODE, ROLE_ENCODE_PREFILL,
 ROLE_ENCODE_PREFILL_DECODE, ROLE_OTHER) = range(9)
FILTER_NONE, FILTER_DECODE, FILTER_PREFILL, FILTER_ENCODE = range(4)
PICKER_MAX_SCORE, PICKER_RANDOM, PICKER_WEIGHTED_RANDOM = range(3)
HANDLER_SINGLE, HANDLER_DISAGG = 0, 1


class ScorerCfg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_int32), ("weight", C.c_double), ("param", C.c_double),
                ("param2", C.c_double)]


class ProfileCfg(C.Structure):
    _fields_ = [("filter", C.c_int32), ("n_scorers", C.c_int32), ("scorers", ScorerCfg * EPP_MAX_SCORERS),
                ("affinity_threshold", C.c_double), ("exploration_probability", C.c_double),
                ("max_ttft_penalty_ms", C.c_double), ("ttft_column", C.c_int32), ("picker", C.c_int32)]


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("device", C.c_int32), ("max_endpoints", C.c_int32),
                ("block_size_tokens", C.c_int32), ("max_prefix_blocks", C.c_int32),
                ("lru_capacity_per_server", C.c_int32), ("handler", C.c_int32), ("always_disagg", C.c_int32),
                ("non_cached_tokens", C.c_int64), ("n_ext_cols", C.c_int32), ("pick_k", C.c_int32),
                ("primary", ProfileCfg), ("prefill", ProfileCfg), ("encode", ProfileCfg), ("tie_seed", C.c_uint64),
                ("encode_enabled", C.c_int32), ("index_commit_interval_us", C.c_int32), ("inflight_load", C.c_int32),
                ("reserved0", C.c_uint32), ("reserved1", C.c_uint64)]


class Decision(C.Structure):
    _fields_ = [("status", C.c_int32), ("pick", C.c_uint32), ("score", C.c_double), ("prefill_pick", C.c_uint32),
                ("tie_count", C.c_uint32), ("total_blocks", C.c_int32), ("match_blocks", C.c_int32)]


class DecisionDetail(C.Structure):
    _fields_ = [("prefill_score", C.c_double), ("prefill_tie_count", C.c_uint32), ("prefill_ran", C.c_uint32),
                ("encode_score", C.c_double), ("encode_pick", C.c_uint32), ("encode_tie_count", C.c_uint32),
                ("encode_ran", C.c_uint32), ("reserved", C.c_uint32)]


class Batch(C.Structure):
    _fields_ = [("n_requests", C.c_int64), ("data", C.c_void_p), ("offsets", C.c_void_p),
                ("uniform_len", C.c_uint64), ("model_ids", C.c_void_p), ("flags", C.c_uint32),
                ("reserved", C.c_uint32), ("lengths", C.c_void_p), ("multimodal", C.c_void_p)]


class Stats(C.Structure):
    _fields_ = [("n_batches", C.c_uint64), ("n_decisions", C.c_uint64), ("index_pairs", C.c_uint64),
                ("index_hashes", C.c_uint64), ("index_slots", C.c_uint64), ("last_h2d_ms", C.c_double),
                ("last_kernels_ms", C.c_double), ("last_d2h_ms", C.c_double), ("last_hash_ms", C.c_double),
                ("last_match_pick_ms", C.c_double), ("last_kernel_launches", C.c_uint64),
                ("device_bytes", C.c_uint64), ("last_kernel_ms", C.c_double * 8), ("last_probes", C.c_uint64),
                ("last_postings", C.c_uint64), ("last_index_apply_ms", C.c_double), ("last_index_build_ms", C.c_double),
                ("last_index_items", C.c_uint64), ("last_index_launches", C.c_uint64), ("last_index_patched", C.c_uint64),
                ("last_hash_bytes_stored", C.c_uint64), ("last_prompt_bytes_read", C.c_uint64)]


class TopkOut(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("k", C.c_int32), ("primary", C.c_void_p), ("primary_scores", C.c_void_p),
                ("prefill", C.c_void_p), ("encode", C.c_void_p)]


EPP_SUBSET_ALL = 0xFFFFFFFF
EPP_SUBSET_MAX_SLOTS = 1024
EPP_PRED_MAX_SLOTS = 1024


class Subset(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("counts", C.c_void_p), ("offsets", C.c_void_p),
                ("slots", C.c_void_p)]


HEADROOM_LEAST, HEADROOM_MOST = 0, 1


class LatencyCfg(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("tier_filter", C.c_int32), ("epsilon_explore_neg", C.c_double),
                ("a1_affinity_threshold", C.c_double), ("a1_exploration_probability", C.c_double),
                ("a1_max_ttft_penalty_ms", C.c_double), ("ttft_weight", C.c_double), ("tpot_weight", C.c_double),
                ("strategy", C.c_int32), ("reserved", C.c_int32), ("composite_kv_weight", C.c_double),
                ("composite_queue_weight", C.c_double), ("composite_prefix_weight", C.c_double)]


class Prediction(C.Structure):
    _fields_ = [("slot", C.c_uint32), ("dispatched", C.c_int32), ("ttft", C.c_double), ("ttft_headroom", C.c_double),
                ("tpot_headroom", C.c_double)]


class Predictions(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("counts", C.c_void_p), ("offsets", C.c_void_p),
                ("entries", C.c_void_p)]


EPP_LABEL_MAX_REQS = 32
LABEL_IN, LABEL_NOT_IN, LABEL_EXISTS, LABEL_DOES_NOT_EXIST, LABEL_BY_LABEL, LABEL_BY_LABEL_OR_ABSENT = range(6)


CONTEXT_LENGTH_LABEL = "llm-d.ai/context-length-range"


class ContextTokens(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("tokens", C.c_void_p)]


EPP_STATUS_REJECTED = -2


class AdmissionCfg(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("latency_slo", C.c_int32), ("probabilistic", C.c_int32),
                ("queue_depth_threshold", C.c_int32), ("kv_cache_util_threshold", C.c_double), ("power", C.c_double),
                ("k", C.c_double)]


class Admission(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("reserved", C.c_uint32), ("priority", C.c_void_p), ("ttft_slo", C.c_void_p),
                ("tpot_slo", C.c_void_p), ("pred_valid", C.c_void_p)]


class LabelReq(C.Structure):
    _fields_ = [("key", C.c_char_p), ("op", C.c_int32), ("n_values", C.c_int32), ("values", C.POINTER(C.c_char_p))]


class BatcherCfg(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("max_batch", C.c_int32), ("max_delay_us", C.c_int32),
                ("index_picks", C.c_int32)]


class BatcherStats(C.Structure):
    _fields_ = [("n_flushes", C.c_uint64), ("n_requests", C.c_uint64), ("n_full_flushes", C.c_uint64),
                ("n_pending", C.c_uint64), ("n_index_errors", C.c_uint64)]


class ShardBest(C.Structure):
    _fields_ = [("score", C.c_double), ("pick", C.c_uint32), ("tie_count", C.c_uint32),
                ("match_blocks", C.c_int32), ("status", C.c_int32)]


assert C.sizeof(Decision) == 32 and C.sizeof(DecisionDetail) == 40 and C.sizeof(ShardBest) == 24
assert C.sizeof(Prediction) == 32

# name -> (restype, argtypes): every symbol include/epp_engine.h declares
SIGNATURES = {
    "epp_abi_version": (C.c_int32, []),
    "epp_last_error": (C.c_char_p, []),
    "epp_engine_create": (C.c_int32, [C.POINTER(Config), C.POINTER(C.c_void_p)]),
    "epp_engine_destroy": (C.c_int32, [C.c_void_p]),
    "epp_config_default": (None, [C.POINTER(Config)]),
    "epp_host_alloc": (C.c_int32, [C.c_size_t, C.POINTER(C.c_void_p)]),
    "epp_host_free": (C.c_int32, [C.c_void_p]),
    "epp_model_register": (C.c_int32, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t,
                                       C.POINTER(C.c_uint32)]),
    "epp_model_seed": (C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64)]),
    "epp_pool_set": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "epp_index_add": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_int32, C.c_void_p, C.c_int32]),
    "epp_index_remove_endpoint": (C.c_int32, [C.c_void_p, C.c_uint32]),
    "epp_index_retain_endpoints": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "epp_index_load_snapshot": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]),
    "epp_index_commit": (C.c_int32, [C.c_void_p]),
    "epp_index_get": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]),
    "epp_hash_prompts": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p]),
    "epp_prefix_match": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p]),
    "epp_pool_set_lora": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    "epp_label_filters_set": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(LabelReq)]),
    "epp_pool_set_labels": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "epp_score": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                              C.c_uint32]),
    "epp_schedule": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_int32]),
    "epp_schedule_with_match": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_void_p, C.c_void_p, C.c_uint32]),
    "epp_schedule_topk": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(TopkOut)]),
    "epp_schedule_with_match_topk": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(TopkOut)]),
    "epp_schedule_subset": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.POINTER(Subset), C.c_void_p, C.c_void_p, C.c_int32,
                                        C.POINTER(TopkOut)]),
    "epp_latency_cfg_default": (None, [C.POINTER(LatencyCfg)]),
    "epp_latency_profile_set": (C.c_int32, [C.c_void_p, C.c_int32, C.POINTER(LatencyCfg)]),
    "epp_schedule_predicted": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.POINTER(Predictions), C.c_void_p, C.c_void_p,
                                           C.c_int32, C.POINTER(TopkOut)]),
    "epp_schedule_with_match_predicted": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(TopkOut),
                                                      C.POINTER(Predictions)]),
    "epp_schedule_subset_predicted": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.POINTER(Subset), C.POINTER(Predictions),
                                                  C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(TopkOut)]),
    "epp_context_length_set": (C.c_int32, [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32]),
    "epp_schedule_ctx": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.POINTER(Subset), C.POINTER(Predictions),
                                     C.POINTER(ContextTokens), C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(TopkOut)]),
    "epp_schedule_with_match_ctx": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(TopkOut),
                                                C.POINTER(Predictions), C.POINTER(ContextTokens)]),
    "epp_admission_cfg_default": (None, [C.POINTER(AdmissionCfg)]),
    "epp_admission_set": (C.c_int32, [C.c_void_p, C.POINTER(AdmissionCfg)]),
    "epp_schedule_admit": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.POINTER(Subset), C.POINTER(Predictions),
                                       C.POINTER(ContextTokens), C.POINTER(Admission), C.c_void_p, C.c_void_p, C.c_int32,
                                       C.POINTER(TopkOut)]),
    "epp_schedule_with_match_admit": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                  C.c_int32, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(TopkOut),
                                                  C.POINTER(Predictions), C.POINTER(ContextTokens), C.POINTER(Admission)]),
    "epp_index_add_picked": (C.c_int32, [C.c_void_p]),
    "epp_nohit_lru_get": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]),
    "epp_inflight_release": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "epp_inflight_reset": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p]),
    "epp_inflight_get": (C.c_int32, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "epp_get_stats": (C.c_int32, [C.c_void_p, C.POINTER(Stats)]),
    "epp_synchronize": (C.c_int32, [C.c_void_p]),
    "epp_event_record": (C.c_int32, [C.c_void_p, C.c_int32]),
    "epp_event_elapsed_ms": (C.c_int32, [C.c_void_p, C.POINTER(C.c_double)]),
    "epp_shard_set": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32]),
    "epp_shard_probe": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p]),
    "epp_shard_pick": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "epp_shard_merge": (C.c_int32, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "epp_shard_p2p_export": (C.c_int32, [C.c_void_p, C.c_int64, C.c_void_p, C.POINTER(C.c_uint64)]),
    "epp_shard_p2p_connect": (C.c_int32, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32]),
    "epp_shard_schedule_p2p": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p]),
    "epp_shard_p2p_phase": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_int32]),
    "epp_shard_set_staged": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_int32)]),
    "epp_shard_merge_detail": (C.c_int32, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "epp_shard_schedule_p2p_detail": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p]),
    "epp_shard_p2p_phase_detail": (C.c_int32, [C.c_void_p, C.POINTER(Batch), C.c_void_p, C.c_void_p, C.c_int32]),
    "epp_shard_set_seeded": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_int32)]),
    "epp_shard_select": (C.c_int32, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]),
    "epp_shard_finish": (C.c_int32, [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "epp_get_config": (C.c_int32, [C.c_void_p, C.POINTER(Config)]),
    "epp_batcher_create": (C.c_int32, [C.c_void_p, C.POINTER(BatcherCfg), C.POINTER(C.c_void_p)]),
    "epp_batcher_destroy": (C.c_int32, [C.c_void_p]),
    "epp_submit": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)]),
    "epp_submit_subset": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                      C.POINTER(C.c_uint64)]),
    "epp_submit_predicted": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                         C.POINTER(C.c_uint64)]),
    "epp_submit_subset_predicted": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32,
                                                C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint64)]),
    "epp_submit_ctx": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                   C.c_uint32, C.c_void_p, C.c_int64, C.POINTER(C.c_uint64)]),
    "epp_submit_admit": (C.c_int32, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_void_p,
                                     C.c_uint32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_double,
                                     C.POINTER(C.c_uint64)]),
    "epp_wait": (C.c_int32, [C.c_void_p, C.c_uint64, C.POINTER(Decision), C.POINTER(DecisionDetail)]),
    "epp_wait_topk": (C.c_int32, [C.c_void_p, C.c_uint64, C.POINTER(Decision), C.POINTER(DecisionDetail), C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "epp_batcher_stats": (C.c_int32, [C.c_void_p, C.POINTER(BatcherStats)]),
    "epp_batcher_last_error": (C.c_char_p, []),
}

_lib = None


def load():
    """dlopen libepp_engine.so and bind every declared symbol.  Raises if the library is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is not built: run `python llm-d-inference-scheduler_b200/build.py` "
                          "(there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
