"""Engine: a thin Python handle over the C ABI (include/epp_engine.h).  All compute happens in the CUDA kernels
behind libepp_engine.so; this module only marshals numpy arrays (host pointers) or torch CUDA tensors (device
pointers, EPP_BATCH_DEVICE_PTRS) into plain pointers and sizes."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _capi as capi

DECISION_DTYPE = np.dtype([("status", "<i4"), ("pick", "<u4"), ("score", "<f8"), ("prefill_pick", "<u4"),
                           ("tie_count", "<u4"), ("total_blocks", "<i4"), ("match_blocks", "<i4")])
DETAIL_DTYPE = np.dtype([("prefill_score", "<f8"), ("prefill_tie_count", "<u4"), ("prefill_ran", "<u4"),
                         ("encode_score", "<f8"), ("encode_pick", "<u4"), ("encode_tie_count", "<u4"),
                         ("encode_ran", "<u4"), ("reserved", "<u4")])
SHARD_BEST_DTYPE = np.dtype([("score", "<f8"), ("pick", "<u4"), ("tie_count", "<u4"), ("match_blocks", "<i4"),
                             ("status", "<i4")])
assert DECISION_DTYPE.itemsize == 32 and DETAIL_DTYPE.itemsize == 40 and SHARD_BEST_DTYPE.itemsize == 24


class EngineError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"epp_engine error {code}: {message}")
        self.code = code
        self.message = message


@dataclass
class ScorerSpec:
    kind: int
    weight: float = 1.0
    param: float = 0.0
    column: int = 0          # ext column read by token-load / active-request
    param2: float = 0.0


@dataclass
class AffinityFilterSpec:
    """prefix-cache-affinity-filter (filter/prefixcacheaffinity/plugin.go:62-66 for the defaults)."""
    affinity_threshold: float = 0.80
    exploration_probability: float = 0.01
    max_ttft_penalty_ms: float = 5000.0
    ttft_column: int = -1    # ext column holding the predicted TTFT per endpoint; -1 = no prediction attached


@dataclass
class ProfileSpec:
    """One SchedulerProfile: role filter and label filters -> [prefix-cache-affinity-filter] -> scorers in order ->
    picker (capi.PICKER_MAX_SCORE / PICKER_RANDOM / PICKER_WEIGHTED_RANDOM).  labels: the label requirements
    [(key, capi.LABEL_* op, [values...]), ...], all ANDed (Engine.label_filters_set)."""
    filter: int = capi.FILTER_NONE
    scorers: list = field(default_factory=list)
    affinity: AffinityFilterSpec | None = None
    picker: int = capi.PICKER_MAX_SCORE
    labels: list = field(default_factory=list)
    latency: dict | None = None      # Engine.latency_profile_set fields of a profile with a latency piece, or None
    context_length: dict | None = None   # Engine.context_length_set fields (label, enable_filtering) of a profile listing
                                         # the context-length scorer, or None (the defaults)


def _fill_profile(dst: capi.ProfileCfg, spec: ProfileSpec):
    if len(spec.scorers) > capi.EPP_MAX_SCORERS:
        raise ValueError("too many scorers")
    dst.filter = spec.filter
    dst.n_scorers = len(spec.scorers)
    for i, s in enumerate(spec.scorers):
        if not isinstance(s, ScorerSpec):
            s = ScorerSpec(*s)
        dst.scorers[i].kind = s.kind
        dst.scorers[i].weight = s.weight
        dst.scorers[i].param = s.param
        dst.scorers[i].column = s.column
        dst.scorers[i].param2 = s.param2
    dst.ttft_column = -1
    dst.picker = spec.picker
    if spec.affinity is not None:
        a = spec.affinity
        dst.affinity_threshold, dst.exploration_probability = a.affinity_threshold, a.exploration_probability
        dst.max_ttft_penalty_ms, dst.ttft_column = a.max_ttft_penalty_ms, a.ttft_column


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _ptr(x):
    if x is None:
        return None
    if _is_torch(x):
        return C.c_void_p(x.data_ptr())
    return x.ctypes.data_as(C.c_void_p)


def pack_subsets(subsets):
    """Per-request endpoint subsets -> the host arrays of epp_subset: (counts u32 [R], offsets u64 [R], slots u32 [...]).
    Entry r is None (the whole pool: EPP_SUBSET_ALL) or a sequence of slot ids, sorted and deduplicated here."""
    R = len(subsets)
    counts = np.full(R, capi.EPP_SUBSET_ALL, dtype=np.uint32)
    offsets = np.zeros(R, dtype=np.uint64)
    parts, n = [], 0
    for r, s in enumerate(subsets):
        if s is None:
            continue
        u = np.unique(np.asarray(s, dtype=np.int64))
        if u.size and (u[0] < 0 or u[-1] > 0xFFFFFFFE):
            raise ValueError(f"request {r}: slot id out of range")
        counts[r] = u.size
        offsets[r] = n
        parts.append(u.astype(np.uint32))
        n += u.size
    slots = np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint32)
    return counts, offsets, np.ascontiguousarray(slots, dtype=np.uint32)


PREDICTION_DTYPE = np.dtype([("slot", "<u4"), ("dispatched", "<i4"), ("ttft", "<f8"), ("ttft_headroom", "<f8"),
                             ("tpot_headroom", "<f8")])
assert PREDICTION_DTYPE.itemsize == C.sizeof(capi.Prediction)


def pack_predictions(predictions):
    """Per-request latency predictions -> the host arrays of epp_predictions: (counts u32 [R], offsets u64 [R], entries
    [n] of PREDICTION_DTYPE).  Entry r is None (no predictions) or an iterable of (slot, ttft, ttft_headroom,
    tpot_headroom, dispatched) -- LatencyPredictionInfo's TTFT(), TTFTHeadroom(), TPOTHeadroom() and
    DispatchedRequestCount() on that slot for request r, or an array of PREDICTION_DTYPE.  Entries are sorted by slot here;
    a slot given twice is an error."""
    R = len(predictions)
    counts = np.zeros(R, dtype=np.uint32)
    offsets = np.zeros(R, dtype=np.uint64)
    parts, n = [], 0
    for r, p in enumerate(predictions):
        offsets[r] = n
        if p is None:
            continue
        if isinstance(p, np.ndarray) and p.dtype == PREDICTION_DTYPE:
            a = np.sort(p, order="slot", kind="stable")
            if a.size > 1 and (np.diff(a["slot"].astype(np.int64)) == 0).any():
                raise ValueError(f"request {r}: a slot has two predictions")
            if a.size and a["slot"][-1] == 0xFFFFFFFF:
                raise ValueError(f"request {r}: slot id out of range")
            counts[r] = a.size
            parts.append(a)
            n += a.size
            continue
        rows = sorted((int(sl), float(t), float(th), float(tp), int(d)) for sl, t, th, tp, d in p)
        a = np.zeros(len(rows), dtype=PREDICTION_DTYPE)
        for i, (sl, t, th, tp, d) in enumerate(rows):
            if sl < 0 or sl > 0xFFFFFFFE:
                raise ValueError(f"request {r}: slot id {sl} out of range")
            if i and sl == rows[i - 1][0]:
                raise ValueError(f"request {r}: slot {sl} has two predictions")
            a[i] = (sl, d, t, th, tp)
        counts[r] = len(rows)
        parts.append(a)
        n += len(rows)
    entries = np.concatenate(parts) if parts else np.zeros(0, dtype=PREDICTION_DTYPE)
    return counts, offsets, np.ascontiguousarray(entries)


def _context_struct(context_tokens, R):
    """epp_context_tokens over R int64 entries -> (struct, the array it points to: keep it alive through the call)."""
    arr = np.ascontiguousarray(np.asarray(context_tokens, dtype=np.int64).reshape(-1))
    if arr.shape[0] != R:
        raise ValueError(f"context_tokens has {arr.shape[0]} entries for {R} requests")
    ct = capi.ContextTokens()
    ct.struct_size = C.sizeof(capi.ContextTokens)
    ct.tokens = arr.ctypes.data if R else None
    return ct, arr


def _admission_struct(admission, R, predictions=None):
    """epp_admission for R requests -> (struct, the arrays it points to: keep them alive through the call).
    admission: a dict with any of "priority" (R ints, < 0 = sheddable), "ttft_slo" / "tpot_slo" (R doubles, the parsed
    x-slo-ttft-ms / x-slo-tpot-ms headers) and "pred_valid" (R entries, each None or one validity byte -- bit 0 TTFTValid,
    bit 1 TPOTValid -- per entry of that request's predictions, in the order given to pack_predictions, which sorts both
    alike)."""
    keep = []
    a = capi.Admission()
    a.struct_size = C.sizeof(capi.Admission)
    for name, dt in (("priority", np.int32), ("ttft_slo", np.float64), ("tpot_slo", np.float64)):
        if admission.get(name) is None:
            continue
        arr = np.ascontiguousarray(np.asarray(admission[name], dtype=dt).reshape(-1))
        if arr.shape[0] != R:
            raise ValueError(f"admission {name} has {arr.shape[0]} entries for {R} requests")
        keep.append(arr)
        setattr(a, name, arr.ctypes.data if R else None)
    pv = admission.get("pred_valid")
    if pv is not None:
        if len(pv) != R:
            raise ValueError(f"admission pred_valid has {len(pv)} entries for {R} requests")
        parts = []
        for r, v in enumerate(pv):
            p = None if predictions is None else predictions[r]
            n = 0 if p is None else len(p)
            v = np.zeros(0, dtype=np.uint8) if v is None else np.asarray(v, dtype=np.uint8).reshape(-1)
            if v.shape[0] != n:
                raise ValueError(f"request {r}: {v.shape[0]} validity bytes for {n} predictions")
            if n:
                slots = p["slot"] if isinstance(p, np.ndarray) and p.dtype == PREDICTION_DTYPE else [int(e[0]) for e in p]
                v = v[np.argsort(np.asarray(slots, dtype=np.int64), kind="stable")]
            parts.append(v)
        arr = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, dtype=np.uint8))
        if arr.shape[0] == 0:
            arr = np.zeros(1, dtype=np.uint8)          # a valid pointer for a call whose requests have no entries
        keep.append(arr)
        a.pred_valid = arr.ctypes.data
    return a, keep


def _prediction_entries(predictions):
    """One request's predictions (a PREDICTION_DTYPE array, or (slot, ttft, ttft_headroom, tpot_headroom, dispatched)
    tuples) as a contiguous PREDICTION_DTYPE array."""
    if isinstance(predictions, np.ndarray) and predictions.dtype == PREDICTION_DTYPE:
        return np.ascontiguousarray(predictions)
    ent = np.zeros(len(predictions), dtype=PREDICTION_DTYPE)
    for i, (sl, tt, th, tp, d) in enumerate(predictions):
        if not 0 <= int(sl) <= 0xFFFFFFFE:
            raise ValueError(f"slot id {sl} out of range")
        ent[i] = (int(sl), int(d), float(tt), float(th), float(tp))
    return ent


def _predictions_struct(packed):
    p = capi.Predictions()
    p.struct_size = C.sizeof(capi.Predictions)
    p.counts, p.offsets, p.entries = (_ptr(a) for a in packed)
    return p


class Engine:
    def __init__(self, max_endpoints: int, primary: ProfileSpec | None = None, prefill: ProfileSpec | None = None,
                 *, device: int = 0, block_size_tokens: int = 16, max_prefix_blocks: int = 256,
                 lru_capacity_per_server: int = 31250, non_cached_tokens: int = 0, always_disagg: bool = False,
                 n_ext_cols: int = 0, tie_seed: int = 0, encode: ProfileSpec | None = None, pick_k: int = 0,
                 index_commit_interval_us: int = 0, inflight_load: bool = False):
        self._lib = capi.load()
        cfg = capi.Config()
        self._lib.epp_config_default(C.byref(cfg))
        cfg.device = device
        cfg.max_endpoints = max_endpoints
        cfg.block_size_tokens = block_size_tokens
        cfg.max_prefix_blocks = max_prefix_blocks
        cfg.lru_capacity_per_server = lru_capacity_per_server
        cfg.non_cached_tokens = non_cached_tokens
        cfg.always_disagg = int(always_disagg)
        cfg.n_ext_cols = n_ext_cols
        if primary is not None:
            _fill_profile(cfg.primary, primary)
        if prefill is not None:
            cfg.handler = capi.HANDLER_DISAGG
            _fill_profile(cfg.prefill, prefill)
        if encode is not None:
            cfg.encode_enabled = 1
            _fill_profile(cfg.encode, encode)
        cfg.tie_seed = tie_seed
        cfg.pick_k = pick_k
        cfg.index_commit_interval_us = index_commit_interval_us
        cfg.inflight_load = int(inflight_load)
        self.cfg = cfg
        self.E = max_endpoints
        self.B = max_prefix_blocks
        self.shard_stages = 1           # records per request of the endpoint-sharded protocol (shard_set_staged)
        self.shard_seeded = False       # the sharded protocol resolves the seeded tie rule (shard_set_seeded)
        self._h = C.c_void_p()
        self._check(self._lib.epp_engine_create(C.byref(cfg), C.byref(self._h)))
        for p, spec in enumerate((primary, prefill, encode)):
            if spec is not None and spec.labels:
                self.label_filters_set(p, spec.labels)
            if spec is not None and spec.latency is not None:
                self.latency_profile_set(p, **spec.latency)
            if spec is not None and spec.context_length is not None:
                self.context_length_set(p, **spec.context_length)

    # ---- plumbing ----
    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, (self._lib.epp_last_error() or b"").decode())

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.epp_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- models / pool / index ----
    def register_model(self, model: bytes, salt: bytes = b"") -> int:
        mid = C.c_uint32()
        self._check(self._lib.epp_model_register(self._h, model, len(model), salt, len(salt), C.byref(mid)))
        return mid.value

    def model_seed(self, model_id: int) -> int:
        out = C.c_uint64()
        self._check(self._lib.epp_model_seed(self._h, model_id, C.byref(out)))
        return out.value

    def pool_set(self, ids, role, kv_usage, waiting, running=None, ext=None):
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        n = ids.shape[0]
        role = np.ascontiguousarray(role, dtype=np.uint8)
        kv = np.ascontiguousarray(kv_usage, dtype=np.float64)
        w = np.ascontiguousarray(waiting, dtype=np.int32)
        run = None if running is None else np.ascontiguousarray(running, dtype=np.int32)
        ex = None if ext is None else np.ascontiguousarray(ext, dtype=np.float64).reshape(-1, n)
        assert role.shape[0] == n and kv.shape[0] == n and w.shape[0] == n
        self._check(self._lib.epp_pool_set(self._h, n, _ptr(ids), _ptr(role), _ptr(kv), _ptr(w), _ptr(run), _ptr(ex)))

    def index_add(self, ep: int, hashes, num_gpu_blocks: int = 0):
        hs = np.ascontiguousarray(hashes, dtype=np.uint64)
        self._check(self._lib.epp_index_add(self._h, ep, hs.shape[0], _ptr(hs), num_gpu_blocks))

    def index_remove_endpoint(self, ep: int):
        self._check(self._lib.epp_index_remove_endpoint(self._h, ep))

    def index_load_snapshot(self, hashes, eps):
        hs = np.ascontiguousarray(hashes, dtype=np.uint64)
        es = np.ascontiguousarray(eps, dtype=np.uint32)
        assert hs.shape == es.shape
        self._check(self._lib.epp_index_load_snapshot(self._h, hs.shape[0], _ptr(hs), _ptr(es)))

    def index_retain_endpoints(self, active_ids):
        """CleanUpInactivePods (plugin.go:99-122): drop every indexed endpoint that is not in active_ids."""
        a = np.ascontiguousarray(active_ids, dtype=np.uint32)
        self._check(self._lib.epp_index_retain_endpoints(self._h, a.shape[0], _ptr(a)))

    def index_commit(self):
        self._check(self._lib.epp_index_commit(self._h))

    def index_get(self, h: int) -> set:
        out = np.zeros(4096, dtype=np.uint32)
        n = C.c_int32()
        self._check(self._lib.epp_index_get(self._h, h, _ptr(out), out.shape[0], C.byref(n)))
        return set(int(x) for x in out[:min(n.value, out.shape[0])])

    def index_add_picked(self):
        self._check(self._lib.epp_index_add_picked(self._h))

    def nohit_lru_get(self) -> list:
        """The no-hit-lru scorer's LRU, oldest first (golang-lru Cache.Keys): slot ids."""
        out = np.zeros(self.E, dtype=np.uint32)
        n = C.c_int32()
        self._check(self._lib.epp_nohit_lru_get(self._h, _ptr(out), out.shape[0], C.byref(n)))
        return [int(x) for x in out[:min(n.value, out.shape[0])]]

    # ---- inflight-load producer (engines created with inflight_load=True) ----
    def inflight_release(self, eps, prompt_lens):
        """ResponseBody (producer.go:131-168): 1 request and est(prompt_lens[i]) tokens off slot eps[i] each;
        EPP_NO_ENDPOINT entries are skipped."""
        e = np.ascontiguousarray(eps, dtype=np.uint32).reshape(-1)
        ln = np.ascontiguousarray(prompt_lens, dtype=np.uint64).reshape(-1)
        assert e.shape == ln.shape
        self._check(self._lib.epp_inflight_release(self._h, e.shape[0], _ptr(e), _ptr(ln)))

    def inflight_reset(self, ids):
        """Endpoint deletion (producer.go:86-97): both counters of the slots become 0."""
        a = np.ascontiguousarray(ids, dtype=np.uint32).reshape(-1)
        self._check(self._lib.epp_inflight_reset(self._h, a.shape[0], _ptr(a)))

    def inflight_get(self):
        """-> (requests int64[E], tokens int64[E]): InFlightLoad per slot, after every call made so far."""
        req = np.zeros(self.E, dtype=np.int64)
        tok = np.zeros(self.E, dtype=np.int64)
        self._check(self._lib.epp_inflight_get(self._h, self.E, _ptr(req), _ptr(tok)))
        return req, tok

    # ---- batches ----
    def _batch(self, data, offsets=None, uniform_len=None, model_ids=None, n_requests=None, lengths=None, multimodal=None):
        """data: bytes-like numpy array / torch CUDA tensor (any dtype, viewed as bytes)."""
        b = capi.Batch()
        dev = _is_torch(data)
        keep = [data]
        if dev:
            if not data.is_cuda:
                raise ValueError("torch batches must be CUDA tensors (device-pointer mode)")
            b.flags = capi.EPP_BATCH_DEVICE_PTRS
            nbytes = data.numel() * data.element_size()
        else:
            data = np.ascontiguousarray(data)
            keep[0] = data
            nbytes = data.nbytes
        b.data = _ptr(data)
        if offsets is not None:
            if dev:
                assert _is_torch(offsets) and offsets.is_cuda
                R = offsets.numel() - 1
            else:
                offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
                R = offsets.shape[0] - 1
            keep.append(offsets)
            b.offsets = _ptr(offsets)
        else:
            if uniform_len is None:
                raise ValueError("offsets or uniform_len required")
            R = n_requests if n_requests is not None else (nbytes // uniform_len if uniform_len else 0)
            b.uniform_len = uniform_len
        if model_ids is not None:
            if not dev:
                model_ids = np.ascontiguousarray(model_ids, dtype=np.uint32)
            keep.append(model_ids)
            b.model_ids = _ptr(model_ids)
        if lengths is not None:
            if not dev:
                lengths = np.ascontiguousarray(lengths, dtype=np.uint64)
            keep.append(lengths)
            b.lengths = _ptr(lengths)
        if multimodal is not None:
            if not dev:
                multimodal = np.ascontiguousarray(multimodal, dtype=np.uint8)
            keep.append(multimodal)
            b.multimodal = _ptr(multimodal)
        b.n_requests = R
        return b, R, dev, keep

    def hash_prompts(self, data, offsets=None, uniform_len=None, model_ids=None, n_requests=None, lengths=None, out=None):
        """a1 hashPrompt -> (hashes [R, max_prefix_blocks] u64, nblocks [R] i32)."""
        b, R, dev, keep = self._batch(data, offsets, uniform_len, model_ids, n_requests, lengths)
        if dev:
            import torch
            hashes = torch.empty((max(R, 1), self.B), dtype=torch.int64, device=data.device) if out is None else out[0]
            nb = torch.empty(max(R, 1), dtype=torch.int32, device=data.device) if out is None else out[1]
        else:
            hashes = np.zeros((R, self.B), dtype=np.uint64)
            nb = np.zeros(R, dtype=np.int32)
        self._check(self._lib.epp_hash_prompts(self._h, C.byref(b), _ptr(hashes), _ptr(nb)))
        return hashes, nb

    def prefix_match(self, data, offsets=None, uniform_len=None, model_ids=None, n_requests=None, lengths=None):
        """a1-a4 Produce -> (match [R, E] i32, total [R] i32)."""
        b, R, dev, keep = self._batch(data, offsets, uniform_len, model_ids, n_requests, lengths)
        if dev:
            import torch
            match = torch.empty((max(R, 1), self.E), dtype=torch.int32, device=data.device)
            total = torch.empty(max(R, 1), dtype=torch.int32, device=data.device)
        else:
            match = np.zeros((R, self.E), dtype=np.int32)
            total = np.zeros(R, dtype=np.int32)
        self._check(self._lib.epp_prefix_match(self._h, C.byref(b), _ptr(match), _ptr(total)))
        return match, total

    def score(self, match, total, profile: int = 0, scorer_index: int = -1, model_ids=None):
        """a5-a9 Scorer.Score / weighted sum -> [R, E] f64 (host arrays)."""
        match = np.ascontiguousarray(match, dtype=np.int32).reshape(-1, self.E)
        total = np.ascontiguousarray(total, dtype=np.int32)
        R = match.shape[0]
        mids = None if model_ids is None else np.ascontiguousarray(model_ids, dtype=np.uint32)
        out = np.zeros((R, self.E), dtype=np.float64)
        self._check(self._lib.epp_score(self._h, R, _ptr(match), _ptr(total), _ptr(mids), profile, scorer_index, _ptr(out), 0))
        return out

    def pool_set_lora(self, ids, max_active_models, n_models_loaded, members=()):
        """LoRA residency for the lora-affinity scorer; members = iterable of (endpoint slot, model id, state) with
        state 1 = active, 2 = waiting (fwkdl.Metrics.ActiveModels / WaitingModels / MaxActiveModels)."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        mx = np.ascontiguousarray(max_active_models, dtype=np.int32)
        nl = np.ascontiguousarray(n_models_loaded, dtype=np.int32)
        mem = np.asarray(list(members), dtype=np.int64).reshape(-1, 3)
        mep = np.ascontiguousarray(mem[:, 0], dtype=np.uint32)
        mmo = np.ascontiguousarray(mem[:, 1], dtype=np.uint32)
        mst = np.ascontiguousarray(mem[:, 2], dtype=np.uint8)
        self._check(self._lib.epp_pool_set_lora(self._h, ids.shape[0], _ptr(ids), _ptr(mx), _ptr(nl), mem.shape[0],
                                                _ptr(mep), _ptr(mmo), _ptr(mst)))

    def label_filters_set(self, profile: int, reqs):
        """The label requirements of profile 0 (primary / decode), 1 (prefill) or 2 (encode), ANDed with its role
        filter: reqs = [(key, op, [values...]), ...], op one of capi.LABEL_* (include/epp_engine.h "Label filters").
        Only before the first pool_set / pool_set_labels."""
        reqs = list(reqs)
        arr = (capi.LabelReq * max(len(reqs), 1))()
        keep = []
        for i, (key, op, values) in enumerate(reqs):
            vals = [v.encode() if isinstance(v, str) else bytes(v) for v in values]
            va = (C.c_char_p * max(len(vals), 1))(*vals)
            keep.append(va)
            arr[i].key = key.encode() if isinstance(key, str) else bytes(key)
            arr[i].op = op
            arr[i].n_values = len(vals)
            arr[i].values = C.cast(va, C.POINTER(C.c_char_p))
        self._check(self._lib.epp_label_filters_set(self._h, profile, len(reqs), arr))

    def pool_set_labels(self, ids, labels):
        """EndpointMetadata.Labels of slots ids[i] = labels[i] (a dict str -> str, or None); other slots have none."""
        ids = np.ascontiguousarray(ids, dtype=np.uint32)
        assert len(labels) == ids.shape[0]
        if any("\n" in k or "=" in k or "\n" in v for lb in labels for k, v in (lb or {}).items()):
            raise ValueError("a label key holds '=' or a newline, or a value holds a newline")
        parts = [b"".join(f"{k}={v}\n".encode() for k, v in (lb or {}).items()) for lb in labels]
        offs = np.zeros(len(parts) + 1, dtype=np.uint64)
        np.cumsum([len(p) for p in parts], out=offs[1:])
        text = np.frombuffer(b"".join(parts) or b"\0", dtype=np.uint8)
        self._check(self._lib.epp_pool_set_labels(self._h, ids.shape[0], _ptr(ids), _ptr(offs), _ptr(text)))

    def latency_profile_set(self, profile: int, **fields):
        """The latency configuration of profile 0 (primary / decode), 1 (prefill) or 2 (encode): the epp_latency_cfg
        fields given as keywords (tier_filter, epsilon_explore_neg, a1_affinity_threshold, a1_exploration_probability,
        a1_max_ttft_penalty_ms, ttft_weight, tpot_weight, strategy, composite_kv_weight, composite_queue_weight,
        composite_prefix_weight), the others at the reference's defaults (include/epp_engine.h "Latency predictions").
        Only before the first pool_set / pool_set_labels."""
        cfg = capi.LatencyCfg()
        self._lib.epp_latency_cfg_default(C.byref(cfg))
        names = {n for n, _ in capi.LatencyCfg._fields_} - {"struct_size", "reserved"}
        for k, v in fields.items():
            if k not in names:
                raise TypeError(f"unknown latency configuration field {k!r}")
            setattr(cfg, k, v)
        self._check(self._lib.epp_latency_profile_set(self._h, profile, C.byref(cfg)))

    def admission_set(self, latency_slo: bool = False, probabilistic: bool = False, **fields):
        """The engine's admitters (include/epp_engine.h "Admission"): the latency-slo-admitter and / or the
        probabilistic-admitter with the epp_admission_cfg fields given as keywords (queue_depth_threshold,
        kv_cache_util_threshold, power, k), the others at the reference's defaults.  Only before the first pool_set /
        pool_set_labels."""
        cfg = capi.AdmissionCfg()
        self._lib.epp_admission_cfg_default(C.byref(cfg))
        cfg.latency_slo = int(latency_slo)
        cfg.probabilistic = int(probabilistic)
        names = {n for n, _ in capi.AdmissionCfg._fields_} - {"struct_size", "latency_slo", "probabilistic"}
        for k, v in fields.items():
            if k not in names:
                raise TypeError(f"unknown admission configuration field {k!r}")
            setattr(cfg, k, v)
        self._check(self._lib.epp_admission_set(self._h, C.byref(cfg)))

    def context_length_set(self, profile: int, label: str | None = None, enable_filtering: bool = False):
        """The context-length-aware plugin of profile 0 (primary / decode), 1 (prefill) or 2 (encode): its range label key
        (None = capi.CONTEXT_LENGTH_LABEL) and whether it also filters (include/epp_engine.h "Context length")."""
        self._check(self._lib.epp_context_length_set(self._h, profile, None if label is None else label.encode(),
                                                     int(enable_filtering)))

    def schedule(self, data, offsets=None, uniform_len=None, model_ids=None, n_requests=None, keep_hashes=False,
                 detail=True, out=None, lengths=None, asynchronous=False, multimodal=None, topk=False, subsets=None,
                 predictions=None, context_tokens=None, admission=None):
        """a1-a14 Scheduler.Schedule for a batch -> (decisions, details).  asynchronous=True (CUDA tensors only)
        enqueues the batch and returns; the outputs are complete after synchronize().  topk=True (engines created with
        pick_k > 1) also returns the dict of the pickers' first-k lists (maxscore/picker.go:104-115): "primary",
        "primary_scores", "prefill", "encode", each [R][pick_k], padded with EPP_NO_ENDPOINT / 0.
        subsets: None, or a list of R entries, each None (the whole pool) or a sequence of slot ids: the request's
        candidates (the gateway's endpoint subset, include/epp_engine.h "Endpoint subsets"); epp_schedule_subset.
        predictions: None, or a list of R entries in the form pack_predictions takes (include/epp_engine.h "Latency
        predictions"); epp_schedule_predicted.  Both together: epp_schedule_subset_predicted (a latency engine's
        restricted requests decided with their predictions).
        context_tokens: None, or R request context lengths (-1 = the default from the prompt length, include/epp_engine.h
        "Context length"); with it every call goes through epp_schedule_ctx.
        admission: None, or the requests' admission inputs as _admission_struct takes them (include/epp_engine.h
        "Admission", engines with admission_set); with it the call goes through epp_schedule_admit and rejected requests
        come back with status capi.EPP_STATUS_REJECTED."""
        b, R, dev, keep = self._batch(data, offsets, uniform_len, model_ids, n_requests, lengths, multimodal)
        if asynchronous:
            b.flags |= capi.EPP_BATCH_ASYNC
        if dev:
            import torch
            dec = out if out is not None else torch.empty((max(R, 1), 32), dtype=torch.uint8, device=data.device)
            det = torch.empty((max(R, 1), 40), dtype=torch.uint8, device=data.device) if detail else None
        else:
            dec = np.zeros(R, dtype=DECISION_DTYPE) if out is None else out
            det = np.zeros(R, dtype=DETAIL_DTYPE) if detail else None
        lists, tk = self._topk_out(R, data.device if dev else None) if topk else (None, None)
        if predictions is not None and len(predictions) != R:
            raise ValueError(f"predictions has {len(predictions)} entries for {R} requests")
        if subsets is not None and len(subsets) != R:
            raise ValueError(f"subsets has {len(subsets)} entries for {R} requests")
        if predictions is not None:
            ppacked = pack_predictions(predictions)     # host arrays, kept alive until the call returns
            pr = _predictions_struct(ppacked)
        if subsets is not None:
            spacked = pack_subsets(subsets)             # host arrays, kept alive until the call returns
            sub = capi.Subset()
            sub.struct_size = C.sizeof(capi.Subset)
            sub.counts, sub.offsets, sub.slots = (_ptr(a) for a in spacked)
        if admission is not None:
            ad, ad_keep = _admission_struct(admission, R, predictions)
            ct, ctx_arr = _context_struct(context_tokens, R) if context_tokens is not None else (None, None)
            self._check(self._lib.epp_schedule_admit(self._h, C.byref(b), C.byref(sub) if subsets is not None else None,
                                                     C.byref(pr) if predictions is not None else None,
                                                     C.byref(ct) if ct is not None else None, C.byref(ad), _ptr(dec),
                                                     _ptr(det), int(keep_hashes), C.byref(tk) if topk else None))
        elif context_tokens is not None:
            ct, ctx_arr = _context_struct(context_tokens, R)
            self._check(self._lib.epp_schedule_ctx(self._h, C.byref(b), C.byref(sub) if subsets is not None else None,
                                                   C.byref(pr) if predictions is not None else None, C.byref(ct), _ptr(dec),
                                                   _ptr(det), int(keep_hashes), C.byref(tk) if topk else None))
        elif predictions is not None and subsets is not None:
            self._check(self._lib.epp_schedule_subset_predicted(self._h, C.byref(b), C.byref(sub), C.byref(pr), _ptr(dec),
                                                                _ptr(det), int(keep_hashes), C.byref(tk) if topk else None))
        elif predictions is not None:
            self._check(self._lib.epp_schedule_predicted(self._h, C.byref(b), C.byref(pr), _ptr(dec), _ptr(det),
                                                         int(keep_hashes), C.byref(tk) if topk else None))
        elif subsets is not None:
            self._check(self._lib.epp_schedule_subset(self._h, C.byref(b), C.byref(sub), _ptr(dec), _ptr(det),
                                                      int(keep_hashes), C.byref(tk) if topk else None))
        elif not topk:
            self._check(self._lib.epp_schedule(self._h, C.byref(b), _ptr(dec), _ptr(det), int(keep_hashes)))
        else:
            self._check(self._lib.epp_schedule_topk(self._h, C.byref(b), _ptr(dec), _ptr(det), int(keep_hashes), C.byref(tk)))
        return (dec, det, lists) if topk else (dec, det)

    def _topk_out(self, R: int, device=None):
        """Destination arrays of the pickers' first-k lists (numpy, or torch on `device`) + the epp_topk_out record."""
        k = int(self.cfg.pick_k)
        n = max(R, 1)
        if device is not None:
            import torch
            lists = {name: torch.empty((n, k), dtype=torch.int32, device=device) for name in ("primary", "prefill", "encode")}
            lists["primary_scores"] = torch.empty((n, k), dtype=torch.float64, device=device)
        else:
            lists = {name: np.zeros((R, k), dtype=np.uint32) for name in ("primary", "prefill", "encode")}
            lists["primary_scores"] = np.zeros((R, k), dtype=np.float64)
        tk = capi.TopkOut()
        tk.struct_size = C.sizeof(capi.TopkOut)
        tk.k = k
        for name in ("primary", "primary_scores", "prefill", "encode"):
            setattr(tk, name, _ptr(lists[name]).value if R else None)
        return lists, tk

    def schedule_with_match(self, match, total, input_len_bytes=None, block_size_tokens: int = 0, model_ids=None,
                            topk=False, predictions=None, context_tokens=None, admission=None):
        match = np.ascontiguousarray(match, dtype=np.int32).reshape(-1, self.E)
        total = np.ascontiguousarray(total, dtype=np.int32)
        R = match.shape[0]
        il = None if input_len_bytes is None else np.ascontiguousarray(input_len_bytes, dtype=np.int64)
        dec = np.zeros(R, dtype=DECISION_DTYPE)
        det = np.zeros(R, dtype=DETAIL_DTYPE)
        mids = None if model_ids is None else np.ascontiguousarray(model_ids, dtype=np.uint32)
        if admission is not None:
            ad, ad_keep = _admission_struct(admission, R, predictions)
        ct, ctx_arr = _context_struct(context_tokens, R) if context_tokens is not None else (None, None)
        if predictions is not None and len(predictions) != R:
            raise ValueError(f"predictions has {len(predictions)} entries for {R} requests")
        packed = pack_predictions(predictions) if predictions is not None else None
        pr = _predictions_struct(packed) if packed is not None else None
        lists, tk = self._topk_out(R) if topk else (None, None)
        args = (self._h, R, _ptr(match), _ptr(total), _ptr(mids), _ptr(il), block_size_tokens, _ptr(dec), _ptr(det), 0)
        tkp = C.byref(tk) if topk else None
        prp = C.byref(pr) if pr is not None else None
        if admission is not None:
            rc = self._lib.epp_schedule_with_match_admit(*args, tkp, prp, C.byref(ct) if ct is not None else None,
                                                         C.byref(ad))
        elif ct is not None:
            rc = self._lib.epp_schedule_with_match_ctx(*args, tkp, prp, C.byref(ct))
        elif pr is not None:
            rc = self._lib.epp_schedule_with_match_predicted(*args, tkp, prp)
        elif topk:
            rc = self._lib.epp_schedule_with_match_topk(*args, tkp)
        else:
            rc = self._lib.epp_schedule_with_match(*args)
        self._check(rc)
        return (dec, det, lists) if topk else (dec, det)

    def synchronize(self):
        self._check(self._lib.epp_synchronize(self._h))

    def event_record(self, which: int):
        """CUDA event on the engine's launch stream (0 = start, 1 = stop)."""
        self._check(self._lib.epp_event_record(self._h, which))

    def event_elapsed_ms(self) -> float:
        ms = C.c_double(0.0)
        self._check(self._lib.epp_event_elapsed_ms(self._h, C.byref(ms)))
        return ms.value

    def stats(self) -> dict:
        s = capi.Stats()
        self._check(self._lib.epp_get_stats(self._h, C.byref(s)))
        d = {k: getattr(s, k) for k, _ in capi.Stats._fields_}
        d["last_kernel_ms"] = list(s.last_kernel_ms)
        return d

    # ---- endpoint-sharded mode (device pointers only) ----
    def shard_set(self, ep_begin: int, ep_end: int):
        self._check(self._lib.epp_shard_set(self._h, ep_begin, ep_end))
        self.shard_stages = 1
        self.shard_seeded = False

    def shard_set_staged(self, ep_begin: int, ep_end: int) -> int:
        """shard_set that also takes the disagg handler -> S, the records per request of shard_pick (1 single profile,
        2 decode + prefill, 3 with encode); shard_pick's out_best is then [R, S * 24] bytes."""
        s = C.c_int32(0)
        self._check(self._lib.epp_shard_set_staged(self._h, ep_begin, ep_end, C.byref(s)))
        self.shard_stages = s.value
        self.shard_seeded = False
        return s.value

    def shard_set_seeded(self, ep_begin: int, ep_end: int) -> int:
        """shard_set_staged with the engine's tie_seed rule across the shards (epp_engine.h, "Seeded ties") -> S.  A batch
        then takes shard_select and shard_finish (a third exchange) instead of shard_merge, and the peer-memory exchange
        four phases."""
        s = C.c_int32(0)
        self._check(self._lib.epp_shard_set_seeded(self._h, ep_begin, ep_end, C.byref(s)))
        self.shard_stages = s.value
        self.shard_seeded = True
        return s.value

    def shard_probe(self, data, out_masks, offsets=None, uniform_len=None, model_ids=None, n_requests=None,
                    lengths=None, multimodal=None):
        b, R, dev, keep = self._batch(data, offsets, uniform_len, model_ids, n_requests, lengths, multimodal)
        self._check(self._lib.epp_shard_probe(self._h, C.byref(b), _ptr(out_masks)))
        return R

    def shard_pick(self, n_requests, global_masks, out_best):
        self._check(self._lib.epp_shard_pick(self._h, n_requests, _ptr(global_masks), _ptr(out_best)))

    def shard_p2p_export(self, max_requests: int):
        """-> (64-byte CUDA IPC handle, raw device pointer) of this rank's exchange buffer."""
        handle = np.zeros(64, dtype=np.uint8)
        ptr = C.c_uint64(0)
        self._check(self._lib.epp_shard_p2p_export(self._h, max_requests, _ptr(handle), C.byref(ptr)))
        return handle, ptr.value

    def shard_p2p_connect(self, n_ranks: int, rank: int, peers, ipc_handles: bool = True):
        """peers: [n_ranks, 64] uint8 handles (other processes) or [n_ranks] uint64 pointers (same process)."""
        a = np.ascontiguousarray(peers, dtype=np.uint8 if ipc_handles else np.uint64)
        self._check(self._lib.epp_shard_p2p_connect(self._h, n_ranks, rank, _ptr(a), int(ipc_handles)))

    def shard_schedule_p2p(self, data, out_decisions, offsets=None, uniform_len=None, model_ids=None, n_requests=None,
                           lengths=None, multimodal=None, out_detail=None):
        """out_detail: [R, 40] uint8 CUDA tensor of epp_decision_detail (prefill and encode fields), or None."""
        b, R, dev, keep = self._batch(data, offsets, uniform_len, model_ids, n_requests, lengths, multimodal)
        self._check(self._lib.epp_shard_schedule_p2p_detail(self._h, C.byref(b), _ptr(out_decisions), _ptr(out_detail)))
        return R

    def shard_p2p_phase(self, data, out_decisions, phase: int, offsets=None, uniform_len=None, model_ids=None,
                        n_requests=None, lengths=None, multimodal=None, out_detail=None):
        """One phase (0, 1, 2; and 3 on a seeded engine) of shard_schedule_p2p, synchronised: for ranks that share a
        GPU."""
        b, R, dev, keep = self._batch(data, offsets, uniform_len, model_ids, n_requests, lengths, multimodal)
        self._check(self._lib.epp_shard_p2p_phase_detail(self._h, C.byref(b), _ptr(out_decisions), _ptr(out_detail), phase))
        return R

    def shard_merge(self, n_requests, n_ranks, all_best, out_decisions, out_detail=None):
        """all_best: [n_ranks, R, S * 24] records; out_detail as in shard_schedule_p2p."""
        self._check(self._lib.epp_shard_merge_detail(self._h, n_requests, n_ranks, _ptr(all_best), _ptr(out_decisions),
                                                     _ptr(out_detail)))

    def shard_select(self, n_requests, n_ranks, all_best, out_sel):
        """Seeded engines: all_best [n_ranks, R, S * 24] records -> out_sel [R, S * 8] bytes, this rank's entries
        (epp_shard_sel: the member it owns, else EPP_NO_ENDPOINT)."""
        self._check(self._lib.epp_shard_select(self._h, n_requests, n_ranks, _ptr(all_best), _ptr(out_sel)))

    def shard_finish(self, n_requests, n_ranks, all_best, all_sel, out_decisions, out_detail=None):
        """Seeded engines: the decisions from the records and every rank's entries ([n_ranks, R, S * 8], stacked in the
        order of all_best)."""
        self._check(self._lib.epp_shard_finish(self._h, n_requests, n_ranks, _ptr(all_best), _ptr(all_sel),
                                               _ptr(out_decisions), _ptr(out_detail)))


class Batcher:
    """The in-library micro-batcher (epp_submit / epp_wait): any number of threads submit single prompts and block for
    their decision; batches are formed and flushed inside libepp_engine.so (csrc/batcher.cu)."""

    def __init__(self, engine: Engine, max_batch: int = 256, max_delay_us: int = 200, index_picks: bool = False):
        self._lib = engine._lib
        self._engine = engine                      # keep the engine alive: the batcher must be destroyed first
        cfg = capi.BatcherCfg()
        cfg.struct_size = C.sizeof(capi.BatcherCfg)
        cfg.max_batch = max_batch
        cfg.max_delay_us = max_delay_us
        cfg.index_picks = int(index_picks)
        self._b = C.c_void_p()
        self._check(self._lib.epp_batcher_create(engine._h, C.byref(cfg), C.byref(self._b)))

    def _check(self, rc: int):
        if rc != 0:
            raise EngineError(rc, (self._lib.epp_batcher_last_error() or b"").decode())

    def submit(self, prompt, model_id: int = 0, multimodal: bool = False, subset=None, predictions=None,
               context_tokens=None, admission=None) -> int:
        """subset: None (the whole pool) or a sequence of slot ids, the request's candidates (epp_submit_subset).
        predictions: None or the request's entries in the form pack_predictions takes (epp_submit_predicted).  Both
        together: epp_submit_subset_predicted.  context_tokens: None, or the request's context length (-1 = the default);
        with it the request goes through epp_submit_ctx with whatever else it carries.  admission: None, or a dict with
        the request's "priority", "ttft_slo", "tpot_slo" and "pred_valid" (one byte per prediction, in the order given);
        with it the request goes through epp_submit_admit with whatever else it carries."""
        buf = np.ascontiguousarray(prompt).view(np.uint8).reshape(-1) if not isinstance(prompt, (bytes, bytearray)) else prompt
        n = len(buf)
        ptr = buf.ctypes.data_as(C.c_void_p) if isinstance(buf, np.ndarray) else C.cast(C.c_char_p(bytes(buf)), C.c_void_p)
        t = C.c_uint64()
        ent = None if predictions is None else _prediction_entries(predictions)
        n_ent = 0 if ent is None else ent.shape[0]
        if admission is not None:
            pv = admission.get("pred_valid")
            pv = None if pv is None else np.ascontiguousarray(np.asarray(pv, dtype=np.uint8).reshape(-1))
            if pv is not None and pv.shape[0] != n_ent:
                raise ValueError(f"{pv.shape[0]} validity bytes for {n_ent} predictions")
        sl = None if subset is None else np.ascontiguousarray(np.asarray(subset, dtype=np.uint32).reshape(-1))
        if sl is not None and sl.shape[0] == 0:
            sl = np.zeros(1, dtype=np.uint32)[:0]          # a non-NULL pointer: an empty subset, not the whole pool
        n_sl = 0 if sl is None else sl.shape[0]
        if admission is not None:
            rc = self._lib.epp_submit_admit(
                self._b, model_id, ptr, n, int(multimodal), n_sl, _ptr(sl), n_ent, _ptr(ent), _ptr(pv),
                -1 if context_tokens is None else int(context_tokens), int(admission.get("priority", 0)),
                float(admission.get("ttft_slo", 0.0)), float(admission.get("tpot_slo", 0.0)), C.byref(t))
        elif context_tokens is not None:
            rc = self._lib.epp_submit_ctx(self._b, model_id, ptr, n, int(multimodal), n_sl, _ptr(sl), n_ent, _ptr(ent),
                                          int(context_tokens), C.byref(t))
        elif ent is not None and sl is not None:
            rc = self._lib.epp_submit_subset_predicted(self._b, model_id, ptr, n, int(multimodal), n_sl, _ptr(sl), n_ent,
                                                       _ptr(ent), C.byref(t))
        elif ent is not None:
            rc = self._lib.epp_submit_predicted(self._b, model_id, ptr, n, int(multimodal), n_ent, _ptr(ent), C.byref(t))
        elif sl is not None:
            rc = self._lib.epp_submit_subset(self._b, model_id, ptr, n, int(multimodal), n_sl, _ptr(sl), C.byref(t))
        else:
            rc = self._lib.epp_submit(self._b, model_id, ptr, n, int(multimodal), C.byref(t))
        self._check(rc)
        return t.value

    def wait(self, ticket: int):
        """-> (decision, detail) as 1-element structured arrays."""
        d = capi.Decision()
        dd = capi.DecisionDetail()
        self._check(self._lib.epp_wait(self._b, ticket, C.byref(d), C.byref(dd)))
        dec = np.frombuffer(bytes(d), dtype=DECISION_DTYPE)[0]
        det = np.frombuffer(bytes(dd), dtype=DETAIL_DTYPE)[0]
        return dec, det

    def wait_topk(self, ticket: int):
        """-> (decision, detail, {"primary": [...], "prefill": [...], "encode": [...]}): the first-k lists of the
        request's profiles (engines created with pick_k > 1), EPP_NO_ENDPOINT entries dropped."""
        d = capi.Decision()
        dd = capi.DecisionDetail()
        k = int(self._engine.cfg.pick_k)
        rows = {name: np.zeros(max(k, 1), dtype=np.uint32) for name in ("primary", "prefill", "encode")}
        self._check(self._lib.epp_wait_topk(self._b, ticket, C.byref(d), C.byref(dd), _ptr(rows["primary"]),
                                            _ptr(rows["prefill"]), _ptr(rows["encode"])))
        lists = {n: [int(x) for x in r if int(x) != capi.EPP_NO_ENDPOINT] for n, r in rows.items()}
        return np.frombuffer(bytes(d), dtype=DECISION_DTYPE)[0], np.frombuffer(bytes(dd), dtype=DETAIL_DTYPE)[0], lists

    def schedule(self, prompt, model_id: int = 0, multimodal: bool = False):
        """Scheduler.Schedule for ONE request (what a goroutine of the reference calls): submit + wait."""
        return self.wait(self.submit(prompt, model_id, multimodal))

    def stats(self) -> dict:
        st = capi.BatcherStats()
        self._check(self._lib.epp_batcher_stats(self._b, C.byref(st)))
        return {k: getattr(st, k) for k, _ in capi.BatcherStats._fields_}

    def close(self):
        if getattr(self, "_b", None) and self._b.value:
            self._lib.epp_batcher_destroy(self._b)
            self._b = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PinnedBuffer:
    """Pinned host memory from epp_host_alloc as a numpy uint8 array (`.array`): what a shim stages prompts in.  Small
    batches whose prompts live in such memory take the engine's single-launch zero-copy path (csrc/cycle_small.cu)."""

    def __init__(self, nbytes: int):
        self._lib = capi.load()
        self._p = C.c_void_p()
        rc = self._lib.epp_host_alloc(max(int(nbytes), 1), C.byref(self._p))
        if rc != 0:
            raise EngineError(rc, (self._lib.epp_last_error() or b"").decode())
        self.array = np.ctypeslib.as_array(C.cast(self._p, C.POINTER(C.c_uint8)), shape=(max(int(nbytes), 1),))

    def close(self):
        if getattr(self, "_p", None) and self._p.value:
            self.array = None
            self._lib.epp_host_free(self._p)
            self._p = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def decisions_from_torch(t) -> np.ndarray:
    """View a [R, 32] uint8 CUDA tensor of epp_decision records as a host structured array."""
    return t.cpu().numpy().view(DECISION_DTYPE).reshape(-1)
