// Package eppcuda binds libepp_engine.so (include/epp_engine.h, C ABI v5) into the llm-d EPP and implements the
// reference's own interfaces on top of it:
//
//	requestcontrol.Scheduler    pkg/epp/requestcontrol/director.go:69-71          -> Scheduler (scheduler.go)
//	requestcontrol.DataProducer pkg/epp/framework/interface/requestcontrol/plugins.go:69-72 -> PrefixProducer (plugins.go)
//	scheduling.Scorer           pkg/epp/framework/interface/scheduling/plugins.go:68-72     -> WeightedScorer (plugins.go)
//	plugin.Register factories   pkg/epp/framework/interface/plugin/registry.go:25-30        -> Register (plugins.go)
//
// The batching that the per-request Go API needs lives INSIDE the library (epp_submit / epp_wait, csrc/batcher.cu): a
// goroutine calls Schedule for one request and blocks for its decision; this package contains no batching logic.
//
// cgo pointer rules: every buffer handed to C is either C memory (C.malloc / epp_host_alloc) or a Go slice WITHOUT
// inner Go pointers passed for the duration of one call; no C struct ever holds a Go pointer.
//
// This package cannot be compiled in the build container (no Go toolchain, no network; the reference itself is
// CGO_ENABLED=0).  It is written against the reference at 520af478 and kept small so that a maintainer can vet it by
// reading: every exported method is a handful of lines around one C call.
package eppcuda

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../llm-d-inference-scheduler_b200 -lepp_engine
#include <stdlib.h>
#include "epp_engine.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"sync"
	"unsafe"

	"k8s.io/apimachinery/pkg/types"

	fwkdl "github.com/llm-d/llm-d-router/pkg/epp/framework/interface/datalayer"
)

// ScorerSpec mirrors epp_scorer_cfg (one WeightedScorer of a SchedulerProfile, in profile order).
type ScorerSpec struct {
	Kind   int // C.EPP_SCORER_*
	Weight float64
	Param  float64
	Column int
	Param2 float64
}

// AffinitySpec mirrors the prefix-cache-affinity-filter parameters (filter/prefixcacheaffinity/plugin.go:45-66).
type AffinitySpec struct {
	AffinityThreshold      float64
	ExplorationProbability float64
	MaxTTFTPenaltyMs       float64
	TTFTColumn             int // ext column carrying LatencyPredictionInfo.TTFT; -1 = attribute absent
}

// ProfileSpec mirrors epp_profile_cfg: role filter and label filters -> [prefix-cache-affinity-filter] -> scorers in
// order -> picker.
type ProfileSpec struct {
	Filter   int // C.EPP_FILTER_*
	Scorers  []ScorerSpec
	Affinity *AffinitySpec
	Picker   int // C.EPP_PICKER_* (0 = max-score-picker); see RandomPicker / WeightedRandomPicker
	// Labels: the requirements of the profile's label filters (ProfileLabels of its LabelFilter plugins, labels.go),
	// all ANDed with Filter; epp_label_filters_set
	Labels []LabelReq
	// Latency: the profile's tier filter, first affinity filter and latency-scorer (ProfilePlacement, latency.go);
	// epp_latency_profile_set.  nil: none.
	Latency *LatencySpec
	// ContextLength: the profile's context-length-aware plugin (ContextLengthPlacement, contextlength.go); it must also
	// be listed in Scorers as C.EPP_SCORER_CONTEXT_LENGTH with its weight.  epp_context_length_set.  nil: none.
	ContextLength *ContextLengthSpec
}

// Config mirrors epp_config (EndpointPickerConfig fields that define this path).
type Config struct {
	Device               int
	MaxEndpoints         int
	BlockSizeTokens      int
	MaxPrefixBlocks      int
	LRUCapacityPerServer int
	NonCachedTokens      int64
	AlwaysDisagg         bool
	TieSeed              uint64 // 0 = lowest slot of the arg-max set (tests); production: any non-zero value
	PickK                int    // max-score-picker maxNumOfEndpoints; <= 1: one target endpoint per profile
	IndexCommitMicros    int    // picks become visible to later requests at most this much later (0 = before the next batch)
	Primary              ProfileSpec
	Prefill              *ProfileSpec // non-nil: disagg handler (decode -> decider -> prefill)
	Encode               *ProfileSpec // non-nil (with Prefill): encode stage for multimodal requests
	MaxBatch             int          // micro-batcher: requests per flush at most
	MaxDelayMicros       int          // ... and how long the oldest request of a batch may wait
	// InFlightLoad runs the inflight-load-producer on the device: every Schedule adds its targets' load, the
	// InFlightLoadProducer (plugins.go) releases it, and the token-load / active-request scorers read it (Column ignored)
	InFlightLoad bool
}

// Engine owns one epp_engine + its micro-batcher and the endpoint-name <-> slot-id table.
type Engine struct {
	h   *C.epp_engine
	b   *C.epp_batcher
	cfg Config

	mu     sync.RWMutex
	latency bool // some profile has a latency piece: Scheduler.Schedule passes each request's predictions
	ctxLen  bool // some profile has the context-length-aware plugin: Scheduler.Schedule passes each request's context length
	slotOf map[types.NamespacedName]uint32
	nameOf []types.NamespacedName // by slot; zero value = free
	free   []uint32
	models map[string]uint32 // TargetModel (+ cache salt) -> epp_model_register id
	keys   map[string]bool   // label keys some profile's label filter references (SetPool sends only these)

	inflight sync.WaitGroup // Schedule calls inside epp_submit / epp_wait (Close waits for them)
	loads    sync.Map       // *scheduling.InferenceRequest -> inflightEntry, with Config.InFlightLoad (plugins.go)
}

func lastError() error { return errors.New(C.GoString(C.epp_last_error())) }

func fillProfile(dst *C.epp_profile_cfg, p ProfileSpec) error {
	if len(p.Scorers) > C.EPP_MAX_SCORERS {
		return fmt.Errorf("eppcuda: %d scorers in one profile (max %d)", len(p.Scorers), C.EPP_MAX_SCORERS)
	}
	dst.filter = C.int32_t(p.Filter)
	dst.n_scorers = C.int32_t(len(p.Scorers))
	for i, s := range p.Scorers {
		dst.scorers[i].kind = C.int32_t(s.Kind)
		dst.scorers[i].column = C.int32_t(s.Column)
		dst.scorers[i].weight = C.double(s.Weight)
		dst.scorers[i].param = C.double(s.Param)
		dst.scorers[i].param2 = C.double(s.Param2)
	}
	dst.ttft_column = -1
	dst.picker = C.int32_t(p.Picker)
	if a := p.Affinity; a != nil {
		dst.affinity_threshold = C.double(a.AffinityThreshold)
		dst.exploration_probability = C.double(a.ExplorationProbability)
		dst.max_ttft_penalty_ms = C.double(a.MaxTTFTPenaltyMs)
		dst.ttft_column = C.int32_t(a.TTFTColumn)
	}
	return nil
}

// New creates the engine on cfg.Device and starts its micro-batcher.  There is no CPU fallback: without a usable CUDA
// device this returns the library's EPP_ERR_NO_DEVICE message.
func New(cfg Config) (*Engine, error) {
	var c C.epp_config
	C.epp_config_default(&c)
	c.device = C.int32_t(cfg.Device)
	c.max_endpoints = C.int32_t(cfg.MaxEndpoints)
	if cfg.BlockSizeTokens > 0 {
		c.block_size_tokens = C.int32_t(cfg.BlockSizeTokens)
	}
	if cfg.MaxPrefixBlocks > 0 {
		c.max_prefix_blocks = C.int32_t(cfg.MaxPrefixBlocks)
	}
	if cfg.LRUCapacityPerServer > 0 {
		c.lru_capacity_per_server = C.int32_t(cfg.LRUCapacityPerServer)
	}
	c.non_cached_tokens = C.int64_t(cfg.NonCachedTokens)
	if cfg.AlwaysDisagg {
		c.always_disagg = 1
	}
	c.tie_seed = C.uint64_t(cfg.TieSeed)
	if cfg.PickK > 1 {
		c.pick_k = C.int32_t(cfg.PickK)
	}
	c.index_commit_interval_us = C.int32_t(cfg.IndexCommitMicros)
	if cfg.InFlightLoad {
		c.inflight_load = 1
	}
	if err := fillProfile(&c.primary, cfg.Primary); err != nil {
		return nil, err
	}
	if cfg.Prefill != nil {
		c.handler = C.EPP_HANDLER_DISAGG
		if err := fillProfile(&c.prefill, *cfg.Prefill); err != nil {
			return nil, err
		}
		if cfg.Encode != nil {
			c.encode_enabled = 1
			if err := fillProfile(&c.encode, *cfg.Encode); err != nil {
				return nil, err
			}
		}
	}
	e := &Engine{cfg: cfg, slotOf: map[types.NamespacedName]uint32{}, models: map[string]uint32{},
		nameOf: make([]types.NamespacedName, cfg.MaxEndpoints), keys: labelKeys(cfg)}
	for s := cfg.MaxEndpoints - 1; s >= 0; s-- {
		e.free = append(e.free, uint32(s))
	}
	if rc := C.epp_engine_create(&c, &e.h); rc != C.EPP_OK {
		return nil, fmt.Errorf("eppcuda: epp_engine_create: %w", lastError())
	}
	for i, p := range []*ProfileSpec{&cfg.Primary, cfg.Prefill, cfg.Encode} {
		if p == nil || (i == 2 && cfg.Prefill == nil) {
			continue
		}
		if err := e.setLabelFilters(i, p.Labels); err != nil {
			C.epp_engine_destroy(e.h)
			return nil, err
		}
		if err := e.setLatency(i, p); err != nil {
			C.epp_engine_destroy(e.h)
			return nil, err
		}
		if err := e.setContextLength(i, p); err != nil {
			C.epp_engine_destroy(e.h)
			return nil, err
		}
	}
	var bc C.epp_batcher_cfg
	bc.struct_size = C.uint32_t(unsafe.Sizeof(bc))
	bc.max_batch = C.int32_t(max(1, cfg.MaxBatch))
	bc.max_delay_us = C.int32_t(cfg.MaxDelayMicros)
	bc.index_picks = 1 // PreRequest of the approximate-prefix producer, applied between flushes on the device
	if rc := C.epp_batcher_create(e.h, &bc, &e.b); rc != C.EPP_OK {
		err := errors.New(C.GoString(C.epp_batcher_last_error()))
		C.epp_engine_destroy(e.h)
		return nil, fmt.Errorf("eppcuda: epp_batcher_create: %w", err)
	}
	return e, nil
}

// Close waits for the Schedule calls in flight, then stops the batcher (which flushes what is pending) and only then
// destroys the engine.
func (e *Engine) Close() {
	e.inflight.Wait()
	if e.b != nil {
		C.epp_batcher_destroy(e.b)
		e.b = nil
	}
	if e.h != nil {
		C.epp_engine_destroy(e.h)
		e.h = nil
	}
}

// modelID registers TargetModel || cacheSalt once (hashing.go:71-78: the seed of the hash chain) and returns its id.
func (e *Engine) modelID(model, salt string) (uint32, error) {
	key := model + "\x00" + salt
	e.mu.RLock()
	id, ok := e.models[key]
	e.mu.RUnlock()
	if ok {
		return id, nil
	}
	e.mu.Lock()
	defer e.mu.Unlock()
	if id, ok = e.models[key]; ok {
		return id, nil
	}
	var out C.uint32_t
	mb, sb := []byte(model), []byte(salt)
	var mp, sp *C.uint8_t
	if len(mb) > 0 {
		mp = (*C.uint8_t)(unsafe.Pointer(&mb[0]))
	}
	if len(sb) > 0 {
		sp = (*C.uint8_t)(unsafe.Pointer(&sb[0]))
	}
	if rc := C.epp_model_register(e.h, mp, C.size_t(len(mb)), sp, C.size_t(len(sb)), &out); rc != C.EPP_OK {
		return 0, fmt.Errorf("eppcuda: epp_model_register: %w", lastError())
	}
	e.models[key] = uint32(out)
	return uint32(out), nil
}

// roleOf maps the llm-d.ai/role label (filter/bylabel/roles.go:10-44) to epp_role.
func roleOf(labels map[string]string) C.uint8_t {
	v, ok := labels["llm-d.ai/role"]
	if !ok {
		return C.EPP_ROLE_NONE
	}
	switch v {
	case "decode":
		return C.EPP_ROLE_DECODE
	case "prefill":
		return C.EPP_ROLE_PREFILL
	case "prefill-decode":
		return C.EPP_ROLE_PREFILL_DECODE
	case "both":
		return C.EPP_ROLE_BOTH
	case "encode":
		return C.EPP_ROLE_ENCODE
	case "encode-prefill":
		return C.EPP_ROLE_ENCODE_PREFILL
	case "encode-prefill-decode":
		return C.EPP_ROLE_ENCODE_PREFILL_DECODE
	}
	return C.EPP_ROLE_OTHER
}

// SetPool replaces the pool-state snapshot (called by the 50 ms scrape loop with Datastore.PodList()).  Endpoints
// that left the pool lose their slot: their index entries are removed ON THE DEVICE before the slot can be handed
// to another endpoint (RemovePod, indexer.go:167-182), both under the same lock.  With InFlightLoad their in-flight
// counters are reset there too (the producer's endpoint-delete event, producer.go:86-97).
func (e *Engine) SetPool(pods []fwkdl.Endpoint) error {
	e.mu.Lock()
	defer e.mu.Unlock()
	seen := make(map[types.NamespacedName]bool, len(pods))
	for _, p := range pods {
		seen[p.GetMetadata().NamespacedName] = true
	}
	for name, slot := range e.slotOf {
		if !seen[name] {
			if rc := C.epp_index_remove_endpoint(e.h, C.uint32_t(slot)); rc != C.EPP_OK {
				return fmt.Errorf("eppcuda: epp_index_remove_endpoint: %w", lastError())
			}
			if e.cfg.InFlightLoad {
				s := C.uint32_t(slot)
				if rc := C.epp_inflight_reset(e.h, 1, &s); rc != C.EPP_OK {
					return fmt.Errorf("eppcuda: epp_inflight_reset: %w", lastError())
				}
			}
			delete(e.slotOf, name)
			e.nameOf[slot] = types.NamespacedName{}
			e.free = append(e.free, slot)
		}
	}
	n := len(pods)
	if n == 0 {
		C.epp_pool_set(e.h, 0, nil, nil, nil, nil, nil, nil)
		if len(e.keys) > 0 {
			C.epp_pool_set_labels(e.h, 0, nil, nil, nil)
		}
		return nil
	}
	var text []byte
	offsets := make([]C.uint64_t, n+1)
	ids := make([]C.uint32_t, n)
	role := make([]C.uint8_t, n)
	kv := make([]C.double, n)
	waiting := make([]C.int32_t, n)
	running := make([]C.int32_t, n)
	for i, p := range pods {
		name := p.GetMetadata().NamespacedName
		slot, ok := e.slotOf[name]
		if !ok {
			if len(e.free) == 0 {
				return fmt.Errorf("eppcuda: pool has more than %d endpoints", e.cfg.MaxEndpoints)
			}
			slot = e.free[len(e.free)-1]
			e.free = e.free[:len(e.free)-1]
			e.slotOf[name] = slot
			e.nameOf[slot] = name
		}
		m := p.GetMetrics()
		ids[i] = C.uint32_t(slot)
		role[i] = roleOf(p.GetMetadata().Labels)
		if len(e.keys) > 0 {
			var err error
			if text, err = appendLabels(text, p.GetMetadata().Labels, e.keys); err != nil {
				return err
			}
			offsets[i+1] = C.uint64_t(len(text))
		}
		kv[i] = C.double(m.KVCacheUsagePercent)
		waiting[i] = C.int32_t(m.WaitingQueueSize)
		running[i] = C.int32_t(m.RunningRequestsSize)
	}
	if rc := C.epp_pool_set(e.h, C.int32_t(n), &ids[0], &role[0], &kv[0], &waiting[0], &running[0], nil); rc != C.EPP_OK {
		return fmt.Errorf("eppcuda: epp_pool_set: %w", lastError())
	}
	if len(e.keys) > 0 {
		return e.setPoolLabels(ids, text, offsets)
	}
	return nil
}

// Decision is epp_decision + epp_decision_detail with slots resolved by the caller.
type Decision struct {
	Status                          int32
	Pick, PrefillPick, EncodePick   uint32
	Score                           float64
	TieCount                        uint32
	MatchBlocks, TotalBlocks        int32
	PrefillRan, EncodeRan           bool
	// PickK > 1: the first-k slots of each profile in picker order (maxscore/picker.go:104-115); nil otherwise
	Primary, Prefill, Encode []uint32
}

const NoEndpoint = uint32(C.EPP_NO_ENDPOINT)

// InFlightRelease takes one request and the token estimate of a promptLen-byte prompt off each slot
// (epp_inflight_release: ResponseBody of the inflight-load-producer).  NoEndpoint entries are skipped.  No CUDA call.
func (e *Engine) InFlightRelease(slots []uint32, promptLen uint64) error {
	if len(slots) == 0 {
		return nil
	}
	lens := make([]C.uint64_t, len(slots))
	for i := range lens {
		lens[i] = C.uint64_t(promptLen)
	}
	if rc := C.epp_inflight_release(e.h, C.int32_t(len(slots)), (*C.uint32_t)(unsafe.Pointer(&slots[0])), &lens[0]); rc != C.EPP_OK {
		return fmt.Errorf("eppcuda: epp_inflight_release: %w", lastError())
	}
	return nil
}

// schedule = epp_submit + epp_wait for ONE request.  prompt is read during the submit call only (the library copies
// the bytes it hashes into its pinned staging buffer).
func (e *Engine) schedule(model uint32, prompt []byte, multimodal bool) (Decision, error) {
	return e.scheduleSubset(model, prompt, multimodal, nil)
}

// scheduleSubset = schedule for a request whose candidates are the endpoints of `slots` (sorted; the gateway's endpoint
// subset, epp_submit_subset), or the whole pool when slots is nil.  At most C.EPP_SUBSET_MAX_SLOTS slots.
func (e *Engine) scheduleSubset(model uint32, prompt []byte, multimodal bool, slots []uint32) (Decision, error) {
	return e.submitAndWait(func(ticket *C.uint64_t) C.int32_t {
		var p unsafe.Pointer
		if len(prompt) > 0 {
			p = unsafe.Pointer(&prompt[0])
		}
		mm := C.uint32_t(0)
		if multimodal {
			mm = 1
		}
		if slots == nil {
			return C.epp_submit(e.b, C.uint32_t(model), p, C.uint64_t(len(prompt)), mm, ticket)
		}
		var sp *C.uint32_t
		if len(slots) > 0 {
			sp = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
		}
		return C.epp_submit_subset(e.b, C.uint32_t(model), p, C.uint64_t(len(prompt)), mm, C.uint32_t(len(slots)), sp, ticket)
	})
}

// submitAndWait runs one submit call of the batcher, then waits for the request's decision.
func (e *Engine) submitAndWait(submit func(ticket *C.uint64_t) C.int32_t) (Decision, error) {
	e.inflight.Add(1)
	defer e.inflight.Done()
	var ticket C.uint64_t
	if rc := submit(&ticket); rc != C.EPP_OK {
		return Decision{}, errors.New(C.GoString(C.epp_batcher_last_error()))
	}
	var d C.epp_decision
	var dd C.epp_decision_detail
	var lists [3][]uint32
	if k := e.cfg.PickK; k > 1 {
		buf := make([]C.uint32_t, 3*k) // plain integers: a Go allocation without Go pointers may be passed to C
		if rc := C.epp_wait_topk(e.b, ticket, &d, &dd, &buf[0], &buf[k], &buf[2*k]); rc != C.EPP_OK {
			return Decision{}, errors.New(C.GoString(C.epp_batcher_last_error()))
		}
		for q := 0; q < 3; q++ {
			for j := 0; j < k && uint32(buf[q*k+j]) != NoEndpoint; j++ {
				lists[q] = append(lists[q], uint32(buf[q*k+j]))
			}
		}
	} else if rc := C.epp_wait(e.b, ticket, &d, &dd); rc != C.EPP_OK {
		return Decision{}, errors.New(C.GoString(C.epp_batcher_last_error()))
	}
	return Decision{Status: int32(d.status), Pick: uint32(d.pick), PrefillPick: uint32(d.prefill_pick),
		EncodePick: uint32(dd.encode_pick), Score: float64(d.score), TieCount: uint32(d.tie_count),
		MatchBlocks: int32(d.match_blocks), TotalBlocks: int32(d.total_blocks), PrefillRan: dd.prefill_ran != 0,
		EncodeRan: dd.encode_ran != 0, Primary: lists[0], Prefill: lists[1], Encode: lists[2]}, nil
}
