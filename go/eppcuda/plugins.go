package eppcuda

/*
#include "epp_engine.h"
*/
import "C"

import (
	"context"
	"encoding/json"
	"errors"
	"unsafe"

	fwkdl "github.com/llm-d/llm-d-router/pkg/epp/framework/interface/datalayer"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/plugin"
	fwkrc "github.com/llm-d/llm-d-router/pkg/epp/framework/interface/requestcontrol"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/scheduling"
	attrprefix "github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/datalayer/attribute/prefix"
)

// Plugin-parity mode: the engine behind the reference's per-plugin interfaces, one request per call (R = 1 batches
// through epp_prefix_match / epp_score).  Slower than Scheduler (no batching) -- it exists so that a deployment can
// replace ONE plugin (the prefix producer or a scorer) and keep the rest of its Go profile unchanged.
const (
	PrefixProducerType = "cuda-approx-prefix-cache-producer"
	WeightedScorerType = "cuda-weighted-scorer"
)

var shared *Engine // set by Register

// Register installs the factories (plugin.Register, registry.go:25-30).  Call it next to RegisterAllPlugins
// (cmd/epp/main.go:59) after the engine has been created.  It also replaces the factories of label-selector-filter,
// by-label-selector and by-label with ones whose plugins carry the engine's compiled requirements (labels.go).
func Register(e *Engine) {
	shared = e
	registerLabelFilters()
	registerLatencyPlugins()
	registerContextLengthPlugin()
	plugin.Register(PrefixProducerType, func(name string, _ json.RawMessage, _ plugin.Handle) (plugin.Plugin, error) {
		if shared == nil {
			return nil, errors.New("eppcuda: engine not created")
		}
		return &PrefixProducer{name: name, e: shared}, nil
	})
	plugin.Register(WeightedScorerType, func(name string, params json.RawMessage, _ plugin.Handle) (plugin.Plugin, error) {
		var p struct {
			Profile int `json:"profile"` // 0 primary, 1 prefill, 2 encode
			Scorer  int `json:"scorer"`  // index inside the profile, -1 = the ordered weighted sum
		}
		p.Scorer = -1
		if len(params) > 0 {
			if err := json.Unmarshal(params, &p); err != nil {
				return nil, err
			}
		}
		return &WeightedScorer{name: name, e: shared, profile: p.Profile, scorer: p.Scorer}, nil
	})
	plugin.Register(InFlightLoadProducerType, func(name string, _ json.RawMessage, _ plugin.Handle) (plugin.Plugin, error) {
		if shared == nil {
			return nil, errors.New("eppcuda: engine not created")
		}
		if !shared.cfg.InFlightLoad {
			return nil, errors.New("eppcuda: the engine was created without Config.InFlightLoad")
		}
		return &InFlightLoadProducer{name: name, e: shared}, nil
	})
}

// InFlightLoadProducerType is the reference's plugin type of the in-flight load producer
// (requestcontrol/dataproducer/inflightload/producer.go).
const InFlightLoadProducerType = "inflight-load-producer"

// inflightEntry is what Scheduler.Schedule stashes per request for the producer's release: the prefill target, the
// other targets (decode / primary, encode) and the prompt length the engine's token estimate was made from.
type inflightEntry struct {
	promptLen uint64
	prefill   uint32
	others    []uint32
}

// InFlightLoadProducer implements requestcontrol.ResponseBodyProcessor (plugins.go:62-65).  Its PreRequest runs inside
// the engine (every Schedule adds its targets' load on the device) and its endpoint-delete hook inside Engine.SetPool;
// ResponseBody releases the load the way producer.go:131-168 does: the prefill target at the first chunk, the others at
// the end of the stream.  The token estimate reads the prompt length, where the reference reads the request body size.
type InFlightLoadProducer struct {
	name string
	e    *Engine
}

var _ fwkrc.ResponseBodyProcessor = (*InFlightLoadProducer)(nil)

func (p *InFlightLoadProducer) TypedName() plugin.TypedName {
	return plugin.TypedName{Type: InFlightLoadProducerType, Name: p.name}
}

func (p *InFlightLoadProducer) ResponseBody(_ context.Context, request *scheduling.InferenceRequest, resp *fwkrc.Response,
	_ *fwkdl.EndpointMetadata) {
	if request == nil || resp == nil {
		return
	}
	v, ok := p.e.loads.Load(request)
	if !ok {
		return
	}
	ent := v.(inflightEntry)
	if resp.StartOfStream {
		_ = p.e.InFlightRelease([]uint32{ent.prefill}, ent.promptLen)
	}
	if resp.EndOfStream {
		p.e.loads.Delete(request)
		_ = p.e.InFlightRelease(ent.others, ent.promptLen)
	}
}

// TokenLoadScorer turns the parameters of a "token-load-scorer" entry (tokenload.Config: queueThresholdTokens, <= 0
// means 4194304) into the engine's scorer.  With Config.InFlightLoad it reads the engine's counters.
func TokenLoadScorer(weight float64, params json.RawMessage) (ScorerSpec, error) {
	var p struct {
		QueueThresholdTokens int64 `json:"queueThresholdTokens"`
	}
	if len(params) > 0 {
		if err := json.Unmarshal(params, &p); err != nil {
			return ScorerSpec{}, err
		}
	}
	return ScorerSpec{Kind: int(C.EPP_SCORER_TOKEN_LOAD), Weight: weight, Param: float64(p.QueueThresholdTokens)}, nil
}

// ActiveRequestScorer turns the parameters of an "active-request-scorer" entry (activerequest.Parameters: idleThreshold,
// maxBusyScore with default 1.0; requestTimeout is accepted and ignored, the producer's release ends a request) into the
// engine's scorer.  With Config.InFlightLoad it reads the engine's counters.
func ActiveRequestScorer(weight float64, params json.RawMessage) (ScorerSpec, error) {
	p := struct {
		RequestTimeout string  `json:"requestTimeout"`
		IdleThreshold  int     `json:"idleThreshold"`
		MaxBusyScore   float64 `json:"maxBusyScore"`
	}{MaxBusyScore: 1.0}
	if len(params) > 0 {
		if err := json.Unmarshal(params, &p); err != nil {
			return ScorerSpec{}, err
		}
	}
	return ScorerSpec{Kind: int(C.EPP_SCORER_ACTIVE_REQUEST), Weight: weight, Param: p.MaxBusyScore,
		Param2: float64(p.IdleThreshold)}, nil
}

// NoHitLRUType is the reference's plugin type of the no-hit-lru scorer (scorer/nohitlru/no_hit_lru.go).
const NoHitLRUType = "no-hit-lru-scorer"

// NoHitLRUScorer turns the parameters of a "no-hit-lru-scorer" entry (nohitlru.Parameters: lruSize, prefixPluginType,
// prefixPluginName) into the engine's scorer of the profile.  The prefix plugin names are accepted and ignored: the
// engine's own prefix match decides whether a request is cold.  lruSize <= 0 means 1024 (no_hit_lru.go:93-95); every
// profile that lists the scorer must use the same lruSize, because they share one LRU (epp_engine_create rejects others).
func NoHitLRUScorer(weight float64, params json.RawMessage) (ScorerSpec, error) {
	var p struct {
		LRUSize          int    `json:"lruSize"`
		PrefixPluginType string `json:"prefixPluginType"`
		PrefixPluginName string `json:"prefixPluginName"`
	}
	if len(params) > 0 {
		if err := json.Unmarshal(params, &p); err != nil {
			return ScorerSpec{}, err
		}
	}
	return ScorerSpec{Kind: int(C.EPP_SCORER_NO_HIT_LRU), Weight: weight, Param: float64(p.LRUSize)}, nil
}

// RandomPickerType and WeightedRandomPickerType are the reference's plugin types of the two random pickers
// (picker/random/picker.go, picker/weightedrandom/picker.go).
const (
	RandomPickerType         = "random-picker"
	WeightedRandomPickerType = "weighted-random-picker"
)

// pickerMaxEndpoints parses picker.PickerParameters (maxNumOfEndpoints); <= 0 means 1, as in the reference factories.
func pickerMaxEndpoints(params json.RawMessage) (int, error) {
	p := struct {
		MaxNumOfEndpoints int `json:"maxNumOfEndpoints"`
	}{MaxNumOfEndpoints: 1}
	if len(params) > 0 {
		if err := json.Unmarshal(params, &p); err != nil {
			return 0, err
		}
	}
	if p.MaxNumOfEndpoints <= 0 {
		p.MaxNumOfEndpoints = 1
	}
	return p.MaxNumOfEndpoints, nil
}

// RandomPicker turns a "random-picker" entry into the profile's picker kind and maxNumOfEndpoints (Config.PickK; the
// engine has one maxNumOfEndpoints for all profiles).
func RandomPicker(params json.RawMessage) (kind int, maxNumOfEndpoints int, err error) {
	k, err := pickerMaxEndpoints(params)
	return int(C.EPP_PICKER_RANDOM), k, err
}

// WeightedRandomPicker turns a "weighted-random-picker" entry into the profile's picker kind and maxNumOfEndpoints.
func WeightedRandomPicker(params json.RawMessage) (kind int, maxNumOfEndpoints int, err error) {
	k, err := pickerMaxEndpoints(params)
	return int(C.EPP_PICKER_WEIGHTED_RANDOM), k, err
}

// NoHitLRUKeys returns the slots of the scorer's LRU, oldest first (golang-lru Cache.Keys, epp_nohit_lru_get).
func (e *Engine) NoHitLRUKeys() ([]uint32, error) {
	out := make([]uint32, e.cfg.MaxEndpoints)
	var n C.int32_t
	if rc := C.epp_nohit_lru_get(e.h, (*C.uint32_t)(unsafe.Pointer(&out[0])), C.int32_t(len(out)), &n); rc != C.EPP_OK {
		return nil, lastError()
	}
	if int(n) < len(out) {
		out = out[:n]
	}
	return out, nil
}

// matchRow runs epp_prefix_match for one request: dense matchBlocks per slot + totalBlocks.
func (e *Engine) matchRow(model uint32, prompt []byte) ([]int32, int32, error) {
	match := make([]int32, e.cfg.MaxEndpoints)
	var total C.int32_t
	var b C.epp_batch
	b.n_requests = 1
	b.uniform_len = C.uint64_t(len(prompt))
	if len(prompt) > 0 {
		b.data = unsafe.Pointer(&prompt[0]) // Go memory without inner pointers, for the duration of the call
	}
	// model_ids stays NULL for model 0; other models go through a one-element C array
	var mid *C.uint32_t
	if model != 0 {
		mid = (*C.uint32_t)(C.malloc(4))
		defer C.free(unsafe.Pointer(mid))
		*mid = C.uint32_t(model)
		b.model_ids = mid
	}
	if rc := C.epp_prefix_match(e.h, &b, (*C.int32_t)(unsafe.Pointer(&match[0])), &total); rc != C.EPP_OK {
		return nil, 0, lastError()
	}
	return match, int32(total), nil
}

// PrefixProducer implements requestcontrol.DataProducer (plugins.go:69-72): it leaves a *PrefixCacheMatchInfo under
// PrefixCacheMatchInfoKey on every endpoint, like approximateprefix.Produce (plugin.go:135-160).
type PrefixProducer struct {
	name string
	e    *Engine
}

var _ fwkrc.DataProducer = (*PrefixProducer)(nil)

func (p *PrefixProducer) TypedName() plugin.TypedName {
	return plugin.TypedName{Type: PrefixProducerType, Name: p.name}
}

func (p *PrefixProducer) Produces() map[string]any {
	return map[string]any{attrprefix.PrefixCacheMatchInfoKey: attrprefix.PrefixCacheMatchInfo{}}
}

func (p *PrefixProducer) Produce(_ context.Context, request *scheduling.InferenceRequest, pods []scheduling.Endpoint) error {
	prompt, err := UserInputBytes(request)
	if err != nil {
		return err
	}
	model, err := p.e.modelID(request.TargetModel, "")
	if err != nil {
		return err
	}
	match, total, err := p.e.matchRow(model, prompt)
	if err != nil {
		return err
	}
	p.e.mu.RLock()
	defer p.e.mu.RUnlock()
	for _, ep := range pods {
		m := 0
		if slot, ok := p.e.slotOf[ep.GetMetadata().NamespacedName]; ok {
			m = int(match[slot])
		}
		ep.Put(attrprefix.PrefixCacheMatchInfoKey, attrprefix.NewPrefixCacheMatchInfo(m, int(total), p.e.cfg.BlockSizeTokens))
	}
	return nil
}

// WeightedScorer implements scheduling.Scorer (plugins.go:68-72) with epp_score on the match info a producer attached.
type WeightedScorer struct {
	name            string
	e               *Engine
	profile, scorer int
}

var _ scheduling.Scorer = (*WeightedScorer)(nil)

func (s *WeightedScorer) TypedName() plugin.TypedName {
	return plugin.TypedName{Type: WeightedScorerType, Name: s.name}
}
func (s *WeightedScorer) Category() scheduling.ScorerCategory { return scheduling.Balance }

func (s *WeightedScorer) Score(_ context.Context, _ *scheduling.CycleState, _ *scheduling.InferenceRequest,
	pods []scheduling.Endpoint) map[scheduling.Endpoint]float64 {
	out := make(map[scheduling.Endpoint]float64, len(pods))
	E := s.e.cfg.MaxEndpoints
	match := make([]int32, E)
	total := int32(0)
	s.e.mu.RLock()
	for _, ep := range pods {
		if v, ok := ep.Get(attrprefix.PrefixCacheMatchInfoKey); ok {
			if info, ok := v.(*attrprefix.PrefixCacheMatchInfo); ok {
				if slot, ok := s.e.slotOf[ep.GetMetadata().NamespacedName]; ok {
					match[slot] = int32(info.MatchBlocks())
					total = int32(info.TotalBlocks())
				}
			}
		}
	}
	s.e.mu.RUnlock()
	scores := make([]float64, E)
	if rc := C.epp_score(s.e.h, 1, (*C.int32_t)(unsafe.Pointer(&match[0])), (*C.int32_t)(unsafe.Pointer(&total)), nil,
		C.int32_t(s.profile), C.int32_t(s.scorer), (*C.double)(unsafe.Pointer(&scores[0])), 0); rc != C.EPP_OK {
		return out // a scorer cannot fail in the reference's interface: missing endpoints contribute 0
	}
	s.e.mu.RLock()
	defer s.e.mu.RUnlock()
	for _, ep := range pods {
		if slot, ok := s.e.slotOf[ep.GetMetadata().NamespacedName]; ok && scores[slot] >= 0 {
			out[ep] = scores[slot]
		}
	}
	return out
}
