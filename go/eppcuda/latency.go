package eppcuda

/*
#include "epp_engine.h"
*/
import "C"

import (
	"context"
	"encoding/json"
	"errors"
	"fmt"
	"sort"
	"unsafe"

	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/plugin"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/scheduling"
	attrlatency "github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/datalayer/attribute/latency"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/scheduling/filter/sloheadroomtier"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/scheduling/scorer/latency"
)

// Latency predictions (include/epp_engine.h "Latency predictions"): the slo-headroom-tier-filter and the latency-scorer
// decided by the engine from each request's LatencyPredictionInfo on its candidates.

// LatencySpec mirrors epp_latency_cfg: the tier filter, the affinity filter placed before it (A1) and the latency
// scorer's configuration.  The affinity filter after the tier filter (A2) is ProfileSpec.Affinity.
type LatencySpec struct {
	Tier   *sloheadroomtier.Config // nil: no tier filter
	A1     *AffinitySpec           // needs Tier
	Scorer *latency.Config         // the latency-scorer's configuration (nil: the reference's DefaultConfig)
}

// TierFilter is the slo-headroom-tier-filter as a plugin of a profile the engine runs.  Its Filter is the reference's
// own (for a profile the Go scheduler runs); the engine reads Config.
type TierFilter struct {
	Config sloheadroomtier.Config
	ref    plugin.Plugin
}

func (f *TierFilter) TypedName() plugin.TypedName { return f.ref.TypedName() }
func (f *TierFilter) Filter(ctx context.Context, cs *scheduling.CycleState, r *scheduling.InferenceRequest,
	eps []scheduling.Endpoint) []scheduling.Endpoint {
	return f.ref.(scheduling.Filter).Filter(ctx, cs, r, eps)
}

// LatencyScorer is the latency-scorer as a plugin of a profile the engine runs (Score is the reference's own).
type LatencyScorer struct {
	Config latency.Config
	ref    plugin.Plugin
}

func (s *LatencyScorer) TypedName() plugin.TypedName       { return s.ref.TypedName() }
func (s *LatencyScorer) Category() scheduling.ScorerCategory { return scheduling.Balance }
func (s *LatencyScorer) Score(ctx context.Context, cs *scheduling.CycleState, r *scheduling.InferenceRequest,
	eps []scheduling.Endpoint) map[scheduling.Endpoint]float64 {
	return s.ref.(scheduling.Scorer).Score(ctx, cs, r, eps)
}

// registerLatencyPlugins replaces both factories.  Each builds the reference's plugin first, so parameters are
// validated with the reference's errors, then unmarshals the same parameters into the exported Config.
func registerLatencyPlugins() {
	plugin.Register(sloheadroomtier.PluginType, func(name string, raw json.RawMessage, h plugin.Handle) (plugin.Plugin, error) {
		ref, err := sloheadroomtier.Factory(name, raw, h)
		if err != nil {
			return nil, err
		}
		cfg := sloheadroomtier.DefaultConfig
		if len(raw) > 0 {
			if err := json.Unmarshal(raw, &cfg); err != nil {
				return nil, fmt.Errorf("failed to unmarshal config: %w", err)
			}
		}
		return &TierFilter{Config: cfg, ref: ref}, nil
	})
	plugin.Register(latency.LatencyScorerType, func(name string, raw json.RawMessage, h plugin.Handle) (plugin.Plugin, error) {
		ref, err := latency.Factory(name, raw, h)
		if err != nil {
			return nil, err
		}
		cfg := latency.DefaultConfig
		if len(raw) > 0 {
			if err := json.Unmarshal(raw, &cfg); err != nil {
				return nil, fmt.Errorf("failed to unmarshal config: %w", err)
			}
		}
		return &LatencyScorer{Config: cfg, ref: ref}, nil
	})
}

// ChainStage is one filter of a profile in order, as ProfilePlacement reads it: a TierFilter, an affinity filter (its
// AffinitySpec) or anything else (role and label filters, which may only come first).
type ChainStage struct {
	Tier          *TierFilter
	Affinity      *AffinitySpec
	ContextLength *ContextLengthAware // taken out of the chain by ContextLengthPlacement first
}

// ProfilePlacement places a profile's affinity and tier filters on the engine's chain
// [role + labels] -> [A1] -> [T] -> [A2]: it returns ProfileSpec.Affinity (A2, or the only affinity filter) and the
// LatencySpec's Tier and A1.  Without a tier filter the chain is today's: at most one affinity filter, and it comes last.
func ProfilePlacement(stages []ChainStage) (a2 *AffinitySpec, lat *LatencySpec, err error) {
	tier := -1
	var affs []int
	for i, s := range stages {
		switch {
		case s.Tier != nil:
			if tier >= 0 {
				return nil, nil, errors.New("eppcuda: at most one slo-headroom-tier-filter per profile")
			}
			tier = i
		case s.Affinity != nil:
			affs = append(affs, i)
		default:
			if tier >= 0 || len(affs) > 0 {
				return nil, nil, errors.New("eppcuda: role and label filters come before the affinity and tier filters")
			}
		}
	}
	if tier < 0 {
		if len(affs) > 1 || (len(affs) == 1 && affs[0] != len(stages)-1) {
			return nil, nil, errors.New("eppcuda: the prefix-cache-affinity-filter comes last")
		}
		if len(affs) == 1 {
			a2 = stages[affs[0]].Affinity
		}
		return a2, nil, nil
	}
	cfg := stages[tier].Tier.Config
	lat = &LatencySpec{Tier: &cfg}
	for _, i := range affs {
		switch {
		case i == tier-1:
			lat.A1 = stages[i].Affinity
		case i == tier+1 && i == len(stages)-1:
			a2 = stages[i].Affinity
		default:
			return nil, nil, errors.New("eppcuda: an affinity filter goes right before or right after the slo-headroom-tier-filter, and nothing follows the one after it")
		}
	}
	if tier != len(stages)-1 && a2 == nil {
		return nil, nil, errors.New("eppcuda: only one prefix-cache-affinity-filter may follow the slo-headroom-tier-filter")
	}
	return a2, lat, nil
}

func (e *Engine) setLatency(profile int, p *ProfileSpec) error {
	if p.Latency == nil {
		return nil
	}
	var c C.epp_latency_cfg
	C.epp_latency_cfg_default(&c)
	if t := p.Latency.Tier; t != nil {
		c.tier_filter = 1
		c.epsilon_explore_neg = C.double(t.EpsilonExploreNeg)
	}
	if a := p.Latency.A1; a != nil {
		c.a1_affinity_threshold = C.double(a.AffinityThreshold)
		c.a1_exploration_probability = C.double(a.ExplorationProbability)
		c.a1_max_ttft_penalty_ms = C.double(a.MaxTTFTPenaltyMs)
	}
	if s := p.Latency.Scorer; s != nil {
		c.ttft_weight = C.double(s.TTFTWeight)
		c.tpot_weight = C.double(s.TPOTWeight)
		c.strategy = C.EPP_HEADROOM_LEAST
		if s.HeadroomSelectionStrategy == latency.StrategyMost { // any other value: the switch's default, "least"
			c.strategy = C.EPP_HEADROOM_MOST
		}
		c.composite_kv_weight = C.double(s.CompositeKVWeight)
		c.composite_queue_weight = C.double(s.CompositeQueueWeight)
		c.composite_prefix_weight = C.double(s.CompositePrefixWeight)
	}
	if rc := C.epp_latency_profile_set(e.h, C.int32_t(profile), &c); rc != C.EPP_OK {
		return fmt.Errorf("eppcuda: epp_latency_profile_set: %w", lastError())
	}
	e.latency = true
	return nil
}

// predictions packs each candidate's LatencyPredictionInfo into the engine's entries (the batcher sorts them).
// Candidates without the attribute, or without a slot, have no entry.
func (e *Engine) predictions(candidates []scheduling.Endpoint) []C.epp_prediction {
	var out []C.epp_prediction
	e.mu.RLock()
	defer e.mu.RUnlock()
	for _, ep := range candidates {
		raw, ok := ep.Get(attrlatency.LatencyPredictionInfoKey)
		if !ok {
			continue
		}
		info, ok := raw.(*attrlatency.LatencyPredictionInfo)
		if !ok || info == nil {
			continue
		}
		slot, ok := e.slotOf[ep.GetMetadata().NamespacedName]
		if !ok {
			continue
		}
		out = append(out, C.epp_prediction{slot: C.uint32_t(slot), dispatched: C.int32_t(info.DispatchedRequestCount()),
			ttft: C.double(info.TTFT()), ttft_headroom: C.double(info.TTFTHeadroom()),
			tpot_headroom: C.double(info.TPOTHeadroom())})
	}
	sort.Slice(out, func(i, j int) bool { return out[i].slot < out[j].slot })
	return out
}

// schedulePredicted = schedule with the request's predictions (epp_submit_predicted).
func (e *Engine) schedulePredicted(model uint32, prompt []byte, multimodal bool, pred []C.epp_prediction) (Decision, error) {
	if len(pred) > int(C.EPP_PRED_MAX_SLOTS) {
		return Decision{}, fmt.Errorf("eppcuda: %d predictions, more than EPP_PRED_MAX_SLOTS", len(pred))
	}
	return e.submitAndWait(func(ticket *C.uint64_t) C.int32_t {
		var p unsafe.Pointer
		if len(prompt) > 0 {
			p = unsafe.Pointer(&prompt[0])
		}
		mm := C.uint32_t(0)
		if multimodal {
			mm = 1
		}
		var pp *C.epp_prediction
		if len(pred) > 0 {
			pp = &pred[0]
		}
		return C.epp_submit_predicted(e.b, C.uint32_t(model), p, C.uint64_t(len(prompt)), mm, C.uint32_t(len(pred)), pp, ticket)
	})
}

// scheduleSubsetPredicted = schedulePredicted for a request whose candidates are the endpoints of `slots` (sorted, at
// most C.EPP_SUBSET_MAX_SLOTS), with the predictions of those candidates (epp_submit_subset_predicted).
func (e *Engine) scheduleSubsetPredicted(model uint32, prompt []byte, multimodal bool, slots []uint32,
	pred []C.epp_prediction) (Decision, error) {
	if len(pred) > int(C.EPP_PRED_MAX_SLOTS) {
		return Decision{}, fmt.Errorf("eppcuda: %d predictions, more than EPP_PRED_MAX_SLOTS", len(pred))
	}
	return e.submitAndWait(func(ticket *C.uint64_t) C.int32_t {
		var p unsafe.Pointer
		if len(prompt) > 0 {
			p = unsafe.Pointer(&prompt[0])
		}
		mm := C.uint32_t(0)
		if multimodal {
			mm = 1
		}
		var sp *C.uint32_t
		if len(slots) > 0 {
			sp = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
		}
		var pp *C.epp_prediction
		if len(pred) > 0 {
			pp = &pred[0]
		}
		return C.epp_submit_subset_predicted(e.b, C.uint32_t(model), p, C.uint64_t(len(prompt)), mm, C.uint32_t(len(slots)),
			sp, C.uint32_t(len(pred)), pp, ticket)
	})
}
