package eppcuda

// #include "epp_engine.h"
import "C"

import (
	"context"
	"errors"
	"sort"

	"k8s.io/apimachinery/pkg/types"

	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/scheduling"
	"github.com/llm-d/llm-d-router/pkg/epp/requestcontrol"
)

// The two request-side helpers of the reference that this path needs are unexported there:
//   getUserInputBytes     approximateprefix/hashing.go:107-136   (the bytes hashPrompt hashes)
//   hasMultimodalContent  profilehandler/disagg/multimodal_helpers.go:8-22 (input of the encode decider)
// The integration exports them (a one-line wrapper each, see INTEGRATION.md) and wires them here.
var (
	UserInputBytes       func(*scheduling.InferenceRequest) ([]byte, error)
	HasMultimodalContent func(*scheduling.InferenceRequest) bool
)

// Profile names of the SchedulingResult (the disagg handler's defaults, disagg_profile_handler.go:27-40).
type ProfileNames struct{ Primary, Prefill, Encode string }

// Scheduler implements requestcontrol.Scheduler (director.go:69-71) on the engine.  It is injected where the
// reference builds its scheduler (cmd/epp/runner/runner.go:336, 376).
type Scheduler struct {
	Engine   *Engine
	Names    ProfileNames
	// the reference scheduler: used only for a candidate the engine has no slot for (not in its pool snapshot yet), or a
	// subset of more than EPP_SUBSET_MAX_SLOTS endpoints
	Fallback requestcontrol.Scheduler
	// the engine-backed admitters (admission.go), or nil: Schedule then uses the decision AdmitRequest kept
	Admitter *Admitter
}

var _ requestcontrol.Scheduler = (*Scheduler)(nil)

// Schedule: one request in, one SchedulingResult out (scheduling/scheduler.go:54-102 with the single or disagg profile
// handler).  Errors map like the reference's: no decode endpoint -> "failed to find available decode workers"
// (disagg_profile_handler.go:335-338), which the director turns into ResourceExhausted (director.go:245).
func (s *Scheduler) Schedule(ctx context.Context, request *scheduling.InferenceRequest,
	candidates []scheduling.Endpoint) (*scheduling.SchedulingResult, error) {
	if request == nil {
		return nil, errors.New("request is nil")
	}
	byName := make(map[types.NamespacedName]scheduling.Endpoint, len(candidates))
	for _, ep := range candidates {
		byName[ep.GetMetadata().NamespacedName] = ep
	}
	if len(byName) == 0 { // an empty subset decides nothing (the director answers ServiceUnavailable before this)
		return nil, errors.New("failed to find available decode workers")
	}
	// A director-side subset (candidates.Locate with x-gateway-destination-endpoint-subset metadata, director.go:222-243)
	// goes to the engine as the sorted slots of the candidates (epp_submit_subset, or epp_submit_subset_predicted on a
	// latency engine); the whole pool as no subset.
	s.Engine.mu.RLock()
	slots := make([]uint32, 0, len(byName)) // non-nil: no candidates is an empty subset (status -1), never the whole pool
	known := true
	for name := range byName {
		slot, ok := s.Engine.slotOf[name]
		if !ok {
			known = false
			break
		}
		slots = append(slots, slot)
	}
	whole := known && len(slots) == len(s.Engine.slotOf)
	s.Engine.mu.RUnlock()
	// a candidate the snapshot does not know, or a subset too large for the batcher's staging: the fallback scheduler
	if !known || (!whole && len(slots) > int(C.EPP_SUBSET_MAX_SLOTS)) {
		if s.Fallback != nil {
			return s.Fallback.Schedule(ctx, request, candidates)
		}
		return nil, errors.New("eppcuda: a candidate is not in the engine's pool snapshot (or the subset is too large) and no fallback scheduler is set")
	}
	if whole {
		slots = nil
	} else {
		sort.Slice(slots, func(i, j int) bool { return slots[i] < slots[j] })
	}
	prompt, err := UserInputBytes(request)
	if err != nil {
		return nil, err
	}
	salt := ""
	if request.Body != nil {
		salt = request.Body.CacheSalt()
	}
	model, err := s.Engine.modelID(request.TargetModel, salt)
	if err != nil {
		return nil, err
	}
	mm := HasMultimodalContent != nil && HasMultimodalContent(request)
	var d Decision
	admitted := false
	if s.Admitter != nil { // the decision the engine made when it admitted the request (admission.go)
		d, admitted = s.Admitter.take(request)
	}
	if admitted {
	} else if s.Engine.ctxLen {
		var pred []C.epp_prediction
		if s.Engine.latency {
			pred = s.Engine.predictions(candidates)
		}
		d, err = s.Engine.scheduleCtx(model, prompt, mm, slots, pred, ContextLength(request))
	} else if s.Engine.latency && slots == nil {
		d, err = s.Engine.schedulePredicted(model, prompt, mm, s.Engine.predictions(candidates))
	} else if s.Engine.latency {
		d, err = s.Engine.scheduleSubsetPredicted(model, prompt, mm, slots, s.Engine.predictions(candidates))
	} else {
		d, err = s.Engine.scheduleSubset(model, prompt, mm, slots)
	}
	if err != nil {
		return nil, err
	}
	if d.Status != 0 {
		return nil, errors.New("failed to find available decode workers")
	}
	res := &scheduling.SchedulingResult{PrimaryProfileName: s.Names.Primary,
		ProfileResults: map[string]*scheduling.ProfileRunResult{}}
	// TargetEndpoints: the pick, or with maxNumOfEndpoints > 1 the first-k list in picker order (the pick first)
	put := func(profile string, pick uint32, list []uint32) {
		if profile == "" || pick == NoEndpoint {
			return
		}
		if list == nil {
			list = []uint32{pick}
		}
		var targets []scheduling.Endpoint
		s.Engine.mu.RLock()
		for _, slot := range list {
			if ep, ok := byName[s.Engine.nameOf[slot]]; ok {
				targets = append(targets, ep)
			} else if slot == pick {
				targets = nil // the pick left the pool since the snapshot
				break
			}
		}
		s.Engine.mu.RUnlock()
		if len(targets) > 0 {
			res.ProfileResults[profile] = &scheduling.ProfileRunResult{TargetEndpoints: targets}
		}
	}
	put(s.Names.Primary, d.Pick, d.Primary)
	put(s.Names.Prefill, d.PrefillPick, d.Prefill)
	put(s.Names.Encode, d.EncodePick, d.Encode)
	if s.Engine.cfg.InFlightLoad {
		// the engine already added the load of every target (PreRequest); the InFlightLoadProducer releases these
		// slots when the response comes back
		s.Engine.loads.Store(request, inflightEntry{promptLen: uint64(len(prompt)), prefill: d.PrefillPick,
			others: []uint32{d.Pick, d.EncodePick}})
	}
	if _, ok := res.ProfileResults[s.Names.Primary]; !ok {
		return nil, errors.New("failed to find available decode workers") // the pick left the pool since the snapshot
	}
	return res, nil
}
