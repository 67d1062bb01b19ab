package eppcuda

import (
	"context"
	"errors"

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
	Fallback requestcontrol.Scheduler // the reference scheduler: used when the director passes a SUBSET of the pool
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
	// the engine scores its whole pool snapshot; a director-side subset (candidates.Locate with subsetting metadata)
	// is the reference scheduler's job
	s.Engine.mu.RLock()
	whole := len(byName) == len(s.Engine.slotOf)
	s.Engine.mu.RUnlock()
	if !whole {
		if s.Fallback != nil {
			return s.Fallback.Schedule(ctx, request, candidates)
		}
		return nil, errors.New("eppcuda: candidate list is not the engine's pool snapshot and no fallback scheduler is set")
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
	d, err := s.Engine.schedule(model, prompt, mm)
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
