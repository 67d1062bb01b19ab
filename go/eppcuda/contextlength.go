package eppcuda

/*
#include <stdlib.h>
#include "epp_engine.h"
*/
import "C"

import (
	"context"
	"encoding/json"
	"errors"
	"fmt"
	"unsafe"

	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/plugin"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/scheduling"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/scheduling/scorer/contextlengthaware"
)

// Context length (include/epp_engine.h "Context length"): the context-length-aware scorer and filter decided by the
// engine from each endpoint's range label and each request's context length.

// ContextLengthSpec mirrors epp_context_length_set: the range label key and whether the plugin also filters.
type ContextLengthSpec struct {
	Label           string
	EnableFiltering bool
}

// ContextLengthAware is the context-length-aware plugin of a profile the engine runs.  Filter and Score are the
// reference's own (for a profile the Go scheduler runs); the engine reads Spec.
type ContextLengthAware struct {
	Spec ContextLengthSpec
	ref  plugin.Plugin
}

func (p *ContextLengthAware) TypedName() plugin.TypedName       { return p.ref.TypedName() }
func (p *ContextLengthAware) Category() scheduling.ScorerCategory { return scheduling.Affinity }
func (p *ContextLengthAware) Filter(ctx context.Context, cs *scheduling.CycleState, r *scheduling.InferenceRequest,
	eps []scheduling.Endpoint) []scheduling.Endpoint {
	return p.ref.(scheduling.Filter).Filter(ctx, cs, r, eps)
}
func (p *ContextLengthAware) Score(ctx context.Context, cs *scheduling.CycleState, r *scheduling.InferenceRequest,
	eps []scheduling.Endpoint) map[scheduling.Endpoint]float64 {
	return p.ref.(scheduling.Scorer).Score(ctx, cs, r, eps)
}

// registerContextLengthPlugin replaces the factory.  It builds the reference's plugin first, so parameters are validated
// with the reference's errors, then unmarshals the same parameters over the same defaults.
func registerContextLengthPlugin() {
	plugin.Register(contextlengthaware.ContextLengthAwareType, func(name string, raw json.RawMessage, h plugin.Handle) (plugin.Plugin, error) {
		ref, err := contextlengthaware.Factory(name, raw, h)
		if err != nil {
			return nil, err
		}
		params := struct {
			Label           string `json:"label"`
			EnableFiltering bool   `json:"enableFiltering"`
		}{Label: contextlengthaware.DefaultContextLengthLabel}
		if raw != nil {
			if err := json.Unmarshal(raw, &params); err != nil {
				return nil, fmt.Errorf("failed to parse the parameters of the '%s' plugin - %w", contextlengthaware.ContextLengthAwareType, err)
			}
		}
		return &ContextLengthAware{Spec: ContextLengthSpec{Label: params.Label, EnableFiltering: params.EnableFiltering}, ref: ref}, nil
	})
}

// ContextLengthPlacement takes a profile's context-length-aware filter stages out of its chain: AddPlugins
// (scheduler_profile.go:76-95) places a weighted instance both among the scorers and among the filters.  A filtering
// instance is a per-endpoint predicate of the first stage, so it may not follow an affinity or tier filter; one instance
// per profile.  rest is the chain for ProfilePlacement; spec is nil without an instance.
func ContextLengthPlacement(stages []ChainStage) (spec *ContextLengthSpec, rest []ChainStage, err error) {
	gate := false
	for _, s := range stages {
		switch {
		case s.ContextLength != nil:
			if spec != nil {
				return nil, nil, errors.New("eppcuda: at most one context-length-aware instance per profile")
			}
			if gate && s.ContextLength.Spec.EnableFiltering {
				return nil, nil, errors.New("eppcuda: a filtering context-length-aware comes before the affinity and tier filters")
			}
			sp := s.ContextLength.Spec
			spec = &sp
		case s.Tier != nil || s.Affinity != nil:
			gate = true
			rest = append(rest, s)
		default:
			rest = append(rest, s)
		}
	}
	return spec, rest, nil
}

// ContextLength restates getContextLength (context_length_aware.go): the token count of TokenizedPrompt when it has
// tokens, else int(float64(chars) * 0.25) over the chat messages' and the completions prompt's raw text.
func ContextLength(r *scheduling.InferenceRequest) int64 {
	if r == nil || r.Body == nil {
		return 0
	}
	if tp := r.Body.TokenizedPrompt; tp != nil && len(tp.TokenIDs) > 0 {
		return int64(len(tp.TokenIDs))
	}
	chars := 0
	if r.Body.ChatCompletions != nil {
		for _, m := range r.Body.ChatCompletions.Messages {
			chars += len(m.Content.Raw)
		}
	}
	if r.Body.Completions != nil {
		chars += len(r.Body.Completions.Prompt.Raw)
	}
	return int64(int(float64(chars) * 0.25))
}

func (e *Engine) setContextLength(profile int, p *ProfileSpec) error {
	if p.ContextLength == nil {
		return nil
	}
	label := C.CString(p.ContextLength.Label)
	defer C.free(unsafe.Pointer(label))
	filt := C.int32_t(0)
	if p.ContextLength.EnableFiltering {
		filt = 1
	}
	if rc := C.epp_context_length_set(e.h, C.int32_t(profile), label, filt); rc != C.EPP_OK {
		return fmt.Errorf("eppcuda: epp_context_length_set: %w", lastError())
	}
	e.ctxLen = true
	e.keys[p.ContextLength.Label] = true // SetPool sends every pod's range label
	return nil
}

// scheduleCtx = schedule with everything a request may carry (epp_submit_ctx): its subset (nil: the whole pool), its
// predictions (latency engines) and its context length.
func (e *Engine) scheduleCtx(model uint32, prompt []byte, multimodal bool, slots []uint32, pred []C.epp_prediction,
	ctxTokens int64) (Decision, error) {
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
		var empty C.uint32_t
		if slots != nil {
			sp = &empty // an empty subset is not the whole pool
			if len(slots) > 0 {
				sp = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
			}
		}
		var pp *C.epp_prediction
		if len(pred) > 0 {
			pp = &pred[0]
		}
		return C.epp_submit_ctx(e.b, C.uint32_t(model), p, C.uint64_t(len(prompt)), mm, C.uint32_t(len(slots)), sp,
			C.uint32_t(len(pred)), pp, C.int64_t(ctxTokens), ticket)
	})
}
