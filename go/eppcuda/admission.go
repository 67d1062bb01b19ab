package eppcuda

/*
#include <stdlib.h>
#include "epp_engine.h"
*/
import "C"

import (
	"context"
	"errors"
	"sort"
	"strconv"
	"sync"
	"unsafe"

	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/scheduling"
	attrlatency "github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/datalayer/attribute/latency"
)

// Admission (include/epp_engine.h "Admission"): the latency-slo-admitter and the probabilistic-admitter decided by the
// engine after its picks, so a rejected request leaves no in-flight adds, no-hit-lru Adds or indexed picks behind.

// AdmissionSpec mirrors epp_admission_cfg; zero thresholds take the reference's defaults.
type AdmissionSpec struct {
	LatencySLO, Probabilistic bool
	QueueDepthThreshold       int
	KVCacheUtilThreshold      float64
	Power, K                  float64
}

// SetAdmission applies the admitters (before the first SetPool).
func (e *Engine) SetAdmission(spec AdmissionSpec) error {
	var cfg C.epp_admission_cfg
	C.epp_admission_cfg_default(&cfg)
	if spec.LatencySLO {
		cfg.latency_slo = 1
	}
	if spec.Probabilistic {
		cfg.probabilistic = 1
	}
	if spec.QueueDepthThreshold != 0 {
		cfg.queue_depth_threshold = C.int32_t(spec.QueueDepthThreshold)
	}
	if spec.KVCacheUtilThreshold != 0 {
		cfg.kv_cache_util_threshold = C.double(spec.KVCacheUtilThreshold)
	}
	if spec.Power != 0 {
		cfg.power = C.double(spec.Power)
	}
	if spec.K != 0 {
		cfg.k = C.double(spec.K)
	}
	if rc := C.epp_admission_set(e.h, &cfg); rc != C.EPP_OK {
		return errors.New(C.GoString(C.epp_last_error()))
	}
	return nil
}

// Admitter is a requestcontrol.Admitter backed by the engine.  AdmitRequest submits the request with its admission
// inputs and waits: a rejected request returns the error; an admitted one keeps its decision for the Schedule call the
// director makes next for the same request (Scheduler.Schedule takes it from there).
type Admitter struct {
	S       *Scheduler
	decided sync.Map // *scheduling.InferenceRequest -> Decision
}

// parseFloatHeaderValue (latencyslo/plugin.go:150-158).
func parseFloatHeaderValue(s string) float64 {
	if s == "" {
		return 0
	}
	v, err := strconv.ParseFloat(s, 64)
	if err != nil {
		return 0
	}
	return v
}

// AdmitRequest of requestcontrol.Admitter.
func (a *Admitter) AdmitRequest(ctx context.Context, request *scheduling.InferenceRequest, endpoints []scheduling.Endpoint) error {
	if request == nil {
		return nil
	}
	e := a.S.Engine
	prompt, err := UserInputBytes(request)
	if err != nil {
		return err
	}
	salt := ""
	if request.Body != nil {
		salt = request.Body.CacheSalt()
	}
	model, err := e.modelID(request.TargetModel, salt)
	if err != nil {
		return err
	}
	e.mu.RLock()
	var slots []uint32
	for _, ep := range endpoints {
		if slot, ok := e.slotOf[ep.GetMetadata().NamespacedName]; ok {
			slots = append(slots, slot)
		}
	}
	whole := len(slots) == len(e.slotOf)
	e.mu.RUnlock()
	if whole {
		slots = nil
	} else {
		sort.Slice(slots, func(i, j int) bool { return slots[i] < slots[j] })
		if slots == nil {
			slots = []uint32{}
		}
	}
	pred, valid := e.predictionsWithValidity(endpoints)
	var ctxTokens int64 = -1
	if e.ctxLen {
		ctxTokens = ContextLength(request)
	}
	mm := HasMultimodalContent != nil && HasMultimodalContent(request)
	d, err := e.submitAndWait(func(ticket *C.uint64_t) C.int32_t {
		var p unsafe.Pointer
		if len(prompt) > 0 {
			p = unsafe.Pointer(&prompt[0])
		}
		m := C.uint32_t(0)
		if mm {
			m = 1
		}
		var sp *C.uint32_t
		var empty C.uint32_t
		if slots != nil {
			sp = &empty
			if len(slots) > 0 {
				sp = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
			}
		}
		var pp *C.epp_prediction
		var vp *C.uint8_t
		if len(pred) > 0 {
			pp = &pred[0]
			vp = (*C.uint8_t)(unsafe.Pointer(&valid[0]))
		}
		return C.epp_submit_admit(e.b, C.uint32_t(model), p, C.uint64_t(len(prompt)), m, C.uint32_t(len(slots)), sp,
			C.uint32_t(len(pred)), pp, vp, C.int64_t(ctxTokens), C.int32_t(request.Objectives.Priority),
			C.double(parseFloatHeaderValue(request.Headers["x-slo-ttft-ms"])),
			C.double(parseFloatHeaderValue(request.Headers["x-slo-tpot-ms"])), ticket)
	})
	if err != nil {
		return err
	}
	if d.Status == C.EPP_STATUS_REJECTED {
		return errors.New("no valid endpoint available to serve the request")
	}
	a.decided.Store(request, d)
	return nil
}

// take returns (and forgets) the decision AdmitRequest made for the request.
func (a *Admitter) take(request *scheduling.InferenceRequest) (Decision, bool) {
	v, ok := a.decided.LoadAndDelete(request)
	if !ok {
		return Decision{}, false
	}
	return v.(Decision), true
}

// predictionsWithValidity is predictions plus each entry's validity byte (bit 0 TTFTValid, bit 1 TPOTValid), in the
// same (slot) order.
func (e *Engine) predictionsWithValidity(candidates []scheduling.Endpoint) ([]C.epp_prediction, []uint8) {
	type pv struct {
		p C.epp_prediction
		v uint8
	}
	var all []pv
	e.mu.RLock()
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
		var v uint8
		if info.IsValid() {
			v = 3
		}
		all = append(all, pv{C.epp_prediction{slot: C.uint32_t(slot), dispatched: C.int32_t(info.DispatchedRequestCount()),
			ttft: C.double(info.TTFT()), ttft_headroom: C.double(info.TTFTHeadroom()),
			tpot_headroom: C.double(info.TPOTHeadroom())}, v})
	}
	e.mu.RUnlock()
	sort.Slice(all, func(i, j int) bool { return all[i].p.slot < all[j].p.slot })
	pred := make([]C.epp_prediction, len(all))
	valid := make([]uint8, len(all))
	for i, x := range all {
		pred[i], valid[i] = x.p, x.v
	}
	return pred, valid
}
