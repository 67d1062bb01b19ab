package eppcuda

/*
#include <stdlib.h>
#include "epp_engine.h"
*/
import "C"

import (
	"encoding/json"
	"fmt"
	"strings"
	"unsafe"

	metav1 "k8s.io/apimachinery/pkg/apis/meta/v1"
	"k8s.io/apimachinery/pkg/selection"

	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/plugin"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/interface/scheduling"
	"github.com/llm-d/llm-d-router/pkg/epp/framework/plugins/scheduling/filter/bylabel"
)

// Label filters (include/epp_engine.h "Label filters"): label-selector-filter, its deprecated alias by-label-selector,
// and by-label.  Each is built by the reference's own factory, so it validates exactly as the reference does, and is
// compiled through metav1.LabelSelectorAsSelector(...).Requirements() into the engine's requirements.  A profile lists
// them in ProfileSpec.Labels (all ANDed with its role filter, before the affinity filter); SetPool sends every pod's
// labels through epp_pool_set_labels when some profile has one.

// LabelReq mirrors epp_label_req: Op is C.EPP_LABEL_*.
type LabelReq struct {
	Key    string
	Op     int
	Values []string
}

// LabelFilter is a registered label filter: the reference's filter (scheduling.Filter, used as is by a Go profile in
// plugin-parity mode) and its compiled requirements (ProfileSpec.Labels, decided by the engine).
type LabelFilter struct {
	scheduling.Filter
	Reqs []LabelReq
}

var _ scheduling.Filter = (*LabelFilter)(nil)

// selectorReqs compiles a metav1.LabelSelector: matchLabels k: v is k In [v]; an empty selector has no requirement.
// A nil selector is labels.Nothing(): two requirements no endpoint meets together.
func selectorReqs(ls *metav1.LabelSelector) ([]LabelReq, error) {
	sel, err := metav1.LabelSelectorAsSelector(ls)
	if err != nil {
		return nil, err
	}
	rs, selectable := sel.Requirements()
	if !selectable {
		return nothingReqs("llm-d.ai/role"), nil
	}
	out := make([]LabelReq, 0, len(rs))
	for _, r := range rs {
		q := LabelReq{Key: r.Key(), Values: r.ValuesUnsorted()}
		switch r.Operator() {
		case selection.In, selection.Equals, selection.DoubleEquals:
			q.Op = int(C.EPP_LABEL_IN)
		case selection.NotIn, selection.NotEquals:
			q.Op = int(C.EPP_LABEL_NOT_IN)
		case selection.Exists:
			q.Op, q.Values = int(C.EPP_LABEL_EXISTS), nil
		case selection.DoesNotExist:
			q.Op, q.Values = int(C.EPP_LABEL_DOES_NOT_EXIST), nil
		default:
			return nil, fmt.Errorf("eppcuda: label selector operator %q is not supported", r.Operator())
		}
		out = append(out, q)
	}
	return out, nil
}

// nothingReqs keeps no endpoint: Exists and DoesNotExist on the same key.
func nothingReqs(key string) []LabelReq {
	return []LabelReq{{Key: key, Op: int(C.EPP_LABEL_EXISTS)}, {Key: key, Op: int(C.EPP_LABEL_DOES_NOT_EXIST)}}
}

func selectorFilter(name string, raw json.RawMessage, deprecated bool) (plugin.Plugin, error) {
	var p plugin.Plugin
	var err error
	if deprecated {
		p, err = bylabel.DeprecatedSelectorFactory(name, raw, nil) //nolint:staticcheck // the registered alias
	} else {
		p, err = bylabel.SelectorFactory(name, raw, nil)
	}
	if err != nil {
		return nil, err
	}
	ls := metav1.LabelSelector{}
	if raw != nil {
		if err := json.Unmarshal(raw, &ls); err != nil {
			return nil, err
		}
	}
	reqs, err := selectorReqs(&ls)
	if err != nil {
		return nil, err
	}
	return &LabelFilter{Filter: p.(scheduling.Filter), Reqs: reqs}, nil
}

// LabelSelectorFilterFactory is the factory of "label-selector-filter" (selector.go:34-42).
func LabelSelectorFilterFactory(name string, raw json.RawMessage, _ plugin.Handle) (plugin.Plugin, error) {
	return selectorFilter(name, raw, false)
}

// DeprecatedSelectorFactory is the factory of "by-label-selector" (selector.go:44-60).
func DeprecatedSelectorFactory(name string, raw json.RawMessage, _ plugin.Handle) (plugin.Plugin, error) {
	return selectorFilter(name, raw, true)
}

// ByLabelFactory is the factory of "by-label" (filter.go:34-57): label absent and allowsNoLabel, or labels[label]
// among validValues, where an absent label reads "".
func ByLabelFactory(name string, raw json.RawMessage, _ plugin.Handle) (plugin.Plugin, error) {
	p, err := bylabel.Factory(name, raw, nil) //nolint:staticcheck // the registered deprecated type
	if err != nil {
		return nil, err
	}
	var q struct {
		Label         string   `json:"label"`
		ValidValues   []string `json:"validValues"`
		AllowsNoLabel bool     `json:"allowsNoLabel"`
	}
	if raw != nil {
		if err := json.Unmarshal(raw, &q); err != nil {
			return nil, err
		}
	}
	op := C.EPP_LABEL_BY_LABEL
	if q.AllowsNoLabel {
		op = C.EPP_LABEL_BY_LABEL_OR_ABSENT
	}
	return &LabelFilter{Filter: p.(scheduling.Filter),
		Reqs: []LabelReq{{Key: q.Label, Op: int(op), Values: q.ValidValues}}}, nil
}

// registerLabelFilters replaces the reference's factories of the three types (register.go:24-27) with ones whose
// plugins also carry the compiled requirements.
func registerLabelFilters() {
	plugin.Register(bylabel.LabelSelectorFilterType, LabelSelectorFilterFactory)
	plugin.Register(bylabel.ByLabelSelectorType, DeprecatedSelectorFactory)
	plugin.Register(bylabel.ByLabelType, ByLabelFactory)
}

// ProfileLabels collects the requirements of a profile's label filters, in any order (they are ANDed).
func ProfileLabels(filters ...scheduling.Filter) []LabelReq {
	var out []LabelReq
	for _, f := range filters {
		if lf, ok := f.(*LabelFilter); ok {
			out = append(out, lf.Reqs...)
		}
	}
	return out
}

// setLabelFilters is epp_label_filters_set for one profile.  Every string and array is C memory, freed on return.
func (e *Engine) setLabelFilters(profile int, reqs []LabelReq) error {
	if len(reqs) == 0 {
		return nil
	}
	var toFree []unsafe.Pointer
	defer func() {
		for _, p := range toFree {
			C.free(p)
		}
	}()
	cstr := func(s string) *C.char {
		p := C.CString(s)
		toFree = append(toFree, unsafe.Pointer(p))
		return p
	}
	arr := (*[1 << 20]C.epp_label_req)(C.malloc(C.size_t(len(reqs)) * C.size_t(unsafe.Sizeof(C.epp_label_req{}))))
	toFree = append(toFree, unsafe.Pointer(arr))
	for i, q := range reqs {
		arr[i].key = cstr(q.Key)
		arr[i].op = C.int32_t(q.Op)
		arr[i].n_values = C.int32_t(len(q.Values))
		arr[i].values = nil
		if len(q.Values) > 0 {
			vs := (*[1 << 20]*C.char)(C.malloc(C.size_t(len(q.Values)) * C.size_t(unsafe.Sizeof((*C.char)(nil)))))
			toFree = append(toFree, unsafe.Pointer(vs))
			for j, v := range q.Values {
				vs[j] = cstr(v)
			}
			arr[i].values = &vs[0]
		}
	}
	if rc := C.epp_label_filters_set(e.h, C.int32_t(profile), C.int32_t(len(reqs)), &arr[0]); rc != C.EPP_OK {
		return fmt.Errorf("eppcuda: epp_label_filters_set(profile %d): %w", profile, lastError())
	}
	return nil
}

// labelKeys is the set of keys some profile's requirement references: only those are sent to the engine.
func labelKeys(cfg Config) map[string]bool {
	keys := map[string]bool{}
	for _, p := range []*ProfileSpec{&cfg.Primary, cfg.Prefill, cfg.Encode} {
		if p == nil {
			continue
		}
		for _, q := range p.Labels {
			keys[q.Key] = true
		}
	}
	return keys
}

// appendLabels appends a pod's referenced labels as "key=value\n" lines (epp_pool_set_labels).
func appendLabels(text []byte, labels map[string]string, keys map[string]bool) ([]byte, error) {
	for k, v := range labels {
		if !keys[k] {
			continue
		}
		if strings.ContainsAny(k, "=\n") || strings.Contains(v, "\n") {
			return nil, fmt.Errorf("eppcuda: label %q holds '=' or a newline", k)
		}
		text = append(text, k...)
		text = append(text, '=')
		text = append(text, v...)
		text = append(text, '\n')
	}
	return text, nil
}

// setPoolLabels is epp_pool_set_labels over the slots of one SetPool call.  text and offsets are Go memory without
// inner pointers, passed for the duration of the call.
func (e *Engine) setPoolLabels(ids []C.uint32_t, text []byte, offsets []C.uint64_t) error {
	if len(text) == 0 {
		text = []byte{0} // a valid pointer for an all-empty label set
	}
	if rc := C.epp_pool_set_labels(e.h, C.int32_t(len(ids)), &ids[0], &offsets[0], (*C.uint8_t)(unsafe.Pointer(&text[0]))); rc != C.EPP_OK {
		return fmt.Errorf("eppcuda: epp_pool_set_labels: %w", lastError())
	}
	return nil
}
