// K2History: the V2 analyzer's k2 priority chain (computeK2, internal/engines/analyzers/saturation_v2/analyzer.go:218-262)
// with its rolling history kept on the device (wva_k2_resolve, include/wva_b200.h).  COMPILE-UNVERIFIED like the rest of
// this package.  The caller lives inside package saturation_v2: it keeps the name -> id maps (modelIDs as history groups,
// accelerator names with "" as an id, namespace|model|variant store slots), calls Resolve once per cycle, applies the
// capacity store Updates once per slot from SlotLastRep / SlotEffective, and keeps FindCompatible and the zero-replica
// fallback on the host.
package wvab200

/*
#include "wva_b200.h"
*/
import "C"

type K2History struct {
	ctx    *Ctx
	h      *C.wva_k2_history
	nSlots int
	nKeys  int
}

// NewK2History registers hgModelOff [H+1] / hgModels [G] (history group -> model groups in visiting order),
// hgAccOff [H+1] / hgAcc (history group -> distinct accelerator ids) and the number of store slots.
func (x *Ctx) NewK2History(hgModelOff, hgModels, hgAccOff, hgAcc []int32, nSlots int) (*K2History, error) {
	var h *C.wva_k2_history
	rc := C.wva_k2_history_create(x.c, C.int64_t(len(hgModelOff)-1), C.int64_t(len(hgModels)), C.int64_t(nSlots),
		(*C.int32_t)(ptrOrNil(hgModelOff)), (*C.int32_t)(ptrOrNil(hgModels)), (*C.int32_t)(ptrOrNil(hgAccOff)),
		(*C.int32_t)(ptrOrNil(hgAcc)), &h)
	if err := x.err(rc, "wva_k2_history_create"); err != nil {
		return nil, err
	}
	return &K2History{ctx: x, h: h, nSlots: nSlots, nKeys: int(C.wva_k2_history_keys(h))}, nil
}

func (k *K2History) Close() { C.wva_k2_history_destroy(k.h) }

// K2Cycle is one cycle's input in wva_k2_in order; OutPos may be nil.
type K2Cycle struct {
	ModelReplicaOff                              []int32
	TotalKvTokens, TokensInUse, QueueLength      []int64
	AvgInputTokens, AvgOutputTokens              []float64
	Accelerator, Slot, OutPos                    []int32
	NOut                                         int
	SlotMaxBatchedTokens, SlotMaxNumSeqs         []int64
	QueueLengthThreshold, KvCacheThreshold       []float64
}

// K2Result: RepK2 in slice order (-1 without capacity data), OutRepK2 scattered to OutPos (the rep_k2 column of the
// wva_saturation_v2_in layout), and per store slot the last data replica of the cycle (-1 = none) and its capacity.
type K2Result struct {
	RepK2, RepEffective, OutRepK2 []int64
	SlotLastRep                   []int32
	SlotEffective                 []int64
}

func (k *K2History) Resolve(c *K2Cycle) (*K2Result, error) {
	P := len(c.TotalKvTokens)
	r := &K2Result{RepK2: make([]int64, P), RepEffective: make([]int64, P), SlotLastRep: make([]int32, k.nSlots),
		SlotEffective: make([]int64, k.nSlots)}
	in := C.wva_k2_in{n_model_groups: C.int64_t(len(c.ModelReplicaOff) - 1), n_replicas: C.int64_t(P),
		model_replica_off: (*C.int32_t)(ptrOrNil(c.ModelReplicaOff)),
		rep_total_kv_tokens: (*C.int64_t)(ptrOrNil(c.TotalKvTokens)), rep_tokens_in_use: (*C.int64_t)(ptrOrNil(c.TokensInUse)),
		rep_queue_length: (*C.int64_t)(ptrOrNil(c.QueueLength)), rep_avg_input_tokens: (*C.double)(ptrOrNil(c.AvgInputTokens)),
		rep_avg_output_tokens: (*C.double)(ptrOrNil(c.AvgOutputTokens)), rep_accelerator: (*C.int32_t)(ptrOrNil(c.Accelerator)),
		rep_slot: (*C.int32_t)(ptrOrNil(c.Slot)), rep_out_pos: (*C.int32_t)(ptrOrNil(c.OutPos)), n_out: C.int64_t(c.NOut),
		slot_max_batched_tokens: (*C.int64_t)(ptrOrNil(c.SlotMaxBatchedTokens)), slot_max_num_seqs: (*C.int64_t)(ptrOrNil(c.SlotMaxNumSeqs)),
		cfg_queue_threshold: (*C.double)(ptrOrNil(c.QueueLengthThreshold)), cfg_kv_threshold: (*C.double)(ptrOrNil(c.KvCacheThreshold))}
	out := C.wva_k2_out{rep_k2: (*C.int64_t)(ptrOrNil(r.RepK2)), rep_effective: (*C.int64_t)(ptrOrNil(r.RepEffective)),
		slot_last_rep: (*C.int32_t)(ptrOrNil(r.SlotLastRep)), slot_effective: (*C.int64_t)(ptrOrNil(r.SlotEffective))}
	if c.OutPos != nil {
		r.OutRepK2 = make([]int64, c.NOut)
		out.out_rep_k2 = (*C.int64_t)(ptrOrNil(r.OutRepK2))
	}
	if err := k.ctx.err(C.wva_k2_resolve(k.h, &in, &out), "wva_k2_resolve"); err != nil {
		return nil, err
	}
	return r, nil
}

// K2Keys is the export / import format: per key history group, accelerator id, bucket (0 short, 1 medium, 2 long),
// count and 10 values oldest first.
type K2Keys struct {
	HG, Acc, Bucket, Count []int32
	Values                 []float64
}

func (k *K2History) Export() (*K2Keys, error) {
	n := k.nKeys
	e := &K2Keys{HG: make([]int32, n), Acc: make([]int32, n), Bucket: make([]int32, n), Count: make([]int32, n),
		Values: make([]float64, n*10)}
	rc := C.wva_k2_history_export(k.h, (*C.int32_t)(ptrOrNil(e.HG)), (*C.int32_t)(ptrOrNil(e.Acc)),
		(*C.int32_t)(ptrOrNil(e.Bucket)), (*C.int32_t)(ptrOrNil(e.Count)), (*C.double)(ptrOrNil(e.Values)))
	return e, k.ctx.err(rc, "wva_k2_history_export")
}

func (k *K2History) Import(e *K2Keys) error {
	rc := C.wva_k2_history_import(k.h, C.int64_t(len(e.HG)), (*C.int32_t)(ptrOrNil(e.HG)), (*C.int32_t)(ptrOrNil(e.Acc)),
		(*C.int32_t)(ptrOrNil(e.Bucket)), (*C.int32_t)(ptrOrNil(e.Count)), (*C.double)(ptrOrNil(e.Values)))
	return k.ctx.err(rc, "wva_k2_history_import")
}
