// IngestV2: the V2 engine's cycle (optimizeV2, internal/engines/saturation/engine.go:397-488) from the six Prometheus
// vectors of CollectReplicaMetrics to the final VariantDecisions, in two graph launches around the host capacity store
// (wva_ingest_v2_*, include/wva_b200.h).  COMPILE-UNVERIFIED like the rest of this package.
//
// Per cycle the caller (package saturation, in place of collectV2ModelRequest -> Optimize -> the enforcer bridge):
//   Begin; SetKv / SetQueue / SetCacheConfig / SetAvg* for each sample; the per-cycle columns through g.Cols;
//   Analyze; the host step: for every variant whose store slot s has g.Res.SlotLastRep[s] >= 0, capacityStore.Update
//   once (the pod is g.Res.RepPod of that replica), then for the variants with g.Res.VarNoData the zero-replica fallback
//   (analyzer.go:317-415, with g.Res.ModAvg*Tokens) written into g.Cols.VarFallbackCapacity; Decide; then the
//   decisions of the models with g.Res.ModHasRequest, with the Reason strings and applyEnforcedTargetsToDecisions
//   (engine_v2.go:106-127) from g.Res.VarOptimizerTarget / g.Res.VarTarget.
package wvab200

/*
#include "wva_b200.h"
*/
import "C"

import (
	"math"
	"runtime"
	"sort"
	"strconv"
	"unsafe"
)

type IngestV2 struct {
	h      *C.wva_ingest_v2
	cols   C.wva_ingest_v2_columns
	res    C.wva_ingest_v2_results
	slotOf map[string]int32 // pod name -> slot
	ns     int
	Cols   IngestV2Columns // Go views of the per-cycle columns (page-locked C memory: cgo pointer rules do not apply)
	Res    IngestV2Results // Go views of the results; valid after the launch that fills them, until the next one
}

// IngestV2Columns: the columns the caller writes every cycle besides the samples, in registry order.  Only
// VarFallbackCapacity may change between Analyze and Decide: Decide uploads it alone, the others go up with Analyze.
type IngestV2Columns struct {
	VarCost                                   []float64 // [V] ReplicaMetrics.Cost of the variant's pods
	VarCurrent, VarPending, VarNameRank       []int32   // [V] VariantReplicaState; rank of the name within its model
	CfgKvThreshold, CfgQueueThreshold         []float64 // [M] SaturationScalingConfig
	CfgScaleUpThreshold, CfgScaleDownBoundary []float64 // [M]
	ModScaleToZeroEnabled, ModRequestError    []uint8   // [M] enforcer inputs
	ModRequestCount                           []float64 // [M]
	SlotMaxBatchedTokens, SlotMaxNumSeqs      []int64   // [store slots] VLLMParams at the start of the cycle
	VarFallbackCapacity                       []float64 // [V] written by the host step between Analyze and Decide
}

// IngestV2Results: what Analyze returns for the host step, and what Decide returns for the decisions.
type IngestV2Results struct {
	VariantReplicaOff, RepPod, SlotLastRep           []int32 // [V+1], [pods], [store slots]
	RepTotalKvTokens, SlotEffective                  []int64 // [pods], [store slots]
	VarNoData, ModHasRequest, ModEnforced            []uint8 // [V], [M], [M]
	ModAvgInputTokens, ModAvgOutputTokens            []float64
	VarOptimizerTarget, VarTarget, VarReady          []int32 // [V]
	VarAction                                        []int8  // [V]
	VarPerReplicaCapacity, VarTotalCapacity          []float64
	VarTotalDemand, VarUtilization                   []float64
	ModTotalSupply, ModTotalDemand, ModUtilization   []float64
	ModRequiredCapacity, ModSpareCapacity            []float64
}

// NewIngestV2: models in registry order; variants[m] the VariantAutoscaling names of model m; pods[variant] its pods
// (slotted in ascending name order); varAccelerator / varStoreSlot per variant in registry order (ids of k2's
// registry; the history's model groups must be these models).
func NewIngestV2(ctx *Ctx, models []string, variants map[string][]string, pods map[string][]string, varAccelerator,
	varStoreSlot []int32, k2 *K2History) (*IngestV2, error) {
	g := &IngestV2{slotOf: map[string]int32{}}
	mvo := []C.int32_t{0}
	vso := []C.int32_t{0}
	nv := 0
	for _, m := range models {
		for _, va := range variants[m] {
			ps := append([]string(nil), pods[va]...)
			sort.Strings(ps) // the ReplicaMetrics slice order of the model, variant after variant
			for _, p := range ps {
				g.slotOf[p] = int32(len(g.slotOf))
			}
			vso = append(vso, C.int32_t(len(g.slotOf)))
			nv++
		}
		mvo = append(mvo, C.int32_t(nv))
	}
	rc := C.wva_ingest_v2_create(ctx.c, C.int64_t(len(models)), C.int64_t(nv), C.int64_t(len(g.slotOf)), &mvo[0], &vso[0],
		(*C.int32_t)(ptrOrNil(varAccelerator)), (*C.int32_t)(ptrOrNil(varStoreSlot)), k2.h, &g.h, &g.cols, &g.res)
	if err := ctx.err(rc, "wva_ingest_v2_create"); err != nil {
		return nil, err
	}
	g.ns = len(g.slotOf)
	v, m, ns, c, r := nv, len(models), int(g.cols.n_store_slots), &g.cols, &g.res
	g.Cols = IngestV2Columns{
		VarCost: f64(c.var_cost, v), VarCurrent: i32(c.var_current, v), VarPending: i32(c.var_pending, v),
		VarNameRank: i32(c.var_name_rank, v), CfgKvThreshold: f64(c.cfg_kv_threshold, m),
		CfgQueueThreshold: f64(c.cfg_queue_threshold, m), CfgScaleUpThreshold: f64(c.cfg_scale_up_threshold, m),
		CfgScaleDownBoundary: f64(c.cfg_scale_down_boundary, m), ModScaleToZeroEnabled: u8(c.mod_scale_to_zero_enabled, m),
		ModRequestError: u8(c.mod_request_error, m), ModRequestCount: f64(c.mod_request_count, m),
		SlotMaxBatchedTokens: i64(c.slot_max_batched_tokens, ns), SlotMaxNumSeqs: i64(c.slot_max_num_seqs, ns),
		VarFallbackCapacity: f64(c.var_fallback_capacity, v)}
	g.Res = IngestV2Results{
		VariantReplicaOff: i32(r.variant_replica_off, v+1), RepPod: i32(r.rep_pod, g.ns), SlotLastRep: i32(r.slot_last_rep, ns),
		RepTotalKvTokens: i64(r.rep_total_kv_tokens, g.ns), SlotEffective: i64(r.slot_effective, ns),
		VarNoData: u8(r.var_no_data, v), ModHasRequest: u8(r.mod_has_request, m), ModEnforced: u8(r.mod_enforced, m),
		ModAvgInputTokens: f64(r.mod_avg_input_tokens, m), ModAvgOutputTokens: f64(r.mod_avg_output_tokens, m),
		VarOptimizerTarget: i32(r.var_optimizer_target, v), VarTarget: i32(r.var_target, v), VarReady: i32(r.var_ready, v),
		VarAction: unsafe.Slice((*int8)(unsafe.Pointer(r.var_action)), v),
		VarPerReplicaCapacity: f64(r.var_per_replica_capacity, v), VarTotalCapacity: f64(r.var_total_capacity, v),
		VarTotalDemand: f64(r.var_total_demand, v), VarUtilization: f64(r.var_utilization, v),
		ModTotalSupply: f64(r.mod_total_supply, m), ModTotalDemand: f64(r.mod_total_demand, m),
		ModUtilization: f64(r.mod_utilization, m), ModRequiredCapacity: f64(r.mod_required_capacity, m),
		ModSpareCapacity: f64(r.mod_spare_capacity, m)}
	return g, nil
}

func (g *IngestV2) Close() { C.wva_ingest_v2_destroy(g.h) }

// Begin: start of a cycle (no pod has a sample; avg_*, hit rate and cache config cleared).
func (g *IngestV2) Begin(ctx *Ctx) error { return ctx.err(C.wva_ingest_v2_begin(g.h), "wva_ingest_v2_begin") }

// SlotOf: the pod slot of a pod name (RepPod indexes slots), false for a pod of no variant.
func (g *IngestV2) SlotOf(pod string) (int32, bool) {
	s, ok := g.slotOf[pod]
	return s, ok
}

func f64(p *C.double, n int) []float64 { return unsafe.Slice((*float64)(unsafe.Pointer(p)), n) }
func i64(p *C.int64_t, n int) []int64  { return unsafe.Slice((*int64)(unsafe.Pointer(p)), n) }
func i32(p *C.int32_t, n int) []int32  { return unsafe.Slice((*int32)(unsafe.Pointer(p)), n) }
func u8(p *C.uint8_t, n int) []uint8   { return unsafe.Slice((*uint8)(unsafe.Pointer(p)), n) }

// SetKv / SetQueue: a later sample of a pod overwrites (replica_metrics.go:133-189); unknown pods are skipped.
func (g *IngestV2) SetKv(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok {
		f64(g.cols.kv, g.ns)[s] = v
		u8(g.cols.has, g.ns)[s] |= 1
	}
}
func (g *IngestV2) SetQueue(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok {
		f64(g.cols.queue, g.ns)[s] = v
		u8(g.cols.has, g.ns)[s] |= 2
	}
}

// SetCacheConfig: the num_gpu_blocks / block_size labels of a cache_config_info sample (:192-225).
func (g *IngestV2) SetCacheConfig(pod, blocks, size string) {
	s, ok := g.slotOf[pod]
	if !ok {
		return
	}
	b, z := i64(g.cols.num_gpu_blocks, g.ns), i64(g.cols.block_size, g.ns)
	if blocks != "" {
		if x, err := strconv.ParseInt(blocks, 10, 64); err == nil {
			b[s] = x
		}
	}
	if size != "" {
		if x, err := strconv.ParseInt(size, 10, 64); err == nil {
			z[s] = x
		}
	}
	if b[s] > 0 && z[s] > 0 {
		u8(g.cols.has, g.ns)[s] |= 4
	}
}

func finite(v float64) bool { return !math.IsNaN(v) && !math.IsInf(v, 0) }

// SetAvgOutput / SetAvgInput / SetPrefixHitRate (:228-292): samples the reference rejects overwrite nothing.
func (g *IngestV2) SetAvgOutput(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok && finite(v) {
		f64(g.cols.avg_output_tokens, g.ns)[s] = v
	}
}
func (g *IngestV2) SetAvgInput(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok && finite(v) {
		f64(g.cols.avg_input_tokens, g.ns)[s] = v
	}
}
func (g *IngestV2) SetPrefixHitRate(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok && finite(v) && v >= 0 && v <= 1 {
		f64(g.cols.prefix_hit_rate, g.ns)[s] = v
	}
}

// Analyze: the first graph launch (pack, k2 chain against the history); Decide: the second (analyzer, optimizer,
// enforcer), after the host step has written var_fallback_capacity.
func (g *IngestV2) Analyze(ctx *Ctx) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return ctx.err(C.wva_ingest_v2_analyze(g.h), "wva_ingest_v2_analyze")
}
func (g *IngestV2) Decide(ctx *Ctx) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return ctx.err(C.wva_ingest_v2_decide(g.h), "wva_ingest_v2_decide")
}
