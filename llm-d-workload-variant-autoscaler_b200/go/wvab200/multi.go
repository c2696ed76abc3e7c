// multi.go — cgo bindings of the round-2 entry points of include/wva_b200.h: several GPUs behind one handle
// (wva_group_*), the batched V1 saturation cycle, and the collector's columnar staging with the reconcile cycle as one
// CUDA graph (wva_ingest_*).  COMPILE-UNVERIFIED like wvab200.go (no Go toolchain in the build image or on the GPU
// box); the Python twins that the tests exercise are Group and Ingest in engine.py.
package wvab200

/*
#include <stdlib.h>
#include "wva_b200.h"
*/
import "C"

import (
	"context"
	"fmt"
	"runtime"
	"sort"
	"unsafe"

	"github.com/llm-d/llm-d-workload-variant-autoscaler/internal/interfaces"
	"github.com/llm-d/llm-d-workload-variant-autoscaler/pkg/config"
)

// Group drives n GPUs from this one process: n contexts joined by an NCCL communicator inside the library
// (wva_group_create).  Manager.Optimize over a Group sizes the servers in n contiguous blocks, exchanges candidates /
// partials over NVLink and returns the global solution.
type Group struct{ g *C.wva_group }

func NewGroup(devices []int) (*Group, error) {
	d := make([]C.int32_t, len(devices))
	for i, v := range devices {
		d[i] = C.int32_t(v)
	}
	var g *C.wva_group
	if rc := C.wva_group_create(&d[0], C.int32_t(len(d)), &g); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_group_create%v: %s", devices, C.GoString(C.wva_strerror(rc)))
	}
	return &Group{g: g}, nil
}
func (g *Group) Close()    { C.wva_group_destroy(g.g) }
func (g *Group) Size() int { return int(C.wva_group_size(g.g)) }

// Ctx returns the context of device i (timings, options); it stays owned by the group.
func (g *Group) Ctx(i int) *Ctx { return &Ctx{c: C.wva_group_ctx(g.g, C.int32_t(i))} }

// OptimizeGroup = pkg/manager.Manager.Optimize (manager.go:21-27) over every GPU of the group: the body of
// (*Manager).Optimize in wvab200.go with its three calls wva_load_system / wva_calculate / wva_solve /
// wva_get_solution replaced by the one call below (sys and sol are the wva_system / wva_solution that Optimize builds).
func optimizeGroup(g *Group, sys *C.wva_system, sol *C.wva_solution) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	if rc := C.wva_group_optimize(g.g, sys, sol); rc != C.WVA_OK {
		return fmt.Errorf("wva_group_optimize: %s", C.GoString(C.wva_strerror(rc)))
	}
	return nil
}

var _ *config.AllocationSolution // (the solution type Optimize returns)

// ---------------------------------------------------------------------------------------------------------------
// Batched V1 saturation: every model of a reconcile cycle in ONE launch.  The reference's engine loops over model
// groups (internal/engines/saturation/engine.go:281-289) and calls AnalyzeModelSaturation + CalculateSaturationTargets
// per model; a maintainer replaces that loop by one AnalyzeBatch call and fans the results back out.
type ModelInput struct {
	ModelID, Namespace string
	Replicas           []interfaces.ReplicaMetrics
	Config             interfaces.SaturationScalingConfig
	States             []interfaces.VariantReplicaState
}

type ModelOutput struct {
	Analysis *interfaces.ModelSaturationAnalysis
	Targets  map[string]int
}

func (a *SaturationAnalyzer) AnalyzeBatch(ctx context.Context, models []ModelInput) ([]ModelOutput, error) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	// CSR model -> variant (ascending VariantName) -> replica (metric slice order)
	var mvo, vro []C.int32_t
	var kv []C.double
	var q []C.int64_t
	var cost []C.double
	var cur, des, pen []C.int32_t
	var hasState []C.uint8_t
	cfg := [4][]C.double{}
	names := make([][]string, len(models))
	mvo = append(mvo, 0)
	vro = append(vro, 0)
	for mi, m := range models {
		b := groupByVariant(m.Replicas) // wvab200.go: variant names sorted, metrics per variant in slice order
		names[mi] = b.variants
		st := map[string]interfaces.VariantReplicaState{}
		for _, s := range m.States {
			st[s.VariantName] = s
		}
		for _, name := range b.variants {
			for _, r := range b.metrics[name] {
				kv = append(kv, C.double(r.KvCacheUsage))
				q = append(q, C.int64_t(r.QueueLength))
			}
			vro = append(vro, C.int32_t(len(kv)))
			cost = append(cost, C.double(b.metrics[name][0].Cost))
			s, ok := st[name]
			cur = append(cur, C.int32_t(s.CurrentReplicas))
			des = append(des, C.int32_t(s.DesiredReplicas))
			pen = append(pen, C.int32_t(s.PendingReplicas))
			if ok {
				hasState = append(hasState, 1)
			} else {
				hasState = append(hasState, 0)
			}
		}
		mvo = append(mvo, C.int32_t(len(cost)))
		cfg[0] = append(cfg[0], C.double(m.Config.KvCacheThreshold))
		cfg[1] = append(cfg[1], C.double(m.Config.QueueLengthThreshold))
		cfg[2] = append(cfg[2], C.double(m.Config.KvSpareTrigger))
		cfg[3] = append(cfg[3], C.double(m.Config.QueueSpareTrigger))
	}
	M, V, P := len(models), len(cost), len(kv)
	in := C.wva_saturation_in{n_models: C.int64_t(M), n_variants: C.int64_t(V), n_replicas: C.int64_t(P),
		model_variant_off: &mvo[0], variant_replica_off: &vro[0],
		rep_kv: (*C.double)(ptrOrNil(kv)), rep_queue: (*C.int64_t)(ptrOrNil(q)),
		var_cost: (*C.double)(ptrOrNil(cost)), var_current: (*C.int32_t)(ptrOrNil(cur)),
		var_desired: (*C.int32_t)(ptrOrNil(des)), var_pending: (*C.int32_t)(ptrOrNil(pen)),
		var_has_state: (*C.uint8_t)(ptrOrNil(hasState)),
		cfg_kv_threshold: &cfg[0][0], cfg_queue_threshold: &cfg[1][0], cfg_kv_trigger: &cfg[2][0], cfg_queue_trigger: &cfg[3][0]}
	target := make([]C.int32_t, V+1)
	nonSat := make([]C.int32_t, V+1)
	avgKv := make([]C.double, V+1)
	avgQ := make([]C.double, V+1)
	flags := make([]C.uint8_t, M+1)
	modKv := make([]C.double, M+1)
	modQ := make([]C.double, M+1)
	out := C.wva_saturation_out{var_target: &target[0], var_non_saturated: &nonSat[0], var_avg_spare_kv: &avgKv[0],
		var_avg_spare_queue: &avgQ[0], mod_flags: &flags[0], mod_avg_spare_kv: &modKv[0], mod_avg_spare_queue: &modQ[0]}
	if err := a.ctx.err(C.wva_saturation_v1(a.ctx.c, &in, &out), "wva_saturation_v1"); err != nil {
		return nil, err
	}
	res := make([]ModelOutput, M)
	for mi := range models {
		t := map[string]int{}
		for k, name := range names[mi] {
			if v := int(target[int(mvo[mi])+k]); v >= 0 {
				t[name] = v
			}
		}
		res[mi] = ModelOutput{Targets: t, Analysis: &interfaces.ModelSaturationAnalysis{
			ModelID: models[mi].ModelID, Namespace: models[mi].Namespace,
			ShouldScaleUp: flags[mi]&C.WVA_SAT_SCALE_UP != 0, ScaleDownSafe: flags[mi]&C.WVA_SAT_SCALE_DOWN_SAFE != 0,
			AvgSpareKvCapacity: float64(modKv[mi]), AvgSpareQueueLength: float64(modQ[mi])}}
	}
	return res, nil
}

// ---------------------------------------------------------------------------------------------------------------
// Ingest: the collector's columnar staging.  Built once per deployment epoch from the pods the reference would list
// (internal/collector/source/pod_va_mapper.go:32 FindVAForPod resolved here, once per pod); every cycle the Prometheus
// response parser calls Set* with the pod name of each sample (one map look-up) and Commit() launches the captured graph.
type Ingest struct {
	h      *C.wva_ingest
	cols   C.wva_ingest_columns
	res    C.wva_ingest_results
	dcols  C.wva_ingest_decision_columns // decision mode only (NewIngestDecisions)
	dres   C.wva_ingest_decision_results
	slotOf map[string]int32 // pod name -> slot
	kv, q  []float64
	has    []uint8
	nv, nm int
}

// models: sorted model ids; variants[m]: sorted VariantAutoscaling names of model m; pods[variant]: its pod names.
func NewIngest(ctx *Ctx, models []string, variants map[string][]string, pods map[string][]string) (*Ingest, error) {
	return newIngest(ctx, models, variants, pods, -1)
}

// NewIngestDecisions: the same registry in decision mode (wva_ingest_create_decisions) — Commit() then runs the rest of
// optimizeV1 (engine.go:322-392: EnforcePolicy per model, convertSaturationTargetsToDecisions, the GPU limiter over all
// decisions) inside the graph.  nTypes = accelerator types of the GPU inventory, in sorted name order.
func NewIngestDecisions(ctx *Ctx, models []string, variants map[string][]string, pods map[string][]string, nTypes int) (*Ingest, error) {
	return newIngest(ctx, models, variants, pods, nTypes)
}

func newIngest(ctx *Ctx, models []string, variants map[string][]string, pods map[string][]string, nTypes int) (*Ingest, error) {
	ing := &Ingest{slotOf: map[string]int32{}}
	mvo := []C.int32_t{0}
	vso := []C.int32_t{0}
	nv := 0
	for _, m := range models {
		for _, va := range variants[m] {
			ps := append([]string(nil), pods[va]...)
			sort.Strings(ps) // canonical order of the per-variant float64 sums
			for _, p := range ps {
				ing.slotOf[p] = int32(len(ing.slotOf))
			}
			vso = append(vso, C.int32_t(len(ing.slotOf)))
			nv++
		}
		mvo = append(mvo, C.int32_t(nv))
	}
	var rc C.int32_t
	if nTypes < 0 {
		rc = C.wva_ingest_create(ctx.c, C.int64_t(len(models)), C.int64_t(nv), C.int64_t(len(ing.slotOf)), &mvo[0], &vso[0],
			&ing.h, &ing.cols, &ing.res)
	} else {
		rc = C.wva_ingest_create_decisions(ctx.c, C.int64_t(len(models)), C.int64_t(nv), C.int64_t(len(ing.slotOf)),
			C.int32_t(nTypes), &mvo[0], &vso[0], &ing.h, &ing.cols, &ing.res, &ing.dcols, &ing.dres)
	}
	if err := ctx.err(rc, "wva_ingest_create"); err != nil {
		return nil, err
	}
	ing.nv, ing.nm = nv, len(models)
	n := len(ing.slotOf)
	ing.kv = unsafe.Slice((*float64)(unsafe.Pointer(ing.cols.kv)), n) // page-locked C memory: cgo pointer rules do not apply
	ing.q = unsafe.Slice((*float64)(unsafe.Pointer(ing.cols.queue)), n)
	ing.has = unsafe.Slice((*uint8)(unsafe.Pointer(ing.cols.has)), n)
	return ing, nil
}
func (g *Ingest) Close() { C.wva_ingest_destroy(g.h) }
func (g *Ingest) Begin() { C.wva_ingest_begin(g.h) }

// SetKv / SetQueue: one sample of registration.QueryKvCacheUsage / QueryQueueLength (replica_metrics.go:120-175);
// unknown pods are skipped as the reference skips pods that match no deployment (:323-328).
func (g *Ingest) SetKv(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok {
		g.kv[s] = v
		g.has[s] |= 1
	}
}
func (g *Ingest) SetQueue(pod string, v float64) {
	if s, ok := g.slotOf[pod]; ok {
		g.q[s] = v
		g.has[s] |= 2
	}
}

// Commit: metric batch -> decisions, one CUDA graph launch.  Targets are read from g.res (page-locked) by the caller.
func (g *Ingest) Commit() error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	if rc := C.wva_ingest_commit(g.h); rc != C.WVA_OK {
		return fmt.Errorf("wva_ingest_commit: %s", C.GoString(C.wva_strerror(rc)))
	}
	return nil
}

// IngestDecisionInputs: the per-cycle columns of the decision mode, indexed like the registry (variants / models) and
// the inventory's sorted types.  AcceleratorType -1 = "" or a type without a pool.
type IngestDecisionInputs struct {
	AcceleratorType, GPUsPerReplica []int32 // [V]
	ScaleToZeroEnabled, RequestError  []bool  // [M]
	RequestCount                      []float64 // [M]
	TypeLimit                         []int32 // [T] TypeInventory limits after Refresh
	EnableLimiter                     bool
}

// SetDecisionInputs copies one cycle's decision columns into the page-locked arena (before Commit).
func (g *Ingest) SetDecisionInputs(in *IngestDecisionInputs) {
	v, m, t := g.nv, g.nm, int(g.dcols.n_types)
	copy(unsafe.Slice((*int32)(unsafe.Pointer(g.dcols.var_accelerator_type)), v), in.AcceleratorType)
	copy(unsafe.Slice((*int32)(unsafe.Pointer(g.dcols.var_gpus_per_replica)), v), in.GPUsPerReplica)
	s2z := unsafe.Slice((*uint8)(unsafe.Pointer(g.dcols.mod_scale_to_zero_enabled)), m)
	rerr := unsafe.Slice((*uint8)(unsafe.Pointer(g.dcols.mod_request_error)), m)
	for i := 0; i < m; i++ {
		s2z[i], rerr[i] = 0, 0
		if in.ScaleToZeroEnabled[i] {
			s2z[i] = 1
		}
		if in.RequestError[i] {
			rerr[i] = 1
		}
	}
	copy(unsafe.Slice((*float64)(unsafe.Pointer(g.dcols.mod_request_count)), m), in.RequestCount)
	if t > 0 {
		copy(unsafe.Slice((*int32)(unsafe.Pointer(g.dcols.type_limit)), t), in.TypeLimit)
	}
	en := int32(0)
	if in.EnableLimiter {
		en = 1
	}
	*(*int32)(unsafe.Pointer(g.dcols.enable_limiter)) = en
}

// IngestDecision: the numeric fields of one interfaces.VariantDecision after the cycle; the caller attaches the names
// (VariantName, ModelID, Namespace, AcceleratorName) from the registry and the Reason / DecisionSteps strings.
type IngestDecision struct {
	Variant                                  int // registry index
	OriginalTarget, Target, GPUsAllocated    int
	Action                                   int // 1 scale-up, -1 scale-down, 0 no-change (before the limiter)
	WasLimited                               bool
}

// Decisions: the cycle's final decisions in registry order, valid after Commit until the next Commit.
func (g *Ingest) Decisions() []IngestDecision {
	v := g.nv
	has := unsafe.Slice((*uint8)(unsafe.Pointer(g.dres.has_decision)), v)
	orig := unsafe.Slice((*int32)(unsafe.Pointer(g.dres.original_target)), v)
	tgt := unsafe.Slice((*int32)(unsafe.Pointer(g.dres.target)), v)
	gpus := unsafe.Slice((*int32)(unsafe.Pointer(g.dres.gpus_allocated)), v)
	lim := unsafe.Slice((*uint8)(unsafe.Pointer(g.dres.was_limited)), v)
	act := unsafe.Slice((*int8)(unsafe.Pointer(g.dres.action)), v)
	var out []IngestDecision
	for i := 0; i < v; i++ {
		if has[i] == 0 {
			continue
		}
		out = append(out, IngestDecision{Variant: i, OriginalTarget: int(orig[i]), Target: int(tgt[i]),
			GPUsAllocated: int(gpus[i]), Action: int(act[i]), WasLimited: lim[i] != 0})
	}
	return out
}
