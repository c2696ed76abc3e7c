// Package wvab200 is the cgo shim that binds the H100 hot path (include/wva_b200.h) behind the
// reference's own Go seams.  COMPILE-UNVERIFIED: the project's build has no Go toolchain, so this file
// has never been compiled; it documents, in code, the
// binding a maintainer adds.  Build needs CGO_ENABLED=1 (the reference's Dockerfile:25 uses 0), glibc,
// libcudart and libwva_b200.so on the loader path.
//
// Seams replaced (paths in the reference tree):
//
//	pkg/manager.Manager.Optimize                 -> (*Manager).Optimize
//	internal/interfaces.SaturationAnalyzer       -> (*SaturationAnalyzer)
//	internal/engines/pipeline.Limiter            -> (*Limiter).Limit
package wvab200

/*
#cgo CFLAGS: -I${SRCDIR}/../../../include
#cgo LDFLAGS: -L${SRCDIR}/../../csrc -lwva_b200 -lcudart
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

	intconfig "github.com/llm-d/llm-d-workload-variant-autoscaler/internal/config"
	"github.com/llm-d/llm-d-workload-variant-autoscaler/internal/engines/pipeline"
	"github.com/llm-d/llm-d-workload-variant-autoscaler/internal/interfaces"
	"github.com/llm-d/llm-d-workload-variant-autoscaler/pkg/config"
)

// Ctx owns one GPU context.  A Ctx is single-caller, like pkg/core's global TheSystem.
type Ctx struct{ c *C.wva_ctx }

func New(device int) (*Ctx, error) {
	var c *C.wva_ctx
	if rc := C.wva_create(C.int32_t(device), &c); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_create: %s", C.GoString(C.wva_strerror(rc)))
	}
	return &Ctx{c: c}, nil
}

func (x *Ctx) Close() { C.wva_destroy(x.c) }

// PinnedFloat64 / PinnedInt64 return slices over page-locked C memory (wva_host_alloc): a collector that writes its
// per-replica SoA batch into them gets DMA at link speed through every entry point (BASELINE config 5).  The memory is C memory — cgo's pointer rules do not apply — and lives until Free.
type Pinned struct{ p unsafe.Pointer }

func PinnedBytes(n int) (*Pinned, error) {
	var p unsafe.Pointer
	if rc := C.wva_host_alloc(C.size_t(n), &p); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_host_alloc(%d): %s", n, C.GoString(C.wva_strerror(rc)))
	}
	return &Pinned{p: p}, nil
}
func (b *Pinned) Float64(n int) []float64 { return unsafe.Slice((*float64)(b.p), n) }
func (b *Pinned) Int64(n int) []int64     { return unsafe.Slice((*int64)(b.p), n) }
func (b *Pinned) Int32(n int) []int32     { return unsafe.Slice((*int32)(b.p), n) }
func (b *Pinned) Free()                   { C.wva_host_free(b.p); b.p = nil }

func (x *Ctx) err(rc C.int32_t, what string) error {
	if rc == C.WVA_OK {
		return nil
	}
	// a non-nil error lets the existing retry / safety-net paths fire
	// (internal/engines/executor/polling.go:56-86, engines/saturation/engine.go:1022-1095)
	return fmt.Errorf("%s: %s %s", what, C.GoString(C.wva_strerror(rc)), C.GoString(C.wva_last_error(x.c)))
}

// UpdateServers replaces the per-cycle server columns of the loaded system (ServerLoadSpec and CurrentAlloc, in the
// server index order of the loaded system; all [S]) in place; Recalculate then re-sizes or re-values only the servers
// they changed, with the candidates of a full wva_calculate (INTEGRATION.md §3, per-cycle use).
func (x *Ctx) UpdateServers(arrival []float32, inTokens, outTokens, curAcc, curReplicas []int32, curCost []float32) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	n := len(arrival)
	if len(inTokens) != n || len(outTokens) != n || len(curAcc) != n || len(curReplicas) != n || len(curCost) != n {
		return fmt.Errorf("UpdateServers: the six columns differ in length")
	}
	if n == 0 {
		return x.err(C.wva_update_servers(x.c, nil, nil, nil, nil, nil, nil), "wva_update_servers")
	}
	var pin runtime.Pinner // C copies the columns before returning
	defer pin.Unpin()
	for _, p := range []unsafe.Pointer{unsafe.Pointer(&arrival[0]), unsafe.Pointer(&inTokens[0]), unsafe.Pointer(&outTokens[0]),
		unsafe.Pointer(&curAcc[0]), unsafe.Pointer(&curReplicas[0]), unsafe.Pointer(&curCost[0])} {
		pin.Pin(p)
	}
	return x.err(C.wva_update_servers(x.c, (*C.float)(unsafe.Pointer(&arrival[0])), (*C.int32_t)(unsafe.Pointer(&inTokens[0])),
		(*C.int32_t)(unsafe.Pointer(&outTokens[0])), (*C.int32_t)(unsafe.Pointer(&curAcc[0])),
		(*C.int32_t)(unsafe.Pointer(&curReplicas[0])), (*C.float)(unsafe.Pointer(&curCost[0]))), "wva_update_servers")
}

// Recalculate returns how many servers of this context's block were re-sized and re-valued.
func (x *Ctx) Recalculate() (resized, revalued int64, err error) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var r, v C.int64_t
	err = x.err(C.wva_recalculate(x.c, &r, &v), "wva_recalculate")
	return int64(r), int64(v), err
}

// GridUpdate brings the replica grid resident from the last wva_grid_run up to date with the UpdateServers calls since
// then, re-evaluating only the servers whose load changed, with the grid of a full wva_grid_run (INTEGRATION.md §3,
// per-cycle use).  It returns how many servers of this context's block were re-evaluated.
func (x *Ctx) GridUpdate() (regridded int64, err error) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	var n C.int64_t
	err = x.err(C.wva_grid_update(x.c, &n), "wva_grid_update")
	return int64(n), err
}

// ServerColumns are the 15 server columns of a wva_system, one entry per server in ascending-name order.
type ServerColumns struct {
	Model, Priority, MinReplicas, MaxBatch       []int32
	KeepAcc, TargetPresent                       []uint8
	SLOTTFT, SLOITL, SLOTPS, Arrival             []float32
	InTokens, OutTokens, CurAcc, CurReplicas     []int32
	CurCost                                      []float32
}

// UpdateServerSet replaces the server set of the loaded system in place (System.AddServerFromSpec / RemoveServer for a
// whole cycle): prev[i] is the loaded index of new server i, or -1 for a new one; cols are the new set's columns.
// Accelerators, models and perf data stay those of the loaded system (INTEGRATION.md §3, per-cycle use).  Recalculate
// and GridUpdate then bring the candidates and the resident grid up to date.
func (x *Ctx) UpdateServerSet(prev []int32, cols *ServerColumns) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	n := len(prev)
	for _, l := range []int{len(cols.Model), len(cols.Priority), len(cols.MinReplicas), len(cols.MaxBatch), len(cols.KeepAcc),
		len(cols.TargetPresent), len(cols.SLOTTFT), len(cols.SLOITL), len(cols.SLOTPS), len(cols.Arrival), len(cols.InTokens),
		len(cols.OutTokens), len(cols.CurAcc), len(cols.CurReplicas), len(cols.CurCost)} {
		if l != n {
			return fmt.Errorf("UpdateServerSet: a column's length differs from len(prev)")
		}
	}
	var pin runtime.Pinner // C copies the columns before returning
	defer pin.Unpin()
	p32 := func(s []int32) *C.int32_t {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.int32_t)(unsafe.Pointer(&s[0]))
	}
	pf := func(s []float32) *C.float {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.float)(unsafe.Pointer(&s[0]))
	}
	pu := func(s []uint8) *C.uint8_t {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.uint8_t)(unsafe.Pointer(&s[0]))
	}
	sys := C.wva_system{
		n_servers: C.int32_t(n),
		srv_model: p32(cols.Model), srv_priority: p32(cols.Priority), srv_min_replicas: p32(cols.MinReplicas),
		srv_max_batch: p32(cols.MaxBatch), srv_keep_acc: pu(cols.KeepAcc), srv_target_present: pu(cols.TargetPresent),
		srv_slo_ttft: pf(cols.SLOTTFT), srv_slo_itl: pf(cols.SLOITL), srv_slo_tps: pf(cols.SLOTPS), srv_arrival: pf(cols.Arrival),
		srv_in_tokens: p32(cols.InTokens), srv_out_tokens: p32(cols.OutTokens),
		srv_cur_acc: p32(cols.CurAcc), srv_cur_replicas: p32(cols.CurReplicas), srv_cur_cost: pf(cols.CurCost),
	}
	return x.err(C.wva_update_server_set(x.c, C.int32_t(n), p32(prev), &sys), "wva_update_server_set")
}

// TableColumns are the accelerator columns ([A], accelerator index order) and the perf tables ([M*A], row-major by
// model) of a wva_system.
type TableColumns struct {
	AccCost                                       []float32
	AccMultiplicity, AccType                      []int32
	PerfAlpha, PerfBeta, PerfGamma                []float32
	PerfMaxBatch, PerfAtTokens, PerfAccCount      []int32
	PerfPresent                                   []uint8
}

// UpdateTables replaces the accelerator costs, multiplicities and types and the ModelAcceleratorPerfData of the loaded
// system in place; nAcc, nTypes and nModels must be the loaded ones (a change of shape is a reload).  Recalculate and
// GridUpdate then re-size and re-evaluate only the (server, accelerator) pairs that read a changed row (INTEGRATION.md
// §3, per-cycle use).  It returns how many pairs of this context's block the call marked for re-sizing.
// COMPILE-UNVERIFIED, like the rest of this file.
func (x *Ctx) UpdateTables(nAcc, nTypes, nModels int, t *TableColumns) (marked int64, err error) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	for _, l := range []int{len(t.AccCost), len(t.AccMultiplicity), len(t.AccType)} {
		if l != nAcc {
			return 0, fmt.Errorf("UpdateTables: an accelerator column's length differs from nAcc")
		}
	}
	for _, l := range []int{len(t.PerfAlpha), len(t.PerfBeta), len(t.PerfGamma), len(t.PerfMaxBatch), len(t.PerfAtTokens),
		len(t.PerfAccCount), len(t.PerfPresent)} {
		if l != nModels*nAcc {
			return 0, fmt.Errorf("UpdateTables: a perf column's length differs from nModels * nAcc")
		}
	}
	var pin runtime.Pinner // C copies the columns before returning
	defer pin.Unpin()
	p32 := func(s []int32) *C.int32_t {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.int32_t)(unsafe.Pointer(&s[0]))
	}
	pf := func(s []float32) *C.float {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.float)(unsafe.Pointer(&s[0]))
	}
	pu := func(s []uint8) *C.uint8_t {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.uint8_t)(unsafe.Pointer(&s[0]))
	}
	sys := C.wva_system{
		n_acc: C.int32_t(nAcc), n_types: C.int32_t(nTypes), n_models: C.int32_t(nModels),
		acc_cost: pf(t.AccCost), acc_multiplicity: p32(t.AccMultiplicity), acc_type: p32(t.AccType),
		perf_alpha: pf(t.PerfAlpha), perf_beta: pf(t.PerfBeta), perf_gamma: pf(t.PerfGamma),
		perf_max_batch: p32(t.PerfMaxBatch), perf_at_tokens: p32(t.PerfAtTokens), perf_acc_count: p32(t.PerfAccCount),
		perf_present: pu(t.PerfPresent),
	}
	var n C.int64_t
	err = x.err(C.wva_update_tables(x.c, &sys, &n), "wva_update_tables")
	return int64(n), err
}

// index maps built from SORTED names: ascending index is then a valid Go map order and the
// name-based tie-breaks of the reference become index comparisons.
type index struct {
	names []string
	of    map[string]int32
}

func newIndex(names []string) index {
	s := append([]string(nil), names...)
	sort.Strings(s)
	ix := index{names: s, of: make(map[string]int32, len(s))}
	for i, n := range s {
		ix.of[n] = int32(i)
	}
	return ix
}

// Manager mirrors pkg/manager.Manager (manager.go:13-27): Optimize = Calculate + Solve + AllocateByType.
type Manager struct {
	ctx  *Ctx
	spec *config.SystemSpec
	acc  index
	srv  index
}

func NewManager(ctx *Ctx, spec *config.SystemSpec) *Manager { return &Manager{ctx: ctx, spec: spec} }

// Optimize flattens the SystemSpec (what System.SetFromSpec + the lookups of CreateAllocation resolve,
// pkg/core/system.go:82-89, allocation.go:43-71), runs the device path and returns the
// config.AllocationSolution that System.GenerateSolution (system.go:303-319) would.
func (m *Manager) Optimize() (*config.AllocationSolution, error) {
	runtime.LockOSThread() // the ctx sets its CUDA device per call; keep the thread for the duration
	defer runtime.UnlockOSThread()
	d := m.spec
	accNames := make([]string, len(d.Accelerators.Spec))
	typeSet := map[string]struct{}{}
	for i, a := range d.Accelerators.Spec {
		accNames[i] = a.Name
		typeSet[a.Type] = struct{}{}
	}
	for _, c := range d.Capacity.Count {
		typeSet[c.Type] = struct{}{}
	}
	typeNames := make([]string, 0, len(typeSet))
	for t := range typeSet {
		typeNames = append(typeNames, t)
	}
	modelSet := map[string]struct{}{}
	for _, p := range d.Models.PerfData {
		modelSet[p.Name] = struct{}{}
	}
	modelNames := make([]string, 0, len(modelSet))
	for n := range modelSet {
		modelNames = append(modelNames, n)
	}
	srvNames := make([]string, len(d.Servers.Spec))
	for i, s := range d.Servers.Spec {
		srvNames[i] = s.Name
	}
	acc, typ, mod, srv := newIndex(accNames), newIndex(typeNames), newIndex(modelNames), newIndex(srvNames)
	m.acc, m.srv = acc, srv
	A, T, M, S := len(acc.names), len(typ.names), len(mod.names), len(srv.names)

	accCost := make([]float32, A)
	accMult, accType, typeCount := make([]int32, A), make([]int32, A), make([]int32, T)
	for _, a := range d.Accelerators.Spec {
		i := acc.of[a.Name]
		accCost[i], accMult[i], accType[i] = a.Cost, int32(a.Multiplicity), typ.of[a.Type]
	}
	for _, c := range d.Capacity.Count {
		typeCount[typ.of[c.Type]] = int32(c.Count)
	}
	alpha, beta, gamma := make([]float32, M*A), make([]float32, M*A), make([]float32, M*A)
	maxB, atTok, accCnt, present := make([]int32, M*A), make([]int32, M*A), make([]int32, M*A), make([]uint8, M*A)
	for _, p := range d.Models.PerfData {
		a, ok := acc.of[p.Acc]
		if !ok {
			continue
		}
		i := int(mod.of[p.Name])*A + int(a)
		alpha[i], beta[i], gamma[i] = p.ServiceParms.Alpha, p.ServiceParms.Beta, p.ServiceParms.Gamma
		maxB[i], atTok[i], accCnt[i], present[i] = int32(p.MaxBatchSize), int32(p.AtTokens), int32(p.AccCount), 1
	}
	// service classes: priority clamp (serviceclass.go:28-31) and per-model targets
	type tgt struct{ itl, ttft, tps float32 }
	prio := map[string]int32{}
	targets := map[string]map[string]tgt{}
	for _, c := range d.ServiceClasses.Spec {
		p := int32(c.Priority)
		if p < config.DefaultHighPriority || p > config.DefaultLowPriority {
			p = config.DefaultServiceClassPriority
		}
		prio[c.Name] = p
		targets[c.Name] = map[string]tgt{}
		for _, mt := range c.ModelTargets {
			targets[c.Name][mt.Model] = tgt{mt.SLO_ITL, mt.SLO_TTFT, mt.SLO_TPS}
		}
	}
	i32 := func() []int32 { return make([]int32, S) }
	f32 := func() []float32 { return make([]float32, S) }
	sModel, sPrio, sMin, sMaxB, sIn, sOut, sCurAcc, sCurRep := i32(), i32(), i32(), i32(), i32(), i32(), i32(), i32()
	sTTFT, sITL, sTPS, sArr, sCurCost := f32(), f32(), f32(), f32(), f32()
	sKeep, sTgt := make([]uint8, S), make([]uint8, S)
	for _, s := range d.Servers.Spec {
		i := srv.of[s.Name]
		class := s.Class
		if class == "" {
			class = config.DefaultServiceClassName // server.go:38-41
		}
		if mi, ok := mod.of[s.Model]; ok {
			sModel[i] = mi
		} else {
			sModel[i] = -1
		}
		if p, ok := prio[class]; ok {
			sPrio[i] = p
		} else {
			sPrio[i] = config.DefaultServiceClassPriority // server.go:92-97
		}
		if t, ok := targets[class][s.Model]; ok {
			sTgt[i], sTTFT[i], sITL[i], sTPS[i] = 1, t.ttft, t.itl, t.tps
		}
		sMin[i], sMaxB[i] = int32(s.MinNumReplicas), int32(s.MaxBatchSize)
		if s.KeepAccelerator {
			sKeep[i] = 1
		}
		ld := s.CurrentAlloc.Load
		sArr[i], sIn[i], sOut[i] = ld.ArrivalRate, int32(ld.AvgInTokens), int32(ld.AvgOutTokens)
		switch a, ok := acc.of[s.CurrentAlloc.Accelerator]; {
		case s.CurrentAlloc.Accelerator == "":
			sCurAcc[i] = C.WVA_CUR_ACC_EMPTY
		case ok:
			sCurAcc[i] = a
		default:
			sCurAcc[i] = C.WVA_CUR_ACC_UNKNOWN
		}
		sCurRep[i], sCurCost[i] = int32(s.CurrentAlloc.NumReplicas), s.CurrentAlloc.Cost
	}
	var pin runtime.Pinner // Go slices are passed for the duration of the call only; C copies them
	defer pin.Unpin()
	p32 := func(s []int32) *C.int32_t {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.int32_t)(unsafe.Pointer(&s[0]))
	}
	pf := func(s []float32) *C.float {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.float)(unsafe.Pointer(&s[0]))
	}
	pu := func(s []uint8) *C.uint8_t {
		if len(s) == 0 {
			return nil
		}
		pin.Pin(&s[0])
		return (*C.uint8_t)(unsafe.Pointer(&s[0]))
	}
	sys := C.wva_system{
		n_acc: C.int32_t(A), n_types: C.int32_t(T), n_models: C.int32_t(M), n_servers: C.int32_t(S),
		acc_cost: pf(accCost), acc_multiplicity: p32(accMult), acc_type: p32(accType), type_count: p32(typeCount),
		perf_alpha: pf(alpha), perf_beta: pf(beta), perf_gamma: pf(gamma),
		perf_max_batch: p32(maxB), perf_at_tokens: p32(atTok), perf_acc_count: p32(accCnt), perf_present: pu(present),
		srv_model: p32(sModel), srv_priority: p32(sPrio), srv_min_replicas: p32(sMin), srv_max_batch: p32(sMaxB),
		srv_keep_acc: pu(sKeep), srv_target_present: pu(sTgt),
		srv_slo_ttft: pf(sTTFT), srv_slo_itl: pf(sITL), srv_slo_tps: pf(sTPS), srv_arrival: pf(sArr),
		srv_in_tokens: p32(sIn), srv_out_tokens: p32(sOut),
		srv_cur_acc: p32(sCurAcc), srv_cur_replicas: p32(sCurRep), srv_cur_cost: pf(sCurCost),
		saturation_policy: C.int32_t(config.SaturatedAllocationPolicyEnum(d.Optimizer.Spec.SaturationPolicy)),
	}
	if d.Optimizer.Spec.Unlimited {
		sys.unlimited = 1
	}
	if d.Optimizer.Spec.DelayedBestEffort {
		sys.delayed_best_effort = 1
	}
	if err := m.ctx.err(C.wva_load_system(m.ctx.c, &sys), "wva_load_system"); err != nil {
		return nil, err
	}
	if err := m.ctx.err(C.wva_calculate(m.ctx.c), "wva_calculate"); err != nil {
		return nil, err
	}
	if err := m.ctx.err(C.wva_solve(m.ctx.c), "wva_solve"); err != nil {
		return nil, err
	}
	state := make([]uint8, S)
	oAcc, oRep, oBatch := i32(), i32(), i32()
	oCost, oITL, oTTFT := f32(), f32(), f32()
	out := C.wva_solution{state: pu(state), acc: p32(oAcc), num_replicas: p32(oRep), batch_size: p32(oBatch),
		cost: pf(oCost), itl: pf(oITL), ttft: pf(oTTFT)}
	if err := m.ctx.err(C.wva_get_solution(m.ctx.c, &out), "wva_get_solution"); err != nil {
		return nil, err
	}
	sol := &config.AllocationSolution{Spec: make(map[string]config.AllocationData, S)}
	for _, s := range d.Servers.Spec {
		i := srv.of[s.Name]
		if state[i] == C.WVA_ALLOC_NONE {
			continue // nil allocation: absent from the solution (system.go:308-311)
		}
		name := ""
		if state[i] == C.WVA_ALLOC_ACC {
			name = acc.names[oAcc[i]]
		}
		sol.Spec[s.Name] = config.AllocationData{Accelerator: name, NumReplicas: int(oRep[i]), MaxBatch: int(oBatch[i]),
			Cost: oCost[i], ITLAverage: oITL[i], TTFTAverage: oTTFT[i], Load: s.CurrentAlloc.Load}
	}
	return sol, nil
}

// SaturationAnalyzer satisfies interfaces.SaturationAnalyzer (saturation_analyzer.go:246-267): one model per call,
// exactly like the swap point Engine.RunSaturationAnalysis (engines/saturation/engine.go:779-795).  Batch callers
// (all models of a cycle in one launch) use AnalyzeBatch.
type SaturationAnalyzer struct{ ctx *Ctx }

func NewSaturationAnalyzer(ctx *Ctx) *SaturationAnalyzer { return &SaturationAnalyzer{ctx: ctx} }

type modelBatch struct {
	variants []string // ascending VariantName
	metrics  map[string][]interfaces.ReplicaMetrics
}

func groupByVariant(rm []interfaces.ReplicaMetrics) modelBatch {
	b := modelBatch{metrics: map[string][]interfaces.ReplicaMetrics{}}
	for _, r := range rm {
		b.metrics[r.VariantName] = append(b.metrics[r.VariantName], r) // slice order kept: sums are order dependent
	}
	for v := range b.metrics {
		b.variants = append(b.variants, v)
	}
	sort.Strings(b.variants)
	return b
}

func (a *SaturationAnalyzer) AnalyzeModelSaturation(ctx context.Context, modelID, namespace string,
	rm []interfaces.ReplicaMetrics, cfg interfaces.SaturationScalingConfig) (*interfaces.ModelSaturationAnalysis, error) {
	res, _, err := a.run(modelID, namespace, rm, cfg, nil)
	return res, err
}

func (a *SaturationAnalyzer) CalculateSaturationTargets(an *interfaces.ModelSaturationAnalysis,
	states []interfaces.VariantReplicaState) map[string]int {
	// the device computes analysis and targets in one pass; the analysis object carries its inputs back
	src, ok := analysisInputs[an]
	if !ok {
		return nil
	}
	_, targets, _ := a.run(an.ModelID, an.Namespace, src.rm, src.cfg, states)
	return targets
}

type analysisSrc struct {
	rm  []interfaces.ReplicaMetrics
	cfg interfaces.SaturationScalingConfig
}

var analysisInputs = map[*interfaces.ModelSaturationAnalysis]analysisSrc{}

func (a *SaturationAnalyzer) run(modelID, ns string, rm []interfaces.ReplicaMetrics, cfg interfaces.SaturationScalingConfig,
	states []interfaces.VariantReplicaState) (*interfaces.ModelSaturationAnalysis, map[string]int, error) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	b := groupByVariant(rm)
	stateOf := map[string]interfaces.VariantReplicaState{}
	for _, s := range states {
		stateOf[s.VariantName] = s
		if _, ok := b.metrics[s.VariantName]; !ok { // a state without metrics is still a variant of the model
			b.variants = append(b.variants, s.VariantName)
		}
	}
	sort.Strings(b.variants)
	V := len(b.variants)
	mvo := []int32{0, int32(V)}
	vro := make([]int32, V+1)
	var kv []float64
	var q []int64
	cost, cur, des, pen, has := make([]float64, V), make([]int32, V), make([]int32, V), make([]int32, V), make([]uint8, V)
	for i, v := range b.variants {
		for _, r := range b.metrics[v] {
			kv, q = append(kv, r.KvCacheUsage), append(q, int64(r.QueueLength))
		}
		vro[i+1] = int32(len(kv))
		if ms := b.metrics[v]; len(ms) > 0 {
			cost[i] = ms[0].Cost // analyzer.go:146-148
		}
		if s, ok := stateOf[v]; ok {
			cur[i], des[i], pen[i], has[i] = int32(s.CurrentReplicas), int32(s.DesiredReplicas), int32(s.PendingReplicas), 1
		}
	}
	c4 := [4][]float64{{cfg.KvCacheThreshold}, {cfg.QueueLengthThreshold}, {cfg.KvSpareTrigger}, {cfg.QueueSpareTrigger}}
	P := len(kv)
	target, rc, nsat := make([]int32, V), make([]int32, V), make([]int32, V)
	maxKv, avgKv, avgQ := make([]float64, V), make([]float64, V), make([]float64, V)
	maxQ := make([]int64, V)
	sat := make([]uint8, P)
	var mTot, mNon [1]int32
	var mKv, mQ [1]float64
	var flags [1]uint8
	in := C.wva_saturation_in{n_models: 1, n_variants: C.int64_t(V), n_replicas: C.int64_t(P),
		model_variant_off: (*C.int32_t)(unsafe.Pointer(&mvo[0])), variant_replica_off: (*C.int32_t)(unsafe.Pointer(&vro[0])),
		rep_kv: (*C.double)(ptrOrNil(kv)), rep_queue: (*C.int64_t)(ptrOrNil(q)),
		var_cost: (*C.double)(ptrOrNil(cost)), var_current: (*C.int32_t)(ptrOrNil(cur)),
		var_desired: (*C.int32_t)(ptrOrNil(des)), var_pending: (*C.int32_t)(ptrOrNil(pen)),
		var_has_state: (*C.uint8_t)(ptrOrNil(has)),
		cfg_kv_threshold: (*C.double)(unsafe.Pointer(&c4[0][0])), cfg_queue_threshold: (*C.double)(unsafe.Pointer(&c4[1][0])),
		cfg_kv_trigger: (*C.double)(unsafe.Pointer(&c4[2][0])), cfg_queue_trigger: (*C.double)(unsafe.Pointer(&c4[3][0]))}
	out := C.wva_saturation_out{var_target: (*C.int32_t)(ptrOrNil(target)), var_replica_count: (*C.int32_t)(ptrOrNil(rc)),
		var_non_saturated: (*C.int32_t)(ptrOrNil(nsat)), var_max_kv: (*C.double)(ptrOrNil(maxKv)),
		var_max_queue: (*C.int64_t)(ptrOrNil(maxQ)), var_avg_spare_kv: (*C.double)(ptrOrNil(avgKv)),
		var_avg_spare_queue: (*C.double)(ptrOrNil(avgQ)), rep_saturated: (*C.uint8_t)(ptrOrNil(sat)),
		mod_total_replicas: (*C.int32_t)(unsafe.Pointer(&mTot[0])), mod_non_saturated: (*C.int32_t)(unsafe.Pointer(&mNon[0])),
		mod_avg_spare_kv: (*C.double)(unsafe.Pointer(&mKv[0])), mod_avg_spare_queue: (*C.double)(unsafe.Pointer(&mQ[0])),
		mod_flags: (*C.uint8_t)(unsafe.Pointer(&flags[0]))}
	if err := a.ctx.err(C.wva_saturation_v1(a.ctx.c, &in, &out), "wva_saturation_v1"); err != nil {
		return nil, nil, err
	}
	an := &interfaces.ModelSaturationAnalysis{ModelID: modelID, Namespace: ns, TotalReplicas: int(mTot[0]),
		NonSaturatedCount: int(mNon[0]), AvgSpareKvCapacity: mKv[0], AvgSpareQueueLength: mQ[0],
		ShouldScaleUp: flags[0]&C.WVA_SAT_SCALE_UP != 0, ScaleDownSafe: flags[0]&C.WVA_SAT_SCALE_DOWN_SAFE != 0}
	if an.ShouldScaleUp {
		an.ScaleUpReason = scaleUpReason(mKv[0], mQ[0], cfg)
	}
	targets := map[string]int{}
	for i, v := range b.variants {
		if ms := b.metrics[v]; len(ms) > 0 {
			va := interfaces.VariantSaturationAnalysis{VariantName: v, AcceleratorName: ms[0].AcceleratorName, Cost: cost[i],
				ReplicaCount: int(rc[i]), NonSaturatedCount: int(nsat[i]), MaxKvCacheUsage: maxKv[i], MaxQueueLength: int(maxQ[i]),
				AvgSpareKvCapacity: avgKv[i], AvgSpareQueueLength: avgQ[i], SaturatedReplicas: []string{}}
			for j := vro[i]; j < vro[i+1]; j++ {
				if sat[j] != 0 {
					va.SaturatedReplicas = append(va.SaturatedReplicas, ms[j-vro[i]].PodName)
				}
			}
			an.VariantAnalyses = append(an.VariantAnalyses, va)
		}
		if target[i] >= 0 {
			targets[v] = int(target[i])
		}
	}
	analysisInputs[an] = analysisSrc{rm: rm, cfg: cfg}
	return an, targets, nil
}

// scaleUpReason formats the reason exactly as analyzer.go:199-225; the decision itself comes from the device.
func scaleUpReason(kv, q float64, cfg interfaces.SaturationScalingConfig) string {
	kvT, qT := kv < cfg.KvSpareTrigger, q < cfg.QueueSpareTrigger
	switch {
	case kvT && qT:
		return fmt.Sprintf("both KV spare (%.3f < %.3f) and queue spare (%.1f < %.1f)", kv, cfg.KvSpareTrigger, q, cfg.QueueSpareTrigger)
	case kvT:
		return fmt.Sprintf("KV spare Saturation low (%.3f < %.3f)", kv, cfg.KvSpareTrigger)
	case qT:
		return fmt.Sprintf("queue spare Saturation low (%.1f < %.1f)", q, cfg.QueueSpareTrigger)
	}
	return ""
}

func ptrOrNil[T any](s []T) unsafe.Pointer {
	if len(s) == 0 {
		return nil
	}
	return unsafe.Pointer(&s[0])
}

// Limiter satisfies pipeline.Limiter (limiter_interfaces.go:72-80): mutates the decisions in place exactly as
// DefaultLimiter.Limit (default_limiter.go:42-81).  limits = TypeInventory.limitByType after Refresh.
type Limiter struct {
	ctx    *Ctx
	name   string
	limits func(ctx context.Context) (map[string]int, error)
}

func (l *Limiter) Name() string { return l.name }

func (l *Limiter) Limit(ctx context.Context, ds []*interfaces.VariantDecision) error {
	if len(ds) == 0 {
		return nil
	}
	lim, err := l.limits(ctx)
	if err != nil {
		return fmt.Errorf("failed to refresh inventory: %w", err)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	names := make([]string, 0, len(lim))
	for t := range lim {
		names = append(names, t)
	}
	typ := newIndex(names)
	D, T := len(ds), len(typ.names)
	at, cur, tgt, gpr := make([]int32, D), make([]int32, D), make([]int32, D), make([]int32, D)
	spare, cost := make([]float64, D), make([]float64, D)
	for i, d := range ds {
		if t, ok := typ.of[d.AcceleratorName]; ok && d.AcceleratorName != "" {
			at[i] = t
		} else {
			at[i] = -1 // "" or a type without a pool: nothing can be allocated (type_inventory.go:353-361)
		}
		cur[i], tgt[i], gpr[i] = int32(d.CurrentReplicas), int32(d.TargetReplicas), int32(d.GPUsPerReplica)
		spare[i], cost[i] = d.SpareCapacity, d.Cost
	}
	limits := make([]int32, T)
	for t, n := range lim {
		limits[typ.of[t]] = int32(n)
	}
	oT, oG, oL := make([]int32, D), make([]int32, D), make([]uint8, D)
	rc := C.wva_limit(l.ctx.c, C.int64_t(D), C.int32_t(T), (*C.int32_t)(ptrOrNil(at)), (*C.int32_t)(ptrOrNil(cur)),
		(*C.int32_t)(ptrOrNil(tgt)), (*C.int32_t)(ptrOrNil(gpr)), (*C.double)(ptrOrNil(spare)), (*C.double)(ptrOrNil(cost)),
		(*C.int32_t)(ptrOrNil(limits)), (*C.int32_t)(ptrOrNil(oT)), (*C.int32_t)(ptrOrNil(oG)), (*C.uint8_t)(ptrOrNil(oL)))
	if err := l.ctx.err(rc, "wva_limit"); err != nil {
		return fmt.Errorf("allocation algorithm failed: %w", err)
	}
	for i, d := range ds {
		d.TargetReplicas, d.GPUsAllocated, d.WasLimited = int(oT[i]), int(oG[i]), oL[i] != 0
		if d.WasLimited {
			d.LimitedBy = l.name
		}
		d.AddDecisionStep(l.name, stepReason(d), d.WasLimited) // default_limiter.go:84-113
	}
	return nil
}

func stepReason(d *interfaces.VariantDecision) string {
	ch := d.TargetReplicas - d.CurrentReplicas
	switch {
	case ch <= 0:
		return fmt.Sprintf("no scale-up (target=%d, current=%d)", d.TargetReplicas, d.CurrentReplicas)
	case d.WasLimited:
		return fmt.Sprintf("limited: allocated %d GPUs for +%d replicas", d.GPUsAllocated, ch)
	default:
		return fmt.Sprintf("allocated %d GPUs for +%d replicas", d.GPUsAllocated, ch)
	}
}

// ---- V2 pipeline (SURVEY 8f.1-2) ----------------------------------------------------------------------------------------
//
// CostAwareOptimizer satisfies pipeline.ScalingOptimizer (optimizer_interfaces.go:23-30) like the reference's
// CostAwareOptimizer (cost_aware_optimizer.go:39-72): every model of the cycle in one launch.  Index space per model =
// Result.VariantCapacities slice order (ties of the reference's unstable sorts resolve to it).
type CostAwareOptimizer struct{ ctx *Ctx }

func NewCostAwareOptimizer(ctx *Ctx) *CostAwareOptimizer { return &CostAwareOptimizer{ctx: ctx} }
func (o *CostAwareOptimizer) Name() string                { return "cost-aware" }

func (o *CostAwareOptimizer) Optimize(ctx context.Context, reqs []pipeline.ModelScalingRequest,
	_ []*pipeline.ResourceConstraints) []interfaces.VariantDecision {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	mvo := []int32{0}
	var required, spare, cost, capacity []float64
	var has []uint8
	var cur []int32
	for _, r := range reqs {
		st := map[string]interfaces.VariantReplicaState{}
		for _, s := range r.VariantStates {
			st[s.VariantName] = s
		}
		if r.Result != nil {
			for _, vc := range r.Result.VariantCapacities {
				cur = append(cur, int32(st[vc.VariantName].CurrentReplicas))
				cost, capacity = append(cost, vc.Cost), append(capacity, vc.PerReplicaCapacity)
			}
			required, spare, has = append(required, r.Result.RequiredCapacity), append(spare, r.Result.SpareCapacity), append(has, 1)
		} else {
			required, spare, has = append(required, 0), append(spare, 0), append(has, 0)
		}
		mvo = append(mvo, int32(len(cur)))
	}
	target := make([]int32, len(cur))
	rc := C.wva_cost_aware_optimize(o.ctx.c, C.int64_t(len(reqs)), C.int64_t(len(cur)), (*C.int32_t)(unsafe.Pointer(&mvo[0])),
		(*C.double)(ptrOrNil(required)), (*C.double)(ptrOrNil(spare)), (*C.uint8_t)(ptrOrNil(has)), (*C.int32_t)(ptrOrNil(cur)),
		(*C.double)(ptrOrNil(cost)), (*C.double)(ptrOrNil(capacity)), (*C.int32_t)(ptrOrNil(target)))
	if o.ctx.err(rc, "wva_cost_aware_optimize") != nil {
		return nil // the engine's safety net emits the previous decisions (engine.go:1022-1095)
	}
	var out []interfaces.VariantDecision
	for m, r := range reqs {
		if r.Result == nil {
			continue
		}
		st := map[string]interfaces.VariantReplicaState{}
		for _, s := range r.VariantStates {
			st[s.VariantName] = s
		}
		for k, vc := range r.Result.VariantCapacities {
			t, c := int(target[int(mvo[m])+k]), st[vc.VariantName].CurrentReplicas
			d := interfaces.VariantDecision{VariantName: vc.VariantName, ModelID: r.ModelID, Namespace: r.Namespace,
				AcceleratorName: vc.AcceleratorName, Cost: vc.Cost, CurrentReplicas: c, TargetReplicas: t}
			switch { // buildDecisions, cost_aware_optimizer.go:241-276
			case t > c:
				d.Action, d.Reason = interfaces.ActionScaleUp, fmt.Sprintf("V2 scale-up (optimizer: cost-aware, required: %.0f)", r.Result.RequiredCapacity)
			case t < c:
				d.Action, d.Reason = interfaces.ActionScaleDown, fmt.Sprintf("V2 scale-down (optimizer: cost-aware, spare: %.0f)", r.Result.SpareCapacity)
			default:
				d.Action, d.Reason = interfaces.ActionNoChange, "V2 steady state"
			}
			out = append(out, d)
		}
	}
	return out
}

// Enforcer mirrors pipeline.Enforcer.EnforcePolicy (enforcer.go:55-83).  The request-count lookup and the
// scale-to-zero configuration stay in Go; index order = ascending variant name (the tie-break compares names).
type Enforcer struct {
	ctx          *Ctx
	requestCount pipeline.RequestCountFuncType
}

func NewEnforcer(ctx *Ctx, f pipeline.RequestCountFuncType) *Enforcer { return &Enforcer{ctx: ctx, requestCount: f} }

func (e *Enforcer) EnforcePolicy(ctx context.Context, modelID, namespace string, targets map[string]int,
	analyses []interfaces.VariantSaturationAnalysis, s2z intconfig.ScaleToZeroConfigData) (map[string]int, bool) {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	names := make([]string, 0, len(targets))
	for n := range targets {
		names = append(names, n)
	}
	sort.Strings(names)
	costOf := map[string]float64{}
	for _, va := range analyses {
		costOf[va.VariantName] = va.Cost
	}
	enabled := intconfig.IsScaleToZeroEnabled(s2z, modelID)
	var count float64
	var failed uint8
	if enabled {
		c, err := e.requestCount(ctx, modelID, namespace, intconfig.ScaleToZeroRetentionPeriod(s2z, modelID))
		if err != nil {
			failed = 1
		}
		count = c
	}
	mvo := []int32{0, int32(len(names))}
	cost, has, tgt := make([]float64, len(names)), make([]uint8, len(names)), make([]int32, len(names))
	for i, n := range names {
		if c, ok := costOf[n]; ok {
			cost[i], has[i] = c, 1
		}
		tgt[i] = int32(targets[n])
	}
	on := uint8(0)
	if enabled {
		on = 1
	}
	var applied uint8
	rc := C.wva_enforce(e.ctx.c, 1, C.int64_t(len(names)), (*C.int32_t)(unsafe.Pointer(&mvo[0])), (*C.uint8_t)(unsafe.Pointer(&on)),
		(*C.double)(unsafe.Pointer(&count)), (*C.uint8_t)(unsafe.Pointer(&failed)), (*C.double)(ptrOrNil(cost)),
		(*C.uint8_t)(ptrOrNil(has)), (*C.int32_t)(ptrOrNil(tgt)), (*C.uint8_t)(unsafe.Pointer(&applied)))
	if e.ctx.err(rc, "wva_enforce") != nil {
		return targets, false
	}
	for i, n := range names {
		targets[n] = int(tgt[i])
	}
	return targets, applied != 0
}

// The V2 analyzer wrapper (`wva_saturation_v2`) belongs INSIDE package saturation_v2: the k2 priority chain, its
// rolling history and the capacity store are unexported there (analyzer.go:17-24, history.go, capacity_store.go) and
// stay as they are; `computeReplicaCapacity` keeps calling `computeK2` and the store, the five arithmetic lines around
// them and `aggregateByVariant`'s sums / median move behind the call.  `pipeline.py SaturationAnalyzerV2` is the
// executable statement of that split.
