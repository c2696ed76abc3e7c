// capi.cu — implementation of the C-ABI declared in include/wva_b200.h.
// Host-side plumbing only (context, device arenas, launches, timing); all of the
// arithmetic lives in the kernels included below.  No CPU fallback exists: every
// entry point either runs CUDA kernels or returns an error status.
#include "../../include/wva_b200.h"
#include "wva_core.cuh"
#include "sizer_kernel.cuh"
#include "sizer_warp_kernel.cuh"
#include "sizer_lane_kernel.cuh"
#include "sizer_pool_kernel.cuh"
#include "sizer_probe.cuh"
#include "solve_kernels.cuh"
#include "grid_kernel.cuh"
#include "saturation_kernel.cuh"
#include "limiter_kernel.cuh"
#include "pipeline_v2_kernel.cuh"
#include "k2_history_kernel.cuh"
#include "overflow_slow_kernel.cuh"
#include "greedy_solve.cuh"
#include "greedy_sweep.cuh"
#include "mm1k_kernel.cuh"
#include "recalc_kernel.cuh"
#include "ingest_scatter.hpp"

#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

using namespace wva;

// ------------------------------------------------------------------ small helpers
// growable allocation that its owner frees by being deleted (with the owner's device current): device memory (DevBuf)
// or pinned host staging (PinBuf)
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf(Buf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf& operator=(Buf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~Buf() { if (p) Free(p); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) Free(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 256;
    cudaError_t e = Alloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
};
inline cudaError_t dev_alloc(void** p, size_t n) { return cudaMalloc(p, n); }
inline cudaError_t pin_alloc(void** p, size_t n) { return cudaMallocHost(p, n); }
using DevBuf = Buf<dev_alloc, cudaFree>;
using PinBuf = Buf<pin_alloc, cudaFreeHost>;

// ------------------------------------------------------------------ column lists
// Every struct-of-arrays of the C-ABI is declared once, in the order its arena is laid out: X(field, count, flags).  The
// public struct (include/wva_b200.h) and its device view share the field names, so one visitor per list walks any of
// them: each_<list>(n, f, s...) calls f(count, flags, s.field...) for every column.  Element sizes come from the fields.
// Counts are written over the extents `n`; over the entities BEFORE a block (servers before a rank's block, models /
// variants / replicas before a group member's block) a column's count is its offset to that block.
struct Ext { size_t A = 0, T = 0, M = 0, S = 0, V = 0, P = 0, R = 0, N = 0; };   // P: pairs or replicas, R: grid levels,
                                                                                // N: capacity-store slots
enum { COL_OPT = 1,       // input the caller may leave NULL: its view is NULL too
       COL_DETAIL = 2,    // V1 saturation analysis field: written only by a detail run
       COL_CYCLE = 4,     // server column wva_update_servers replaces in place (ServerLoadSpec and CurrentAlloc)
       COL_SRV = 8,       // server column ([S]): wva_update_server_set replaces the set of them
       COL_TAB = 16 };    // accelerator or perf table column: wva_update_tables replaces them in place
#define SRV_CYCLE (COL_SRV | COL_CYCLE)

// The model tables come first and the server columns last: a new server set keeps the arena's prefix as it is.
#define SYS_COLS(X)                                                                                                    \
  X(acc_cost, n.A, COL_TAB) X(acc_multiplicity, n.A, COL_TAB) X(acc_type, n.A, COL_TAB) X(type_count, n.T, 0)          \
  X(perf_alpha, n.M * n.A, COL_TAB) X(perf_beta, n.M * n.A, COL_TAB) X(perf_gamma, n.M * n.A, COL_TAB)                 \
  X(perf_max_batch, n.M * n.A, COL_TAB) X(perf_at_tokens, n.M * n.A, COL_TAB) X(perf_acc_count, n.M * n.A, COL_TAB)    \
  X(perf_present, n.M * n.A, COL_TAB)                                                                                  \
  X(srv_model, n.S, COL_SRV) X(srv_priority, n.S, COL_SRV) X(srv_min_replicas, n.S, COL_SRV)                           \
  X(srv_max_batch, n.S, COL_SRV) X(srv_keep_acc, n.S, COL_SRV) X(srv_target_present, n.S, COL_SRV)                     \
  X(srv_slo_ttft, n.S, COL_SRV) X(srv_slo_itl, n.S, COL_SRV) X(srv_slo_tps, n.S, COL_SRV)                              \
  X(srv_arrival, n.S, SRV_CYCLE) X(srv_in_tokens, n.S, SRV_CYCLE) X(srv_out_tokens, n.S, SRV_CYCLE)                    \
  X(srv_cur_acc, n.S, SRV_CYCLE) X(srv_cur_replicas, n.S, SRV_CYCLE) X(srv_cur_cost, n.S, SRV_CYCLE)
#define CAND_COLS(X)                                                                                                   \
  X(state, n.P, 0) X(num_replicas, n.P, 0) X(batch_size, n.P, 0) X(cost, n.P, 0) X(value, n.P, 0) X(itl, n.P, 0)      \
  X(ttft, n.P, 0) X(rho, n.P, 0) X(max_arrv_rate, n.P, 0) X(n_solves, n.P, COL_OPT)
#define SOL_COLS(X)                                                                                                    \
  X(state, n.S, 0) X(acc, n.S, 0) X(num_replicas, n.S, 0) X(batch_size, n.S, 0) X(cost, n.S, 0) X(value, n.S, 0)      \
  X(itl, n.S, 0) X(ttft, n.S, 0) X(rho, n.S, 0) X(max_arrv_rate, n.S, 0)
// the variant and model columns of wva_saturation_in, which the ingest column arena lays out in the same order
#define SAT_IN_SHARED_COLS(X)                                                                                          \
  X(var_cost, n.V, 0) X(var_current, n.V, 0) X(var_desired, n.V, 0) X(var_pending, n.V, 0)                             \
  X(cfg_kv_threshold, n.M, 0) X(cfg_queue_threshold, n.M, 0) X(cfg_kv_trigger, n.M, 0) X(cfg_queue_trigger, n.M, 0)
#define SAT_IN_COLS(X)                                                                                                 \
  X(model_variant_off, n.M + 1, 0) X(variant_replica_off, n.V + 1, 0) X(rep_kv, n.P, 0) X(rep_queue, n.P, 0)           \
  X(var_cost, n.V, 0) X(var_current, n.V, 0) X(var_desired, n.V, 0) X(var_pending, n.V, 0)                             \
  X(var_has_state, n.V, COL_OPT)                                                                                       \
  X(cfg_kv_threshold, n.M, 0) X(cfg_queue_threshold, n.M, 0) X(cfg_kv_trigger, n.M, 0) X(cfg_queue_trigger, n.M, 0)
#define SAT_OUT_COLS(X)                                                                                                \
  X(var_target, n.V, 0) X(var_replica_count, n.V, COL_DETAIL) X(var_non_saturated, n.V, COL_DETAIL)                    \
  X(var_max_kv, n.V, COL_DETAIL) X(var_max_queue, n.V, COL_DETAIL) X(var_avg_spare_kv, n.V, COL_DETAIL)                \
  X(var_avg_spare_queue, n.V, COL_DETAIL) X(rep_saturated, n.P, COL_DETAIL) X(mod_total_replicas, n.M, COL_DETAIL)     \
  X(mod_non_saturated, n.M, COL_DETAIL) X(mod_avg_spare_kv, n.M, COL_DETAIL) X(mod_avg_spare_queue, n.M, COL_DETAIL)   \
  X(mod_flags, n.M, 0)
#define V2_IN_COLS(X)                                                                                                  \
  X(model_variant_off, n.M + 1, 0) X(variant_replica_off, n.V + 1, 0) X(rep_total_kv_tokens, n.P, 0)                   \
  X(rep_tokens_in_use, n.P, 0) X(rep_queue_length, n.P, 0) X(rep_avg_input_tokens, n.P, 0)                             \
  X(rep_avg_output_tokens, n.P, 0) X(rep_prefix_hit_rate, n.P, 0) X(rep_k2, n.P, 0) X(rep_slice_order, n.P, COL_OPT)   \
  X(var_current, n.V, 0) X(var_pending, n.V, 0) X(var_fallback_capacity, n.V, 0) X(cfg_kv_threshold, n.M, 0)          \
  X(cfg_scale_up_threshold, n.M, 0) X(cfg_scale_down_boundary, n.M, 0) X(sched_queue_size, n.M, COL_OPT)               \
  X(sched_queue_bytes, n.M, COL_OPT)
#define V2_OUT_COLS(X)                                                                                                 \
  X(rep_k1, n.P, 0) X(rep_effective, n.P, 0) X(rep_demand, n.P, 0) X(rep_saturated, n.P, 0) X(var_ready, n.V, 0)      \
  X(var_per_replica_capacity, n.V, 0) X(var_total_capacity, n.V, 0) X(var_total_demand, n.V, 0)                        \
  X(var_utilization, n.V, 0) X(mod_total_supply, n.M, 0) X(mod_total_demand, n.M, 0) X(mod_utilization, n.M, 0)        \
  X(mod_required_capacity, n.M, 0) X(mod_spare_capacity, n.M, 0)
// the replica grid's optional outputs (wva_grid_run with full != 0)
#define GRID_COLS(X)                                                                                                   \
  X(ok, n.P * n.R, 0) X(ttft, n.P * n.R, 0) X(itl, n.P * n.R, 0) X(rho, n.P * n.R, 0) X(tput, n.P * n.R, 0)
// The ingest arenas (wva_ingest_create / wva_ingest_v2_create), over S pod slots and N store slots: the caller's host
// image and the device image of each arena share the offsets.  The decision-mode lists follow the plain ones in the
// same arenas.
#define INGEST_COLS(X) X(kv, n.S, 0) X(queue, n.S, 0) X(has, n.S, 0) SAT_IN_SHARED_COLS(X)
#define INGEST_RES_COLS(X)                                                                                             \
  X(partials, 8, 0) X(var_target, n.V, 0) X(var_replica_count, n.V, 0) X(var_non_saturated, n.V, 0)                  \
  X(var_avg_spare_kv, n.V, 0) X(var_avg_spare_queue, n.V, 0) X(mod_flags, n.M, 0) X(mod_total_replicas, n.M, 0)
#define INGEST_DEC_COLS(X)                                                                                             \
  X(var_accelerator_type, n.V, 0) X(var_gpus_per_replica, n.V, 0) X(mod_scale_to_zero_enabled, n.M, 0)                \
  X(mod_request_count, n.M, 0) X(mod_request_error, n.M, 0) X(type_limit, n.T + 1, 0) X(enable_limiter, 1, 0)
#define INGEST_DEC_RES_COLS(X)                                                                                         \
  X(has_decision, n.V, 0) X(original_target, n.V, 0) X(target, n.V, 0) X(gpus_allocated, n.V, 0)                     \
  X(was_limited, n.V, 0) X(action, n.V, 0) X(mod_enforcer_applied, n.M, 0)
#define INGEST_V2_COLS(X)                                                                                              \
  X(kv, n.S, 0) X(queue, n.S, 0) X(num_gpu_blocks, n.S, 0) X(block_size, n.S, 0) X(avg_output_tokens, n.S, 0)         \
  X(avg_input_tokens, n.S, 0) X(prefix_hit_rate, n.S, 0) X(has, n.S, 0) X(var_cost, n.V, 0) X(var_current, n.V, 0)    \
  X(var_pending, n.V, 0) X(var_name_rank, n.V, 0) X(cfg_kv_threshold, n.M, 0) X(cfg_queue_threshold, n.M, 0)          \
  X(cfg_scale_up_threshold, n.M, 0) X(cfg_scale_down_boundary, n.M, 0) X(mod_scale_to_zero_enabled, n.M, 0)           \
  X(mod_request_count, n.M, 0) X(mod_request_error, n.M, 0) X(slot_max_batched_tokens, n.N, 0)                        \
  X(slot_max_num_seqs, n.N, 0)
// the analyze launch's results (the replica columns hold every slot, with room to spare)
#define INGEST_V2_ANALYZE_COLS(X)                                                                                      \
  X(variant_replica_off, n.V + 2, 0) X(rep_pod, n.S + 4, 0) X(rep_total_kv_tokens, n.S + 2, 0)                        \
  X(slot_last_rep, n.N, 0) X(slot_effective, n.N, 0) X(var_no_data, n.V, 0) X(mod_has_request, n.M, 0)               \
  X(mod_avg_input_tokens, n.M, 0) X(mod_avg_output_tokens, n.M, 0)
// the decide launch's results: its own, then the analyzer's outputs (SatV2Out's fields)
#define INGEST_V2_DECIDE_COLS(X)                                                                                       \
  X(var_optimizer_target, n.V, 0) X(var_target, n.V, 0) X(var_action, n.V, 0) X(mod_enforced, n.M, 0)
#define INGEST_V2_DECIDE_SAT_COLS(X)                                                                                   \
  X(var_ready, n.V, 0) X(var_per_replica_capacity, n.V, 0) X(var_total_capacity, n.V, 0) X(var_total_demand, n.V, 0)  \
  X(var_utilization, n.V, 0) X(mod_total_supply, n.M, 0) X(mod_total_demand, n.M, 0) X(mod_utilization, n.M, 0)       \
  X(mod_required_capacity, n.M, 0) X(mod_spare_capacity, n.M, 0)

#define COL_VISIT_(field, count, flags) f((size_t)(count), flags, s.field...);
#define COL_VISITOR_(name, LIST) \
  template <class F, class... Structs> static void name(const Ext& n, F&& f, Structs&&... s) { LIST(COL_VISIT_) }
COL_VISITOR_(each_sys, SYS_COLS)
COL_VISITOR_(each_cand, CAND_COLS)
COL_VISITOR_(each_sol, SOL_COLS)
COL_VISITOR_(each_sat_shared, SAT_IN_SHARED_COLS)
COL_VISITOR_(each_sat_in, SAT_IN_COLS)
COL_VISITOR_(each_sat_out, SAT_OUT_COLS)
COL_VISITOR_(each_v2_in, V2_IN_COLS)
COL_VISITOR_(each_v2_out, V2_OUT_COLS)
COL_VISITOR_(each_grid, GRID_COLS)
COL_VISITOR_(each_ingest, INGEST_COLS)
COL_VISITOR_(each_ingest_res, INGEST_RES_COLS)
COL_VISITOR_(each_ingest_dec, INGEST_DEC_COLS)
COL_VISITOR_(each_ingest_dec_res, INGEST_DEC_RES_COLS)
COL_VISITOR_(each_ingest_v2, INGEST_V2_COLS)
COL_VISITOR_(each_ingest_v2_analyze, INGEST_V2_ANALYZE_COLS)
COL_VISITOR_(each_ingest_v2_decide, INGEST_V2_DECIDE_COLS)
COL_VISITOR_(each_ingest_v2_decide_sat, INGEST_V2_DECIDE_SAT_COLS)
#undef COL_VISITOR_
#undef COL_VISIT_

// Column functors: f(count, flags, view field, caller's field).  They are called through the lists above, and directly
// for the few columns that belong to one entry point only.

// bump allocator over one arena: every sub-array 256-byte aligned.  As a functor it lays out the next column and, once
// the arena has a base, points the view's field at it; a pass without a base only sizes the arena.
struct Layout {
  char* base = nullptr;
  size_t off = 0;
  size_t take(size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; }
  template <class T, class... H> void operator()(size_t n, int, T*& p, H&&...) {
    const size_t o = take(n * sizeof(T));
    if (base) p = (T*)(base + o);
  }
};
// copies the columns the caller supplied (non-NULL, not empty) into the view (H2D) or out of it (D2H); keeps the first error
struct Copy {
  cudaStream_t s;
  cudaMemcpyKind kind;
  cudaError_t e = cudaSuccess;
  template <class T, class H> void operator()(size_t n, int, T* d, H* h) {
    if (!h || !n || e != cudaSuccess) return;
    const bool up = kind == cudaMemcpyHostToDevice;
    e = cudaMemcpyAsync(up ? (void*)d : (void*)h, up ? (const void*)h : (const void*)d, n * sizeof(T), kind, s);
  }
};
// lays out an input arena and copies the caller's arrays into it; an optional column the caller left NULL is NULL
struct Upload : Layout {
  Copy copy;
  explicit Upload(cudaStream_t s) : copy{s, cudaMemcpyHostToDevice} {}
  template <class T, class H> void operator()(size_t n, int flags, T*& d, H* h) {
    const size_t o = take(n * sizeof(T));
    if (!base) return;
    d = (h || !(flags & COL_OPT)) ? (T*)(base + o) : nullptr;
    copy(n, flags, d, h);
  }
};
// true once a column that is not optional and not empty was left NULL by the caller
struct Missing {
  bool any = false;
  template <class T, class H> void operator()(size_t n, int flags, T*, H* h) { any |= n && !h && !(flags & COL_OPT); }
};

// visits the server columns of S servers that carry every bit of `flag` (COL_SRV: all of them; COL_CYCLE: the per-cycle
// ones) and nothing else
template <int FLAG, class F, class... Structs> static void each_srv(size_t S, F&& f, Structs&&... s) {
  Ext n;
  n.S = S;
  each_sys(n, [&](size_t c, int flags, auto&&... col) { if ((flags & FLAG) == FLAG) f(c, flags, col...); }, s...);
}
template <class F, class... Structs> static void each_cycle(size_t S, F&& f, Structs&&... s) {
  each_srv<COL_CYCLE>(S, f, s...);
}
template <class F, class... Structs> static void each_server(size_t S, F&& f, Structs&&... s) {
  each_srv<COL_SRV>(S, f, s...);
}

// visits the accelerator and perf table columns of A accelerators and M models (not type_count: wva_set_capacity's)
template <class F, class... Structs> static void each_table(size_t A, size_t M, F&& f, Structs&&... s) {
  Ext n;
  n.A = A; n.M = M;
  each_sys(n, [&](size_t c, int flags, auto&&... col) { if (flags & COL_TAB) f(c, flags, col...); }, s...);
}

// The preconditions of the table columns, shared by wva_load_system and wva_update_tables: every array non-NULL,
// acc_type in [0, T), and the service coefficients of every present perf row finite and >= 0.  Returns the violated
// rule, or nullptr.
static const char* check_table_columns(const wva_system& s, size_t A, size_t T, size_t M) {
  Missing miss;
  SysView none = {};
  each_table(A, M, miss, none, s);
  if (miss.any) return "a required array is NULL";
  for (size_t a = 0; a < A; a++)
    if (s.acc_type[a] < 0 || s.acc_type[a] >= (int)T) return "acc_type out of range";
  // ServiceParms (pkg/analyzer/queueanalyzer.go:33-38) are measured service-time coefficients: finite and >= 0.  A
  // negative or NaN coefficient makes arrival rates negative (QueueModel.Solve's gate, queuemodel.go:31) or NaN and
  // the sizing meaningless; it is rejected here instead of being carried into the kernels.
  for (size_t i = 0; i < M * A; i++) {
    if (!s.perf_present[i]) continue;
    const float a = s.perf_alpha[i], b = s.perf_beta[i], g = s.perf_gamma[i];
    if (!(a >= 0.0f && b >= 0.0f && g >= 0.0f) || a > 3.0e38f || b > 3.0e38f || g > 3.0e38f)
      return "perf_alpha / perf_beta / perf_gamma must be finite and >= 0";
  }
  return nullptr;
}

// The preconditions of the per-cycle columns, shared by wva_load_system and wva_update_servers: every array non-NULL
// and srv_cur_acc an accelerator index or a WVA_CUR_ACC_* sentinel.  Returns the violated rule, or nullptr.
static const char* check_cycle_columns(const wva_system& s, size_t S, int A) {
  Missing miss;
  SysView none = {};
  each_cycle(S, miss, none, s);
  if (miss.any) return "a required array is NULL";
  for (size_t i = 0; i < S; i++)
    if (s.srv_cur_acc[i] >= A || s.srv_cur_acc[i] < WVA_CUR_ACC_UNKNOWN) return "srv_cur_acc out of range";
  return nullptr;
}
// The preconditions of all server columns, shared by wva_load_system and wva_update_server_set: the per-cycle ones, and
// every other server array non-NULL with srv_model below M (-1 = unknown model).  Returns the violated rule, or nullptr.
static const char* check_server_columns(const wva_system& s, size_t S, int A, int M) {
  Missing miss;
  SysView none = {};
  each_server(S, miss, none, s);
  if (miss.any) return "a required array is NULL";
  for (size_t i = 0; i < S; i++)
    if (s.srv_model[i] >= M) return "srv_model out of range";
  return check_cycle_columns(s, S, A);
}

// Sizes an arena with a pass of `lay` over a copy of `f` that has no base, reserves it, then runs `lay` over `f` with the
// arena as its base.  Nothing is bound and nothing copied unless the reservation succeeds.
template <class F, class Lay> static cudaError_t lay_out(DevBuf& buf, F& f, Lay&& lay) {
  F sizing = f;
  lay(sizing);
  const cudaError_t e = buf.reserve(sizing.off + 256);
  if (e == cudaSuccess) { f.base = (char*)buf.p; lay(f); }
  return e;
}

// Lays out an arena that has a page-locked host image and a device image at the same offsets: f(count, flags, host
// field, device field) binds both to the column.  The two fields may differ in type, not in element size.
struct Twin : Layout {
  char* host = nullptr;
  template <class T, class U> void operator()(size_t n, int, T*& h, U*& d) {
    static_assert(sizeof(T) == sizeof(U), "one element size in both images");
    const size_t o = take(n * sizeof(T));
    if (base) { h = (T*)(host + o); d = (U*)(base + o); }
  }
};
// lay_out for a Twin: the host image (zeroed) and the device image reserved, then every column bound.  Returns the
// arena's bytes (0 if a reservation fails: `e` says why).
template <class Lay> static size_t lay_out(PinBuf& hbuf, DevBuf& dbuf, Lay&& lay, cudaError_t& e) {
  Twin f;
  lay(f);
  const size_t bytes = f.off + 256;
  if ((e = hbuf.reserve(bytes)) != cudaSuccess || (e = dbuf.reserve(bytes)) != cudaSuccess) return 0;
  memset(hbuf.p, 0, bytes);
  f = Twin{};
  f.base = (char*)dbuf.p; f.host = (char*)hbuf.p;
  lay(f);
  return bytes;
}

struct GridState {   // results of the last wva_grid_run, resident in HBM
  int R = 0;
  bool full = false, ran = false;
  bool current = false;        // the resident grid comes from wva_grid_run / wva_grid_update on the loaded system
  DevBuf buf, defer;
  GridOut view = {};
  GridCounters* ctr = nullptr;
  int* nmax = nullptr;         // device word of the max batch pass
  GridOverflowList ovf = {};   // the block's float64-overflow list, also used by wva_grid_update
};
// Lays out the grid buffer of P pairs at R levels through `f`: the counters, the max batch word, the frontier, the
// float64-overflow list (grid_kernel.cuh: GridOverflowList; 16 levels per pair on average, as the deferral list) and,
// with full outputs, the level arrays last.
template <class F> static void grid_columns(F& f, size_t P, int R, bool full, GridCounters*& ctr, int*& nmax, GridOut& view,
                                            GridOverflowList& ovf) {
  const size_t n = P * (size_t)R;
  ovf.cap = std::min<unsigned long long>({(unsigned long long)n, (unsigned long long)P * 16 + 1024, 0x7fffffffull});
  Ext levels;
  levels.P = P; levels.R = (size_t)R;
  f(1, 0, ctr); f(1, 0, nmax); f(P, 0, view.frontier); f(ovf.cap, 0, ovf.items);
  if (full) each_grid(levels, f, view);
}
struct SatState {    // resident inputs / outputs of the saturation model
  bool uploaded = false, ran = false;
  long long M = 0, V = 0, P = 0;
  DevBuf in, out, desc;
  SatIn vin = {};
  SatOut vout = {};
};

struct wva_ctx {
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[8] = {};
  std::string last_error;
  long long launches = 0;
  wva_timing timing = {};

  // queueing system
  bool loaded = false, calculated = false, solved = false;
  bool sized = false;               // the resident candidates come from wva_calculate / wva_recalculate on this ctx
  bool marked = false;              // `marks` holds the marks of a wva_update_servers since then (else all clear)
  bool grid_marked = false;         // `grid_marks` holds the load changes since the last wva_grid_run / wva_grid_update
  bool table_marked = false;        // tmarks.size_* hold the table changes since the last wva_calculate / wva_recalculate
  bool table_grid_marked = false;   // tmarks.grid_row holds those since the last wva_grid_run / wva_grid_update
  bool force_lane_sizer = false;
  int gang_refill = -1;             // lock-step lane sizer: a warp refills only when all its lanes are idle; -1 = by size
  int length_sort = -1;             // lane sizer pulls items through the probe-sorted permutation (sizer_probe.cuh); -1 = by size
  int table_mode = 0;        // WVA_OPT_TABLE_MODE
  int greedy_mode = 0;       // WVA_OPT_GREEDY_MODE
  int grid_defer = 0;        // WVA_OPT_GRID_DEFER
  int lane_sizer_mode = 2;   // the sizer mode WVA_OPT_FORCE_LANE_SIZER forces while force_lane_sizer is set (launch_sizer)
  int A = 0, T = 0, M = 0, S = 0;
  uint8_t unlimited = 1, delayed = 0;
  int policy = 0;
  DevBuf sys_arena, cand_arena, sol_arena, scratch, gtab, greedy_ws, split_ws, order_ws, pool_ws;
  DevBuf marks, grid_marks, cycle_in, recalc_ws, gather_ws;   // wva_update_servers / wva_recalculate / wva_grid_update
  DevBuf table_marks, pairs_ws;     // wva_update_tables: its marks (tmarks); the pair list of a table-marked update
  TableMarks tmarks = {};
  PinBuf stage_in, stage_out;
  SysView sys = {};
  CandView cand = {};
  SolView sol = {};
  long long* d_type_count = nullptr;
  double* d_type_cost = nullptr;
  SizerCounters* d_ctr = nullptr;   // in scratch
  // generic io arenas for saturation / limiter / grid / mm1k
  DevBuf io_in, io_out;
  GridState grid;
  SatState sat;
  // multi-GPU (comm.inl): one NCCL communicator, contiguous block of servers per rank
  void* comm = nullptr;             // ncclComm_t
  int world = 1, rank = 0;
  int shard_rows = 0;               // servers per rank block = ceil(S / world)
  int shard_lo = 0, shard_hi = 0;   // this ctx sizes servers [shard_lo, shard_hi)
  int shard_status = 0;             // status of the rank's last wva_calculate, agreed on by all ranks in wva_solve
  DevBuf comm_ws;
};

// views of the rank's block of servers: srv_* arrays and the candidate rows are plain arrays indexed by server, so a
// block is the same struct with offset pointers and n_servers = block size (models / accelerators stay global)
static Ext before_block(const wva_ctx* ctx) {   // the servers before the block (no models, accelerators or types)
  Ext n;
  n.S = (size_t)ctx->shard_lo; n.P = (size_t)ctx->shard_lo * ctx->A;
  return n;
}
static const auto advance = [](size_t n, int, auto*& p) { p += n; };
static SysView shard_sys(const wva_ctx* ctx) {
  SysView v = ctx->sys;
  each_sys(before_block(ctx), advance, v);
  v.n_servers = ctx->shard_hi - ctx->shard_lo;
  return v;
}
static CandView shard_cand(const wva_ctx* ctx) { CandView c = ctx->cand; each_cand(before_block(ctx), advance, c); return c; }
static SolView shard_sol(const wva_ctx* ctx) { SolView o = ctx->sol; each_sol(before_block(ctx), advance, o); return o; }
static int32_t comm_exchange_and_solve(wva_ctx* ctx);   // comm.inl
static int32_t comm_reduce_sat_partials(wva_ctx* ctx, long long* d_partials, long long* d_all);
static int32_t comm_agree_status(wva_ctx* ctx, int my_status, int* agreed);
static void comm_release(wva_ctx* ctx);

#define CK(call)                                                                         \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      ctx->last_error = std::string(#call) + ": " + cudaGetErrorString(e__);             \
      return (e__ == cudaErrorMemoryAllocation) ? WVA_ERR_NOMEM : WVA_ERR_CUDA;          \
    }                                                                                    \
  } while (0)

static float elapsed(wva_ctx* ctx, int a, int b) {
  float ms = 0;
  cudaEventElapsedTime(&ms, ctx->ev[a], ctx->ev[b]);
  return ms;
}

extern "C" {

const char* wva_strerror(int32_t code) {
  switch (code) {
    case WVA_OK: return "ok";
    case WVA_ERR_ARG: return "invalid argument";
    case WVA_ERR_CUDA: return "CUDA error";
    case WVA_ERR_NO_DEVICE: return "no usable CUDA device (this library has no CPU fallback)";
    case WVA_ERR_STATE: return "call order violated";
    case WVA_ERR_NOMEM: return "out of memory";
    case WVA_ERR_LIMIT: return "size exceeds kernel limits";
    default: return "unknown status";
  }
}

int32_t wva_create(int32_t device, wva_ctx** out) {
  if (!out) return WVA_ERR_ARG;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0 || device < 0 || device >= n) return WVA_ERR_NO_DEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return WVA_ERR_NO_DEVICE;
  if (prop.major != 9 || prop.minor != 0) return WVA_ERR_NO_DEVICE;  // kernels are built for sm_90a only
  if (cudaSetDevice(device) != cudaSuccess) return WVA_ERR_NO_DEVICE;
  wva_ctx* ctx = new (std::nothrow) wva_ctx();
  if (!ctx) return WVA_ERR_NOMEM;
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return WVA_ERR_CUDA; }
  for (auto& e : ctx->ev)
    if (cudaEventCreate(&e) != cudaSuccess) { delete ctx; return WVA_ERR_CUDA; }
  *out = ctx;
  return WVA_OK;
}

int32_t wva_destroy(wva_ctx* ctx) {
  if (!ctx) return WVA_ERR_ARG;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  comm_release(ctx);
  for (auto& e : ctx->ev) if (e) cudaEventDestroy(e);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return WVA_OK;
}

const char* wva_last_error(const wva_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }
int64_t wva_launch_count(const wva_ctx* ctx) { return ctx ? ctx->launches : 0; }

int32_t wva_last_timing(const wva_ctx* ctx, wva_timing* out) {
  if (!ctx || !out) return WVA_ERR_ARG;
  *out = ctx->timing;
  return WVA_OK;
}

// ------------------------------------------------------------------ load
int32_t wva_load_system(wva_ctx* ctx, const wva_system* s) {
  if (!ctx || !s) return WVA_ERR_ARG;
  if (s->n_acc < 0 || s->n_types < 0 || s->n_models < 0 || s->n_servers < 0) return WVA_ERR_ARG;
  if (s->n_types > WVA_MAX_TYPES) { ctx->last_error = "wva_load_system: more than 64 capacity types"; return WVA_ERR_LIMIT; }
  CK(cudaSetDevice(ctx->device));
  const size_t A = s->n_acc, T = s->n_types, M = s->n_models, S = s->n_servers;
  Ext n;
  n.A = A; n.T = T; n.M = M; n.S = S;
  Missing miss;
  each_sys(n, miss, ctx->sys, *s);
  if (miss.any) { ctx->last_error = "wva_load_system: a required array is NULL"; return WVA_ERR_ARG; }
  // validate indices the kernels dereference (after the NULL checks above)
  if (const char* bad = check_table_columns(*s, A, T, M)) { ctx->last_error = std::string("wva_load_system: ") + bad; return WVA_ERR_ARG; }
  if (const char* bad = check_server_columns(*s, S, (int)A, (int)M)) { ctx->last_error = std::string("wva_load_system: ") + bad; return WVA_ERR_ARG; }
  // one H2D copy of the whole arena, staged in pinned memory at the arena's offsets
  Layout L;
  each_sys(n, L, ctx->sys);
  const size_t total = L.off + 256;
  CK(ctx->stage_in.reserve(total));
  CK(ctx->sys_arena.reserve(total));
  char* h = (char*)ctx->stage_in.p;
  L = Layout{(char*)ctx->sys_arena.p};
  each_sys(n, [&](size_t c, int, auto*& d, auto* src) { if (c) memcpy(h + L.off, src, c * sizeof(*d)); L(c, 0, d); }, ctx->sys, *s);
  CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  CK(cudaMemcpyAsync(ctx->sys_arena.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  SysView& v = ctx->sys;
  v.n_acc = (int)A; v.n_types = (int)T; v.n_models = (int)M; v.n_servers = (int)S;
  ctx->A = (int)A; ctx->T = (int)T; ctx->M = (int)M; ctx->S = (int)S;
  ctx->unlimited = s->unlimited; ctx->delayed = s->delayed_best_effort; ctx->policy = s->saturation_policy;

  // candidate + solution arenas.  With a communicator the rank owns the block of servers [shard_lo, shard_hi) and the
  // arrays are padded to world equal blocks, so that the all-gather can run in place on them.
  ctx->shard_rows = ctx->world > 1 ? (int)((S + ctx->world - 1) / ctx->world) : (int)S;
  ctx->shard_lo = ctx->world > 1 ? (int)std::min(S, (size_t)ctx->rank * ctx->shard_rows) : 0;
  ctx->shard_hi = ctx->world > 1 ? (int)std::min(S, (size_t)(ctx->rank + 1) * ctx->shard_rows) : (int)S;
  const size_t S_pad = ctx->world > 1 ? (size_t)ctx->shard_rows * ctx->world : S;
  Ext pad;
  pad.S = S_pad; pad.P = S_pad * A;
  Layout C;
  CK(lay_out(ctx->cand_arena, C, [&](Layout& f) { each_cand(pad, f, ctx->cand); }));
  Layout O;
  CK(lay_out(ctx->sol_arena, O, [&](Layout& f) { each_sol(pad, f, ctx->sol); f(T, 0, ctx->d_type_count); f(T, 0, ctx->d_type_cost); }));
  CK(cudaMemsetAsync(ctx->sol_arena.p, 0, ctx->sol_arena.cap, ctx->stream));   // padding is copied out with the arena
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->loaded = true; ctx->calculated = false; ctx->solved = false;
  ctx->sized = false; ctx->marked = false;
  ctx->grid.current = false; ctx->grid_marked = false;
  ctx->table_marked = false; ctx->table_grid_marked = false;
  return WVA_OK;
}

// ------------------------------------------------------------------ calculate
}  // extern "C" (templates need C++ linkage)
template <int THREADS, bool SMEM>
static cudaError_t launch_sizer(wva_ctx* ctx, int mode, const SysView& sys_v, const CandView& cand_v, const int* list,
                                int blocks, size_t smem, unsigned long long n_pairs, int nmax, float* gtab, int* ovf_list) {
  // mode 1 = flattened state machine (a burst of single chain states per round); 2 = lock-step rounds; 3 = lock-step
  // with two chains per lane; 4 = lock-step, every pair split into a TTFT item and an ITL item (mid-size systems); 5 =
  // split items whose second chain evaluates the predicted next bisection point (wva_core.cuh spec2_*)
  cudaError_t e;
  SplitWs sw = {nullptr, nullptr, nullptr};
  const bool split = mode == 4 || mode == 5;
  if (split) {
    Layout L;
    e = lay_out(ctx->split_ws, L, [&](Layout& f) { f(2 * n_pairs, 0, sw.res); f(2 * n_pairs, 0, sw.solves); f(n_pairs, 0, sw.cnt); });
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(sw.cnt, 0, (size_t)n_pairs * 4, ctx->stream);
    if (e != cudaSuccess) return e;
  }
  // length-sorted queue: float32 probe -> (N, expected chain length) keys -> descending radix sort of the item ids
  const unsigned* order = nullptr;
  const unsigned long long n_items = split ? 2 * n_pairs : n_pairs;
  // the sorted queue + gang refill pays between ~130 and ~1500 pairs per SM (the items then fill 1.5-15 waves and
  // longest-first ordering shortens the tail); below, every lane holds one item and the probe is pure overhead; far
  // above, the gain no longer covers the probe's variance.  With the table in global memory it is kept at any size.
  // The flattened mode (1) takes neither.
  const bool by_size = n_pairs > (unsigned long long)ctx->sm_count * 130 &&
                       (n_pairs <= (unsigned long long)ctx->sm_count * 1500 || !SMEM);
  const bool do_sort = mode != 1 && (ctx->length_sort < 0 ? by_size : ctx->length_sort != 0);
  const bool do_gang = mode != 1 && (ctx->gang_refill < 0 ? by_size : ctx->gang_refill != 0);
  if (do_sort && n_items >= 64 && n_items < (1ull << 31)) {
    size_t tmp = 0;
    cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp, (unsigned*)nullptr, (unsigned*)nullptr, (unsigned*)nullptr,
                                              (unsigned*)nullptr, (int)n_items, 0, 32, ctx->stream);
    unsigned *k_in = nullptr, *k_out = nullptr, *v_in = nullptr, *v_out = nullptr;
    unsigned char* d_tmp = nullptr;
    Layout L;
    e = lay_out(ctx->order_ws, L, [&](Layout& f) {
      f(n_items, 0, k_in); f(n_items, 0, k_out); f(n_items, 0, v_in); f(n_items, 0, v_out); f(tmp, 0, d_tmp);
    });
    if (e != cudaSuccess) return e;
    const unsigned pb = (unsigned)((n_items + 127) / 128);
    if (split) sizer_probe_kernel<true><<<pb, 128, 0, ctx->stream>>>(sys_v, list, n_items, nmax, k_in, v_in);
    else sizer_probe_kernel<false><<<pb, 128, 0, ctx->stream>>>(sys_v, list, n_items, nmax, k_in, v_in);
    e = cub::DeviceRadixSort::SortPairsDescending(d_tmp, tmp, k_in, k_out, v_in, v_out, (int)n_items, 0, 32, ctx->stream);
    if (e != cudaSuccess) return e;
    ctx->launches += 4;
    order = v_out;
  }
  // <THREADS, SMEM, DUAL, SPLIT, FLAT>; mode 2 with its table in global memory runs the same body under a 128-register
  // cap (2 blocks per SM)
  auto k = mode == 1 ? sizer_lane_kernel<THREADS, SMEM, false, false, true>
         : mode == 3 ? sizer_lane_kernel<THREADS, SMEM, true, false, false>
         : mode == 4 ? sizer_lane_kernel<THREADS, SMEM, false, true, false>
         : mode == 5 ? sizer_lane_kernel<THREADS, SMEM, true, true, false>
         : THREADS == 256 && !SMEM ? sizer_lane_kernel_gtab_2blk
                                   : sizer_lane_kernel<THREADS, SMEM, false, false, false>;
  e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k<<<blocks, THREADS, smem, ctx->stream>>>(sys_v, cand_v, list, n_pairs, nmax, gtab, ctx->d_ctr, ovf_list, sw, order,
                                            do_gang ? 1 : 0);
  ctx->launches++;
  return cudaGetLastError();
}
template <int WARPS>
static cudaError_t launch_sizer_warp(wva_ctx* ctx, const SysView& sys_v, const CandView& cand_v, const int* list, int blocks,
                                     size_t smem, unsigned long long n_pairs, int nmax, int* ovf_list) {
  auto k = sizer_warp_kernel<WARPS>;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k<<<blocks, WARPS * 32, smem, ctx->stream>>>(sys_v, cand_v, list, n_pairs, nmax, ctx->d_ctr, ovf_list);
  ctx->launches++;
  return cudaGetLastError();
}
extern "C" {

/* test / profiling hook: 1 forces the lane-per-pair sizer regardless of the system size */
int32_t wva_set_option(wva_ctx* ctx, int32_t option, int32_t value) {
  if (!ctx) return WVA_ERR_ARG;
  if (option == WVA_OPT_FORCE_LANE_SIZER) {
    ctx->force_lane_sizer = value != 0;
    if (value >= 1 && value <= 6) ctx->lane_sizer_mode = value;
    return WVA_OK;
  }
  if (option == WVA_OPT_LENGTH_SORT) { ctx->length_sort = value < 0 ? -1 : (value != 0); return WVA_OK; }
  if (option == WVA_OPT_GANG_REFILL) { ctx->gang_refill = value < 0 ? -1 : (value != 0); return WVA_OK; }
  if (option == WVA_OPT_GRID_DEFER) { if (value < 0 || value > 2) return WVA_ERR_ARG; ctx->grid_defer = value; return WVA_OK; }
  if (option == WVA_OPT_GREEDY_MODE) { if (value < 0 || value > 2) return WVA_ERR_ARG; ctx->greedy_mode = value; return WVA_OK; }
  if (option == WVA_OPT_TABLE_MODE) { if (value < 0 || value > 2) return WVA_ERR_ARG; ctx->table_mode = value; return WVA_OK; }
  return WVA_ERR_ARG;
}

#ifdef WVA_POOL_PHASES
/* profiling build only (tools/perf_pool_phases.py): copies the pool sizer's phase sums out (out != NULL) and clears them */
int32_t wva_pool_phases(wva_ctx* ctx, uint64_t* out) {
  if (!ctx) return WVA_ERR_ARG;
  CK(cudaSetDevice(ctx->device));
  CK(cudaDeviceSynchronize());
  if (out) CK(cudaMemcpyFromSymbol(out, g_pool_phase, sizeof(g_pool_phase)));
  static const unsigned long long zero[PH_N] = {};
  CK(cudaMemcpyToSymbol(g_pool_phase, zero, sizeof(zero)));
  return WVA_OK;
}
#endif

}  // extern "C"

// CreateAllocation for every (server, accelerator) pair of the view sys_v into the rows of cand_v, or, with a device
// list of n_list pair indices of the view, for those pairs only (each written at its own row): the sizer picked by the
// number of pairs, then the float64-overflow slow path.  Sets the sizer fields of ctx->timing (calculate_ms: ev[2] to
// ev[3], the sizer launches).
static int32_t size_views(wva_ctx* ctx, const SysView& sys_v, const CandView& cand_v, const int* list = nullptr,
                          unsigned long long n_list = 0) {
  const unsigned long long n_pairs = list ? n_list : (unsigned long long)sys_v.n_servers * ctx->A;
  // scratch: counters + nmax reduction + overflow list.  The split sizer modes process a pair as TWO items and each may
  // append the pair (both chains of an alpha-dominated pair overflow at lambda_max): 2 entries per pair.
  int *d_nmax = nullptr, *d_ovf = nullptr;
  Layout L;
  CK(lay_out(ctx->scratch, L, [&](Layout& f) { f(1, 0, ctx->d_ctr); f(1, 0, d_nmax); f(2 * n_pairs + 256, 0, d_ovf); }));
  CK(cudaMemsetAsync(ctx->scratch.p, 0, 512, ctx->stream));
  CK(cudaEventRecord(ctx->ev[2], ctx->stream));
  if (n_pairs > 0) {
    // 1) largest batch size any pair will use -> table geometry
    int blocks = (int)((n_pairs + 255) / 256);
    if (blocks > 4096) blocks = 4096;
    max_batch_kernel<<<blocks, 256, 0, ctx->stream>>>(sys_v, list, n_pairs, d_nmax);
    ctx->launches++;
    int nmax = 0;
    CK(cudaMemcpyAsync(&nmax, d_nmax, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (nmax < 1) nmax = 1;
    const int NLIMIT = 1 << 16;
    if (nmax > NLIMIT) nmax = NLIMIT;  // pairs beyond it are flagged through limit_hit
    const size_t SMEM_PER_SM = 224 * 1024;
    // 2) the lane sizer's mode, unless forced.  Mid-size systems (measured: up to ~200 pairs per SM) leave lanes idle:
    // split every pair into a TTFT item and an ITL item, which halves the chain of dependent solves per work item.
    // Crossovers (natural queue order): split items up to ~180 pairs per SM, split items with a speculative second
    // chain (mode 5) up to ~380, whole pairs (mode 2, the searches share evaluations) beyond
    const int mode = ctx->force_lane_sizer ? ctx->lane_sizer_mode
                   : (n_pairs <= (unsigned long long)ctx->sm_count * 180) ? 4
                   : (n_pairs <= (unsigned long long)ctx->sm_count * 380) ? 5 : 2;
    // 3) the sizer.  Large systems: the pool sizer (sizer_pool_kernel.cuh) regroups the pending solves of 1024 pairs
    // per SM by length every time a warp goes back for work (88-92 % live lane-steps instead of 49-62 %); it overtakes
    // the lane sizer from ~640 pairs per SM
    const bool pool_auto = !ctx->force_lane_sizer && n_pairs > (unsigned long long)ctx->sm_count * 640 && nmax <= 4096;
    const size_t warp_tab = (size_t)nmax * 20;
    cudaError_t e = cudaSuccess;
    if (pool_auto || (ctx->force_lane_sizer && mode == 6)) {
      const int P = POOL_PMAX;
      const size_t pool_bytes = (size_t)ctx->sm_count * P * sizeof(PoolEntry);
      CK(ctx->pool_ws.reserve(pool_bytes + 512));
      PoolEntry* pool = (PoolEntry*)ctx->pool_ws.p;
      CK(cudaFuncSetAttribute(sizer_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PoolSmem)));
      sizer_pool_kernel<<<ctx->sm_count, POOL_THREADS, sizeof(PoolSmem), ctx->stream>>>(sys_v, cand_v, list, n_pairs, nmax, P,
                                                                                        pool, ctx->d_ctr, d_ovf);
      ctx->launches++;
      cudaError_t pe = cudaGetLastError();
      if (pe != cudaSuccess) { ctx->last_error = std::string("pool sizer launch: ") + cudaGetErrorString(pe); return WVA_ERR_CUDA; }
      ctx->timing.sizer_kernel = 4;
    } else if (n_pairs <= (unsigned long long)ctx->sm_count * 32 && warp_tab * 4 + 1024 <= SMEM_PER_SM && !ctx->force_lane_sizer) {
      // Small / medium systems are bound by the critical path of their slowest pair: the warp-per-pair sizer
      // (speculative bisection, sizer_warp_kernel.cuh) while the system is small (measured crossover against the
      // lock-step lane sizer: ~32 pairs per SM) and its per-warp tables (20 B x nmax) fit in shared memory.
      ctx->timing.sizer_kernel = 1;
      if (warp_tab * 8 <= 48 * 1024) {
        int per_sm = (int)(SMEM_PER_SM / (warp_tab * 8 + 1024)); if (per_sm > 6) per_sm = 6; if (per_sm < 1) per_sm = 1;
        e = launch_sizer_warp<8>(ctx, sys_v, cand_v, list, ctx->sm_count * per_sm, warp_tab * 8, n_pairs, nmax, d_ovf);
      } else {
        int per_sm = (int)(SMEM_PER_SM / (warp_tab * 4 + 1024)); if (per_sm > 8) per_sm = 8; if (per_sm < 1) per_sm = 1;
        e = launch_sizer_warp<4>(ctx, sys_v, cand_v, list, ctx->sm_count * per_sm, warp_tab * 4, n_pairs, nmax, d_ovf);
      }
    } else {
      // The lane sizer.  Its head table (4 B x nmax per lane) lives in shared memory when at least 64 lanes fit on an
      // SM; lanes per SM are maximised over CTA sizes {256,192,128,64} (1 KB per CTA is reserved by the driver).
      // Otherwise the table goes to global memory.
      const size_t per_lane = (size_t)nmax * 4;
      const int sizes[4] = {256, 192, 128, 64};
      int best_threads = 0, best_per_sm = 0;
      for (int i = 0; i < 4; i++) {
        size_t cta = per_lane * sizes[i] + 1024;
        int per_sm = (int)(SMEM_PER_SM / cta);
        if (per_sm * sizes[i] > 1024) per_sm = 1024 / sizes[i];
        if (per_sm * sizes[i] > best_threads * best_per_sm) { best_threads = sizes[i]; best_per_sm = per_sm; }
      }
      // small problems are latency bound: spread the items over every SM with as few lanes per SM as needed instead
      // of filling the first SMs (lanes pull one item each from the queue)
      const unsigned long long n_items = (mode >= 4) ? 2 * n_pairs : n_pairs;
      const unsigned long long lanes_needed = (n_items + ctx->sm_count - 1) / ctx->sm_count;
      if (best_per_sm >= 1 && lanes_needed <= 256 && lanes_needed < (unsigned long long)best_threads * best_per_sm) {
        int t = 64;
        while ((unsigned long long)t < lanes_needed) t += 64;
        if (per_lane * t + 1024 <= SMEM_PER_SM) { best_threads = t; best_per_sm = 1; }
      }
      // Head table placement: N = 256 leaves 192 lanes per SM in shared memory (1.5 warps per scheduler), slower than
      // the table in global memory / L2 with two 256-thread blocks per SM under a 128-register cap; at N = 128 (384
      // lanes in shared memory) and N = 64 shared memory wins.
      if (best_per_sm >= 1 && ctx->table_mode != 2 && (ctx->table_mode == 1 || best_threads * best_per_sm > 256 || n_pairs <= (unsigned long long)ctx->sm_count * 512)) {
        int blocks = ctx->sm_count * best_per_sm;
        size_t smem = per_lane * best_threads;
        ctx->timing.sizer_kernel = 2;
        switch (best_threads) {
          case 256: e = launch_sizer<256, true>(ctx, mode, sys_v, cand_v, list, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
          case 192: e = launch_sizer<192, true>(ctx, mode, sys_v, cand_v, list, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
          case 128: e = launch_sizer<128, true>(ctx, mode, sys_v, cand_v, list, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
          default: e = launch_sizer<64, true>(ctx, mode, sys_v, cand_v, list, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
        }
      } else {
        int blk = ctx->sm_count * 2;
        ctx->timing.sizer_kernel = 3;
        CK(ctx->gtab.reserve((size_t)blk * 256 * per_lane));
        e = launch_sizer<256, false>(ctx, mode, sys_v, cand_v, list, blk, 0, n_pairs, nmax, (float*)ctx->gtab.p, d_ovf);
      }
    }
    if (e != cudaSuccess) { ctx->last_error = std::string("sizer launch: ") + cudaGetErrorString(e); return WVA_ERR_CUDA; }
  }
  CK(cudaEventRecord(ctx->ev[3], ctx->stream));
  SizerCounters hc;
  CK(cudaMemcpyAsync(&hc, ctx->d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.calculate_ms = elapsed(ctx, 2, 3);
  ctx->timing.chain_solves = (int64_t)hc.solves;
  ctx->timing.chain_states = (int64_t)hc.states;
  if (getenv("WVA_SIZER_DEBUG") && hc.lockstep_slots)
    fprintf(stderr, "sizer: live lane-steps %llu of %llu lock-step slots (%.1f %%)\n", hc.states, hc.lockstep_slots,
            100.0 * (double)hc.states / (double)hc.lockstep_slots);
  if (getenv("WVA_SIZER_DEBUG"))
    fprintf(stderr, "sizer: %llu of %llu chain solves not certified (E12), redone by the exact solver\n", hc.certify_fallbacks,
            hc.solves);
  ctx->timing.overflow_pairs = (int64_t)hc.overflow_pairs;
  ctx->timing.certify_fallbacks = (int64_t)hc.certify_fallbacks;
  if (hc.limit_hit) { ctx->last_error = "a (server, accelerator) pair needs a max batch size above 65536"; return WVA_ERR_LIMIT; }
  if (hc.overflow_pairs) {
    // float64 overflow-rescale branch (mm1modelstatedependent.go:84-89,96-104): exact slow path
    int32_t rc = run_overflow_slow_path(sys_v, cand_v, d_ovf, (int)hc.overflow_pairs, ctx->stream, &ctx->launches);
    if (rc != 0) { ctx->last_error = "overflow slow path failed"; return WVA_ERR_CUDA; }
    CK(cudaStreamSynchronize(ctx->stream));
  }
  return WVA_OK;
}

extern "C" {

int32_t wva_calculate(wva_ctx* ctx) {
  if (!ctx) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_calculate before wva_load_system"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  ctx->shard_status = WVA_ERR_CUDA;   // until this call returns WVA_OK (agreed on by all ranks in wva_solve)
  ctx->sized = false;
  const int32_t rc = size_views(ctx, shard_sys(ctx), shard_cand(ctx));
  if (rc != WVA_OK) return rc;
  ctx->calculated = true; ctx->solved = false;
  ctx->sized = true; ctx->marked = false;   // every pair sized from the resident columns: the marks are void
  ctx->table_marked = false;
  ctx->shard_status = WVA_OK;
  return WVA_OK;
}

// ------------------------------------------------------------------ per-cycle update
int32_t wva_update_servers(wva_ctx* ctx, const float* srv_arrival, const int32_t* srv_in_tokens,
                           const int32_t* srv_out_tokens, const int32_t* srv_cur_acc, const int32_t* srv_cur_replicas,
                           const float* srv_cur_cost) {
  if (!ctx) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_update_servers before wva_load_system"; return WVA_ERR_STATE; }
  wva_system in = {};
  in.srv_arrival = srv_arrival; in.srv_in_tokens = srv_in_tokens; in.srv_out_tokens = srv_out_tokens;
  in.srv_cur_acc = srv_cur_acc; in.srv_cur_replicas = srv_cur_replicas; in.srv_cur_cost = srv_cur_cost;
  const size_t S = (size_t)ctx->S;
  if (const char* bad = check_cycle_columns(in, S, ctx->A)) { ctx->last_error = std::string("wva_update_servers: ") + bad; return WVA_ERR_ARG; }
  if (S == 0) return WVA_OK;
  CK(cudaSetDevice(ctx->device));
  // the six columns staged at their offsets of one pinned buffer, one H2D copy, then one classify-and-write pass
  SysView nu = ctx->sys;
  Layout L;
  each_cycle(S, L, nu);
  const size_t total = L.off + 256;
  CK(ctx->stage_in.reserve(total));
  CK(ctx->cycle_in.reserve(total));
  CK(ctx->marks.reserve(S));
  CK(ctx->grid_marks.reserve(S));
  char* h = (char*)ctx->stage_in.p;
  L = Layout{(char*)ctx->cycle_in.p};
  each_cycle(S, [&](size_t c, int, auto*& d, auto* src) { memcpy(h + L.off, src, c * sizeof(*d)); L(c, 0, d); }, nu, in);
  CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  CK(cudaMemcpyAsync(ctx->cycle_in.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
  if (!ctx->marked) CK(cudaMemsetAsync(ctx->marks.p, 0, S, ctx->stream));
  if (!ctx->grid_marked) CK(cudaMemsetAsync(ctx->grid_marks.p, 0, S, ctx->stream));
  unsigned char *marks = (unsigned char*)ctx->marks.p, *grid_marks = (unsigned char*)ctx->grid_marks.p;
  classify_servers_kernel<<<(unsigned)((S + 255) / 256), 256, 0, ctx->stream>>>(ctx->sys, nu, ctx->sys, nullptr, ctx->shard_lo,
                                                                               ctx->shard_hi, marks, grid_marks, marks,
                                                                               grid_marks);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // the staging buffer is free for the next call
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->marked = true; ctx->grid_marked = true; ctx->solved = false;
  return WVA_OK;
}

}  // extern "C"

// fills `m` with one entry per column the visitor walks: f(count, flags, from, to) moves `from` to `to`
#define COUNT_COL_(field, count, flags) +1
static_assert(0 SYS_COLS(COUNT_COL_) <= RowMoves::MAXC && 0 CAND_COLS(COUNT_COL_) <= RowMoves::MAXC,
              "RowMoves holds every column of either list");
#undef COUNT_COL_
struct AddMove {
  RowMoves& m;
  template <class T, class U> void operator()(size_t c, int, T* from, U* to) {
    if (!c) return;
    m.src[m.n] = (const char*)from; m.dst[m.n] = (char*)to; m.width[m.n] = (int)sizeof(T);
    m.n++;
  }
};

static void launch_move_rows(wva_ctx* ctx, const RowMoves& m, const int* rows, int n_rows, int per, bool scatter) {
  const unsigned long long n_items = (unsigned long long)n_rows * per;
  const unsigned long long blocks = std::min<unsigned long long>((n_items + 255) / 256, (unsigned long long)ctx->sm_count * 16);
  move_rows_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(m, rows, n_items, per, scatter);
  ctx->launches++;
}

// The pairs of the rank's block that `pred` selects, compacted in pair order into ctx->pairs_ws as indices into the
// block: *list and *n_list.
static int32_t select_pairs(wva_ctx* ctx, const TablePair& pred, int** list, int* n_list) {
  *n_list = 0;
  const long long n_pairs = (long long)(ctx->shard_hi - ctx->shard_lo) * ctx->A;
  if (n_pairs == 0) return WVA_OK;
  if (n_pairs > 0x7fffffffLL) { ctx->last_error = "a block of more than 2^31 - 1 pairs takes no pair list"; return WVA_ERR_LIMIT; }
  thrust::counting_iterator<int> pairs(0);
  size_t tmp = 0;
  CK(cub::DeviceSelect::If(nullptr, tmp, pairs, (int*)nullptr, (int*)nullptr, (int)n_pairs, pred, ctx->stream));
  int* d_cnt = nullptr;
  unsigned char* d_tmp = nullptr;
  Layout L;
  CK(lay_out(ctx->pairs_ws, L, [&](Layout& f) { f(n_pairs, 0, *list); f(1, 0, d_cnt); f(tmp, 0, d_tmp); }));
  CK(cub::DeviceSelect::If(d_tmp, tmp, pairs, *list, d_cnt, (int)n_pairs, pred, ctx->stream));
  ctx->launches++;
  CK(cudaMemcpyAsync(n_list, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return WVA_OK;
}

extern "C" {

int32_t wva_recalculate(wva_ctx* ctx, int64_t* n_resized, int64_t* n_revalued) {
  if (!ctx) return WVA_ERR_ARG;
  if (n_resized) *n_resized = 0;
  if (n_revalued) *n_revalued = 0;
  if (!ctx->loaded) { ctx->last_error = "wva_recalculate before wva_load_system"; return WVA_ERR_STATE; }
  if (!ctx->sized) {
    ctx->last_error = "wva_recalculate: the resident candidates do not come from wva_calculate on the loaded system";
    return WVA_ERR_STATE;
  }
  CK(cudaSetDevice(ctx->device));
  ctx->shard_status = WVA_ERR_CUDA;   // until this call returns WVA_OK (agreed on by all ranks in wva_solve)
  ctx->sized = false;                 // until every marked server is brought up to date
  ctx->timing.chain_solves = ctx->timing.chain_states = ctx->timing.overflow_pairs = ctx->timing.certify_fallbacks = 0;
  ctx->timing.sizer_kernel = 0;
  const int lo = ctx->shard_lo, n = ctx->shard_hi - ctx->shard_lo, A = ctx->A;
  CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  // 1) the rank's marked servers compacted, in server order: the re-size list, then the re-value-only list
  int cnt[2] = {0, 0};
  int *resize = nullptr, *revalue = nullptr;
  const unsigned char* marks = ctx->marked && n > 0 ? (const unsigned char*)ctx->marks.p : nullptr;
  if (marks) {
    thrust::counting_iterator<int> servers(lo);
    thrust::discard_iterator<> clean;
    size_t tmp = 0;
    CK(cub::DevicePartition::If(nullptr, tmp, servers, (int*)nullptr, (int*)nullptr, clean, (int*)nullptr, n,
                                MarkedResize{marks}, MarkedRevalueOnly{marks}, ctx->stream));
    int* d_cnt = nullptr;
    unsigned char* d_tmp = nullptr;
    Layout L;
    CK(lay_out(ctx->recalc_ws, L, [&](Layout& f) { f(n, 0, resize); f(n, 0, revalue); f(2, 0, d_cnt); f(tmp, 0, d_tmp); }));
    CK(cub::DevicePartition::If(d_tmp, tmp, servers, resize, revalue, clean, d_cnt, n, MarkedResize{marks},
                                MarkedRevalueOnly{marks}, ctx->stream));
    ctx->launches++;
    CK(cudaMemcpyAsync(cnt, d_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  const int D = cnt[0], R = cnt[1];
  // the current allocation alone changed: TransitionPenalty of every candidate again (before any re-sizing, which writes
  // its pairs' values itself)
  auto revalue_servers = [&]() {
    if (R == 0 || A == 0) return;
    const unsigned long long n_items = (unsigned long long)R * A;
    const unsigned long long blocks = std::min<unsigned long long>((n_items + 255) / 256, (unsigned long long)ctx->sm_count * 16);
    revalue_kernel<<<(unsigned)blocks, 256, 0, ctx->stream>>>(ctx->sys, ctx->cand, revalue, n_items);
    ctx->launches++;
  };
  if (ctx->table_marked) {
    // 2) table marks: every pair of a re-size-marked server and the table-marked pairs of the others, sized in place
    revalue_servers();
    const SysView blk = shard_sys(ctx);
    const TablePair pred{blk.srv_model, marks ? marks + lo : nullptr, MARK_RESIZE, ctx->tmarks.size_row,
                         ctx->tmarks.size_acc, A};
    int* list = nullptr;
    int n_list = 0;
    int32_t rc = select_pairs(ctx, pred, &list, &n_list);
    if (rc == WVA_OK && n_list > 0) rc = size_views(ctx, blk, shard_cand(ctx), list, (unsigned long long)n_list);
    if (rc != WVA_OK) return rc;
  } else if (D > 0) {
    // 2) the D servers' columns gathered into a view of D servers (model, perf and accelerator arrays shared) ...
    Ext g;
    g.S = (size_t)D; g.P = (size_t)D * A;
    SysView gsys = ctx->sys;
    gsys.n_servers = D;
    CandView gcand = {};
    Layout G;
    CK(lay_out(ctx->gather_ws, G, [&](Layout& f) {
      each_server(D, f, gsys);
      each_cand(g, f, gcand);
    }));
    RowMoves in;
    each_sys(g, AddMove{in}, ctx->sys, gsys);
    launch_move_rows(ctx, in, resize, D, 1, false);
    // 3) ... sized by the dispatch of wva_calculate, picked from D ...
    const int32_t rc = size_views(ctx, gsys, gcand);
    if (rc != WVA_OK) return rc;
    // 4) ... and every candidate field written back over the resident rows
    RowMoves out;
    each_cand(g, AddMove{out}, gcand, ctx->cand);
    launch_move_rows(ctx, out, resize, D, A, true);
  }
  if (!ctx->table_marked) revalue_servers();
  if (marks) CK(cudaMemsetAsync(ctx->marks.p, 0, ctx->S, ctx->stream));
  ctx->marked = false; ctx->table_marked = false;
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev[3], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.calculate_ms = elapsed(ctx, 0, 3);
  if (n_resized) *n_resized = D;
  if (n_revalued) *n_revalued = R;
  ctx->calculated = true; ctx->solved = false;
  ctx->sized = true;
  ctx->shard_status = WVA_OK;
  return WVA_OK;
}

}  // extern "C"

// Every column of `m` (per elements per row) laid out for the new set of n_rows rows, from the run list d_runs (its count,
// then the runs' first rows) of `prev`.
static int32_t launch_reindex(wva_ctx* ctx, const RowMoves& m, const int* prev, const int* d_runs, int n_rows, int per) {
  if (m.n == 0 || n_rows == 0) return WVA_OK;
  unsigned long long most = 0;
  for (int c = 0; c < m.n; c++) most = std::max(most, (unsigned long long)n_rows * per * m.width[c]);
  constexpr int CHUNKS = 8;
  const unsigned long long blocks = std::min<unsigned long long>((most + 16 * 256 * CHUNKS - 1) / (16 * 256 * CHUNKS),
                                                                 (unsigned long long)ctx->sm_count * 8);
  reindex_rows_kernel<CHUNKS><<<dim3((unsigned)blocks, (unsigned)m.n), 256, 0, ctx->stream>>>(m, prev, d_runs + 1, d_runs,
                                                                                            n_rows, per);
  ctx->launches++;
  CK(cudaGetLastError());
  return WVA_OK;
}

extern "C" {

int32_t wva_update_server_set(wva_ctx* ctx, int32_t n_servers, const int32_t* prev, const wva_system* servers) {
  if (!ctx) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_update_server_set before wva_load_system"; return WVA_ERR_STATE; }
  const size_t S = (size_t)ctx->S, A = (size_t)ctx->A;
  auto bad_arg = [&](const char* why) { ctx->last_error = std::string("wva_update_server_set: ") + why; return WVA_ERR_ARG; };
  if (n_servers < 0 || !servers) return bad_arg("n_servers < 0 or servers NULL");
  const size_t S2 = (size_t)n_servers;
  if (S2 > 0 && !prev) return bad_arg("prev is NULL");
  bool same = S2 == S;
  for (size_t i = 0, next = 0; i < S2; i++) {   // next: the least old index the next kept server may have
    const int p = prev[i];
    if (p < -1 || p >= (int)S) return bad_arg("prev out of range");
    if (p >= 0 && (size_t)p < next) return bad_arg("the kept servers' prev entries are not strictly increasing");
    if (p >= 0) next = (size_t)p + 1;
    same &= p == (int)i;
  }
  if (const char* bad = check_server_columns(*servers, S2, ctx->A, ctx->M)) return bad_arg(bad);
  if (ctx->world > 1 && !same) {
    ctx->last_error = "wva_update_server_set: the server set of a ctx with a communicator cannot change";
    return WVA_ERR_STATE;
  }
  CK(cudaSetDevice(ctx->device));
  // the server columns and prev staged at their offsets of one pinned buffer, one H2D copy
  SysView nu = ctx->sys;
  nu.n_servers = (int)S2;
  int* d_prev = nullptr;
  Layout L;
  each_server(S2, L, nu);
  L(S2, 0, d_prev);
  const size_t total = L.off + 256;
  CK(ctx->stage_in.reserve(total));
  CK(ctx->cycle_in.reserve(total));
  char* h = (char*)ctx->stage_in.p;
  L = Layout{(char*)ctx->cycle_in.p};
  auto stage = [&](size_t c, int, auto*& d, auto* src) { if (c) memcpy(h + L.off, src, c * sizeof(*d)); L(c, 0, d); };
  each_server(S2, stage, nu, *servers);
  stage(S2, 0, d_prev, prev);
  if (same) {
    // the same set: one classify-and-write pass in place, as wva_update_servers
    CK(ctx->marks.reserve(S));
    CK(ctx->grid_marks.reserve(S));
    CK(cudaEventRecord(ctx->ev[0], ctx->stream));
    CK(cudaMemcpyAsync(ctx->cycle_in.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
    unsigned char *marks = (unsigned char*)ctx->marks.p, *grid_marks = (unsigned char*)ctx->grid_marks.p;
    if (S > 0) {
      classify_servers_kernel<<<(unsigned)((S + 255) / 256), 256, 0, ctx->stream>>>(
          ctx->sys, nu, ctx->sys, nullptr, ctx->shard_lo, ctx->shard_hi, ctx->marked ? marks : nullptr,
          ctx->grid_marked ? grid_marks : nullptr, marks, grid_marks);
      ctx->launches++;
    }
  } else {
    // A new set (one rank): every arena reserved before anything moves, so that a failed reservation changes nothing
    GridState& g = ctx->grid;
    Ext n;
    n.A = A; n.T = (size_t)ctx->T; n.M = (size_t)ctx->M; n.S = S2; n.P = S2 * A;
    DevBuf sys_arena, cand_arena, sol_arena, marks_buf, grid_marks_buf, grid_buf;
    SysView sys = ctx->sys;
    sys.n_servers = (int)S2;
    CandView cand = {};
    SolView sol = {};
    long long* type_count = nullptr;
    double* type_cost = nullptr;
    Layout SL, CL, OL, GL;
    size_t prefix = 0;   // the model tables: the arena up to its first server column
    CK(lay_out(sys_arena, SL, [&](Layout& f) {
      each_sys(n, [&](size_t c, int flags, auto*& p) { if ((flags & COL_SRV) && !prefix) prefix = f.off; f(c, flags, p); }, sys);
    }));
    CK(lay_out(cand_arena, CL, [&](Layout& f) { each_cand(n, f, cand); }));
    CK(lay_out(sol_arena, OL, [&](Layout& f) { each_sol(n, f, sol); f(n.T, 0, type_count); f(n.T, 0, type_cost); }));
    CK(marks_buf.reserve(S2));
    CK(grid_marks_buf.reserve(S2));
    GridCounters* gctr = nullptr;
    int* gnmax = nullptr;
    GridOut gview = {};
    GridOverflowList govf = {};
    if (g.current) CK(lay_out(grid_buf, GL, [&](Layout& f) { grid_columns(f, n.P, g.R, g.full, gctr, gnmax, gview, govf); }));
    size_t tmp = 0;
    CK(cub::DeviceSelect::If(nullptr, tmp, thrust::counting_iterator<int>(0), (int*)nullptr, (int*)nullptr, (int)S2,
                             RunHead{d_prev}, ctx->stream));
    int* d_runs = nullptr;
    unsigned char* d_tmp = nullptr;
    Layout W;
    CK(lay_out(ctx->recalc_ws, W, [&](Layout& f) { f(S2 + 1, 0, d_runs); f(tmp, 0, d_tmp); }));
    CK(cudaEventRecord(ctx->ev[0], ctx->stream));
    CK(cudaMemcpyAsync(ctx->cycle_in.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
    // the model tables as they are; every server column through the classify pass, the marks carried over
    if (prefix) CK(cudaMemcpyAsync(sys_arena.p, ctx->sys_arena.p, prefix, cudaMemcpyDeviceToDevice, ctx->stream));
    if (S2 > 0) {
      classify_servers_kernel<<<(unsigned)((S2 + 255) / 256), 256, 0, ctx->stream>>>(
          ctx->sys, nu, sys, d_prev, 0, (int)S2, ctx->marked ? (const unsigned char*)ctx->marks.p : nullptr,
          ctx->grid_marked ? (const unsigned char*)ctx->grid_marks.p : nullptr, (unsigned char*)marks_buf.p,
          (unsigned char*)grid_marks_buf.p);
      ctx->launches++;
    }
    // the runs of prev (count word, then each run's first new row), then the candidate rows and the frontier (A per
    // server) and the grid levels (A * R per server) moved run by run
    if (S2 > 0) {
      CK(cub::DeviceSelect::If(d_tmp, tmp, thrust::counting_iterator<int>(0), d_runs + 1, d_runs, (int)S2, RunHead{d_prev},
                               ctx->stream));
      ctx->launches++;
    }
    RowMoves rows, lv;
    each_cand(n, AddMove{rows}, ctx->cand, cand);
    if (g.current) AddMove{rows}(n.P, 0, g.view.frontier, gview.frontier);
    Ext gx;
    gx.P = n.P; gx.R = (size_t)g.R;
    if (g.current && g.full) each_grid(gx, AddMove{lv}, g.view, gview);
    int32_t rc = launch_reindex(ctx, rows, d_prev, d_runs, (int)S2, (int)A);
    if (rc == WVA_OK) rc = launch_reindex(ctx, lv, d_prev, d_runs, (int)S2, (int)A * g.R);
    if (rc != WVA_OK) return rc;
    CK(cudaMemsetAsync(sol_arena.p, 0, sol_arena.cap, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));   // nothing reads the old arenas any more
    std::swap(ctx->sys_arena, sys_arena);
    std::swap(ctx->cand_arena, cand_arena);
    std::swap(ctx->sol_arena, sol_arena);
    std::swap(ctx->marks, marks_buf);
    std::swap(ctx->grid_marks, grid_marks_buf);
    ctx->sys = sys; ctx->cand = cand; ctx->sol = sol;
    ctx->d_type_count = type_count; ctx->d_type_cost = type_cost;
    if (g.current) {
      std::swap(g.buf, grid_buf);
      g.view = gview; g.ctr = gctr; g.nmax = gnmax; g.ovf = govf;
    } else {
      g.ran = false;   // a grid of the old set, not brought along: nothing to fetch
    }
    ctx->S = (int)S2;
    ctx->shard_rows = (int)S2; ctx->shard_lo = 0; ctx->shard_hi = (int)S2;
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // the staging buffer is free for the next call
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->marked = true; ctx->grid_marked = true; ctx->solved = false;
  return WVA_OK;
}

// ------------------------------------------------------------------ table update
int32_t wva_update_tables(wva_ctx* ctx, const wva_system* tables, int64_t* n_marked) {
  if (!ctx) return WVA_ERR_ARG;
  if (n_marked) *n_marked = 0;
  if (!ctx->loaded) { ctx->last_error = "wva_update_tables before wva_load_system"; return WVA_ERR_STATE; }
  auto bad_arg = [&](const char* why) { ctx->last_error = std::string("wva_update_tables: ") + why; return WVA_ERR_ARG; };
  if (!tables) return bad_arg("tables is NULL");
  if (tables->n_acc != ctx->A || tables->n_types != ctx->T || tables->n_models != ctx->M)
    return bad_arg("n_acc, n_types and n_models must be the loaded system's");
  const size_t A = (size_t)ctx->A, M = (size_t)ctx->M, MA = M * A;
  if (const char* bad = check_table_columns(*tables, A, (size_t)ctx->T, M)) return bad_arg(bad);
  CK(cudaSetDevice(ctx->device));
  // the table columns staged at their offsets of one pinned buffer, one H2D copy, then one classify-and-write pass
  SysView nu = ctx->sys;
  Layout L;
  each_table(A, M, L, nu);
  const size_t total = L.off + 256;
  CK(ctx->stage_in.reserve(total));
  CK(ctx->cycle_in.reserve(total));
  TableMarks& tm = ctx->tmarks;
  Layout TL;
  CK(lay_out(ctx->table_marks, TL, [&](Layout& f) { f(MA, 0, tm.size_row); f(A, 0, tm.size_acc); f(MA, 0, tm.grid_row); f(MA + A, 0, tm.fresh); }));
  unsigned long long* d_count = nullptr;
  Layout W;
  CK(lay_out(ctx->pairs_ws, W, [&](Layout& f) { f(1, 0, d_count); }));
  char* h = (char*)ctx->stage_in.p;
  L = Layout{(char*)ctx->cycle_in.p};
  each_table(A, M, [&](size_t c, int, auto*& d, auto* src) { if (c) memcpy(h + L.off, src, c * sizeof(*d)); L(c, 0, d); }, nu, *tables);
  CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  CK(cudaMemcpyAsync(ctx->cycle_in.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
  if (!ctx->table_marked) {
    CK(cudaMemsetAsync(tm.size_row, 0, MA, ctx->stream));
    CK(cudaMemsetAsync(tm.size_acc, 0, A, ctx->stream));
  }
  if (!ctx->table_grid_marked) CK(cudaMemsetAsync(tm.grid_row, 0, MA, ctx->stream));
  CK(cudaMemsetAsync(d_count, 0, sizeof(*d_count), ctx->stream));
  const size_t items = std::max(MA, A);
  if (items > 0) {
    classify_tables_kernel<<<(unsigned)((items + 255) / 256), 256, 0, ctx->stream>>>(ctx->sys, nu, (int)A, (int)M, tm);
    ctx->launches++;
  }
  // the pairs of the block this diff marked for re-sizing
  const SysView blk = shard_sys(ctx);
  const unsigned long long n_pairs = (unsigned long long)blk.n_servers * A;
  if (n_pairs > 0) {
    count_table_pairs_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, ctx->stream>>>(blk.srv_model, (int)A, (int)M, n_pairs,
                                                                                       tm.fresh, d_count);
    ctx->launches++;
  }
  unsigned long long count = 0;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // the staging buffer is free for the next call
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->table_marked = true; ctx->table_grid_marked = true; ctx->solved = false;
  if (n_marked) *n_marked = (int64_t)count;
  return WVA_OK;
}

// ------------------------------------------------------------------ solve
}  // extern "C"

// allocator + AllocateByType on a view (the whole system, or the rank's block of servers)
static int32_t solve_view(wva_ctx* ctx, const SysView& sv, const CandView& cv, const SolView& ov) {
  const int S = sv.n_servers, T = ctx->T;
  if (S > 0) {
    if (ctx->unlimited) {
      int blocks = (int)(((size_t)S * 32 + 255) / 256);
      solve_unlimited_kernel<<<blocks, 256, 0, ctx->stream>>>(sv, cv, ov);
      ctx->launches++;
    } else {
      long long gstats[2] = {0, 0};
      // the static-order sweep (greedy_sweep.cuh) wherever it applies; the literal queue otherwise or on request.
      // (100 k servers x 32, capacity 60 %: the sweep is several times faster than the queue, more so under the
      // best-effort policies)
      const bool sweep = greedy_sweep_covers(sv) && ctx->greedy_mode != 1;
      int32_t rc = sweep ? run_solve_greedy_sweep(sv, cv, ov, ctx->delayed, ctx->policy, &ctx->greedy_ws.p,
                                                  &ctx->greedy_ws.cap, ctx->stream, &ctx->launches, gstats)
                         : run_solve_greedy(sv, cv, ov, ctx->delayed, ctx->policy, &ctx->greedy_ws.p,
                                            &ctx->greedy_ws.cap, ctx->stream, &ctx->launches, gstats);
      if (rc != 0) { ctx->last_error = "SolveGreedy failed"; return rc; }
      ctx->timing.greedy_heap_pushes = gstats[0]; ctx->timing.greedy_events = gstats[1];
    }
  }
  // AllocateByType
  int nparts = (S + 255) / 256;
  if (nparts < 1) nparts = 1;
  const size_t n_part = (size_t)nparts * (T > 0 ? T : 1);
  // reuse scratch beyond its first 1024 bytes (counters)
  unsigned char* counters = nullptr;
  long long* pc = nullptr;
  double* pd = nullptr;
  Layout L;
  CK(lay_out(ctx->scratch, L, [&](Layout& f) { f(1024, 0, counters); f(n_part, 0, pc); f(n_part, 0, pd); }));
  if (T > 0) {
    if (S > 0) {
      by_type_partial_kernel<<<nparts, 256, 0, ctx->stream>>>(sv, ov, pc, pd);
      ctx->launches++;
    } else {
      CK(cudaMemsetAsync(pc, 0, n_part * 8, ctx->stream));
      CK(cudaMemsetAsync(pd, 0, n_part * 8, ctx->stream));
    }
    by_type_final_kernel<<<T, 256, 0, ctx->stream>>>(T, S > 0 ? nparts : 0, pc, pd, ctx->d_type_count, ctx->d_type_cost);
    ctx->launches++;
  }
  CK(cudaGetLastError());
  return WVA_OK;
}

extern "C" {

int32_t wva_solve(wva_ctx* ctx) {
  if (!ctx) return WVA_ERR_ARG;
  if (!ctx->calculated && ctx->world == 1) { ctx->last_error = "wva_solve before wva_calculate"; return WVA_ERR_STATE; }
  if (!ctx->loaded) { ctx->last_error = "wva_solve before wva_load_system"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  CK(cudaEventRecord(ctx->ev[4], ctx->stream));
  ctx->timing.exchange_ms = 0.0f; ctx->timing.greedy_heap_pushes = 0; ctx->timing.greedy_events = 0;
  int32_t rc;
  if (ctx->world > 1) rc = comm_exchange_and_solve(ctx);
  else rc = solve_view(ctx, ctx->sys, ctx->cand, ctx->sol);
  if (rc != WVA_OK) return rc;
  CK(cudaEventRecord(ctx->ev[5], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.solve_ms = elapsed(ctx, 4, 5);
  ctx->solved = true;
  return WVA_OK;
}

// OptimizerSpec / CapacityData of the loaded system replaced in place (sizing reads neither)
int32_t wva_set_optimizer(wva_ctx* ctx, int32_t unlimited, int32_t delayed_best_effort, int32_t saturation_policy) {
  if (!ctx || saturation_policy < WVA_POLICY_NONE || saturation_policy > WVA_POLICY_ROUND_ROBIN) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_set_optimizer before wva_load_system"; return WVA_ERR_STATE; }
  ctx->unlimited = unlimited ? 1 : 0; ctx->delayed = delayed_best_effort ? 1 : 0; ctx->policy = saturation_policy;
  ctx->solved = false;
  return WVA_OK;
}
int32_t wva_set_capacity(wva_ctx* ctx, const int32_t* type_count) {
  if (!ctx || (!type_count && ctx->T > 0)) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_set_capacity before wva_load_system"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  if (ctx->T > 0) {
    CK(cudaMemcpyAsync((void*)ctx->sys.type_count, type_count, (size_t)ctx->T * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  ctx->solved = false;
  return WVA_OK;
}

// ------------------------------------------------------------------ candidates from outside
int32_t wva_set_candidates(wva_ctx* ctx, const wva_candidates* in) {
  if (!ctx || !in) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_set_candidates before wva_load_system"; return WVA_ERR_STATE; }
  Ext n;
  n.P = (size_t)ctx->S * ctx->A;
  const size_t P = n.P;
  Missing miss;
  each_cand(n, miss, ctx->cand, *in);
  if (miss.any) {
    ctx->last_error = "wva_set_candidates: a required array is NULL";
    return WVA_ERR_ARG;
  }
  for (size_t i = 0; i < P; i++)
    if (in->state[i] > WVA_ALLOC_EMPTY || in->num_replicas[i] < 0) {
      ctx->last_error = "wva_set_candidates: state / num_replicas out of range";
      return WVA_ERR_ARG;
    }
  CK(cudaSetDevice(ctx->device));
  CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  Copy up{ctx->stream, cudaMemcpyHostToDevice};
  each_cand(n, up, ctx->cand, *in);
  CK(up.e);
  if (P > 0 && !in->n_solves) CK(cudaMemsetAsync(ctx->cand.n_solves, 0, P * 4, ctx->stream));
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));               // the caller's buffers are free again on return (cgo pointer rule)
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->calculated = true; ctx->solved = false;
  ctx->sized = false;   // the caller's candidates: wva_recalculate cannot bring them up to date
  return WVA_OK;
}

// ------------------------------------------------------------------ readback
int32_t wva_get_candidates(wva_ctx* ctx, wva_candidates* out) {
  if (!ctx || !out) return WVA_ERR_ARG;
  if (!ctx->calculated) { ctx->last_error = "wva_get_candidates before wva_calculate"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  Ext n;
  n.P = (size_t)ctx->S * ctx->A;
  if (n.P == 0) return WVA_OK;
  CK(cudaEventRecord(ctx->ev[6], ctx->stream));
  Copy down{ctx->stream, cudaMemcpyDeviceToHost};
  each_cand(n, down, ctx->cand, *out);
  CK(down.e);
  CK(cudaEventRecord(ctx->ev[7], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.d2h_ms = elapsed(ctx, 6, 7);
  return WVA_OK;
}

int32_t wva_get_solution(wva_ctx* ctx, wva_solution* out) {
  if (!ctx || !out) return WVA_ERR_ARG;
  if (!ctx->solved) { ctx->last_error = "wva_get_solution before wva_solve"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  const size_t S = ctx->S, T = ctx->T;
  // one contiguous D2H of the solution arena into pinned staging, then scatter to the caller
  size_t bytes = ctx->sol_arena.cap;
  CK(ctx->stage_out.reserve(bytes));
  CK(cudaEventRecord(ctx->ev[6], ctx->stream));
  CK(cudaMemcpyAsync(ctx->stage_out.p, ctx->sol_arena.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaEventRecord(ctx->ev[7], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.d2h_ms = elapsed(ctx, 6, 7);
  const char* h = (const char*)ctx->stage_out.p;
  const char* d = (const char*)ctx->sol_arena.p;
  auto H = [&](const void* devp) { return h + ((const char*)devp - d); };
  Ext n;
  n.S = S;
  each_sol(n, [&](size_t c, int, auto* d, auto* o) { if (o) memcpy(o, H(d), c * sizeof(*d)); }, ctx->sol, *out);
  if (out->type_count) memcpy(out->type_count, H(ctx->d_type_count), T * 8);
  if (out->type_cost) memcpy(out->type_cost, H(ctx->d_type_cost), T * 8);
  return WVA_OK;
}

}  // extern "C"

#include "capi_aux.inl"
#include "comm.inl"
#include "ingest.inl"
#include "k2_history.inl"
#include "ingest_v2.inl"
