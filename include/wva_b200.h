/*
 * wva_b200.h — C-ABI of the H100-native (sm_90a) WVA optimization hot path.
 *
 * This is the drop-in boundary a cgo shim binds (see INTEGRATION.md and
 * llm-d-workload-variant-autoscaler_b200/go/).  The reference
 * (llm-d/llm-d-workload-variant-autoscaler @ b08b1c77) has NO FFI boundary of
 * its own — it is 100 % Go — so every entry point below cites the Go
 * function(s) it replaces (paths relative to the reference root).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross this boundary
 *   - the CALLER owns every host buffer; the library copies before returning
 *     and never retains a caller pointer (cgo pointer rule)
 *   - every function returns an int32 status (WVA_OK == 0); an infeasible
 *     (server, accelerator) candidate is DATA (feasible == 0, the Go nil
 *     *Allocation, pkg/core/allocation.go:118-122), never an error
 *   - strings never cross: the shim keeps name<->index maps built from SORTED
 *     names (Go map iteration order is random; sorted-name index order is the
 *     canonical order wherever the reference iterates a map)
 *   - a ctx is single-caller (the reference's math runs on one goroutine,
 *     internal/engines/executor/polling.go:50-54); distinct ctxs are
 *     independent and may be used concurrently
 *   - there is NO CPU fallback: without a usable CUDA device wva_create fails
 */
#ifndef WVA_B200_H
#define WVA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes ------------------------------------------------------- */
enum {
  WVA_OK = 0,
  WVA_ERR_ARG = 1,        /* null pointer / negative size / inconsistent index */
  WVA_ERR_CUDA = 2,       /* a CUDA runtime call or kernel failed              */
  WVA_ERR_NO_DEVICE = 3,  /* no usable sm_90 device (no CPU fallback exists)   */
  WVA_ERR_STATE = 4,      /* call order violated (e.g. solve before calculate) */
  WVA_ERR_NOMEM = 5,      /* host or device allocation failed                  */
  WVA_ERR_LIMIT = 6       /* a size exceeds what the kernels support           */
};

/* saturation policy: pkg/config/config.go:4-41 (SaturatedAllocationPolicy) */
enum {
  WVA_POLICY_NONE = 0,
  WVA_POLICY_PRIORITY_EXHAUSTIVE = 1,
  WVA_POLICY_PRIORITY_ROUND_ROBIN = 2,
  WVA_POLICY_ROUND_ROBIN = 3
};

/* candidate / solution state */
enum {
  WVA_ALLOC_NONE = 0,   /* Go nil *Allocation                                     */
  WVA_ALLOC_ACC = 1,    /* allocation on accelerator index `acc`                  */
  WVA_ALLOC_EMPTY = 2   /* zero-load allocation with accelerator "" and 0 replicas
                           (pkg/core/allocation.go:255-260)                       */
};

/* current-accelerator sentinels (srv_cur_acc) */
#define WVA_CUR_ACC_EMPTY (-1)   /* curAllocation.accelerator == ""               */
#define WVA_CUR_ACC_UNKNOWN (-2) /* non-empty name that matches no accelerator    */

typedef struct wva_ctx wva_ctx;

/*
 * Index-keyed SoA image of config.SystemSpec (pkg/config/types.go:11-149) after
 * System.SetFromSpec (pkg/core/system.go:82-89) resolved the string keys.
 * Sizes: A = n_acc, T = n_types, M = n_models, S = n_servers.
 */
typedef struct wva_system {
  /* accelerators: AcceleratorSpec (types.go:29-37) */
  int32_t n_acc;
  int32_t n_types;                  /* T <= 64: wva_load_system returns WVA_ERR_LIMIT
                                       for more (the allocators keep 64-bit type masks) */
  const float* acc_cost;            /* [A] Cost, cents/hr                         */
  const int32_t* acc_multiplicity;  /* [A] Multiplicity                           */
  const int32_t* acc_type;          /* [A] index of Type in [0,T)                 */
  const int32_t* type_count;        /* [T] CapacityData count (0 when absent)     */

  /* ModelAcceleratorPerfData (types.go:66-73), row-major [M][A] */
  int32_t n_models;
  const float* perf_alpha;          /* [M*A] ServiceParms.Alpha                   */
  const float* perf_beta;           /* [M*A]                                      */
  const float* perf_gamma;          /* [M*A]                                      */
  const int32_t* perf_max_batch;    /* [M*A] MaxBatchSize                         */
  const int32_t* perf_at_tokens;    /* [M*A] AtTokens                             */
  const int32_t* perf_acc_count;    /* [M*A] AccCount (<=0 -> 1, model.go:52-55)  */
  const uint8_t* perf_present;      /* [M*A] 1 if model has perf data on acc      */

  /* servers: ServerSpec (types.go:108-117) with class/target resolved */
  int32_t n_servers;
  const int32_t* srv_model;         /* [S] model index, -1 = unknown model        */
  const int32_t* srv_priority;      /* [S] Server.Priority() (server.go:92-97)    */
  const int32_t* srv_min_replicas;  /* [S] MinNumReplicas                         */
  const int32_t* srv_max_batch;     /* [S] MaxBatchSize override (0 = derive)     */
  const uint8_t* srv_keep_acc;      /* [S] KeepAccelerator                        */
  const uint8_t* srv_target_present;/* [S] class exists and has a target for the model */
  const float* srv_slo_ttft;        /* [S] Target.TTFT ms (0 = no target)         */
  const float* srv_slo_itl;         /* [S] Target.ITL ms                          */
  const float* srv_slo_tps;         /* [S] Target.TPS tokens/s                    */
  const float* srv_arrival;         /* [S] ServerLoadSpec.ArrivalRate, req/min    */
  const int32_t* srv_in_tokens;     /* [S] AvgInTokens                            */
  const int32_t* srv_out_tokens;    /* [S] AvgOutTokens                           */
  const int32_t* srv_cur_acc;       /* [S] CurrentAlloc accelerator index / sentinel */
  const int32_t* srv_cur_replicas;  /* [S] CurrentAlloc.NumReplicas               */
  const float* srv_cur_cost;        /* [S] CurrentAlloc.Cost                      */

  /* OptimizerSpec (types.go:145-149) */
  uint8_t unlimited;
  uint8_t delayed_best_effort;
  int32_t saturation_policy;        /* WVA_POLICY_*                               */
} wva_system;

/*
 * Per-(server, accelerator) candidates = Server.AllAllocations() after
 * Server.Calculate (pkg/core/server.go:55-67); row-major [S][A].
 * Fields mirror core.Allocation (pkg/core/allocation.go:13-24).
 */
typedef struct wva_candidates {
  uint8_t* state;          /* [S*A] WVA_ALLOC_*                                   */
  int32_t* num_replicas;   /* [S*A]                                               */
  int32_t* batch_size;     /* [S*A]                                               */
  float* cost;             /* [S*A]                                               */
  float* value;            /* [S*A] TransitionPenalty(cur -> candidate)           */
  float* itl;              /* [S*A]                                               */
  float* ttft;             /* [S*A] AvgWaitTime + AvgPrefillTime (allocation.go:148) */
  float* rho;              /* [S*A]                                               */
  float* max_arrv_rate;    /* [S*A] maxArrvRatePerReplica, req/msec               */
  int32_t* n_solves;       /* [S*A] chain solves spent on the pair (may be NULL)  */
} wva_candidates;

/*
 * Solution = Server.Allocation() for every server after Manager.Optimize
 * (pkg/manager/manager.go:21-27) + System.AllocateByType (system.go:271-299).
 */
typedef struct wva_solution {
  uint8_t* state;          /* [S] WVA_ALLOC_*                                     */
  int32_t* acc;            /* [S] accelerator index (-1 unless state==ACC)        */
  int32_t* num_replicas;   /* [S]                                                 */
  int32_t* batch_size;     /* [S]                                                 */
  float* cost;             /* [S]                                                 */
  float* value;            /* [S]                                                 */
  float* itl;              /* [S]                                                 */
  float* ttft;             /* [S]                                                 */
  float* rho;              /* [S]                                                 */
  float* max_arrv_rate;    /* [S]                                                 */
  int64_t* type_count;     /* [T] AllocationByType.count                          */
  double* type_cost;       /* [T] AllocationByType.cost (summed in f64)           */
} wva_solution;

/* per-call device timings, milliseconds (CUDA events on the ctx stream) */
typedef struct wva_timing {
  float h2d_ms;
  float calculate_ms;
  float solve_ms;
  float grid_ms;
  float saturation_ms;
  float limit_ms;
  float d2h_ms;
  int64_t chain_solves;    /* chain solves executed by the last calculate/grid    */
  int64_t chain_states;    /* birth-death states visited by the last calculate/grid */
  int64_t overflow_pairs;  /* float64 overflow-rescale slow path: pairs (calculate), levels (grid) */
  float exchange_ms;       /* NCCL exchange of the last wva_solve / wva_saturation_run on a ctx with a communicator
                              (all-gather of the candidate arena or of the solution, all-reduce of the partials) */
  int32_t sizer_kernel;    /* which sizer the last wva_calculate ran: 1 warp per pair, 2 lane per pair (head table in
                              shared memory), 3 lane per pair (table in global memory), 4 pool sizer; 0 nothing to size */
  int64_t greedy_heap_pushes; /* entries the last limited wva_solve pushed into the re-insertion heap (greedy.go:143-163) */
  int64_t greedy_events;      /* head entries the last limited wva_solve processed (greedy.go:112-165 loop trips)    */
  int64_t certify_fallbacks;  /* chain solves of the last calculate/grid whose certified fast solve (DESIGN.md §3 E12)
                                 could not prove the reference's float32 results and that the exact solver redid      */
} wva_timing;

/* ---- lifecycle ----------------------------------------------------------- */
int32_t wva_create(int32_t device, wva_ctx** out);
int32_t wva_destroy(wva_ctx* ctx);
const char* wva_strerror(int32_t code);
/* text of the last CUDA error seen by this ctx ("" if none) */
const char* wva_last_error(const wva_ctx* ctx);
/* number of kernel launches issued by this ctx since creation */
int64_t wva_launch_count(const wva_ctx* ctx);

/* options (wva_set_option): tuning / test hooks, never needed for correctness */
#define WVA_OPT_FORCE_LANE_SIZER 1 /* 0: pick by system size; 1: lane-per-pair, flattened state machine;
                                      2: lane-per-pair, lock-step rounds (what large systems use); 3: two chains
                                      per lane (TTFT and ITL searches together); 4: every pair split into a TTFT
                                      item and an ITL item; 5: split items whose second chain evaluates the
                                      predicted next bisection point; 6: pool sizer — the pending solves of 1024 pairs
                                      per SM regrouped by chain length (what very large systems use) */
#define WVA_OPT_LENGTH_SORT 2      /* 1: the lane sizer visits the work items in probe-sorted order
                                      (csrc/sizer_probe.cuh); 0: natural (server, accelerator) order; -1 (default):
                                      sorted where it was measured to pay (130-1500 pairs per SM).  Order
                                      only — results are identical either way */
#define WVA_OPT_GANG_REFILL 3      /* 1: a warp of the lane sizer takes 32 new items only when all its
                                      lanes are idle (lanes stay in the same bisection step); 0: lanes refill
                                      one by one; -1 (default): as WVA_OPT_LENGTH_SORT.  Scheduling only */
#define WVA_OPT_TABLE_MODE 4       /* lane sizer head table: 0 (default) shared memory when >= 64 lanes per SM fit, else
                                      global memory; 1 force shared memory (when it fits at all); 2 force global memory
                                      (two 256-thread blocks per SM under a 128-register cap).  Placement only */
#define WVA_OPT_GREEDY_MODE 5      /* limited-capacity allocator: 1 the literal queue (sorted array + re-insertion heap,
                                      csrc/greedy_solve.cuh); 0 (default) and 2 the static-order event sweep
                                      (csrc/greedy_sweep.cuh) wherever it applies (<= 1 179 648 servers, <= 64 capacity
                                      types), the queue elsewhere.  Same result either way */
#define WVA_OPT_GRID_DEFER 6       /* replica grid: 0 (default) the near-saturation levels of every pair (lambda / mu_N
                                      > 0.6: the long chains) are deferred to a pass sorted by chain length when the
                                      system has >= 20 000 pairs; 1 never; 2 always.  Scheduling only */
int32_t wva_set_option(wva_ctx* ctx, int32_t option, int32_t value);

/* ---- multi-GPU: model-sharded over one NCCL communicator ----------------- */
/*
 * The path shards by server (SURVEY 8e): rank r of `world` owns the contiguous block of servers
 * [r*ceil(S/world), min(S, (r+1)*ceil(S/world))); accelerator / perf / capacity tables are replicated (every rank loads
 * the SAME wva_system).  On a ctx with a communicator
 *   wva_calculate   sizes only the rank's block (no collective);
 *   wva_solve       limited capacity (SolveGreedy needs every server, pkg/solver/greedy.go:35-105): ONE in-place
 *                   ncclAllGather group over the candidate arena in HBM (no host staging), then the same sweep on
 *                   every rank; unlimited (SolveUnlimited is per server, solver.go:63-79): the rank solves its block,
 *                   ONE ncclAllGather group of the solution arrays + ONE ncclAllReduce(sum) of the by-type
 *                   {count int64, cost float64} partials (System.AllocateByType, pkg/core/system.go:271-299).
 *                   Every rank then holds the global solution (wva_get_solution is identical on all ranks);
 *   wva_saturation_run  analyses the models the rank uploaded and all-reduces the int64 partials
 *                   (wva_saturation_out.partials_all).
 * NCCL is dlopen'ed (libnccl.so.2) on first use: single-GPU callers need no NCCL at all.  The 128-byte id is created
 * on one rank (wva_comm_unique_id) and carried to the others by the host (the Go shim: any channel it likes).
 * wva_comm_init_rank must precede wva_load_system (arenas are sized for the padded all-gather).
 */
#define WVA_COMM_ID_BYTES 128
int32_t wva_comm_unique_id(uint8_t id[WVA_COMM_ID_BYTES]);
int32_t wva_comm_init_rank(wva_ctx* ctx, int32_t world, int32_t rank, const uint8_t id[WVA_COMM_ID_BYTES]);
/* the block of servers this ctx sizes: [*lo, *hi) (the whole system without a communicator) */
int32_t wva_comm_shard(const wva_ctx* ctx, int32_t* lo, int32_t* hi);

/*
 * One host process driving several GPUs (what a Go controller does): n contexts, one per device, joined by one NCCL
 * communicator (ncclCommInitRank from n host threads).  wva_group_optimize = Manager.Optimize over the group: every
 * device loads the system, sizes its block of servers, the exchange above runs over NVLink, the allocator runs, and
 * the global solution is copied out once (from device 0).  wva_group_saturation_v1 splits the batch of models into n
 * contiguous blocks (device i analyses block i, outputs land at the block's offsets of the caller's arrays) and
 * all-reduces the partials.  wva_group_ctx exposes the per-device contexts for everything else (timings, options).
 */
typedef struct wva_group wva_group;
int32_t wva_group_create(const int32_t* devices, int32_t n, wva_group** out);
int32_t wva_group_destroy(wva_group* g);
int32_t wva_group_size(const wva_group* g);
wva_ctx* wva_group_ctx(wva_group* g, int32_t i);
int32_t wva_group_optimize(wva_group* g, const wva_system* sys, wva_solution* out);

/* ---- queueing sizing + allocator ---------------------------------------- */
/* System.SetFromSpec (pkg/core/system.go:82-89): copies the SoA to HBM. */
int32_t wva_load_system(wva_ctx* ctx, const wva_system* sys);
/* OptimizerSpec (pkg/config/types.go:145-149) and CapacityData (types.go:40-50) of the LOADED system, replaced in
 * place: the candidates of a wva_calculate stay valid (sizing reads neither), only wva_solve must run again —
 * what Optimizer.Optimize does when the same System is solved under another spec (pkg/solver/optimizer.go:24-36). */
int32_t wva_set_optimizer(wva_ctx* ctx, int32_t unlimited, int32_t delayed_best_effort, int32_t saturation_policy);
int32_t wva_set_capacity(wva_ctx* ctx, const int32_t* type_count /* [T] */);
/* System.Calculate (pkg/core/system.go:258-268) -> Server.Calculate (server.go:55-67)
 * -> CreateAllocation (allocation.go:27-155) for every (server, accelerator). */
int32_t wva_calculate(wva_ctx* ctx);
/* Replace the per-cycle server columns of the loaded system in place: ServerLoadSpec and CurrentAlloc
 * (pkg/config/types.go), i.e. what AddServerInfoToSystemData (internal/utils/utils.go:204-240) rewrites every cycle.
 * All six arrays are [S] and required; srv_cur_acc follows wva_load_system's rule (else WVA_ERR_ARG and nothing
 * changes).  WVA_ERR_STATE before wva_load_system.  A device pass compares the new values bitwise with the resident
 * ones (-0.0 vs 0.0 and differing NaN payloads are changes) and marks each server of the ctx's block: re-size when
 * arrival, in_tokens or out_tokens changed, or cur_acc changed on a keepAccelerator server; re-value when only the
 * current allocation changed.  Marks accumulate until the next wva_calculate or wva_recalculate.  The servers whose
 * load changed also get a grid mark, which accumulates until the next wva_grid_run or wva_grid_update.  The candidates
 * and the resident grid are left as they were; wva_solve, wva_grid_run and wva_analyze_grid read the new columns. */
int32_t wva_update_servers(wva_ctx* ctx, const float* srv_arrival, const int32_t* srv_in_tokens,
                           const int32_t* srv_out_tokens, const int32_t* srv_cur_acc, const int32_t* srv_cur_replicas,
                           const float* srv_cur_cost);
/* Bring the candidates up to date with every wva_update_servers since the last wva_calculate / wva_recalculate:
 * re-size the servers whose sizing inputs changed (the sizer wva_calculate would pick for that many servers, on a
 * gathered copy of their columns) and re-value the ones whose current allocation alone changed.  With table marks of
 * wva_update_tables pending, the pairs of the re-size-marked servers and the table-marked pairs are re-sized in place
 * instead (the sizer picked for that many pairs), after the re-valuation; the counts stay whole servers.  The candidates are
 * bit-equal to those of a wva_calculate, except n_solves, which counts the solves of the sizer that last sized the pair
 * (the sizers spend different numbers of solves on the same result).  *n_resized / *n_revalued (either may be NULL) get the two counts of the ctx's
 * block.  WVA_ERR_STATE unless the resident candidates come from wva_calculate / wva_recalculate on the loaded system:
 * after wva_load_system until the next wva_calculate, after wva_set_candidates, and after a failed sizing.  Timing as
 * for wva_calculate, with calculate_ms over the whole call; with nothing to re-size sizer_kernel and the counts are 0. */
int32_t wva_recalculate(wva_ctx* ctx, int64_t* n_resized, int64_t* n_revalued);
/* Replace the server set of the loaded system in place: System.AddServerFromSpec / RemoveServer (pkg/core/system.go)
 * for a whole cycle's servers at once, with every server column re-specified.  `servers` carries the n_servers (S') new
 * servers' 15 srv_* columns, in ascending-name order (INTEGRATION.md §3); its accelerator, model, perf, type and
 * optimizer fields are ignored, the loaded system's tables stay.  prev[i] (may be NULL when S' = 0) is the index of new
 * server i in the loaded system, or -1 for a new server; old indices that appear nowhere are the removed servers.
 * WVA_ERR_ARG, with nothing changed, unless every prev entry is in [-1, S), the non-negative ones are strictly
 * increasing, and the columns pass wva_load_system's server checks (non-NULL, srv_model < M, the srv_cur_acc rule).
 * WVA_ERR_STATE before wva_load_system, and on a ctx with a communicator unless the set is unchanged (S' = S,
 * prev[i] = i): its rank blocks cannot move.
 * Every per-server resident array follows the new set: the server columns, the candidate rows, the resident grid (when
 * it comes from wva_grid_run / wva_grid_update: levels and frontier) and the pending marks of wva_update_servers; the
 * solution is void (wva_get_solution is WVA_ERR_STATE until wva_solve).  A new server's candidates are nil
 * (WVA_ALLOC_NONE, every field 0) and its grid rows not ok with frontier 0, until it is sized or re-gridded.  Each kept
 * server is compared bitwise with its old row and marked as wva_update_servers marks it, widened to every column:
 * re-size when a column sizer_setup reads changed (the load, srv_model, max batch, target, SLOs, min replicas,
 * keepAccelerator, or cur_acc on a server whose keepAccelerator is set before or after), re-value when only the current
 * allocation changed, nothing when only srv_priority changed; a grid mark when a column the grid reads changed (the
 * load, srv_model, max batch, target, SLOs).  New servers get both marks.  wva_recalculate and wva_grid_update then
 * consume the marks as they do after wva_update_servers, with the candidates and grid of wva_load_system +
 * wva_calculate (+ wva_grid_run) on the new system; wva_set_candidates still rules out wva_recalculate.  When the set
 * changes, the new arenas are reserved before anything moves (WVA_ERR_NOMEM changes nothing) and swapped in after the
 * move, so the call needs the old and the new arenas at once: about twice the grid's size with full outputs (2 x 14 GB
 * for 100 000 servers x 32 accelerators at R = 256).  Timing: h2d_ms covers the whole call. */
int32_t wva_update_server_set(wva_ctx* ctx, int32_t n_servers, const int32_t* prev /* [S'] */, const wva_system* servers);
/* Replace the accelerator and model performance tables of the loaded system in place: the accelerator costs an
 * operator edits (internal/utils/utils.go:140-156) and the ModelAcceleratorPerfData a tuner re-estimates every cycle
 * (internal/engines/analyzers/queueingmodel/tuner/tuner.go:189-244).  `tables` carries acc_cost, acc_multiplicity,
 * acc_type ([A]) and the seven perf_* arrays ([M*A]); n_acc, n_types and n_models must be the loaded ones (adding or
 * removing accelerators, types or models is wva_load_system).  Its server columns, type_count (wva_set_capacity) and
 * optimizer fields are ignored.  WVA_ERR_ARG, with nothing changed, on a NULL array, another shape, or a violation of
 * wva_load_system's table checks (acc_type in [0, T), finite alpha / beta / gamma >= 0 on every present perf row).
 * WVA_ERR_STATE before wva_load_system.
 * One H2D copy, then one device pass compares every entry bitwise with the resident one (-0.0 vs 0.0 is a change),
 * writes it over it and marks table rows, not servers, so the marks stay valid across wva_update_server_set:
 *   - a perf row (m, a) for sizing when alpha, beta, gamma, max_batch, at_tokens, acc_count or present changed, and for
 *     the grid when any of them but acc_count changed (the grid reads neither acc_count nor acc_cost);
 *   - an accelerator a for sizing when acc_cost[a] changed (every candidate's cost and value on it);
 *   - nothing for acc_multiplicity and acc_type: only the allocators read them, and the solution is void until
 *     wva_solve.
 * Pair (s, a) of the ctx's block then needs re-sizing when srv_model[s] = m >= 0 and row (m, a) or accelerator a is
 * sizing-marked, and re-gridding when row (m, a) is grid-marked; unknown-model servers read no table.  *n_marked (may be
 * NULL) = the pairs of the block this call's diff marks for re-sizing.  The marks accumulate from call to call:
 * wva_recalculate consumes the sizing marks and wva_grid_update the grid marks, each re-sizing / re-gridding every pair
 * of a server-marked server and the table-marked pairs of the others, in place through a list of pairs, to the
 * candidates and grid of wva_load_system + wva_calculate (+ wva_grid_run) on the updated system.  wva_calculate voids
 * the sizing marks, wva_grid_run the grid marks, wva_load_system both; each call leaves the other kind alone.  With a
 * communicator every rank passes the same tables and marks its own block; no collective is involved.  Timing: h2d_ms
 * covers the whole call. */
int32_t wva_update_tables(wva_ctx* ctx, const wva_system* tables, int64_t* n_marked);
/* Manager.Optimize (pkg/manager/manager.go:21-27): Optimizer.Optimize
 * (pkg/solver/optimizer.go:24-36) -> Solver.Solve (solver.go:32-60) — SolveUnlimited
 * (solver.go:63-79) or SolveGreedy (greedy.go:35-105) — then AllocateByType. */
int32_t wva_solve(wva_ctx* ctx);
/* Server.AllAllocations() of every server (server.go:138-140). */
int32_t wva_get_candidates(wva_ctx* ctx, wva_candidates* out);
/* Install candidates computed elsewhere — on another GPU, for another shard of the servers — in place of a
 * wva_calculate on this context: Server.allAllocations (pkg/core/server.go:21,55-67) is plain per-server data, and
 * Solver.Solve (pkg/solver/solver.go:32-60) reads nothing else of the sizing.  This is the exchange step of the
 * model-sharded limited-capacity solve: every rank sizes its shard, the candidate arrays are all-gathered, and the
 * greedy sweep — which needs all servers — runs on the merged set.  All arrays are [S*A] for the LOADED system and
 * required except n_solves; state must be a WVA_ALLOC_* value and num_replicas >= 0 (else WVA_ERR_ARG). */
int32_t wva_set_candidates(wva_ctx* ctx, const wva_candidates* in);
/* System.GenerateSolution (system.go:303-319) + allocationByType. */
int32_t wva_get_solution(wva_ctx* ctx, wva_solution* out);

/*
 * Replica-grid evaluator: for every (server, accelerator, r in 1..R) one
 * QueueAnalyzer.Analyze(totalRate / r) (pkg/analyzer/queueanalyzer.go:127-167),
 * i.e. exactly the call CreateAllocation makes at allocation.go:140-148 with
 * numReplicas = r.  Outputs (any may be NULL), row-major [S][A][R]:
 *   ok    1 if Analyze returned metrics (rate in range), else 0
 *   ttft  AvgWaitTime + AvgPrefillTime;  itl AvgTokenTime;  rho;  tput Throughput
 * frontier [S*A]: smallest r whose metrics meet every non-zero SLO of the server
 *   (ttft <= slo_ttft, itl <= slo_itl), 0 if none in 1..R — the per-(model,
 *   variant) feasible frontier the north-star design reduces to.
 * Levels whose chain overflows float64 get the reference's rescaled metrics like
 * every other level (timing overflow_pairs counts them); more than
 * min(S*A*R, 16*S*A + 1024) of them in one run is WVA_ERR_LIMIT.  Batch sizes
 * above 10188 are WVA_ERR_LIMIT.
 */
int32_t wva_analyze_grid(wva_ctx* ctx, int32_t R, uint8_t* ok, float* ttft,
                         float* itl, float* rho, float* tput, int32_t* frontier);
/* The same in two steps, so a caller can keep the grid resident in HBM:
 * wva_grid_run evaluates it on the loaded system (full != 0 materialises the
 * per-level arrays, the frontier is always produced); wva_grid_fetch copies the
 * requested arrays to host buffers (NULL = skip). */
int32_t wva_grid_run(wva_ctx* ctx, int32_t R, int32_t full);
int32_t wva_grid_fetch(wva_ctx* ctx, uint8_t* ok, float* ttft, float* itl,
                       float* rho, float* tput, int32_t* frontier);
/* Bring the resident grid of the last wva_grid_run up to date with every wva_update_servers since the last
 * wva_grid_run / wva_grid_update: re-evaluate, at the same R and with the same outputs (full or frontier only), the
 * servers of the ctx's block whose arrival, in_tokens or out_tokens changed (bitwise), and write their rows over the
 * resident ones (in place when every server of the block changed).  *n_regridded (may be NULL) = that number of
 * servers.  The grid is bit-equal to that of a
 * wva_grid_run on the updated system: a server's rows read no current-allocation column.  These grid marks are apart
 * from the sizing marks: wva_calculate / wva_recalculate leave them, and the grid calls leave the sizing marks.  The
 * deferred pass and the batch size limit are decided from the re-evaluated servers; the float64-overflow list has the
 * capacity of a run on the whole block.  WVA_ERR_STATE unless the resident grid comes from wva_grid_run /
 * wva_grid_update on the loaded system: before wva_load_system, after it until the next wva_grid_run, and after a
 * failed grid call.  grid_ms covers the whole call; chain_solves, chain_states, overflow_pairs and certify_fallbacks
 * are those of the re-evaluated servers, 0 when none.  With grid marks of wva_update_tables pending, every pair of a
 * marked server and the pairs whose perf row changed are re-evaluated in place through a list of pairs, from which the
 * deferred pass and the batch size limit are then decided; *n_regridded still counts the marked servers. */
int32_t wva_grid_update(wva_ctx* ctx, int64_t* n_regridded);

/*
 * Closed-form M/M/1/K leg: MM1KModel.Solve (pkg/analyzer/mm1kmodel.go:30-92).
 * n independent (lambda, mu, K) triples -> valid flag + 6 float32 statistics.
 */
int32_t wva_mm1k_eval(wva_ctx* ctx, int64_t n, const float* lambda,
                      const float* mu, const int32_t* K, uint8_t* valid,
                      float* avg_resp, float* avg_wait, float* avg_serv,
                      float* avg_num, float* avg_queue, float* throughput,
                      float* rho);

/* ---- V1 saturation capacity model --------------------------------------- */
/*
 * Saturation inputs: M models, V variants (CSR by model), P replicas (CSR by
 * variant, in the order the reference's metric slice lists them).
 * Replaces saturation.Analyzer.AnalyzeModelSaturation
 * (internal/saturation/analyzer.go:31-131) and CalculateSaturationTargets
 * (analyzer.go:290-439) for a whole batch of models in one call.
 * Variants of a model must be indexed in ascending VariantName order.
 */
typedef struct wva_saturation_in {
  int64_t n_models, n_variants, n_replicas;
  const int32_t* model_variant_off;  /* [M+1]                                     */
  const int32_t* variant_replica_off;/* [V+1] (int64 not needed below 2^31 replicas) */
  /* ReplicaMetrics (internal/interfaces/saturation_analyzer.go:12-22) */
  const double* rep_kv;              /* [P] KvCacheUsage                          */
  const int64_t* rep_queue;          /* [P] QueueLength (Go int)                  */
  /* VariantReplicaState (saturation_analyzer.go:228-243) + Cost */
  const double* var_cost;            /* [V]                                       */
  const int32_t* var_current;        /* [V] CurrentReplicas                       */
  const int32_t* var_desired;        /* [V] DesiredReplicas                       */
  const int32_t* var_pending;        /* [V] PendingReplicas                       */
  const uint8_t* var_has_state;      /* [V] 0 = no VariantReplicaState for the variant
                                        (stateMap lookup yields the zero value); may be NULL = all 1 */
  /* SaturationScalingConfig per model (saturation_scaling.go:8-47) */
  const double* cfg_kv_threshold;    /* [M]                                       */
  const double* cfg_queue_threshold; /* [M]                                       */
  const double* cfg_kv_trigger;      /* [M]                                       */
  const double* cfg_queue_trigger;   /* [M]                                       */
} wva_saturation_in;

typedef struct wva_saturation_out {  /* any pointer may be NULL (skipped)         */
  int32_t* var_target;               /* [V] CalculateSaturationTargets result     */
  /* VariantSaturationAnalysis (saturation_analyzer.go:98-109) */
  int32_t* var_replica_count;        /* [V]                                       */
  int32_t* var_non_saturated;        /* [V]                                       */
  double* var_max_kv;                /* [V]                                       */
  int64_t* var_max_queue;            /* [V]                                       */
  double* var_avg_spare_kv;          /* [V]                                       */
  double* var_avg_spare_queue;       /* [V]                                       */
  uint8_t* rep_saturated;            /* [P] 1 if the replica is in SaturatedReplicas */
  /* ModelSaturationAnalysis (saturation_analyzer.go:74-95) */
  int32_t* mod_total_replicas;       /* [M]                                       */
  int32_t* mod_non_saturated;        /* [M]                                       */
  double* mod_avg_spare_kv;          /* [M]                                       */
  double* mod_avg_spare_queue;       /* [M]                                       */
  uint8_t* mod_flags;                /* [M] bit0 ShouldScaleUp, bit1 ScaleDownSafe,
                                            bit2 model in transition, bit3 kv trigger,
                                            bit4 queue trigger                    */
  int64_t* partials;                 /* [4] n_scale_up, n_scale_down, n_transition,
                                            sum of targets (shard partials for the
                                            all-reduce across GPUs)               */
  int64_t* partials_all;             /* [4] the same summed over every rank of the ctx's communicator (one
                                            ncclAllReduce inside wva_saturation_run); == partials without one */
} wva_saturation_out;

#define WVA_SAT_SCALE_UP 1
#define WVA_SAT_SCALE_DOWN_SAFE 2
#define WVA_SAT_IN_TRANSITION 4
#define WVA_SAT_KV_TRIGGERED 8
#define WVA_SAT_QUEUE_TRIGGERED 16

int32_t wva_saturation_v1(wva_ctx* ctx, const wva_saturation_in* in,
                          const wva_saturation_out* out);
/* the same over a group of devices (see wva_group above): device i analyses the i-th contiguous block of models */
int32_t wva_group_saturation_v1(wva_group* g, const wva_saturation_in* in, const wva_saturation_out* out);
/* The same in three steps (inputs / results stay resident in HBM between them):
 * upload = host -> HBM copy of the metric batch; run = the analysis + targets
 * kernel (detail == 0 writes only var_target, mod_flags and partials); fetch =
 * HBM -> host copy of the requested outputs (NULL = skip). */
int32_t wva_saturation_upload(wva_ctx* ctx, const wva_saturation_in* in);
int32_t wva_saturation_run(wva_ctx* ctx, int32_t detail);
int32_t wva_saturation_fetch(wva_ctx* ctx, const wva_saturation_out* out);

/* ---- Collector -> SoA ingest + streaming reconcile (one CUDA graph per metric batch) ------------------------------- */
/*
 * Replaces the per-model, string-keyed assembly of []ReplicaMetrics — CollectReplicaMetrics
 * (internal/collector/replica_metrics.go:78-403: six Prometheus vectors folded into a map keyed by pod name, every pod
 * matched to its VariantAutoscaling through PodVAMapper.FindVAForPod, source/pod_va_mapper.go:32) — for the V1
 * saturation path.  The string work happens once per pod: the caller registers every pod into a SLOT of its variant
 * (registry = CSR model -> variant -> slot; the slots of a variant in ascending pod-name order, which is the canonical
 * order of the per-variant float64 sums) and keeps a map pod name -> slot.  Every cycle the Prometheus response parser
 * writes each sample into page-locked columns indexed by slot (wva_ingest_write, or directly through `cols`), fills the
 * per-variant state and per-model config columns, and calls wva_ingest_commit: ONE CUDA graph launch uploads the column
 * arena, packs the pods that reported into CSR replica arrays on the device (a pod with neither metric is skipped, a
 * missing metric reads 0, queue = int(value): replica_metrics.go:160,296-318), runs the V1 analysis + targets kernel and
 * downloads the decision arena.  `res` arrays are valid after wva_ingest_commit returns, until the next commit.
 * A registry change (pods added / removed) = destroy + create (ints only).
 */
typedef struct wva_ingest wva_ingest;
enum { WVA_VEC_KV_CACHE_USAGE = 0, WVA_VEC_QUEUE_LENGTH = 1 };   /* registration.QueryKvCacheUsage / QueryQueueLength */
typedef struct wva_ingest_columns {  /* page-locked host memory owned by the wva_ingest; the collector writes it      */
  int64_t n_slots, n_variants, n_models;
  double* kv;                        /* [slots] KvCacheUsage sample value                                            */
  double* queue;                     /* [slots] queue-length sample value (converted with Go's int(float64) on the device) */
  uint8_t* has;                      /* [slots] bit0: a KV sample arrived this cycle, bit1: a queue sample arrived    */
  double* var_cost;                  /* [V] as wva_saturation_in                                                      */
  int32_t* var_current; int32_t* var_desired; int32_t* var_pending;
  double* cfg_kv_threshold; double* cfg_queue_threshold; double* cfg_kv_trigger; double* cfg_queue_trigger;   /* [M] */
} wva_ingest_columns;
typedef struct wva_ingest_results {  /* page-locked host memory owned by the wva_ingest                               */
  int32_t* var_target;               /* [V] CalculateSaturationTargets (-1 = variant absent from the map)             */
  int32_t* var_replica_count;        /* [V] pods of the variant that reported                                         */
  int32_t* var_non_saturated;        /* [V]                                                                           */
  double* var_avg_spare_kv;          /* [V] (VariantDecision.SpareCapacity: the limiter's sort key, engine.go:650-651) */
  double* var_avg_spare_queue;       /* [V]                                                                           */
  uint8_t* mod_flags;                /* [M] WVA_SAT_*                                                                 */
  int32_t* mod_total_replicas;       /* [M]                                                                           */
  int64_t* partials;                 /* [4] as wva_saturation_out                                                     */
} wva_ingest_results;
int32_t wva_ingest_create(wva_ctx* ctx, int64_t n_models, int64_t n_variants, int64_t n_slots,
                          const int32_t* model_variant_off /* [M+1] */, const int32_t* variant_slot_off /* [V+1] */,
                          wva_ingest** out, wva_ingest_columns* cols, wva_ingest_results* res);
int32_t wva_ingest_destroy(wva_ingest* ing);
/* start of a cycle: no pod has reported yet */
int32_t wva_ingest_begin(wva_ingest* ing);
/* one Prometheus-shaped vector keyed by slot, in result order: later samples of a pod overwrite earlier ones (the
 * reference assigns into a map, replica_metrics.go:133-160); slot < 0 = no pod label / unknown pod: skipped.  A vector of
 * 64 K samples or more that is not in registry order is binned by slot range over up to 8 host threads (same result as
 * the serial loop; WVA_INGEST_THREADS overrides the count, 1 = always serial). */
int32_t wva_ingest_write(wva_ingest* ing, int32_t which /* WVA_VEC_* */, int64_t n, const int32_t* slot, const double* value);
/* metric batch -> decisions: one CUDA graph launch (wva_timing.saturation_ms = device time of the whole graph) */
int32_t wva_ingest_commit(wva_ingest* ing);

/*
 * Decision mode: the same graph carried on to the cycle's final decisions — the rest of optimizeV1
 * (internal/engines/saturation/engine.go:322-392) for every model at once, with no host round trip inside:
 *   Enforcer.EnforcePolicy per model (pipeline/enforcer.go:55-183; targets = var_target, -1 = absent from the map;
 *   has_cost = the variant has a reporting pod, analyzer.go:148-149, else DefaultVariantCost 10; variants of a model in
 *   ascending name order) -> convertSaturationTargetsToDecisions (engine.go:589-661) -> DefaultLimiter.Limit over all
 *   decisions of the cycle (pipeline/default_limiter.go:42-81, the pipeline of wva_limit) when enable_limiter != 0.
 * A model none of whose pods reported produces no decision and runs no enforcer (prepareModelData returns nil,
 * engine.go:737-742).  wva_ingest_create_decisions returns the plain `cols` / `res` (filled exactly as by
 * wva_ingest_create: pre-enforcer targets and analyses) plus the views below; begin / write / commit / destroy are
 * shared with the plain mode.  Every decision column is per cycle: the graph reads it at each commit.
 */
typedef struct wva_ingest_decision_columns {   /* page-locked host memory owned by the wva_ingest; filled every cycle  */
  int32_t n_types;                   /* T: accelerator types of the inventory                                          */
  int32_t* var_accelerator_type;     /* [V] index in [0, T) of VariantSaturationAnalysis.AcceleratorName (engine.go:648);
                                      *     -1 (or any value outside [0, T)) = "" or a type without a pool              */
  int32_t* var_gpus_per_replica;     /* [V] VariantReplicaState.GPUsPerReplica (<= 0 reads 1, engine.go:624-628)      */
  uint8_t* mod_scale_to_zero_enabled;/* [M] IsScaleToZeroEnabled for the model (enforcer.go:66)                     */
  double* mod_request_count;         /* [M] requestCountFunc's count over the retention period (enforcer.go:100,109) */
  uint8_t* mod_request_error;        /* [M] the request-count query failed: targets kept (enforcer.go:101-105)       */
  int32_t* type_limit;               /* [T] TypeInventory limitByType after Refresh (default_limiter.go:47-50)       */
  int32_t* enable_limiter;           /* [1] SaturationScalingConfig.EnableLimiter (engine.go:370); 0 = final = original */
} wva_ingest_decision_columns;
typedef struct wva_ingest_decision_results {   /* page-locked host memory owned by the wva_ingest                     */
  uint8_t* has_decision;             /* [V] a VariantDecision exists: reporting model, enforced target >= 0 (:611)   */
  int32_t* original_target;          /* [V] OriginalTargetReplicas = the enforced target (:636); -1 without decision */
  int32_t* target;                   /* [V] TargetReplicas after the limiter (greedy_saturation_algorithm.go:100)     */
  int32_t* gpus_allocated;           /* [V] GPUsAllocated (greedy_saturation_algorithm.go:99)                         */
  uint8_t* was_limited;              /* [V] WasLimited (greedy_saturation_algorithm.go:103-105)                       */
  int8_t* action;                    /* [V] Action before the limiter (:614-622): 1 scale-up, -1 scale-down, 0 no-change */
  uint8_t* mod_enforcer_applied;     /* [M] EnforcePolicy's second result (engine.go:334-341)                        */
} wva_ingest_decision_results;
int32_t wva_ingest_create_decisions(wva_ctx* ctx, int64_t n_models, int64_t n_variants, int64_t n_slots, int32_t n_types,
                                    const int32_t* model_variant_off /* [M+1] */, const int32_t* variant_slot_off /* [V+1] */,
                                    wva_ingest** out, wva_ingest_columns* cols, wva_ingest_results* res,
                                    wva_ingest_decision_columns* dcols, wva_ingest_decision_results* dres);

/* ---- GPU-count limiter ---------------------------------------------------- */
/*
 * DefaultLimiter.Limit (internal/engines/pipeline/default_limiter.go:42-81) with
 * TypeInventory.CreateAllocator / typeAllocator.TryAllocate
 * (type_inventory.go:222-243,347-373) and GreedyBySaturation.Allocate
 * (greedy_saturation_algorithm.go:34-108).  D decisions, T accelerator types.
 * acc_type[d] = -1 (or any value outside [0, T)) encodes AcceleratorName == "".
 * Outputs are the mutated VariantDecision fields.  Any T >= 0 is supported: the
 * type pass sorts as many key bits as T + 2 segments need.
 */
int32_t wva_limit(wva_ctx* ctx, int64_t n_decisions, int32_t n_types,
                  const int32_t* acc_type, const int32_t* current,
                  const int32_t* target, const int32_t* gpus_per_replica,
                  const double* spare_capacity, const double* cost,
                  const int32_t* type_limit, int32_t* out_target,
                  int32_t* out_gpus_allocated, uint8_t* out_was_limited);

/* ---- V2 pipeline: token-capacity analyzer, cost-aware optimizer, enforcer ------- */
/*
 * SaturationAnalyzer.Analyze (internal/engines/analyzers/saturation_v2/analyzer.go:59-138: computeReplicaCapacity
 * :142-211, aggregateByVariant :266-349, estimateSchedulerQueueDemand :471-501, median :505-519) for a batch of
 * models.  The arithmetic only: what the reference keeps in string-keyed state stays with the caller (SURVEY 8f.1) —
 * the k2 priority chain (computeK2 :218-262, rolling history) resolves rep_k2 per replica (on the device with
 * wva_k2_resolve below), the capacity store
 * resolves var_fallback_capacity for variants without ready replicas (:317-324).
 * Variants of a model in VariantStates order; replicas of a variant in ReplicaMetrics order.
 */
typedef struct {
  int64_t n_models, n_variants, n_replicas;
  const int32_t* model_variant_off;     /* [M+1] */
  const int32_t* variant_replica_off;   /* [V+1] */
  const int64_t* rep_total_kv_tokens;   /* [P] ReplicaMetrics.TotalKvCapacityTokens; <= 0: no capacity data, replica skipped */
  const int64_t* rep_tokens_in_use;     /* [P] */
  const int64_t* rep_queue_length;      /* [P] */
  const double* rep_avg_input_tokens;   /* [P] */
  const double* rep_avg_output_tokens;  /* [P] */
  const double* rep_prefix_hit_rate;    /* [P] */
  const int64_t* rep_k2;                /* [P] compute-bound capacity from the caller's chain; < 0 = fall back to k1 */
  const int32_t* rep_slice_order;       /* [P] or NULL: replica indices of each model in ReplicaMetrics slice order
                                           (model m owns positions [vro[mvo[m]], vro[mvo[m+1]])); NULL = as laid out */
  const int32_t* var_current;           /* [V] VariantReplicaState.CurrentReplicas */
  const int32_t* var_pending;           /* [V] PendingReplicas */
  const double* var_fallback_capacity;  /* [V] per-replica capacity when the variant has no replica with data; 0 = none */
  const double* cfg_kv_threshold;       /* [M] SaturationScalingConfig.KvCacheThreshold */
  const double* cfg_scale_up_threshold; /* [M] ScaleUpThreshold */
  const double* cfg_scale_down_boundary;/* [M] ScaleDownBoundary */
  const int64_t* sched_queue_size;      /* [M] or NULL: SchedulerQueueMetrics.QueueSize (NULL = no scheduler queue) */
  const int64_t* sched_queue_bytes;     /* [M] or NULL */
} wva_saturation_v2_in;

typedef struct {            /* any pointer may be NULL */
  int64_t* rep_k1;          /* [P] MemoryBoundCapacity */
  int64_t* rep_effective;   /* [P] EffectiveCapacity = min(k1, k2) */
  int64_t* rep_demand;      /* [P] ReplicaDemand */
  uint8_t* rep_saturated;   /* [P] IsSaturated */
  int32_t* var_ready;       /* [V] VariantCapacity.ReplicaCount */
  double* var_per_replica_capacity; /* [V] */
  double* var_total_capacity;       /* [V] */
  double* var_total_demand;         /* [V] */
  double* var_utilization;          /* [V] */
  double* mod_total_supply;         /* [M] AnalyzerResult.TotalSupply */
  double* mod_total_demand;         /* [M] */
  double* mod_utilization;          /* [M] */
  double* mod_required_capacity;    /* [M] */
  double* mod_spare_capacity;       /* [M] */
} wva_saturation_v2_out;
int32_t wva_saturation_v2(wva_ctx* ctx, const wva_saturation_v2_in* in, const wva_saturation_v2_out* out);

/*
 * CostAwareOptimizer.Optimize (internal/engines/pipeline/cost_aware_optimizer.go:39-197) for a batch of models:
 * scale-up on the most cost-efficient variants (cost / perReplicaCapacity ascending, ceil), scale-down on the most
 * expensive (cost descending, floor, the cheapest variant keeps one replica while no other variant has any).
 * Variants in VariantCapacities slice order (ties of the reference's unstable sorts resolve to that order).
 * var_target[v] = -1 for the variants of a model without a result (req.Result == nil: no decisions).
 */
int32_t wva_cost_aware_optimize(wva_ctx* ctx, int64_t n_models, int64_t n_variants, const int32_t* model_variant_off,
                                const double* mod_required_capacity, const double* mod_spare_capacity,
                                const uint8_t* mod_has_result /* or NULL */, const int32_t* var_current,
                                const double* var_cost, const double* var_per_replica_capacity, int32_t* var_target);

/*
 * Enforcer.EnforcePolicy (internal/engines/pipeline/enforcer.go:55-183) for a batch of models: scale-to-zero when it
 * is enabled and the model had no requests in its retention period (request count and lookup error supplied by the
 * caller), else keep one replica on the cheapest variant when every target is 0.  var_target is updated in place
 * (-1 = the variant is not in the targets map); mod_applied[m] = the bool EnforcePolicy returns.
 */
int32_t wva_enforce(wva_ctx* ctx, int64_t n_models, int64_t n_variants, const int32_t* model_variant_off,
                    const uint8_t* mod_scale_to_zero_enabled, const double* mod_request_count,
                    const uint8_t* mod_request_error /* or NULL */, const double* var_cost,
                    const uint8_t* var_has_cost /* or NULL */, int32_t* var_target, uint8_t* mod_applied);

/*
 * The three V2 stages for every model of a cycle in one call: wva_saturation_v2 -> wva_cost_aware_optimize (every
 * model has a result) -> wva_enforce, chained on the device — one upload of the metrics, three launches, one download
 * of the decisions.  What engine_v2.go / engine.go:461-520 does model by model through maps.  Index space =
 * VariantStates order; var_name_rank[v] = rank of the variant's name within its model (the enforcer's tie-break
 * compares names, enforcer.go:161), NULL when the states are already in name order.  `out` (or any member) may be NULL.
 */
int32_t wva_pipeline_v2(wva_ctx* ctx, const wva_saturation_v2_in* in, const double* var_cost, const int32_t* var_name_rank,
                        const uint8_t* mod_scale_to_zero_enabled, const double* mod_request_count,
                        const uint8_t* mod_request_error /* or NULL */, const wva_saturation_v2_out* out,
                        int32_t* var_target, uint8_t* mod_applied /* or NULL */);

/* ---- V2 k2 priority chain with its rolling history in HBM -------------------- */
/*
 * SaturationAnalyzer.computeK2 (internal/engines/analyzers/saturation_v2/analyzer.go:218-262) for every replica of a
 * cycle, with the analyzer's computeCapacityHistory (history.go, window RollingAverageWindowSize = 10, constants.go)
 * kept on the device for the life of the handle.  What the reference does, and the device reproduces exactly:
 *   - only replicas with TotalKvCapacityTokens > 0 run the chain (:148-150); the others neither read nor write history;
 *     replicas of a variant without a VariantReplicaState still do (Analyze loops over every ReplicaMetrics, :73-84);
 *   - the key is modelID|accelerator|bucket, without the namespace: the model groups (modelID|namespace,
 *     internal/utils/variant.go:64-74) of one modelID share it.  A HISTORY GROUP here is one modelID; its model groups
 *     are visited in registry order (one of Go's map orders), the replicas of a group in ReplicaMetrics slice order,
 *     and an append is seen by every later replica of the same key in the same cycle;
 *   - bucket (types.go:28-37): 0 short (avgOutput < 100), 1 medium (< 500), 2 long (otherwise, NaN included);
 *   - priority 1, observed: queueLen >= int(QueueLengthThreshold) (Go amd64 conversion: NaN / out of range ->
 *     INT64_MIN) && tokensInUse > 0: k2 = tokensInUse, appended to the key's window (the oldest value is dropped at 10);
 *   - priority 2, historical: the window's float64 sum, oldest to newest, / float64(len); > 0: k2 = int64(avg);
 *   - priority 3, derived: estimateCapacityFromParams (:418-437) with the VLLMParams of the store record
 *     namespace|model|variant as of the start of the cycle (the per-replica Update keeps them, :184-196);
 *   - priority 4: k2 = k1 = int64(float64(TotalKvCapacityTokens) * KvCacheThreshold); effective = min(k1, k2).
 * The capacity store itself stays with the caller: FindCompatible (capacity_store.go:153-187) returns the first live
 * record in map order, and the zero-replica fallback (:317-415) reads the store after this cycle's updates.  The
 * resolve returns what the caller needs to apply those updates once per store slot (last write wins, :188-197).
 * Nothing evicts keys (EvictStaleHistory has no caller in the reference); export / import is how a caller drops them.
 *
 * Registry (integers only; a change = export, create, import): H history groups; CSR history group -> model groups
 * (every model group in [0, G) exactly once); CSR history group -> its distinct accelerator ids (the caller maps names,
 * "" included, to ids >= 0); the number of store slots.  The keys of history group h are (accelerator k of h, bucket b)
 * at index (hg_acc_off[h] + k) * 3 + b.
 */
typedef struct wva_k2_history wva_k2_history;
int32_t wva_k2_history_create(wva_ctx* ctx, int64_t n_history_groups, int64_t n_model_groups, int64_t n_slots,
                              const int32_t* hg_model_off /* [H+1] */, const int32_t* hg_models /* [G] */,
                              const int32_t* hg_acc_off /* [H+1] */, const int32_t* hg_acc /* [hg_acc_off[H]] */,
                              wva_k2_history** out);
int32_t wva_k2_history_destroy(wva_k2_history* h);
/* number of history keys: 3 * hg_acc_off[H] */
int64_t wva_k2_history_keys(const wva_k2_history* h);

typedef struct {
  int64_t n_model_groups, n_replicas;       /* G must equal the registry's                                         */
  const int32_t* model_replica_off;         /* [G+1] replicas of model group g in ReplicaMetrics slice order         */
  const int64_t* rep_total_kv_tokens;       /* [P] TotalKvCapacityTokens; <= 0: no capacity data                      */
  const int64_t* rep_tokens_in_use;         /* [P] */
  const int64_t* rep_queue_length;          /* [P] */
  const double* rep_avg_input_tokens;       /* [P] */
  const double* rep_avg_output_tokens;      /* [P] */
  const int32_t* rep_accelerator;           /* [P] accelerator id; must be registered for the group's history group   */
  const int32_t* rep_slot;                  /* [P] store slot of namespace|model|variant, in [0, n_slots)             */
  const int32_t* rep_out_pos;               /* [P] or NULL: position in a wva_saturation_v2_in layout, -1 = not there */
  int64_t n_out;                            /* size of that layout (out_rep_k2)                                       */
  const int64_t* slot_max_batched_tokens;   /* [S] VLLMParams.EffectiveMaxBatchedTokens (0 = no params)               */
  const int64_t* slot_max_num_seqs;         /* [S] VLLMParams.MaxNumSeqs                                              */
  const double* cfg_queue_threshold;        /* [G] SaturationScalingConfig.QueueLengthThreshold                       */
  const double* cfg_kv_threshold;           /* [G] KvCacheThreshold                                                  */
} wva_k2_in;
typedef struct {
  int64_t* rep_k2;          /* [P] computeK2's result; -1 without capacity data (wva_saturation_v2_in.rep_k2 as is)   */
  int64_t* rep_effective;   /* [P] min(k1, k2); 0 without capacity data (may be NULL)                                  */
  int64_t* out_rep_k2;      /* [n_out] rep_k2 scattered to rep_out_pos, -1 elsewhere (NULL unless rep_out_pos given)   */
  int32_t* slot_last_rep;   /* [S] index of the slot's last data replica of the cycle, -1 = none (may be NULL)        */
  int64_t* slot_effective;  /* [S] that replica's EffectiveCapacity, 0 = none (may be NULL)                           */
} wva_k2_out;
/* One cycle: appends to the history once.  Every input is checked before the history changes; a call that returns an
 * error leaves it as it was.  wva_saturation_v2 / wva_pipeline_v2 may then run as often as the caller likes. */
int32_t wva_k2_resolve(wva_k2_history* h, const wva_k2_in* in, const wva_k2_out* out);
/* Every key (wva_k2_history_keys of them): history group, accelerator id, bucket, count (0..10), values [K*10] oldest
 * first (zeros past count). */
int32_t wva_k2_history_export(wva_k2_history* h, int32_t* hg, int32_t* acc, int32_t* bucket, int32_t* count, double* values);
/* Replaces the whole history with n keys in the export format (keys not listed start empty).  A key not registered,
 * listed twice, a bucket outside 0..2 or a count outside 0..10 is WVA_ERR_ARG and changes nothing. */
int32_t wva_k2_history_import(wva_k2_history* h, int64_t n, const int32_t* hg, const int32_t* acc, const int32_t* bucket,
                              const int32_t* count, const double* values);

/* ---- V2 ingest: metric batch -> V2 decisions in two graph launches around the host capacity store -------------------- */
/*
 * The V2 engine's cycle (optimizeV2, internal/engines/saturation/engine.go:397-488) from the six Prometheus vectors of
 * CollectReplicaMetrics (internal/collector/replica_metrics.go:78-403) to the final VariantDecisions, with the same
 * registry as wva_ingest (CSR model -> variant -> pod slot, the slots of a variant in ascending pod-name order: that
 * order is the ReplicaMetrics slice order of the model, variant after variant, the canonical stand-in for the
 * reference's `range podData` map order).  The capacity knowledge store stays with the caller, so a cycle is
 *   begin -> write (samples) + the per-cycle columns -> wva_ingest_v2_analyze -> host step -> wva_ingest_v2_decide.
 *
 * analyze (one graph launch): H2D of the column arena; per pod slot the replica fields (a pod reports iff it has a KV
 * or a queue sample, the missing one reads 0; queue = Go's int(float64); TotalKvCapacityTokens = blocks * size with
 * hasCacheConfig, INT64_MAX on overflow, else 0; TokensInUse = clamp(math.Round(kv * total), 0, total) converted as
 * Go's int64(float64)); the reporting pods packed per variant; the k2 chain of wva_k2_resolve against the handle's
 * history (model group m of the history = model m here); D2H of the per-slot store updates, the variants without a
 * replica with capacity data and the model workload averages (computeModelWorkloadAverages, analyzer.go:438-455).
 * The registry checks of the k2 chain are made once at create; if the chain's error word is set anyway, the history is
 * left as it was (the kernels test it on the device) and analyze returns WVA_ERR_ARG.
 *
 * host step (the caller, between the launches): the store updates once per store slot with slot_last_rep >= 0
 * (analyzer.go:184-196, last write wins), then var_fallback_capacity for the variants with var_no_data (:317-415).
 *
 * Every column but var_fallback_capacity goes up with analyze: only var_fallback_capacity may change between analyze
 * and decide (a write to another column in between is not seen by decide).
 *
 * decide (one graph launch): H2D of var_fallback_capacity; SaturationAnalyzer.Analyze -> CostAwareOptimizer.Optimize
 * -> Enforcer.EnforcePolicy (the kernels of wva_pipeline_v2) for every model with a reporting pod (the others make no
 * ModelScalingRequest: prepareModelData returns nil, engine.go:738-742); D2H of the results.  The optimizer and the
 * enforcer see a variant's cost only when it has a reporting pod (the VariantCapacity's Cost is 0 otherwise).
 * `res` arrays are valid after the launch that fills them, until the next one.  Registry change = destroy + create.
 */
typedef struct wva_ingest_v2 wva_ingest_v2;
enum { WVA_VEC_AVG_OUTPUT_TOKENS = 2, WVA_VEC_AVG_INPUT_TOKENS = 3, WVA_VEC_PREFIX_CACHE_HIT_RATE = 4 };
#define WVA_CACHE_LABEL_ABSENT INT64_MIN     /* a cache_config_info label that is absent or does not parse as int64 */
typedef struct wva_ingest_v2_columns { /* page-locked host memory owned by the wva_ingest_v2; written every cycle   */
  int64_t n_slots, n_variants, n_models, n_store_slots;
  double* kv;                          /* [slots] KvCacheUsage sample                                               */
  double* queue;                       /* [slots] queue-length sample                                               */
  int64_t* num_gpu_blocks;             /* [slots] parsed cache_config_info labels                                   */
  int64_t* block_size;                 /* [slots]                                                                   */
  double* avg_output_tokens;           /* [slots] 0 until a finite sample arrives                                   */
  double* avg_input_tokens;            /* [slots]                                                                   */
  double* prefix_hit_rate;             /* [slots] 0 until a finite sample in [0, 1] arrives                         */
  uint8_t* has;                        /* [slots] bit0 KV sample, bit1 queue sample, bit2 hasCacheConfig            */
  double* var_cost;                    /* [V] ReplicaMetrics.Cost of the variant's pods                             */
  int32_t* var_current; int32_t* var_pending;   /* [V] VariantReplicaState                                          */
  int32_t* var_name_rank;              /* [V] rank of the variant's name among its model's (enforcer tie-break)     */
  double* cfg_kv_threshold; double* cfg_queue_threshold;                 /* [M] SaturationScalingConfig            */
  double* cfg_scale_up_threshold; double* cfg_scale_down_boundary;       /* [M]                                    */
  uint8_t* mod_scale_to_zero_enabled; double* mod_request_count; uint8_t* mod_request_error;   /* [M] enforcer     */
  int64_t* slot_max_batched_tokens;    /* [store slots] VLLMParams.EffectiveMaxBatchedTokens at the cycle's start  */
  int64_t* slot_max_num_seqs;          /* [store slots] VLLMParams.MaxNumSeqs                                       */
  double* var_fallback_capacity;       /* [V] written by the host step, read by decide                              */
} wva_ingest_v2_columns;
typedef struct wva_ingest_v2_results { /* page-locked host memory owned by the wva_ingest_v2                        */
  /* analyze */
  int32_t* variant_replica_off;        /* [V+1] replicas of variant v (its reporting pods, slot order)              */
  int32_t* rep_pod;                    /* [slots] pod slot of replica r (first variant_replica_off[V] valid)        */
  int64_t* rep_total_kv_tokens;        /* [slots] TotalKvCapacityTokens of replica r                                */
  int32_t* slot_last_rep;              /* [store slots] last replica with capacity data of the slot, -1 = none      */
  int64_t* slot_effective;             /* [store slots] its EffectiveCapacity                                       */
  uint8_t* var_no_data;                /* [V] no replica with capacity data: the zero-replica fallback applies      */
  uint8_t* mod_has_request;            /* [M] a pod of the model reported                                           */
  double* mod_avg_input_tokens; double* mod_avg_output_tokens;           /* [M] workload averages                  */
  /* decide */
  int32_t* var_optimizer_target;       /* [V] CostAwareOptimizer's TargetReplicas, -1 without request               */
  int32_t* var_target;                 /* [V] the enforced target, -1 without request                              */
  int8_t* var_action;                  /* [V] sign(enforced target - current)                                       */
  uint8_t* mod_enforced;               /* [M] EnforcePolicy's second result (0 without request)                     */
  int32_t* var_ready;                  /* [V] as wva_saturation_v2_out                                              */
  double* var_per_replica_capacity; double* var_total_capacity; double* var_total_demand; double* var_utilization;
  double* mod_total_supply; double* mod_total_demand; double* mod_utilization;
  double* mod_required_capacity; double* mod_spare_capacity;
} wva_ingest_v2_results;
/* var_accelerator [V]: accelerator id of the variant, registered for its model's history group; var_store_slot [V]:
 * store slot of namespace|model|variant in [0, the history's n_slots).  The history's model groups must be the models. */
int32_t wva_ingest_v2_create(wva_ctx* ctx, int64_t n_models, int64_t n_variants, int64_t n_slots,
                             const int32_t* model_variant_off /* [M+1] */, const int32_t* variant_slot_off /* [V+1] */,
                             const int32_t* var_accelerator, const int32_t* var_store_slot, wva_k2_history* h,
                             wva_ingest_v2** out, wva_ingest_v2_columns* cols, wva_ingest_v2_results* res);
int32_t wva_ingest_v2_destroy(wva_ingest_v2* ing);
/* start of a cycle: no pod has a sample; avg_* and prefix_hit_rate read 0, the cache config is unset */
int32_t wva_ingest_v2_begin(wva_ingest_v2* ing);
/* one vector keyed by slot, in result order (WVA_VEC_*: a later sample of a pod overwrites an earlier one; a
 * non-finite avg_* sample, or a hit rate that is non-finite or outside [0, 1], overwrites nothing); slot < 0 skipped */
int32_t wva_ingest_v2_write(wva_ingest_v2* ing, int32_t which, int64_t n, const int32_t* slot, const double* value);
/* cache_config_info: per sample the parsed labels (WVA_CACHE_LABEL_ABSENT leaves the value as it is); bit2 of `has`
 * is set once both values are > 0 after a sample */
int32_t wva_ingest_v2_write_cache_config(wva_ingest_v2* ing, int64_t n, const int32_t* slot, const int64_t* num_gpu_blocks,
                                         const int64_t* block_size);
int32_t wva_ingest_v2_analyze(wva_ingest_v2* ing);
int32_t wva_ingest_v2_decide(wva_ingest_v2* ing);

/* ---- host memory ----------------------------------------------------------- */
/* Page-locked host buffers for the caller's SoA arrays (the collector writes its batch straight into them): every
 * entry point copies from / to such a buffer by DMA at link speed instead of through the driver's pageable staging
 * (several times faster for a batch of replica metrics).  Any host pointer is accepted everywhere — this is an
 * optimisation, not a requirement.  Not tied to a context; free with wva_host_free. */
int32_t wva_host_alloc(size_t bytes, void** out);
int32_t wva_host_free(void* p);

/* ---- observability -------------------------------------------------------- */
int32_t wva_last_timing(const wva_ctx* ctx, wva_timing* out);

/* microbenchmarks used by bench.py for the compute roofline (ops/s on device) */
int32_t wva_microbench_fp64(wva_ctx* ctx, double* dfma_per_s, double* ddiv_per_s);

#ifdef __cplusplus
}
#endif
#endif /* WVA_B200_H */
