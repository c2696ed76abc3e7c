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
  int32_t n_types;
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

/* ---- GPU-count limiter ---------------------------------------------------- */
/*
 * DefaultLimiter.Limit (internal/engines/pipeline/default_limiter.go:42-81) with
 * TypeInventory.CreateAllocator / typeAllocator.TryAllocate
 * (type_inventory.go:222-243,347-373) and GreedyBySaturation.Allocate
 * (greedy_saturation_algorithm.go:34-108).  D decisions, T accelerator types.
 * acc_type[d] = -1 encodes AcceleratorName == "".  Outputs are the mutated
 * VariantDecision fields.
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
 * the k2 priority chain (computeK2 :218-262, rolling history) resolves rep_k2 per replica, the capacity store
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
