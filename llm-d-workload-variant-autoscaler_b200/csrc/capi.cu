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
#include "overflow_slow_kernel.cuh"
#include "greedy_solve.cuh"
#include "greedy_sweep.cuh"
#include "mm1k_kernel.cuh"
#include "ingest_scatter.hpp"

#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <mutex>
#include <new>
#include <string>
#include <vector>

using namespace wva;

// ------------------------------------------------------------------ small helpers
struct DevBuf {  // growable device allocation
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct PinBuf {  // growable pinned host staging
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 8 + 256;
    cudaError_t e = cudaMallocHost(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// bump allocator over one arena: every sub-array 256-byte aligned
struct Layout {
  size_t off = 0;
  size_t take(size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; }
};

struct GridState {   // results of the last wva_grid_run, resident in HBM
  int R = 0;
  bool full = false, ran = false;
  DevBuf buf, defer;
  GridOut view = {};
  GridCounters* ctr = nullptr;
};
struct SatState {    // resident inputs / outputs of the saturation model
  bool uploaded = false, ran = false;
  long long M = 0, V = 0, P = 0;
  DevBuf in, out, desc;
  SatIn vin = {};
  SatOut vout = {};
  size_t out_bytes = 0;
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
  bool force_lane_sizer = false;
  int gang_refill = -1;             // lock-step lane sizer: a warp refills only when all its lanes are idle; -1 = by size
  int length_sort = -1;             // lane sizer pulls items through the probe-sorted permutation (sizer_probe.cuh); -1 = by size
  int table_mode = 0;        // WVA_OPT_TABLE_MODE
  int greedy_mode = 0;       // WVA_OPT_GREEDY_MODE
  int grid_defer = 0;        // WVA_OPT_GRID_DEFER
  int lane_sizer_mode = 2;   // 1 flattened, 2 lock-step (default), 3 lock-step with two chains per lane (slower: measured)
  int A = 0, T = 0, M = 0, S = 0;
  uint8_t unlimited = 1, delayed = 0;
  int policy = 0;
  DevBuf sys_arena, cand_arena, sol_arena, scratch, gtab, greedy_ws, split_ws, order_ws, pool_ws;
  PinBuf stage_in, stage_out;
  SysView sys = {};
  CandView cand = {};
  SolView sol = {};
  long long* d_type_count = nullptr;
  double* d_type_cost = nullptr;
  SizerCounters* d_ctr = nullptr;   // in scratch
  // generic io arenas for saturation / limiter / grid / mm1k
  DevBuf io_in, io_out;
  PinBuf io_stage_in, io_stage_out;
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
static SysView shard_sys(const wva_ctx* ctx) {
  SysView v = ctx->sys;
  const int lo = ctx->shard_lo;
  v.n_servers = ctx->shard_hi - ctx->shard_lo;
  v.srv_model += lo; v.srv_priority += lo; v.srv_min_replicas += lo; v.srv_max_batch += lo; v.srv_keep_acc += lo;
  v.srv_target_present += lo; v.srv_slo_ttft += lo; v.srv_slo_itl += lo; v.srv_slo_tps += lo; v.srv_arrival += lo;
  v.srv_in_tokens += lo; v.srv_out_tokens += lo; v.srv_cur_acc += lo; v.srv_cur_replicas += lo; v.srv_cur_cost += lo;
  return v;
}
static CandView shard_cand(const wva_ctx* ctx) {
  CandView c = ctx->cand;
  const size_t o = (size_t)ctx->shard_lo * ctx->A;
  c.state += o; c.num_replicas += o; c.batch_size += o; c.cost += o; c.value += o; c.itl += o; c.ttft += o; c.rho += o;
  c.max_arrv_rate += o; c.n_solves += o;
  return c;
}
static SolView shard_sol(const wva_ctx* ctx) {
  SolView c = ctx->sol;
  const size_t o = (size_t)ctx->shard_lo;
  c.state += o; c.acc += o; c.num_replicas += o; c.batch_size += o; c.cost += o; c.value += o; c.itl += o; c.ttft += o;
  c.rho += o; c.max_arrv_rate += o;
  return c;
}
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
  ctx->sys_arena.release(); ctx->cand_arena.release(); ctx->sol_arena.release(); ctx->scratch.release();
  ctx->gtab.release(); ctx->pool_ws.release(); ctx->greedy_ws.release(); ctx->split_ws.release(); ctx->order_ws.release(); ctx->grid.buf.release(); ctx->grid.defer.release(); ctx->sat.in.release(); ctx->sat.out.release(); ctx->sat.desc.release(); ctx->io_in.release(); ctx->io_out.release();
  ctx->stage_in.release(); ctx->stage_out.release(); ctx->io_stage_in.release(); ctx->io_stage_out.release();
  comm_release(ctx); ctx->comm_ws.release();
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
  if (s->n_types > WVA_MAX_TYPES) return WVA_ERR_LIMIT;
  CK(cudaSetDevice(ctx->device));
  const size_t A = s->n_acc, T = s->n_types, M = s->n_models, S = s->n_servers, MA = M * A;
  struct Item { const void* src; size_t bytes; size_t off; };
  Layout L;
  std::vector<Item> items;
  auto add = [&](const void* p, size_t bytes) { Item it{p, bytes, L.take(bytes)}; items.push_back(it); return it.off; };
  size_t o_acc_cost = add(s->acc_cost, A * 4), o_acc_mult = add(s->acc_multiplicity, A * 4),
         o_acc_type = add(s->acc_type, A * 4), o_type_count = add(s->type_count, T * 4);
  size_t o_pa = add(s->perf_alpha, MA * 4), o_pb = add(s->perf_beta, MA * 4), o_pg = add(s->perf_gamma, MA * 4),
         o_pmb = add(s->perf_max_batch, MA * 4), o_pat = add(s->perf_at_tokens, MA * 4),
         o_pac = add(s->perf_acc_count, MA * 4), o_pp = add(s->perf_present, MA);
  size_t o_sm = add(s->srv_model, S * 4), o_sp = add(s->srv_priority, S * 4), o_smr = add(s->srv_min_replicas, S * 4),
         o_smb = add(s->srv_max_batch, S * 4), o_sk = add(s->srv_keep_acc, S), o_stp = add(s->srv_target_present, S),
         o_st = add(s->srv_slo_ttft, S * 4), o_si = add(s->srv_slo_itl, S * 4), o_sps = add(s->srv_slo_tps, S * 4),
         o_sa = add(s->srv_arrival, S * 4), o_sin = add(s->srv_in_tokens, S * 4), o_sout = add(s->srv_out_tokens, S * 4),
         o_sca = add(s->srv_cur_acc, S * 4), o_scr = add(s->srv_cur_replicas, S * 4), o_scc = add(s->srv_cur_cost, S * 4);
  for (auto& it : items) if (it.bytes && !it.src) { ctx->last_error = "wva_load_system: a required array is NULL"; return WVA_ERR_ARG; }
  // validate indices the kernels dereference (after the NULL checks above)
  for (size_t a = 0; a < A; a++)
    if (s->acc_type[a] < 0 || s->acc_type[a] >= (int)T) { ctx->last_error = "wva_load_system: acc_type out of range"; return WVA_ERR_ARG; }
  for (size_t i = 0; i < S; i++) {
    if (s->srv_model[i] >= (int)M) { ctx->last_error = "wva_load_system: srv_model out of range"; return WVA_ERR_ARG; }
    if (s->srv_cur_acc[i] >= (int)A || s->srv_cur_acc[i] < WVA_CUR_ACC_UNKNOWN) { ctx->last_error = "wva_load_system: srv_cur_acc out of range"; return WVA_ERR_ARG; }
  }
  // ServiceParms (pkg/analyzer/queueanalyzer.go:33-38) are measured service-time coefficients: finite and >= 0.  A
  // negative or NaN coefficient makes arrival rates negative (QueueModel.Solve's gate, queuemodel.go:31) or NaN and
  // the sizing meaningless; it is rejected here instead of being carried into the kernels.
  for (size_t i = 0; i < MA; i++) {
    if (!s->perf_present[i]) continue;
    const float a = s->perf_alpha[i], b = s->perf_beta[i], g = s->perf_gamma[i];
    if (!(a >= 0.0f && b >= 0.0f && g >= 0.0f) || a > 3.0e38f || b > 3.0e38f || g > 3.0e38f) {
      ctx->last_error = "wva_load_system: perf_alpha / perf_beta / perf_gamma must be finite and >= 0";
      return WVA_ERR_ARG;
    }
  }
  const size_t total = L.off + 256;
  CK(ctx->stage_in.reserve(total));
  CK(ctx->sys_arena.reserve(total));
  char* h = (char*)ctx->stage_in.p;
  for (auto& it : items) if (it.bytes) memcpy(h + it.off, it.src, it.bytes);
  CK(cudaEventRecord(ctx->ev[0], ctx->stream));
  CK(cudaMemcpyAsync(ctx->sys_arena.p, h, total, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  char* d = (char*)ctx->sys_arena.p;
  SysView& v = ctx->sys;
  v.n_acc = (int)A; v.n_types = (int)T; v.n_models = (int)M; v.n_servers = (int)S;
  v.acc_cost = (const float*)(d + o_acc_cost); v.acc_multiplicity = (const int*)(d + o_acc_mult);
  v.acc_type = (const int*)(d + o_acc_type); v.type_count = (const int*)(d + o_type_count);
  v.perf_alpha = (const float*)(d + o_pa); v.perf_beta = (const float*)(d + o_pb); v.perf_gamma = (const float*)(d + o_pg);
  v.perf_max_batch = (const int*)(d + o_pmb); v.perf_at_tokens = (const int*)(d + o_pat);
  v.perf_acc_count = (const int*)(d + o_pac); v.perf_present = (const unsigned char*)(d + o_pp);
  v.srv_model = (const int*)(d + o_sm); v.srv_priority = (const int*)(d + o_sp);
  v.srv_min_replicas = (const int*)(d + o_smr); v.srv_max_batch = (const int*)(d + o_smb);
  v.srv_keep_acc = (const unsigned char*)(d + o_sk); v.srv_target_present = (const unsigned char*)(d + o_stp);
  v.srv_slo_ttft = (const float*)(d + o_st); v.srv_slo_itl = (const float*)(d + o_si); v.srv_slo_tps = (const float*)(d + o_sps);
  v.srv_arrival = (const float*)(d + o_sa); v.srv_in_tokens = (const int*)(d + o_sin); v.srv_out_tokens = (const int*)(d + o_sout);
  v.srv_cur_acc = (const int*)(d + o_sca); v.srv_cur_replicas = (const int*)(d + o_scr); v.srv_cur_cost = (const float*)(d + o_scc);
  ctx->A = (int)A; ctx->T = (int)T; ctx->M = (int)M; ctx->S = (int)S;
  ctx->unlimited = s->unlimited; ctx->delayed = s->delayed_best_effort; ctx->policy = s->saturation_policy;

  // candidate + solution arenas.  With a communicator the rank owns the block of servers [shard_lo, shard_hi) and the
  // arrays are padded to world equal blocks, so that the all-gather can run in place on them.
  ctx->shard_rows = ctx->world > 1 ? (int)((S + ctx->world - 1) / ctx->world) : (int)S;
  ctx->shard_lo = ctx->world > 1 ? (int)std::min(S, (size_t)ctx->rank * ctx->shard_rows) : 0;
  ctx->shard_hi = ctx->world > 1 ? (int)std::min(S, (size_t)(ctx->rank + 1) * ctx->shard_rows) : (int)S;
  const size_t S_pad = ctx->world > 1 ? (size_t)ctx->shard_rows * ctx->world : S;
  const size_t P = S_pad * A;
  {
    Layout C;
    size_t o_state = C.take(P), o_nr = C.take(P * 4), o_bs = C.take(P * 4), o_cost = C.take(P * 4), o_val = C.take(P * 4),
           o_itl = C.take(P * 4), o_ttft = C.take(P * 4), o_rho = C.take(P * 4), o_mar = C.take(P * 4), o_ns = C.take(P * 4);
    CK(ctx->cand_arena.reserve(C.off + 256));
    char* c = (char*)ctx->cand_arena.p;
    CandView& cv = ctx->cand;
    cv.state = (unsigned char*)(c + o_state); cv.num_replicas = (int*)(c + o_nr); cv.batch_size = (int*)(c + o_bs);
    cv.cost = (float*)(c + o_cost); cv.value = (float*)(c + o_val); cv.itl = (float*)(c + o_itl);
    cv.ttft = (float*)(c + o_ttft); cv.rho = (float*)(c + o_rho); cv.max_arrv_rate = (float*)(c + o_mar);
    cv.n_solves = (int*)(c + o_ns);
  }
  {
    Layout C;
    const size_t SP = S_pad;
    size_t o_state = C.take(SP), o_acc = C.take(SP * 4), o_nr = C.take(SP * 4), o_bs = C.take(SP * 4), o_cost = C.take(SP * 4),
           o_val = C.take(SP * 4), o_itl = C.take(SP * 4), o_ttft = C.take(SP * 4), o_rho = C.take(SP * 4), o_mar = C.take(SP * 4),
           o_tc = C.take(T * 8), o_tk = C.take(T * 8);
    CK(ctx->sol_arena.reserve(C.off + 256));
    CK(cudaMemsetAsync(ctx->sol_arena.p, 0, ctx->sol_arena.cap, ctx->stream));   // padding is copied out with the arena
    char* c = (char*)ctx->sol_arena.p;
    SolView& sv = ctx->sol;
    sv.state = (unsigned char*)(c + o_state); sv.acc = (int*)(c + o_acc); sv.num_replicas = (int*)(c + o_nr);
    sv.batch_size = (int*)(c + o_bs); sv.cost = (float*)(c + o_cost); sv.value = (float*)(c + o_val);
    sv.itl = (float*)(c + o_itl); sv.ttft = (float*)(c + o_ttft); sv.rho = (float*)(c + o_rho);
    sv.max_arrv_rate = (float*)(c + o_mar);
    ctx->d_type_count = (long long*)(c + o_tc); ctx->d_type_cost = (double*)(c + o_tk);
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->loaded = true; ctx->calculated = false; ctx->solved = false;
  return WVA_OK;
}

// ------------------------------------------------------------------ calculate
}  // extern "C" (templates need C++ linkage)
template <int THREADS, bool SMEM>
static cudaError_t launch_sizer(wva_ctx* ctx, int blocks, size_t smem, unsigned long long n_pairs, int nmax, float* gtab,
                                int* ovf_list) {
  const SysView sys_v = shard_sys(ctx);
  const CandView cand_v = shard_cand(ctx);
  // lane_sizer_mode 1 = flattened state machine (sizer_kernel.cuh); 2 = lock-step rounds; 3 = lock-step with two
  // chains per lane; 4 = lock-step, every pair split into a TTFT item and an ITL item (mid-size systems); 5 = split
  // items whose second chain evaluates the predicted next bisection point (wva_core.cuh spec2_*)
  cudaError_t e;
  if (ctx->lane_sizer_mode == 1) {
    auto k = sizer_kernel<THREADS, SMEM>;
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k<<<blocks, THREADS, smem, ctx->stream>>>(sys_v, cand_v, n_pairs, nmax, gtab, ctx->d_ctr, ovf_list);
  } else {
    SplitWs sw = {nullptr, nullptr, nullptr};
    const bool split = ctx->lane_sizer_mode == 4 || ctx->lane_sizer_mode == 5;
    if (split) {
      size_t need = (size_t)n_pairs * 20 + 256;
      e = ctx->split_ws.reserve(need);
      if (e != cudaSuccess) return e;
      sw.res = (float*)ctx->split_ws.p;
      sw.solves = (int*)((char*)ctx->split_ws.p + (size_t)n_pairs * 8);
      sw.cnt = (int*)((char*)ctx->split_ws.p + (size_t)n_pairs * 16);
      e = cudaMemsetAsync(sw.cnt, 0, (size_t)n_pairs * 4, ctx->stream);
      if (e != cudaSuccess) return e;
    }
    // length-sorted queue: float32 probe -> (N, expected chain length) keys -> descending radix sort of the item ids
    const unsigned* order = nullptr;
    const unsigned long long n_items = split ? 2 * n_pairs : n_pairs;
    // the sorted queue + gang refill pays between ~130 and ~1500 pairs per SM (the items then fill 1.5-15 waves and
    // longest-first ordering shortens the tail); below, every lane holds one item and the probe is pure overhead; far
    // above, the gain no longer covers the probe's variance.  With the table in global memory it is kept at any size.
    const bool by_size = n_pairs > (unsigned long long)ctx->sm_count * 130 &&
                         (n_pairs <= (unsigned long long)ctx->sm_count * 1500 || !SMEM);
    const bool do_sort = ctx->length_sort < 0 ? by_size : ctx->length_sort != 0;
    const bool do_gang = ctx->gang_refill < 0 ? by_size : ctx->gang_refill != 0;
    if (do_sort && n_items >= 64 && n_items < (1ull << 31)) {
      size_t tmp = 0;
      cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp, (unsigned*)nullptr, (unsigned*)nullptr, (unsigned*)nullptr,
                                                (unsigned*)nullptr, (int)n_items, 0, 32, ctx->stream);
      const size_t arr = ((size_t)n_items * 4 + 255) & ~(size_t)255;
      e = ctx->order_ws.reserve(4 * arr + tmp + 256);
      if (e != cudaSuccess) return e;
      unsigned* k_in = (unsigned*)ctx->order_ws.p;
      unsigned* k_out = (unsigned*)((char*)ctx->order_ws.p + arr);
      unsigned* v_in = (unsigned*)((char*)ctx->order_ws.p + 2 * arr);
      unsigned* v_out = (unsigned*)((char*)ctx->order_ws.p + 3 * arr);
      void* d_tmp = (char*)ctx->order_ws.p + 4 * arr;
      const unsigned pb = (unsigned)((n_items + 127) / 128);
      if (split) sizer_probe_kernel<true><<<pb, 128, 0, ctx->stream>>>(sys_v, n_items, nmax, k_in, v_in);
      else sizer_probe_kernel<false><<<pb, 128, 0, ctx->stream>>>(sys_v, n_items, nmax, k_in, v_in);
      e = cub::DeviceRadixSort::SortPairsDescending(d_tmp, tmp, k_in, k_out, v_in, v_out, (int)n_items, 0, 32, ctx->stream);
      if (e != cudaSuccess) return e;
      ctx->launches += 4;
      order = v_out;
    }
    auto k = (ctx->lane_sizer_mode == 5) ? sizer_lane_kernel<THREADS, SMEM, true, true>
           : split ? sizer_lane_kernel<THREADS, SMEM, false, true>
           : (ctx->lane_sizer_mode == 3) ? sizer_lane_kernel<THREADS, SMEM, true, false>
                                         : sizer_lane_kernel<THREADS, SMEM, false, false>;
    if (THREADS == 256 && !SMEM && !split && ctx->lane_sizer_mode != 3 && ctx->lane_sizer_mode != 5)
      k = sizer_lane_kernel_gtab_2blk;                 // the same body under a 128-register cap (2 blocks per SM)
    e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k<<<blocks, THREADS, smem, ctx->stream>>>(sys_v, cand_v, n_pairs, nmax, gtab, ctx->d_ctr, ovf_list, sw, order, do_gang ? 1 : 0);
  }
  ctx->launches++;
  return cudaGetLastError();
}
template <int WARPS>
static cudaError_t launch_sizer_warp(wva_ctx* ctx, int blocks, size_t smem, unsigned long long n_pairs, int nmax,
                                     int* ovf_list) {
  auto k = sizer_warp_kernel<WARPS>;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  k<<<blocks, WARPS * 32, smem, ctx->stream>>>(shard_sys(ctx), shard_cand(ctx), n_pairs, nmax, ctx->d_ctr, ovf_list);
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

int32_t wva_calculate(wva_ctx* ctx) {
  if (!ctx) return WVA_ERR_ARG;
  if (!ctx->loaded) { ctx->last_error = "wva_calculate before wva_load_system"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  const SysView sys_v = shard_sys(ctx);
  const CandView cand_v = shard_cand(ctx);
  const unsigned long long n_pairs = (unsigned long long)sys_v.n_servers * ctx->A;
  ctx->shard_status = WVA_ERR_CUDA;   // until this call returns WVA_OK (agreed on by all ranks in wva_solve)
  // scratch: counters + nmax reduction + overflow list.  The split sizer modes process a pair as TWO items and each may
  // append the pair (both chains of an alpha-dominated pair overflow at lambda_max): 2 entries per pair.
  size_t need = 256 + 256 + (size_t)n_pairs * 8 + 1024;
  CK(ctx->scratch.reserve(need));
  ctx->d_ctr = (SizerCounters*)ctx->scratch.p;
  int* d_nmax = (int*)((char*)ctx->scratch.p + 256);
  int* d_ovf = (int*)((char*)ctx->scratch.p + 512);
  CK(cudaMemsetAsync(ctx->scratch.p, 0, 512, ctx->stream));
  CK(cudaEventRecord(ctx->ev[2], ctx->stream));
  if (n_pairs > 0) {
    // 1) largest batch size any pair will use -> table geometry
    int blocks = (int)((n_pairs + 255) / 256);
    if (blocks > 4096) blocks = 4096;
    max_batch_kernel<<<blocks, 256, 0, ctx->stream>>>(sys_v, n_pairs, d_nmax);
    ctx->launches++;
    int nmax = 0;
    CK(cudaMemcpyAsync(&nmax, d_nmax, 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    if (nmax < 1) nmax = 1;
    const int NLIMIT = 1 << 16;
    if (nmax > NLIMIT) nmax = NLIMIT;  // pairs beyond it are flagged through limit_hit
    // 2) pick geometry: the head table (4 B x nmax per lane) lives in shared memory when at
    //    least 64 lanes fit on an SM; lanes per SM are maximised over CTA sizes {256,192,128,64}
    //    (1 KB per CTA is reserved by the driver).  Otherwise the table goes to global memory.
    const size_t SMEM_PER_SM = 224 * 1024;
    const size_t per_lane = (size_t)nmax * 4;
    const int sizes[4] = {256, 192, 128, 64};
    int best_threads = 0, best_per_sm = 0;
    for (int i = 0; i < 4; i++) {
      size_t cta = per_lane * sizes[i] + 1024;
      int per_sm = (int)(SMEM_PER_SM / cta);
      if (per_sm * sizes[i] > 1024) per_sm = 1024 / sizes[i];
      if (per_sm * sizes[i] > best_threads * best_per_sm) { best_threads = sizes[i]; best_per_sm = per_sm; }
    }
    // small problems are latency bound: spread the pairs over every SM with as few lanes per SM
    // as needed instead of filling the first SMs (lanes pull one pair each from the queue)
    // mid-size systems (measured: up to ~200 pairs per SM) still leave lanes idle: split every pair into a
    // TTFT item and an ITL item, which halves the chain of dependent solves per work item
    // crossovers (natural queue order): split items up to ~180 pairs per SM, split items with a speculative second
    // chain (mode 5) up to ~380, whole pairs (mode 2, the searches share evaluations) beyond
    if (!ctx->force_lane_sizer)
      ctx->lane_sizer_mode = (n_pairs <= (unsigned long long)ctx->sm_count * 180) ? 4
                           : (n_pairs <= (unsigned long long)ctx->sm_count * 380) ? 5 : 2;
    // large systems: the pool sizer (sizer_pool_kernel.cuh) regroups the pending solves of 1024 pairs per SM by
    // length every time a warp goes back for work (88-92 % live lane-steps instead of 49-62 %); it overtakes the lane
    // sizer from ~640 pairs per SM
    const bool pool_auto = !ctx->force_lane_sizer && n_pairs > (unsigned long long)ctx->sm_count * 640 && nmax <= 4096;
    if (pool_auto || (ctx->force_lane_sizer && ctx->lane_sizer_mode == 6)) {
      const int P = POOL_PMAX;
      const int row_stride = (nmax + 31) & ~31;
      const size_t pool_bytes = (size_t)ctx->sm_count * P * sizeof(PoolEntry);
      const size_t rows_bytes = (size_t)ctx->sm_count * P * (size_t)row_stride * 4;
      CK(ctx->pool_ws.reserve(pool_bytes + rows_bytes + 512));
      PoolEntry* pool = (PoolEntry*)ctx->pool_ws.p;
      float* rows = (float*)((char*)ctx->pool_ws.p + ((pool_bytes + 255) & ~(size_t)255));
      CK(cudaFuncSetAttribute(sizer_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PoolSmem)));
      sizer_pool_kernel<<<ctx->sm_count, POOL_THREADS, sizeof(PoolSmem), ctx->stream>>>(sys_v, cand_v, n_pairs, nmax, P, pool, rows,
                                                                                        row_stride, ctx->d_ctr, d_ovf);
      ctx->launches++;
      cudaError_t pe = cudaGetLastError();
      if (pe != cudaSuccess) { ctx->last_error = std::string("pool sizer launch: ") + cudaGetErrorString(pe); return WVA_ERR_CUDA; }
      ctx->timing.sizer_kernel = 4;
      goto sizer_done;
    }
    const unsigned long long n_items = (ctx->lane_sizer_mode >= 4) ? 2 * n_pairs : n_pairs;
    const unsigned long long lanes_needed = (n_items + ctx->sm_count - 1) / ctx->sm_count;
    if (best_per_sm >= 1 && lanes_needed <= 256 && lanes_needed < (unsigned long long)best_threads * best_per_sm) {
      int t = 64;
      while ((unsigned long long)t < lanes_needed) t += 64;
      if (per_lane * t + 1024 <= SMEM_PER_SM) { best_threads = t; best_per_sm = 1; }
    }
    cudaError_t e;
    // Small / medium systems are bound by the critical path of their slowest pair: use the
    // warp-per-pair sizer (speculative bisection, sizer_warp_kernel.cuh) while the system is small
    // (measured crossover against the lock-step lane sizer: ~32 pairs per SM) and its per-warp
    // tables (20 B x nmax) fit in shared memory.
    const size_t warp_tab = (size_t)nmax * 20;
    if (n_pairs <= (unsigned long long)ctx->sm_count * 32 && warp_tab * 4 + 1024 <= SMEM_PER_SM && !ctx->force_lane_sizer) {
      if (warp_tab * 8 <= 48 * 1024) {
        int per_sm = (int)(SMEM_PER_SM / (warp_tab * 8 + 1024)); if (per_sm > 6) per_sm = 6; if (per_sm < 1) per_sm = 1;
        e = launch_sizer_warp<8>(ctx, ctx->sm_count * per_sm, warp_tab * 8, n_pairs, nmax, d_ovf);
        ctx->timing.sizer_kernel = 1;
      } else {
        int per_sm = (int)(SMEM_PER_SM / (warp_tab * 4 + 1024)); if (per_sm > 8) per_sm = 8; if (per_sm < 1) per_sm = 1;
        e = launch_sizer_warp<4>(ctx, ctx->sm_count * per_sm, warp_tab * 4, n_pairs, nmax, d_ovf);
        ctx->timing.sizer_kernel = 1;
      }
    } else
    // Head table placement: N = 256 leaves 192 lanes per SM in shared memory (1.5 warps per scheduler), slower than the
    // table in global memory / L2 with two 256-thread blocks per SM under a 128-register cap; at N = 128 (384 lanes in
    // shared memory) and N = 64 shared memory wins.
    if (best_per_sm >= 1 && ctx->table_mode != 2 && (ctx->table_mode == 1 || best_threads * best_per_sm > 256 || n_pairs <= (unsigned long long)ctx->sm_count * 512)) {
      int blocks = ctx->sm_count * best_per_sm;
      size_t smem = per_lane * best_threads;
      ctx->timing.sizer_kernel = 2;
      switch (best_threads) {
        case 256: e = launch_sizer<256, true>(ctx, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
        case 192: e = launch_sizer<192, true>(ctx, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
        case 128: e = launch_sizer<128, true>(ctx, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
        default: e = launch_sizer<64, true>(ctx, blocks, smem, n_pairs, nmax, nullptr, d_ovf); break;
      }
    } else {
      int blk = ctx->sm_count * 2;
      ctx->timing.sizer_kernel = 3;
      CK(ctx->gtab.reserve((size_t)blk * 256 * per_lane));
      e = launch_sizer<256, false>(ctx, blk, 0, n_pairs, nmax, (float*)ctx->gtab.p, d_ovf);
    }
    if (e != cudaSuccess) { ctx->last_error = std::string("sizer launch: ") + cudaGetErrorString(e); return WVA_ERR_CUDA; }
  }
sizer_done:
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
  ctx->calculated = true; ctx->solved = false;
  ctx->shard_status = WVA_OK;
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
  size_t need = (size_t)nparts * (T > 0 ? T : 1) * 16 + 512;
  // reuse scratch beyond its first 1024 bytes (counters)
  CK(ctx->scratch.reserve(1024 + need));
  long long* pc = (long long*)((char*)ctx->scratch.p + 1024);
  double* pd = (double*)((char*)ctx->scratch.p + 1024 + (size_t)nparts * (T > 0 ? T : 1) * 8);
  if (T > 0) {
    if (S > 0) {
      by_type_partial_kernel<<<nparts, 256, 0, ctx->stream>>>(sv, ov, pc, pd);
      ctx->launches++;
    } else {
      CK(cudaMemsetAsync(pc, 0, need - 512, ctx->stream));
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
  const size_t P = (size_t)ctx->S * ctx->A;
  if (P > 0 && (!in->state || !in->num_replicas || !in->batch_size || !in->cost || !in->value || !in->itl || !in->ttft ||
                !in->rho || !in->max_arrv_rate)) {
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
  const CandView& c = ctx->cand;
  struct { void* dst; const void* src; size_t b; } cp[] = {
      {c.state, in->state, P}, {c.num_replicas, in->num_replicas, P * 4}, {c.batch_size, in->batch_size, P * 4},
      {c.cost, in->cost, P * 4}, {c.value, in->value, P * 4}, {c.itl, in->itl, P * 4}, {c.ttft, in->ttft, P * 4},
      {c.rho, in->rho, P * 4}, {c.max_arrv_rate, in->max_arrv_rate, P * 4}};
  if (P > 0) {
    for (auto& x : cp) CK(cudaMemcpyAsync(x.dst, x.src, x.b, cudaMemcpyHostToDevice, ctx->stream));
    if (in->n_solves) CK(cudaMemcpyAsync(c.n_solves, in->n_solves, P * 4, cudaMemcpyHostToDevice, ctx->stream));
    else CK(cudaMemsetAsync(c.n_solves, 0, P * 4, ctx->stream));
  }
  CK(cudaEventRecord(ctx->ev[1], ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));               // the caller's buffers are free again on return (cgo pointer rule)
  ctx->timing.h2d_ms = elapsed(ctx, 0, 1);
  ctx->calculated = true; ctx->solved = false;
  return WVA_OK;
}

// ------------------------------------------------------------------ readback
int32_t wva_get_candidates(wva_ctx* ctx, wva_candidates* out) {
  if (!ctx || !out) return WVA_ERR_ARG;
  if (!ctx->calculated) { ctx->last_error = "wva_get_candidates before wva_calculate"; return WVA_ERR_STATE; }
  CK(cudaSetDevice(ctx->device));
  const size_t P = (size_t)ctx->S * ctx->A;
  if (P == 0) return WVA_OK;
  CK(cudaEventRecord(ctx->ev[6], ctx->stream));
  const CandView& c = ctx->cand;
  struct { void* dst; const void* src; size_t b; } cp[] = {
      {out->state, c.state, P}, {out->num_replicas, c.num_replicas, P * 4}, {out->batch_size, c.batch_size, P * 4},
      {out->cost, c.cost, P * 4}, {out->value, c.value, P * 4}, {out->itl, c.itl, P * 4}, {out->ttft, c.ttft, P * 4},
      {out->rho, c.rho, P * 4}, {out->max_arrv_rate, c.max_arrv_rate, P * 4}, {out->n_solves, c.n_solves, P * 4}};
  for (auto& x : cp)
    if (x.dst) CK(cudaMemcpyAsync(x.dst, x.src, x.b, cudaMemcpyDeviceToHost, ctx->stream));
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
  const SolView& v = ctx->sol;
  if (out->state) memcpy(out->state, H(v.state), S);
  if (out->acc) memcpy(out->acc, H(v.acc), S * 4);
  if (out->num_replicas) memcpy(out->num_replicas, H(v.num_replicas), S * 4);
  if (out->batch_size) memcpy(out->batch_size, H(v.batch_size), S * 4);
  if (out->cost) memcpy(out->cost, H(v.cost), S * 4);
  if (out->value) memcpy(out->value, H(v.value), S * 4);
  if (out->itl) memcpy(out->itl, H(v.itl), S * 4);
  if (out->ttft) memcpy(out->ttft, H(v.ttft), S * 4);
  if (out->rho) memcpy(out->rho, H(v.rho), S * 4);
  if (out->max_arrv_rate) memcpy(out->max_arrv_rate, H(v.max_arrv_rate), S * 4);
  if (out->type_count) memcpy(out->type_count, H(ctx->d_type_count), T * 8);
  if (out->type_cost) memcpy(out->type_cost, H(ctx->d_type_cost), T * 8);
  return WVA_OK;
}

}  // extern "C"

#include "capi_aux.inl"
#include "comm.inl"
#include "ingest.inl"
