// grid_kernel.cuh — replica-grid evaluator: for every (server, accelerator, r) one
// QueueAnalyzer.Analyze(totalRate / r) (pkg/analyzer/queueanalyzer.go:127-167), the
// call CreateAllocation makes at pkg/core/allocation.go:140-148 with numReplicas = r.
//
// Mapping: one warp per (server, accelerator) pair ("one block per model sweeps its
// variant x replica grid" at warp granularity).  The pair's head table (mu_n, 1/mu_n)
// is built once by the warp into shared memory; the 32 lanes then take 32 consecutive
// replica levels per round and solve their chains in lock step (lockstep_solve.cuh):
// broadcast table reads, no per-state control flow, a lane whose terms became no-ops
// idles until the round's longest chain ends.  The per-pair frontier (smallest r meeting
// every SLO) is a warp-shuffle min.
#pragma once
#include "wva_core.cuh"
#include "lockstep_solve.cuh"

namespace wva {

struct GridOut {
  unsigned char* ok;
  float *ttft, *itl, *rho, *tput;
  int* frontier;
};

struct GridCounters {
  unsigned long long next_pair, solves, states, overflow;
  int limit_hit, pad_;
  unsigned long long slots0, slots_rest, rounds;   // 32 x longest chain of the round: first round of a pair / later rounds
  unsigned long long slots_def;                   // the same for the deferred pass
  unsigned long long certify_fallbacks;           // deferred pass: fast solves (E12) redone by the exact solver
  unsigned long long pathological;                // overflow pass: literal solves whose rescale loop the reference never leaves
};

// Levels whose chain overflows float64 (CH_OVERFLOW).  The reference's Analyze still returns metrics for them
// (computeProbabilities rescales, mm1modelstatedependent.go:84-89,96-104), which needs every earlier p[i]: both passes
// append the level's output index pair * R + r - 1 here, and grid_overflow_kernel solves them with literal_solve.
// ctr->overflow counts every level; only the first `cap` are stored, and the host fails the run if any is missing.
struct GridOverflowList {
  unsigned long long* items;
  unsigned long long cap;
};
__device__ __forceinline__ void grid_overflow_push(const GridOverflowList& ol, GridCounters* ctr, unsigned long long o) {
  const unsigned long long k = atomicAdd(&ctr->overflow, 1ull);
  if (k < ol.cap) ol.items[k] = o;
}

// Analyze's outputs for one admitted level (queueanalyzer.go:143-166; ttft as allocation.go:148); true if the level meets
// every SLO of its server
__device__ __forceinline__ bool grid_store(const GridOut& out, size_t o, const PairModel& m, const SolveStats& st, float lambda,
                                           float slo_ttft, float slo_itl, float slo_tps, float lambda_tps) {
  float pf, dec, avg_ttft;
  eval_values(m, st, &avg_ttft, &dec, &pf);
  float rho = f_div(st.avgNumInServers, (float)m.N);
  rho = fminf(fmaxf(rho, 0.0f), 1.0f);
  if (out.ok) out.ok[o] = 1;
  if (out.ttft) out.ttft[o] = f_add(st.avgWaitTime, pf);
  if (out.itl) out.itl[o] = dec;
  if (out.rho) out.rho[o] = rho;
  if (out.tput) out.tput[o] = f_mul(st.throughput, 1000.0f);
  return (slo_ttft <= 0.0f || avg_ttft <= slo_ttft) && (slo_itl <= 0.0f || dec <= slo_itl) &&
         (slo_tps <= 0.0f || lambda <= lambda_tps);
}

// Deferral of the near-saturation levels (large systems).  A pair's chain length is a steep function of lambda / mu_N
// (early exit E4): the one or two lowest admitted levels of a pair run thousands of states next to ~50 for the rest, so a
// warp that takes 32 consecutive levels spends its first round waiting for one lane.  With deferral the pair's warp skips
// the levels whose ratio exceeds `thr`, saves the pair's model (without its head table: m.tab == nullptr), and appends
// (pair, r, class) to a global list; the list is radix-sorted by length class and grid_deferred_kernel solves it 32
// items — of 32 different pairs, similar lengths — at a time, each lane computing its own pair's rates (RateTable).
// Same per-level arithmetic, same outputs.
struct GridSide {            // what an evaluation needs of its pair
  PairModel m;
  float total_rate, slo_ttft, slo_itl, slo_tps, lambda_tps;
  int pad_[3];
};
struct GridDefer {
  GridSide* side;            // [n_pairs], nullptr = no deferral
  unsigned long long* items; // (pair << 16) | r
  unsigned char* cls;        // length class of the item (sort key)
  unsigned long long* n_items;
  unsigned long long cap;
  float thr;
};
__device__ __forceinline__ int grid_class(const PairModel& m, float ratio) {
  if (!(ratio > 1e-6f)) ratio = 1e-6f;
  if (ratio > 0.999999f) ratio = 0.999999f;
  float est = (float)m.N + 37.4f / -__logf(ratio);
  if (est > (float)m.K) est = (float)m.K;
  const int c = (int)(__log2f(fmaxf(est, 32.0f) * (1.0f / 32.0f)) * 8.0f);
  return c < 0 ? 0 : (c > 255 ? 255 : c);
}

// per-pair preparation shared by all lanes of the warp; false -> every level is "not ok"
__device__ __forceinline__ bool grid_setup(PairModel& m, const SysView& s, int srv, int acc, int n_limit,
                                           float* total_rate, float* slo_ttft, float* slo_itl, float* slo_tps,
                                           int* limit_hit) {
  float arrival = s.srv_arrival[srv];
  int in_tok = s.srv_in_tokens[srv], out_tok = s.srv_out_tokens[srv];
  int model = s.srv_model[srv];
  if (arrival < 0.0f || in_tok < 0 || out_tok < 0 || model < 0 || model >= s.n_models) return false;
  size_t pi = (size_t)model * s.n_acc + acc;
  if (!s.perf_present[pi] || !s.srv_target_present[srv] || arrival == 0.0f || out_tok == 0) return false;
  long long N;
  if (s.srv_max_batch[srv] > 0) N = s.srv_max_batch[srv];
  else { N = (long long)s.perf_max_batch[pi] * s.perf_at_tokens[pi] / out_tok; if (N < 1) N = 1; }
  if (N > n_limit) { *limit_hit = 1; return false; }
  model_init(m, s.perf_alpha[pi], s.perf_beta[pi], s.perf_gamma[pi], in_tok, out_tok, (int)N);
  *slo_ttft = s.srv_slo_ttft[srv]; *slo_itl = s.srv_slo_itl[srv]; *slo_tps = s.srv_slo_tps[srv];
  *total_rate = (*slo_tps == 0.0f) ? f_div(arrival, 60.0f) : f_div(*slo_tps, (float)out_tok);
  return true;
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, WARPS == 8 ? 2 : 1)
grid_kernel(SysView s, int R, GridOut out, unsigned long long n_pairs, int nmax, GridCounters* ctr, GridDefer df,
            GridOverflowList ol) {
  extern __shared__ double2 smem_grid[];
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double2* tab = smem_grid + (size_t)warp * nmax;
  float* tabf = (float*)(smem_grid + (size_t)WARPS * nmax) + (size_t)warp * nmax;
  unsigned long long my_solves = 0, my_states = 0, my_s0 = 0, my_sr = 0, my_rounds = 0;

  while (true) {
    unsigned long long pair = 0;
    if (lane == 0) pair = atomicAdd(&ctr->next_pair, 1ull);
    pair = __shfl_sync(full, pair, 0);
    if (pair >= n_pairs) break;
    const int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
    const size_t obase = (size_t)pair * (size_t)R;
    PairModel m;
    float total_rate = 0, slo_ttft = 0, slo_itl = 0, slo_tps = 0;
    int lim = 0;
    bool valid = grid_setup(m, s, srv, acc, nmax, &total_rate, &slo_ttft, &slo_itl, &slo_tps, &lim);
    if (lim && lane == 0) ctr->limit_hit = 1;
    if (!valid) {
      for (int r = lane; r < R; r += 32) {
        if (out.ok) out.ok[obase + r] = 0;
        if (out.ttft) out.ttft[obase + r] = 0.0f;
        if (out.itl) out.itl[obase + r] = 0.0f;
        if (out.rho) out.rho[obase + r] = 0.0f;
        if (out.tput) out.tput[obase + r] = 0.0f;
      }
      if (out.frontier && lane == 0) out.frontier[pair] = 0;
      continue;
    }
    __syncwarp();
    for (int n = lane; n < m.N; n += 32) {
      float mu32 = serv_rate(m, n + 1);
      double mu = (double)mu32;
      tabf[n] = mu32;
      tab[n] = make_double2(mu, rcp_f32den(mu32, mu));
    }
    __syncwarp();
    model_finish(m, tabf, 1);
    const float lambda_tps = f_mul(m.lambda_max, f_sub(1.0f, WVA_STABILITY_SAFETY));
    int front = 0x7fffffff;
    const bool deferring = df.side != nullptr && pair < 0xffffffffull;
    bool saved = false;                                   // the pair's model is written when its first level is deferred
    const float mu_last_f = (float)m.mu_last;
    bool first_round = true;

    // Two levels per lane and round (r0 + lane + 1 and r0 + 32 + lane + 1): the two chains of a lane share every table
    // load and give the FP64 pipe two independent dependency chains; half as many rounds (the chains of a round are ~20
    // states long on average, so the per-round work is a large part of the cost).
    for (int r0 = 0; r0 < R; r0 += 64) {
      int r[2]; bool in_range[2], admitted[2], defer[2], here[2], ovf[2];
      float rate[2], lambda[2];
#pragma unroll
      for (int c = 0; c < 2; c++) {
        r[c] = r0 + 32 * c + lane + 1;
        in_range[c] = r[c] <= R;
        rate[c] = f_div(total_rate, (float)r[c]);
        admitted[c] = in_range[c] && analyze_admits(m, rate[c]);      // queueanalyzer.go:128-136
        lambda[c] = f_div(rate[c], 1000.0f);
        defer[c] = false; ovf[c] = false;
      }
      if (!__any_sync(full, admitted[0] || admitted[1])) {
#pragma unroll
        for (int c = 0; c < 2; c++)
          if (in_range[c]) {
            const size_t o = obase + (size_t)(r[c] - 1);
            if (out.ok) out.ok[o] = 0;
            if (out.ttft) out.ttft[o] = 0.0f;
            if (out.itl) out.itl[o] = 0.0f;
            if (out.rho) out.rho[o] = 0.0f;
            if (out.tput) out.tput[o] = 0.0f;
          }
        continue;
      }
      if (deferring) {
#pragma unroll
        for (int c = 0; c < 2; c++) {
          const float ratio = lambda[c] / mu_last_f;
          const bool want = admitted[c] && ratio > df.thr;
          const unsigned wm = __ballot_sync(full, want);
          if (wm) {
            unsigned long long base = 0;
            if (lane == 0) base = atomicAdd(df.n_items, (unsigned long long)__popc(wm));
            base = __shfl_sync(full, base, 0);
            // the first `room` wanting lanes (by ballot rank) take the slots left in the list and leave the warp; the rest
            // are solved here.  So every slot below min(n_items, cap) is written exactly once.
            const unsigned long long room = base < df.cap ? df.cap - base : 0ull;
            const unsigned rank = __popc(wm & ((1u << lane) - 1u));
            defer[c] = want && rank < room;
            if (defer[c]) {
              const unsigned long long k = base + rank;
              df.items[k] = (pair << 16) | (unsigned long long)r[c];
              df.cls[k] = (unsigned char)grid_class(m, ratio);
            }
            if (room > 0 && !saved) {                       // warp-uniform: the first level of the pair that leaves
              saved = true;
              if (lane == 0) {
                GridSide sd;
                sd.m = m; sd.m.tab = nullptr; sd.m.stride = 0;
                sd.total_rate = total_rate; sd.slo_ttft = slo_ttft; sd.slo_itl = slo_itl; sd.slo_tps = slo_tps; sd.lambda_tps = lambda_tps;
                df.side[pair] = sd;
              }
            }
          }
        }
      }
      here[0] = admitted[0] && !defer[0]; here[1] = admitted[1] && !defer[1];
      SolveStats st[2];
      int sv = 0;
      bool bad = false;
      // a pair with a service rate outside the (E1) divisor range takes the per-lane chain below for every level
      if (!m.e1_ok) bad = here[0] || here[1];
      else if (__any_sync(full, here[0] || here[1])) lockstep_solve_inl<2, WarpTable>(m, WarpTable{tab}, lambda, here, st, sv, bad);
      if (here[0] || here[1]) { my_solves += (here[0] ? 1 : 0) + (here[1] ? 1 : 0); my_states += (unsigned long long)sv; }
      {
        int mxs = (here[0] || here[1]) ? sv : 0;
        for (int o = 16; o; o >>= 1) mxs = max(mxs, __shfl_xor_sync(full, mxs, o));
        if (lane == 0) { if (first_round) my_s0 += 32ull * mxs; else my_sr += 32ull * mxs; my_rounds++; }
        first_round = false;
      }
      if (bad) {
        // a chain of this lane left the exponent window (or the pair needs IEEE divisions): redo its levels one by one
        // through the per-lane state machine; a true float64 overflow goes to the overflow list
#pragma unroll
        for (int c = 0; c < 2; c++)
          if (here[c]) {
            Chain ch;
            chain_start(ch, lambda[c]);
            ch.tail_ok = d_bits(ch.lamg) <= d_bits(m.mu_last);
            while (!chain_step(ch, m, st[c])) {}
            ovf[c] = ch.phase == CH_OVERFLOW;
            if (ovf[c]) grid_overflow_push(ol, ctr, obase + (size_t)(r[c] - 1));
          }
      }
#pragma unroll
      for (int c = 0; c < 2; c++) {
        if (in_range[c] && !defer[c] && !ovf[c]) {
          const size_t o = obase + (size_t)(r[c] - 1);
          if (!admitted[c]) {
            if (out.ok) out.ok[o] = 0;
            if (out.ttft) out.ttft[o] = 0.0f;
            if (out.itl) out.itl[o] = 0.0f;
            if (out.rho) out.rho[o] = 0.0f;
            if (out.tput) out.tput[o] = 0.0f;
          } else if (grid_store(out, o, m, st[c], lambda[c], slo_ttft, slo_itl, slo_tps, lambda_tps) && r[c] < front) {
            front = r[c];
          }
        }
      }
    }
    for (int o = 16; o; o >>= 1) front = min(front, __shfl_down_sync(full, front, o));
    // the deferred and overflow passes may still lower the frontier (atomicMin); grid_frontier_fix maps "none" to 0
    if (out.frontier && lane == 0) out.frontier[pair] = front;
    __syncwarp();
  }
  for (int o = 16; o; o >>= 1) {
    my_solves += __shfl_down_sync(full, my_solves, o);
    my_states += __shfl_down_sync(full, my_states, o);
  }
  if (lane == 0) {
    atomicAdd(&ctr->solves, my_solves); atomicAdd(&ctr->states, my_states);
    atomicAdd(&ctr->slots0, my_s0); atomicAdd(&ctr->slots_rest, my_sr); atomicAdd(&ctr->rounds, my_rounds);
  }
}

// The deferred levels, sorted by length class: lane per (pair, level), 32 different pairs per warp.
__global__ void __launch_bounds__(256, 2)
grid_deferred_kernel(int R, GridOut out, GridDefer df, const unsigned long long* __restrict__ items, unsigned long long n_items,
                     GridCounters* ctr, unsigned long long* next_item, GridOverflowList ol) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  unsigned long long my_solves = 0, my_states = 0, my_slots = 0, my_rounds = 0;
  while (true) {
    unsigned long long i0 = 0;
    if (lane == 0) i0 = atomicAdd(next_item, 32ull);
    i0 = __shfl_sync(full, i0, 0);
    if (i0 >= n_items) break;
    const bool live = i0 + lane < n_items;
    unsigned long long it = live ? items[i0 + lane] : items[i0];
    const unsigned long long pair = it >> 16;
    const int r = (int)(it & 0xffffu);
    const GridSide* sp = df.side + pair;
    PairModel m = sp->m;
    const float total_rate = sp->total_rate, slo_ttft = sp->slo_ttft, slo_itl = sp->slo_itl, slo_tps = sp->slo_tps,
                lambda_tps = sp->lambda_tps;
    const float rate = f_div(total_rate, (float)r);
    const float lambda = f_div(rate, 1000.0f);
    const int nref = __shfl_sync(full, m.N, 0);
    const bool uniform = __all_sync(full, m.N == nref && m.e1_ok);   // else the per-lane chain (IEEE divisions)
    SolveStats st;
    int sv = 0;
    bool bad = false, ovf = false;
    if (uniform) {
      sv = lockstep_solve_fast(m, RateTable{rate_coef(m)}, lambda, live, st, &ctr->certify_fallbacks);
      bad = sv < 0;
      if (bad) sv = -1 - sv;
    } else if (live) {
      Chain c;
      chain_start(c, lambda);
      c.tail_ok = d_bits(c.lamg) <= d_bits(m.mu_last);
      while (!chain_step(c, m, st)) {}
      bad = false; ovf = c.phase == CH_OVERFLOW; sv = c.states;
    }
    if (live && bad) {
      Chain c;
      chain_start(c, lambda);
      c.tail_ok = d_bits(c.lamg) <= d_bits(m.mu_last);
      while (!chain_step(c, m, st)) {}
      ovf = c.phase == CH_OVERFLOW;
    }
    if (live) {
      my_solves++; my_states += (unsigned long long)sv;
      const size_t o = (size_t)pair * (size_t)R + (size_t)(r - 1);
      if (ovf) grid_overflow_push(ol, ctr, o);
      else if (grid_store(out, o, m, st, lambda, slo_ttft, slo_itl, slo_tps, lambda_tps) && out.frontier)
        atomicMin(&out.frontier[pair], r);
    }
    {
      int mxs = live ? sv : 0;
      for (int o = 16; o; o >>= 1) mxs = max(mxs, __shfl_xor_sync(full, mxs, o));
      if (lane == 0) { my_slots += 32ull * mxs; my_rounds++; }
    }
  }
  for (int o = 16; o; o >>= 1) {
    my_solves += __shfl_down_sync(full, my_solves, o);
    my_states += __shfl_down_sync(full, my_states, o);
  }
  if (lane == 0) {
    atomicAdd(&ctr->solves, my_solves); atomicAdd(&ctr->states, my_states);
    atomicAdd(&ctr->slots_def, my_slots); atomicAdd(&ctr->rounds, my_rounds);
  }
}

// The overflow list, one thread per level: the pair's model is rebuilt from the system into a per-thread table, the
// level is solved by the literal stored-p[] algorithm with the reference's rescale branches (p holds K + 1 doubles),
// and its outputs are written as above.
__global__ void __launch_bounds__(64) grid_overflow_kernel(SysView s, int R, GridOut out, const unsigned long long* items,
                                                           int n, int nmax, double* pbuf, float* tabbuf, GridCounters* ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long o = items[i];
  const unsigned long long pair = o / (unsigned)R;
  const int r = (int)(o % (unsigned)R) + 1;
  const int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
  PairModel m;
  float total_rate = 0, slo_ttft = 0, slo_itl = 0, slo_tps = 0;
  int lim = 0;
  if (!grid_setup(m, s, srv, acc, nmax, &total_rate, &slo_ttft, &slo_itl, &slo_tps, &lim)) return;   // listed levels pass it
  float* tab = tabbuf + (size_t)i * nmax;
  double* p = pbuf + (size_t)i * ((size_t)nmax * (WVA_QUEUE_TO_BATCH + 1) + 1);
  model_fill_table(m, tab, 1, 0, 1);
  model_finish(m, tab, 1);
  const float lambda_tps = f_mul(m.lambda_max, f_sub(1.0f, WVA_STABILITY_SAFETY));
  const float lambda = f_div(f_div(total_rate, (float)r), 1000.0f);
  SolveStats st;
  bool patho = false;
  literal_solve(m, lambda, p, st, &patho);
  if (patho) atomicAdd(&ctr->pathological, 1ull);
  if (grid_store(out, o, m, st, lambda, slo_ttft, slo_itl, slo_tps, lambda_tps) && out.frontier) atomicMin(&out.frontier[pair], r);
}

__global__ void __launch_bounds__(256) grid_frontier_fix_kernel(int* frontier, unsigned long long n) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && frontier[i] == 0x7fffffff) frontier[i] = 0;
}

}  // namespace wva
