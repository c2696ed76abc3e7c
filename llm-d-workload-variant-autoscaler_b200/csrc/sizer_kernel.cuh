// sizer_kernel.cuh — System.Calculate on the device: one lane per (server,
// accelerator) candidate, persistent CTAs pulling pairs from a global counter.
//
// SIMT shape: the inner loop body is ONE birth-death state of whatever solve the
// lane is in (pass 1 or pass 2 of any bisection step of any pair), so lanes of a
// warp never wait for each other's solve lengths; only the rare transitions
// (solve finished -> bisection bookkeeping, pair finished -> fetch + BuildModel)
// diverge.  The head table mu_n (float32) of each lane lives in shared memory,
// column-interleaved ([n][thread]) so a lane always hits bank (tid % 32).
#pragma once
#include "wva_core.cuh"

namespace wva {

struct SizerCounters {
  unsigned long long next_pair;      // work queue head
  unsigned long long solves;         // chain solves executed
  unsigned long long states;         // birth-death states visited
  unsigned long long overflow_pairs; // pairs that hit the float64 overflow-rescale branch
  int limit_hit;                     // some pair needs N beyond the build limit
  int pad_;
  unsigned long long lockstep_slots; // lock-step lane sizer: 32 x (longest chain of the warp), summed over rounds
                                     // (states / lockstep_slots = share of the lane-steps that did live work)
  unsigned long long certify_fallbacks; // pool sizer: fast solves (E12) not certified, redone by the exact solver
};

// Largest max-batch-size N any pair that needs sizing will use (allocation.go:79-88):
// decides the table geometry of the sizer launch.
__global__ void __launch_bounds__(256) max_batch_kernel(SysView s, unsigned long long n_pairs, int* out) {
  int best = 0;
  for (unsigned long long pair = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; pair < n_pairs;
       pair += (unsigned long long)gridDim.x * blockDim.x) {
    int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
    int model = s.srv_model[srv];
    if (model < 0) continue;
    size_t pi = (size_t)model * s.n_acc + acc;
    int out_tok = s.srv_out_tokens[srv];
    if (!s.perf_present[pi] || out_tok <= 0 || s.srv_arrival[srv] <= 0.0f) continue;
    long long N;
    if (s.srv_max_batch[srv] > 0) N = s.srv_max_batch[srv];
    else { N = (long long)s.perf_max_batch[pi] * s.perf_at_tokens[pi] / out_tok; if (N < 1) N = 1; }
    if (N > 0x7fffffff) N = 0x7fffffff;
    best = max(best, (int)N);
  }
  for (int o = 16; o; o >>= 1) best = max(best, __shfl_down_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best > 0) atomicMax(out, best);
}

template <int THREADS, bool SMEM_TABLE>
__global__ void __launch_bounds__(THREADS)
sizer_kernel(SysView s, CandView out, unsigned long long n_pairs, int nmax, float* gtab,
             SizerCounters* ctr, int* overflow_list) {
  extern __shared__ float smem_tab[];
  const int lane = threadIdx.x & 31;
  const unsigned full = 0xffffffffu;
  float* tab;
  int stride;
  if (SMEM_TABLE) { tab = smem_tab + threadIdx.x; stride = THREADS; }
  else { tab = gtab + ((size_t)blockIdx.x * THREADS + threadIdx.x); stride = gridDim.x * THREADS; }

  SizerLane z;
  SolveStats st;
  bool live = false, exhausted = false;
  unsigned long long my_solves = 0, my_states = 0;

  while (true) {
    // ---- refill: lanes without work fetch pairs until one needs sizing -----------------
    bool need_table = false;
    if (!live && !exhausted) {
      while (true) {
        unsigned long long pair = atomicAdd(&ctr->next_pair, 1ull);
        if (pair >= n_pairs) { exhausted = true; break; }
        int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
        int lim = 0;
        int rc = sizer_setup(z, s, out, srv, acc, nmax, &lim);
        if (lim) ctr->limit_hit = 1;
        if (rc == SETUP_NEEDS_TABLE) { need_table = true; break; }
      }
    }
    // ---- BuildModel, cooperatively: the warp fills each requesting lane's column --------
    unsigned need = __ballot_sync(full, need_table);
    while (need) {
      int src = __ffs(need) - 1;
      need &= need - 1;
      PairModel b;
      b.alpha = __shfl_sync(full, z.m.alpha, src);
      b.beta = __shfl_sync(full, z.m.beta, src);
      b.in_tok = __shfl_sync(full, z.m.in_tok, src);
      b.out_tok = __shfl_sync(full, z.m.out_tok, src);
      b.slope = __shfl_sync(full, z.m.slope, src);
      b.pre_c = __shfl_sync(full, z.m.pre_c, src);
      b.dec_c = __shfl_sync(full, z.m.dec_c, src);
      b.N = __shfl_sync(full, z.m.N, src);
      // column of lane `src` is this lane's column shifted by (src - lane)
      model_fill_table(b, tab + (src - lane), stride, lane, 32);
    }
    __syncwarp();
    if (need_table) {
      model_finish(z.m, tab, stride);
      live = sizer_begin(z, s, out);
      if (!live) { my_solves += z.solves; }
    }
    if (!__any_sync(full, live || !exhausted)) break;

    // ---- steady state: advance every live lane by a burst of states ----------------------
    // (a burst bounds how often the warp re-converges for refills)
    for (int it = 0; it < 64; it++) {
      if (live) {
        if (chain_step(z.c, z.m, st)) {
          if (z.c.phase == CH_OVERFLOW) {
            unsigned long long k = atomicAdd(&ctr->overflow_pairs, 1ull);
            if (overflow_list) overflow_list[k] = z.srv * s.n_acc + z.acc;
            z.states += z.c.states;
            lane_fail(z, s, out);
            live = false;
          } else {
            live = sizer_on_solve(z, s, out, st);
          }
          if (!live) { my_solves += z.solves; my_states += z.states; }
        }
      }
      // every 8 states: stop when the warp is idle or some lane can refill (warp-uniform)
      if ((it & 7) == 7 && (!__any_sync(full, live) || __any_sync(full, !live && !exhausted))) break;
    }
  }
  // ---- counters -----------------------------------------------------------------------------
  for (int o = 16; o; o >>= 1) {
    my_solves += __shfl_down_sync(full, my_solves, o);
    my_states += __shfl_down_sync(full, my_states, o);
  }
  if (lane == 0) { atomicAdd(&ctr->solves, my_solves); atomicAdd(&ctr->states, my_states); }
}

}  // namespace wva
