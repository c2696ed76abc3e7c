// sizer_kernel.cuh — what the sizer kernels (lane, warp, pool and the overflow slow path) share: the
// counters, the retirement of a float64-overflowing pair, the max-batch reduction that decides the
// head-table geometry, and the warp broadcast of one lane's pair model for cooperative BuildModel.
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

// A pair whose chain overflowed float64 (`states` = states of the failed solve or round): counted, listed for
// overflow_slow_kernel (which redoes it with the reference's rescale) and written as nil until then.
__device__ __forceinline__ void retire_overflow(SizerLane& z, const SysView& s, const CandView& out, SizerCounters* ctr,
                                                int* overflow_list, int states) {
  const unsigned long long k = atomicAdd(&ctr->overflow_pairs, 1ull);
  if (overflow_list) overflow_list[k] = z.srv * s.n_acc + z.acc;
  z.states += states;
  lane_fail(z, s, out);
}

// Largest max-batch-size N any pair that needs sizing will use (allocation.go:79-88):
// decides the table geometry of the sizer launch.  Items are pairs of the view, or entries of `list` (list_pair).
__global__ void __launch_bounds__(256) max_batch_kernel(SysView s, const int* list, unsigned long long n_pairs, int* out) {
  int best = 0;
  for (unsigned long long item = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; item < n_pairs;
       item += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long pair = list_pair(list, item);
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

// Lane `src`'s service-rate coefficients (the fields rate_coef reads) and N, on every lane of the warp.
__device__ __forceinline__ PairModel shfl_model(const PairModel& m, int src) {
  const unsigned full = 0xffffffffu;
  PairModel b;
  b.alpha = __shfl_sync(full, m.alpha, src);
  b.beta = __shfl_sync(full, m.beta, src);
  b.in_tok = __shfl_sync(full, m.in_tok, src);
  b.out_tok = __shfl_sync(full, m.out_tok, src);
  b.slope = __shfl_sync(full, m.slope, src);
  b.pre_c = __shfl_sync(full, m.pre_c, src);
  b.dec_c = __shfl_sync(full, m.dec_c, src);
  b.N = __shfl_sync(full, m.N, src);
  return b;
}

}  // namespace wva
