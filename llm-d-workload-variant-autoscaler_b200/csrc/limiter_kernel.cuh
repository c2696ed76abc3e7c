// limiter_kernel.cuh — GPU-count limiter: DefaultLimiter.Limit
// (internal/engines/pipeline/default_limiter.go:42-81), TypeInventory.CreateAllocator /
// typeAllocator.TryAllocate (type_inventory.go:222-243,347-373) and
// GreedyBySaturation.Allocate (greedy_saturation_algorithm.go:34-108).
//
// The reference's sequential "take min(requested, remaining)" per accelerator type
// is exactly a per-type exclusive prefix sum over the candidates in priority order:
//   remaining_i = max(0, avail_t - sum_{j<i, type t} requested_j).
// Device pipeline: used[t] by integer atomics -> three stable LSD radix passes over ALL
// entries at a fixed size (cost, spare, segment) carrying the entry index (ties end in
// ascending index = the oracle's canonical order; entries that are not candidates carry
// the segment key T + 1 and sort last) -> segmented exclusive scan by type -> scatter
// of the mutated fields.  No step depends on a count read back by the host, so the
// whole pipeline can be captured into a CUDA graph (limiter_enqueue in capi_aux.inl).
// The radix sort / scan / select primitives are CUB (CUDA toolkit); the key
// construction, the allocation rule and the scatter are the kernels below.
#pragma once
#include "wva_core.cuh"
#include <cub/cub.cuh>

namespace wva {

// order-preserving map double -> uint64 (-0 == +0, NaN last)
__device__ __forceinline__ unsigned long long sortable_f64(double x) {
  if (x == 0.0) x = 0.0;
  unsigned long long b = (unsigned long long)__double_as_longlong(x);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}

// One thread per entry: used[t] by integer atomics, identity payload and cost key for the first sort pass, and the
// segment key of the last one.  An entry that is not a decision (has[d] == 0), not a scale-up candidate, or every entry
// when the limiter is off (*enable == 0) gets the key T + 1: it sorts after every real segment and consumes nothing.
__global__ void __launch_bounds__(256) limiter_prepare_kernel(long long D, int T, const int* acc_type, const int* current,
                                                              const int* target, const int* gpr, const double* cost,
                                                              const unsigned char* has, const int* enable, long long* used,
                                                              unsigned long long* k_cost, int* idx, unsigned* seg,
                                                              int* out_target, int* out_gpus, unsigned char* out_limited) {
  long long d = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= D) return;
  const bool dec = !has || has[d];
  const int t = acc_type[d];
  if (dec && t >= 0 && t < T) {  // calculateUsedGPUs default_limiter.go:72-81 (GPUsPerReplica as given)
    long long u = (long long)current[d] * gpr[d];
    if (u) atomicAdd((unsigned long long*)&used[t], (unsigned long long)u);
  }
  const bool cand = dec && (!enable || *enable) && target[d] > current[d];   // filterScaleUpCandidates :50-58
  seg[d] = !cand ? (unsigned)T + 1u : (t >= 0 && t < T) ? (unsigned)t : (unsigned)T;   // "" -> own segment T
  k_cost[d] = sortable_f64(cost[d]);
  idx[d] = (int)d;
  out_target[d] = target[d];
  out_gpus[d] = 0;
  out_limited[d] = 0;
}

// keys of the next pass in the current order: spare capacity, or the segment
__global__ void __launch_bounds__(256) limiter_gather_kernel(int n, const int* order, const double* spare, const unsigned* seg,
                                                             unsigned long long* k_spare, unsigned* k_seg) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int d = order[i];
  if (k_spare) k_spare[i] = sortable_f64(spare[d]);
  if (k_seg) k_seg[i] = seg[d];
}

// requested GPUs in final order (0 past the candidates)
__global__ void __launch_bounds__(256) limiter_request_kernel(int n, int T, const int* order, const unsigned* k_seg,
                                                              const int* current, const int* target, const int* gpr,
                                                              long long* req) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long r = 0;
  if (k_seg[i] <= (unsigned)T) {
    int d = order[i];
    int g = gpr[d]; if (g <= 0) g = 1;            // greedy_saturation_algorithm.go:85-88
    r = (long long)(target[d] - current[d]) * g;
  }
  req[i] = r;
}

// allocateForDecision (greedy_saturation_algorithm.go:79-108) with TryAllocate folded in, candidates only
__global__ void __launch_bounds__(256) limiter_apply_kernel(int n, int T, const int* order, const unsigned* k_seg,
                                                            const long long* req, const long long* prefix,
                                                            const long long* used, const int* type_limit,
                                                            const int* current, const int* target, const int* gpr,
                                                            int* out_target, int* out_gpus, unsigned char* out_limited) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned t = k_seg[i];
  if (t > (unsigned)T) return;
  int d = order[i];
  int g = gpr[d]; if (g <= 0) g = 1;
  long long needed = (long long)target[d] - current[d];
  long long allocated = 0;
  if (t < (unsigned)T) {
    long long avail0 = (long long)type_limit[t] - used[t];      // CreateAllocator type_inventory.go:231-236
    if (avail0 < 0) avail0 = 0;
    long long remaining = avail0 - prefix[i];
    if (remaining < 0) remaining = 0;
    allocated = req[i] < remaining ? req[i] : remaining;         // TryAllocate :358-366
  }
  long long replicas = allocated / g;
  out_gpus[d] = (int)(replicas * g);
  out_target[d] = current[d] + (int)replicas;
  out_limited[d] = replicas < needed ? 1 : 0;
}

}  // namespace wva
