// pipeline_v2_kernel.cuh — the V2 scaling pipeline around the token-capacity analyzer, batched over models:
//
//   saturation_v2_kernel   SaturationAnalyzer.Analyze        internal/engines/analyzers/saturation_v2/analyzer.go:59-138
//   cost_aware_kernel      CostAwareOptimizer.Optimize       internal/engines/pipeline/cost_aware_optimizer.go:39-197
//   enforce_kernel         Enforcer.EnforcePolicy            internal/engines/pipeline/enforcer.go:55-183
//
// All three are per-model, order-dependent scalar algorithms over a handful of variants (float64 sums in slice
// order, "first best" selections, a running `remaining`), so the mapping is one warp per model with a lane per
// variant for the parts that are independent per variant (replica streams, medians) and warp-uniform sequential
// walks, fed by shuffles, for the ordered parts.  HBM-bound: 56 B per replica for the analyzer, ~30 B per variant
// for the other two.
#pragma once
#include "wva_core.cuh"

namespace wva {

struct SatV2In {
  long long n_models, n_variants, n_replicas;
  const int *model_variant_off, *variant_replica_off;
  const long long *rep_total_kv, *rep_tokens_in_use, *rep_queue_len, *rep_k2;
  const double *rep_avg_in, *rep_avg_out, *rep_hit;
  const int* rep_slice_order;
  const int *var_current, *var_pending;
  const double* var_fallback;
  const double *cfg_kv_threshold, *cfg_scale_up, *cfg_scale_down;
  const long long *sched_size, *sched_bytes;
};
struct SatV2Out {
  long long *rep_k1, *rep_effective, *rep_demand; unsigned char* rep_saturated;
  int* var_ready; double *var_cap, *var_total_cap, *var_total_demand, *var_util;
  double *mod_supply, *mod_demand, *mod_util, *mod_required, *mod_spare;
};

// float64 -> int64 as Go does on amd64 (CVTTSD2SQ): NaN / out of range -> 0x8000000000000000
__device__ __forceinline__ long long go_int64(double x) {
  if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return (long long)0x8000000000000000ull;
  return (long long)x;   // cvt.rzi.s64.f64
}

__device__ __forceinline__ double shfl_d(unsigned mask, double v, int src) {
  int lo = __shfl_sync(mask, __double2loint(v), src), hi = __shfl_sync(mask, __double2hiint(v), src);
  return __hiloint2double(hi, lo);
}

// the five input streams of one replica
struct V2Rep { long long cap, in_use, queue, k2; double avg_in; };
__device__ __forceinline__ V2Rep v2_load(const SatV2In& in, int r) {
  V2Rep x;
  x.cap = in.rep_total_kv[r]; x.in_use = in.rep_tokens_in_use[r]; x.queue = in.rep_queue_len[r]; x.k2 = in.rep_k2[r];
  x.avg_in = in.rep_avg_in[r];
  return x;
}
// effective capacity of a replica (0 when it has no capacity data); also its demand
__device__ __forceinline__ bool v2_eval(const V2Rep& x, double kv_thr, long long& k1, long long& eff, long long& demand) {
  k1 = 0; eff = 0; demand = 0;
  if (x.cap <= 0) return false;                                                        // analyzer.go:148-150
  demand = x.in_use;
  if (x.avg_in > 0) demand += x.queue * go_int64(x.avg_in);                            // :153-156
  k1 = go_int64(d_mul((double)x.cap, kv_thr));                                         // :159
  const long long k2 = x.k2 < 0 ? k1 : x.k2;                                           // computeK2 priority 4
  eff = k2 < k1 ? k2 : k1;                                                             // :175-178
  return true;
}
__device__ __forceinline__ bool v2_replica(const SatV2In& in, int r, double kv_thr, long long& k1, long long& eff, long long& demand) {
  if (in.rep_total_kv[r] <= 0) { k1 = 0; eff = 0; demand = 0; return false; }          // the other streams are not read
  return v2_eval(v2_load(in, r), kv_thr, k1, eff, demand);
}

// Three ordered float64 sums over 32 slots at once: the slots go through shared memory ([3][V2_COL] per warp) and lane c
// (c = 0, 1, 2; the other lanes wait) runs chain c as 32 dependent adds fed by LDS — 2 instructions per
// element for the warp instead of the 14 of a shuffle-fed walk.  A slot that must not count holds +0.0 (x + 0.0 == x).
// V2_COL = 34 doubles puts the three columns 4 banks apart: with 32 (same banks) every read was a 3-way conflict, and
// those reads were most of the kernel's L1TEX time.
#define V2_COL 34
__device__ __forceinline__ void ordered_sums3(double* buf, int lane, double a, double b, double c, double& sa, double& sb, double& sc) {
  const unsigned full = 0xffffffffu;
  __syncwarp();
  buf[lane] = a; buf[V2_COL + lane] = b; buf[2 * V2_COL + lane] = c;
  __syncwarp();
  const double2* col = reinterpret_cast<const double2*>(buf + V2_COL * (lane % 3));   // 16-byte aligned: V2_COL is even
  double acc = (lane % 3 == 0) ? sa : ((lane % 3 == 1) ? sb : sc);
  // only lanes 0-2 run the chains: with all 32 lanes shadowing them these 128-bit shared loads (one wavefront per
  // quarter-warp) were half of the L1 data-pipe wavefronts of the kernel; the kernel time did not move — it is bound
  // by issue slots and latency, not by the L1 pipe
  if (lane < 3) {
#pragma unroll
    for (int l = 0; l < 16; l++) { const double2 t = col[l]; acc = d_add(d_add(acc, t.x), t.y); }
  }
  __syncwarp();
  sa = shfl_d(full, acc, 0); sb = shfl_d(full, acc, 1); sc = shfl_d(full, acc, 2);
}

// Replicas of one model staged per warp: a model's replicas are one contiguous range of the replica arrays, so the
// warp reads them COALESCED (lane = replica, 5 input streams, 4 output streams), leaves (effective, demand) in shared
// memory, and the per-variant parts — ordered demand sum, median — run lane-per-variant on shared memory.  Reading the
// replica arrays lane-per-variant straight from global memory (12 sectors per request) kept L1TEX busy at half the
// bandwidth of the staged form, with conflict-free ordered sums and two rounds of loads in flight.  Models with more
// than V2_STAGE replicas still take the lane-per-variant path.
#define V2_STAGE 256
#define V2_NO_DATA 0x7fffffffffffffffLL   // never a real effective capacity: go_int64 < 2^63 - 1, and eff <= k1

// 4 blocks per SM = 64 registers: faster than 1 / 3 / 5 blocks (88 / 72 / 48 registers) at 200 000 models x 32
// variants — occupancy against spills.
#ifndef V2_MINB
#define V2_MINB 4
#endif
#ifndef V2_ROUNDS
#define V2_ROUNDS 2   // rounds of replica loads in flight per lane in the staging phase (3 gains nothing over 2)
#endif
__global__ void __launch_bounds__(256, V2_MINB) saturation_v2_kernel(SatV2In in, SatV2Out out) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  __shared__ __align__(16) double sums_buf[8][3 * V2_COL];
  __shared__ long long stage_eff[8][V2_STAGE], stage_dem[8][V2_STAGE];
  double* buf = sums_buf[threadIdx.x >> 5];
  long long* s_eff = stage_eff[threadIdx.x >> 5];
  long long* s_dem = stage_dem[threadIdx.x >> 5];
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long m = warp0; m < in.n_models; m += nwarps) {
    const int v0 = in.model_variant_off[m], v1 = in.model_variant_off[m + 1];
    const double kv_thr = in.cfg_kv_threshold[m];
    const int R0 = in.variant_replica_off[v0], R1 = in.variant_replica_off[v1];
    const bool staged = R1 - R0 <= V2_STAGE;
    if (staged) {                                                                      // computeReplicaCapacity, lane = replica
      __syncwarp();
      for (int r0 = R0 + lane; r0 < R1; r0 += 32 * V2_ROUNDS) {                         // V2_ROUNDS rounds of loads in flight
        V2Rep x[V2_ROUNDS];
#pragma unroll
        for (int h = 0; h < V2_ROUNDS; h++) x[h] = v2_load(in, r0 + 32 * h < R1 ? r0 + 32 * h : r0);
#pragma unroll
        for (int h = 0; h < V2_ROUNDS; h++) {
          const int r = r0 + 32 * h;
          if (r >= R1) break;
          long long k1, eff, demand;
          const bool has = v2_eval(x[h], kv_thr, k1, eff, demand);
          s_eff[r - R0] = has ? eff : V2_NO_DATA;
          s_dem[r - R0] = demand;
          if (out.rep_k1) out.rep_k1[r] = k1;
          if (out.rep_effective) out.rep_effective[r] = eff;
          if (out.rep_demand) out.rep_demand[r] = demand;
          if (out.rep_saturated) out.rep_saturated[r] = (has && demand >= eff) ? 1 : 0;  // :180
        }
      }
      __syncwarp();
    }
    double total_supply = 0.0, total_anticipated = 0.0, total_demand = 0.0;
    for (int c0 = v0; c0 < v1; c0 += 32) {
      const int v = c0 + lane;
      const bool act = v < v1;
      double demand_sum = 0.0, cap = 0.0, total_cap = 0.0, anticipated = 0.0;
      if (act) {
        const int lo = in.variant_replica_off[v], hi = in.variant_replica_off[v + 1];
        int n_data = 0;
        long long e8[8];                                                               // effective capacities of a small variant
        const bool small = hi - lo <= 8;
#pragma unroll
        for (int j = 0; j < 8; j++) e8[j] = V2_NO_DATA;
        if (staged) {
          for (int r0 = lo; r0 < hi; r0 += 8) {
#pragma unroll
            for (int j = 0; j < 8; j++) {
              const int r = r0 + j;
              if (r >= hi) break;
              const long long eff = s_eff[r - R0];
              if (eff != V2_NO_DATA) { n_data++; demand_sum = d_add(demand_sum, (double)s_dem[r - R0]); if (small) e8[j] = eff; }   // :309-312
            }
          }
        } else {
          for (int r0 = lo; r0 < hi; r0 += 8) {                                        // slice order, straight from global memory
#pragma unroll
            for (int j = 0; j < 8; j++) {
              const int r = r0 + j;
              if (r >= hi) break;
              long long k1, eff, demand;
              const bool has = v2_replica(in, r, kv_thr, k1, eff, demand);
              if (has) { n_data++; demand_sum = d_add(demand_sum, (double)demand); if (small) e8[j] = eff; }
              if (out.rep_k1) out.rep_k1[r] = k1;
              if (out.rep_effective) out.rep_effective[r] = eff;
              if (out.rep_demand) out.rep_demand[r] = demand;
              if (out.rep_saturated) out.rep_saturated[r] = (has && demand >= eff) ? 1 : 0;
            }
          }
        }
        if (n_data > 0) {
          // median (analyzer.go:505-519) by rank counting: the element of rank k has exactly k elements before it in
          // (value, index) order.  Up to 8 replicas: on the registers just filled (absent slots hold +inf and rank last);
          // more: over the staged values, or re-evaluating the replicas — no scratch.
          const int k_hi = n_data / 2, k_lo = (n_data % 2 == 0) ? k_hi - 1 : k_hi;
          long long m_lo = 0, m_hi = 0;
          if (small) {
#pragma unroll
            for (int a = 0; a < 8; a++) {
              int rank = 0;
#pragma unroll
              for (int b = 0; b < 8; b++) rank += (e8[b] < e8[a] || (e8[b] == e8[a] && b < a)) ? 1 : 0;
              if (rank == k_lo) m_lo = e8[a];
              if (rank == k_hi) m_hi = e8[a];
            }
          } else if (staged) {
            for (int r = lo; r < hi; r++) {
              const long long e = s_eff[r - R0];
              if (e == V2_NO_DATA) continue;
              int rank = 0;
              for (int q = lo; q < hi; q++) {
                const long long eq = s_eff[q - R0];                                    // the sentinel never ranks before a value
                if (eq < e || (eq == e && q < r)) rank++;
              }
              if (rank == k_lo) m_lo = e;
              if (rank == k_hi) m_hi = e;
            }
          } else {
            for (int r = lo; r < hi; r++) {
              long long k1, e, d;
              if (!v2_replica(in, r, kv_thr, k1, e, d)) continue;
              int rank = 0;
              for (int q = lo; q < hi; q++) {
                long long k1q, eq, dq;
                if (!v2_replica(in, q, kv_thr, k1q, eq, dq)) continue;
                if (eq < e || (eq == e && q < r)) rank++;
              }
              if (rank == k_lo) m_lo = e;
              if (rank == k_hi) m_hi = e;
            }
          }
          cap = (double)((n_data % 2 == 0) ? (m_lo + m_hi) / 2 : m_hi);
        } else {
          cap = in.var_fallback[v];                                                    // :317-324 (resolved by the caller)
        }
        const int pending = in.var_pending[v];
        int ready = in.var_current[v] - pending;                                        // :300-303
        if (ready < 0) ready = 0;
        total_cap = d_mul((double)ready, cap);
        double util = 0.0;
        if (total_cap > 0) util = d_div(demand_sum, total_cap);
        anticipated = d_mul((double)(ready + pending), cap);                           // Analyze :93-94
        if (out.var_ready) out.var_ready[v] = ready;
        if (out.var_cap) out.var_cap[v] = cap;
        if (out.var_total_cap) out.var_total_cap[v] = total_cap;
        if (out.var_total_demand) out.var_total_demand[v] = demand_sum;
        if (out.var_util) out.var_util[v] = util;
      }
      // model sums in VariantStates order (Analyze :88-96); an inactive slot adds +0.0
      ordered_sums3(buf, lane, total_cap, demand_sum, anticipated, total_supply, total_demand, total_anticipated);
    }
    // scheduler queue demand (estimateSchedulerQueueDemand :471-501), only for the models that have one
    const long long qs = in.sched_size ? in.sched_size[m] : 0, qb = in.sched_bytes ? in.sched_bytes[m] : 0;
    if (in.sched_size && !(qs == 0 && qb == 0)) {
      // computeModelWorkloadAverages (:438-455): float64 sums over the model's replicas in SLICE order; the lanes
      // fetch 32 replicas per round trip, the adds run in order through shuffles
      const int r0 = R0, r1 = R1;
      double ai = 0.0, ao = 0.0, ah = 0.0;
      int cnt = 0;
      for (int b = r0; b < r1; b += 32) {
        const int pos = b + lane;
        double xi = 0.0, xo = 0.0, xh = 0.0;
        bool use = false;
        if (pos < r1) {
          const int r = in.rep_slice_order ? in.rep_slice_order[pos] : pos;
          xi = in.rep_avg_in[r]; xo = in.rep_avg_out[r]; xh = in.rep_hit[r];
          use = xi > 0 || xo > 0;
        }
        const unsigned um = __ballot_sync(full, use);
        ordered_sums3(buf, lane, use ? xi : 0.0, use ? xo : 0.0, use ? xh : 0.0, ai, ao, ah);
        cnt += __popc(um);
      }
      if (cnt > 0) { ai = d_div(ai, (double)cnt); ao = d_div(ao, (double)cnt); ah = d_div(ah, (double)cnt); }
      const double from_bytes = d_div((double)qb, 4.0);                                // BytesPerToken
      const double from_count = d_mul((double)qs, ai);
      double input_tokens = from_bytes;
      if (from_count > input_tokens) input_tokens = from_count;
      input_tokens = d_mul(input_tokens, d_sub(1.0, ah));
      const double output_tokens = d_mul((double)qs, ao);
      total_demand = d_add(total_demand, d_add(input_tokens, output_tokens));
    }
    if (lane == 0) {
      double utilization = 0.0;
      if (total_supply > 0) utilization = d_div(total_demand, total_supply);           // :101-104
      double required = 0.0, spare = 0.0;
      const double up = in.cfg_scale_up[m], down = in.cfg_scale_down[m];
      if (up > 0) required = d_sub(d_div(total_demand, up), total_anticipated);        // :108-113
      if (required < 0) required = 0.0;
      if (down > 0) spare = d_sub(total_supply, d_div(total_demand, down));            // :115-120
      if (spare < 0) spare = 0.0;
      if (out.mod_supply) out.mod_supply[m] = total_supply;
      if (out.mod_demand) out.mod_demand[m] = total_demand;
      if (out.mod_util) out.mod_util[m] = utilization;
      if (out.mod_required) out.mod_required[m] = required;
      if (out.mod_spare) out.mod_spare[m] = spare;
    }
  }
}

// ---- CostAwareOptimizer ---------------------------------------------------------------------------------------------------
// One warp per model.  The variants are visited in sorted order without sorting: "next in (key, index) order after the
// last one" is an arg-min over the lanes (chunks of 32 for wider models), the walk itself is warp-uniform.
__global__ void __launch_bounds__(256) cost_aware_kernel(long long n_models, const int* mvo, const double* required, const double* spare,
                                                         const unsigned char* has_result, const int* current, const double* cost,
                                                         const double* cap, int* target) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const double DMAX = 1.79769313486231570814527423731704357e+308;
  for (long long m = warp0; m < n_models; m += nwarps) {
    const int v0 = mvo[m], v1 = mvo[m + 1], V = v1 - v0;
    if (has_result && !has_result[m]) {                                                // req.Result == nil :49-51
      for (int v = v0 + lane; v < v1; v += 32) target[v] = -1;
      continue;
    }
    const double req = required[m], spr = spare[m];
    const bool up = req > 0, down = !up && spr > 0;
    if (V <= 32) {
      // the usual model: a lane owns its variant — cost, capacity, sort key and target stay in registers, the walk
      // visits the not-yet-visited variant with the smallest (key, index), and each target is written once
      const int v = v0 + lane;
      const bool act = v < v1;
      const double mc = act ? cost[v] : 0.0, mcap = act ? cap[v] : 0.0;
      int tgt = act ? current[v] : 0;                                                  // initTargets
      if (up || down) {
        int cheapest = -1;
        if (down) {                                                                    // findCheapestVariant :191-201
          double c = act ? mc : DMAX;
          int idx = (act && c < DMAX) ? v : -1;
          for (int o = 16; o; o >>= 1) {
            const double oc = shfl_d(full, c, lane ^ o);
            const int oi = __shfl_xor_sync(full, idx, o);
            if (oi >= 0 && (idx < 0 || oc < c || (oc == c && oi < idx))) { c = oc; idx = oi; }
          }
          if (idx >= 0 && c < DMAX) cheapest = idx;
        }
        const double key = up ? (mcap <= 0 ? DMAX : d_div(mc, mcap)) : -mc;            // costEfficiency :233-238 / sortByCostDesc
        bool visited = !act;
        double remaining = up ? req : spr;
        for (int step = 0; step < V && remaining > 0; step++) {
          double k = key; int idx = visited ? -1 : v;
          for (int o = 16; o; o >>= 1) {
            const double ok = shfl_d(full, k, lane ^ o);
            const int oi = __shfl_xor_sync(full, idx, o);
            if (oi >= 0 && (idx < 0 || ok < k || (ok == k && oi < idx))) { k = ok; idx = oi; }
          }
          const int bi = idx;
          if (bi < 0) break;
          if (v == bi) visited = true;
          const double c = shfl_d(full, mcap, bi - v0);
          if (c <= 0) continue;
          if (up) {                                                                    // :88-96
            const long long need = go_int64(ceil(d_div(remaining, c)));
            if (v == bi) tgt = (int)((long long)tgt + need);
            remaining = d_sub(remaining, d_mul((double)need, c));
          } else {                                                                     // :126-160
            const int cur = __shfl_sync(full, tgt, bi - v0);
            int min_rep = 0;
            if (bi == cheapest && !__any_sync(full, act && v != cheapest && tgt > 0)) min_rep = 1;
            const int removable = cur - min_rep;
            if (removable > 0) {
              long long rem = go_int64(floor(d_div(remaining, c)));
              if (rem > removable) rem = removable;
              if (rem > 0) {
                if (v == bi) tgt = cur - (int)rem;
                remaining = d_sub(remaining, d_mul((double)rem, c));
              }
            }
          }
        }
      }
      if (act) target[v] = tgt;
      continue;
    }
    for (int v = v0 + lane; v < v1; v += 32) target[v] = current[v];                   // initTargets
    __syncwarp();
    if (!up && !down) continue;
    int cheapest = -1;
    if (down) {                                                                        // findCheapestVariant :191-201
      double best = DMAX;
      for (int c0 = v0; c0 < v1; c0 += 32) {
        const int v = c0 + lane;
        double c = (v < v1) ? cost[v] : DMAX;
        int idx = (v < v1 && c < DMAX) ? v : -1;
        for (int o = 16; o; o >>= 1) {
          const double oc = shfl_d(full, c, lane ^ o);
          const int oi = __shfl_xor_sync(full, idx, o);
          if (oi >= 0 && (idx < 0 || oc < c || (oc == c && oi < idx))) { c = oc; idx = oi; }
        }
        if (idx >= 0 && c < best) { best = c; cheapest = idx; }
      }
    }
    double remaining = up ? req : spr;
    // last visited (key, index); keys: scale-up = cost efficiency ascending, scale-down = -cost ascending
    double last_key = 0.0; int last_idx = -1;
    for (int step = 0; step < V && remaining > 0; step++) {
      double bk = 0.0; int bi = -1;
      for (int c0 = v0; c0 < v1; c0 += 32) {
        const int v = c0 + lane;
        double k = 0.0; int idx = -1;
        if (v < v1) {
          k = up ? (cap[v] <= 0 ? DMAX : d_div(cost[v], cap[v])) : -cost[v];           // costEfficiency :233-238 / sortByCostDesc
          const bool after = last_idx < 0 || k > last_key || (k == last_key && v > last_idx);
          idx = after ? v : -1;
        }
        for (int o = 16; o; o >>= 1) {
          const double ok = shfl_d(full, k, lane ^ o);
          const int oi = __shfl_xor_sync(full, idx, o);
          if (oi >= 0 && (idx < 0 || ok < k || (ok == k && oi < idx))) { k = ok; idx = oi; }
        }
        if (idx >= 0 && (bi < 0 || k < bk)) { bk = k; bi = idx; }
      }
      if (bi < 0) break;
      last_key = bk; last_idx = bi;
      const double c = cap[bi];
      if (c <= 0) continue;
      if (up) {                                                                        // :88-96
        const long long need = go_int64(ceil(d_div(remaining, c)));
        if (lane == 0) target[bi] = (int)((long long)target[bi] + need);
        remaining = d_sub(remaining, d_mul((double)need, c));
      } else {                                                                         // :126-160
        const int cur = target[bi];
        int min_rep = 0;
        if (bi == cheapest) {
          bool other = false;
          for (int v = v0 + lane; v < v1; v += 32) if (v != cheapest && target[v] > 0) other = true;
          if (!__any_sync(full, other)) min_rep = 1;
        }
        const int removable = cur - min_rep;
        if (removable > 0) {
          long long rem = go_int64(floor(d_div(remaining, c)));
          if (rem > removable) rem = removable;
          if (rem > 0) {
            if (lane == 0) target[bi] = cur - (int)rem;
            remaining = d_sub(remaining, d_mul((double)rem, c));
          }
        }
      }
      __syncwarp();
    }
  }
}

// ---- Enforcer ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) enforce_kernel(long long n_models, const int* mvo, const unsigned char* s2z, const double* req_count,
                                                      const unsigned char* req_err, const double* cost, const unsigned char* has_cost,
                                                      const int* name_rank, int* target, unsigned char* applied) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long m = warp0; m < n_models; m += nwarps) {
    const int v0 = mvo[m], v1 = mvo[m + 1];
    bool app = false;
    if (s2z[m]) {                                                                      // applyScaleToZero :86-127
      const bool err = req_err && req_err[m];
      if (!err && !(req_count[m] > 0)) {
        for (int v = v0 + lane; v < v1; v += 32) if (target[v] >= 0) target[v] = 0;
        app = true;
      }
    } else {                                                                           // ensureMinimumReplicas :130-183
      long long total = 0;
      for (int v = v0 + lane; v < v1; v += 32) { const int t = target[v]; if (t >= 0) total += t; }
      total = __reduce_add_sync(full, (unsigned)(total > 0 ? 1 : 0));
      if (total == 0) {
        // the reference's running "cheapestCost < 0 || cost < cheapestCost || tie -> smaller name" walk, in index order
        // (name_rank: the variants' ranks by name when the index order is not the name order — fused pipeline)
        int cheapest = -1, cheapest_rank = -1; double cc = -1.0;
        for (int c0 = v0; c0 < v1; c0 += 32) {
          const int v = c0 + lane;
          const bool in_map = v < v1 && target[v] >= 0;
          const double c = in_map ? ((has_cost && !has_cost[v]) ? 10.0 : cost[v]) : 0.0;   // saturation.DefaultVariantCost
          const int rk = in_map ? (name_rank ? name_rank[v] : v) : 0;
          unsigned mask = __ballot_sync(full, in_map);
          for (; mask; mask &= mask - 1) {
            const int src = __ffs(mask) - 1;
            const double sc = shfl_d(full, c, src);
            const int sr = __shfl_sync(full, rk, src);
            if (cc < 0 || sc < cc || (sc == cc && sr < cheapest_rank)) { cheapest = c0 + src; cheapest_rank = sr; cc = sc; }
          }
        }
        if (cheapest >= 0) { if (lane == 0) target[cheapest] = 1; app = true; }
      }
    }
    if (lane == 0 && applied) applied[m] = app ? 1 : 0;
  }
}

}  // namespace wva
