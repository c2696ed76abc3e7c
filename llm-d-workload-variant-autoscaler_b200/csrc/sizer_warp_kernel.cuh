// sizer_warp_kernel.cuh — System.Calculate for small / medium systems: one WARP per
// (server, accelerator) candidate, bisection evaluated speculatively across the lanes.
//
// The float32 bisection of the reference (pkg/analyzer/utils.go:26-70) is a chain of
// ~25 dependent chain solves per target; with one lane per pair (sizer_lane_kernel.cuh) the
// wall time of a small system is the critical path of its slowest pair.  Here the lanes
// of a warp evaluate, in one round, every node of the next D levels of the bisection
// tree (the midpoints are pure float32 arithmetic on (lo, hi), so all 2^D - 1 are known
// before any is evaluated); the warp then walks the tree with the evaluated y values,
// taking exactly the branches BinarySearch would take, including its tolerance break,
// the iteration cap and the fixpoint rule (E6).  Results are bit-identical to the
// sequential search; ~6x fewer solves sit on the critical path.
//
// All lanes of a warp share the pair's head table (mu_n, 1/mu_n as float64 pairs in
// shared memory, broadcast reads) and run each solve in lock step: pass 1 for every
// lane, then pass 2 for every lane (no pass divergence inside the warp).
#pragma once
#include "wva_core.cuh"
#include "sizer_kernel.cuh"
#include "lockstep_solve.cuh"

namespace wva {

#if defined(__CUDACC__)

// one solve per lane: in lock step from the shared table, or — for a pair with a service rate outside the (E1) divisor
// range (warp-uniform: one pair per warp) — through the per-lane chain with IEEE divisions (warp_chain_solve)
__device__ __noinline__ void warp_chain_solve(const PairModel& m, float x, bool act, SolveStats& st, int& states, bool& ovf) {
  st = SolveStats{};
  states = 0;
  ovf = false;
  if (!act) return;
  Chain c;
  chain_start(c, x);
  c.tail_ok = d_bits(c.lamg) <= d_bits(m.mu_last);
  while (!chain_step(c, m, st)) {}
  ovf = c.phase == CH_OVERFLOW;
  states = c.states;
}
__device__ __forceinline__ void warp_solve(const PairModel& m, const double2* tab, float x, bool act, SolveStats& st,
                                           int& states, bool& ovf) {
  if (m.e1_ok) lockstep_solve(m, WarpTable{tab}, x, act, st, states, ovf);
  else warp_chain_solve(m, x, act, st, states, ovf);
}

template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
sizer_warp_kernel(SysView s, CandView out, const int* list, unsigned long long n_pairs, int nmax, SizerCounters* ctr,
                  int* overflow_list) {
  extern __shared__ double2 smem_tab2[];
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double2* tab = smem_tab2 + (size_t)warp * nmax;
  float* tabf = (float*)(smem_tab2 + (size_t)WARPS * nmax) + (size_t)warp * nmax;  // float32 copy for model_finish
  long long my_states = 0;
  int sv_states = 0;
  unsigned long long my_solves = 0;

  while (true) {
    unsigned long long item = 0;
    if (lane == 0) item = atomicAdd(&ctr->next_pair, 1ull);
    item = __shfl_sync(full, item, 0);
    if (item >= n_pairs) break;
    const unsigned long long pair = list_pair(list, item);
    const int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
    SizerLane z;   // used for its setup / bookkeeping fields; every lane holds the same copy
    int lim = 0;
    // candidates decided without a solve are written by lane 0 only
    CandView o0 = out;
    int rc = sizer_setup(z, s, o0, srv, acc, nmax, &lim, lane == 0);
    if (lim && lane == 0) ctr->limit_hit = 1;
    if (rc != SETUP_NEEDS_TABLE) continue;
    PairModel& m = z.m;
    __syncwarp();
    for (int n = lane; n < m.N; n += 32) {
      float mu32 = serv_rate(m, n + 1);
      double mu = (double)mu32;
      tabf[n] = mu32;
      tab[n] = make_double2(mu, rcp_f32den(mu32, mu));
    }
    __syncwarp();
    model_finish(m, tabf, 1);
    const size_t idx = (size_t)srv * s.n_acc + acc;
    int solves = 0;
    bool failed = false, ovf_any = false;
    Search& sT = z.sT;
    Search& sI = z.sI;
    SolveStats st;
    bool ovf;
    float y_t, y_i, pf;

    if (searches_begin(z)) {
      if (m.lambda_min > m.lambda_max) failed = true;   // BinarySearch: invalid range (utils.go:29-31)
      else {
        // ---- round 0: both end points (lanes 0,1) + the first 4 levels of the tree shared by both
        //      searches (lanes 2..16); every evaluation yields the TTFT and the ITL value ----------------
        const int D0 = 4;
        float x = 0.0f;
        bool act = false;
        if (lane == 0) { x = m.lambda_min; act = true; }
        else if (lane == 1) { x = m.lambda_max; act = true; }
        else if (lane < 2 + 15) { int node = lane - 1; x = spec_node_x(m.lambda_min, m.lambda_max, node, spec_depth_of(node)); act = true; }
        warp_solve(m, tab, x, act, st, sv_states, ovf); my_states += sv_states;
        solves += 17;
        if (__any_sync(full, act && ovf)) ovf_any = true;
        eval_values(m, st, &y_t, &y_i, &pf);
        if (!ovf_any) {
          for (int k = 0; k < 2; k++) {
            Search& q = k ? sI : sT;
            if (!q.active) continue;
            const float my_y = k ? y_i : y_t;
            if (!search_bracket(q, m, __shfl_sync(full, my_y, 0), __shfl_sync(full, my_y, 1))) failed = true;
            else if (q.active) spec_walk(q, D0, [&](int node) { return __shfl_sync(full, my_y, node + 1); });
          }
        }
        // ---- further rounds: 15-node trees, TTFT on lanes 0..14, ITL on lanes 16..30 (31-node tree on
        //      lanes 0..30 when only one search is still running) ------------------------------------
        while (!failed && !ovf_any && (sT.active || sI.active)) {
          const bool both = sT.active && sI.active;
          const int D = both ? 4 : 5;
          const int half = lane >> 4, hl = lane & 15;
          int node; bool mine_is_I;
          if (both) { node = hl + 1; mine_is_I = half == 1; act = hl < 15; }
          else { node = lane + 1; mine_is_I = sI.active; act = lane < 31; }
          const Search& mq = mine_is_I ? sI : sT;
          x = act ? spec_node_x(mq.lo, mq.hi, node, spec_depth_of(node)) : 0.0f;
          warp_solve(m, tab, x, act, st, sv_states, ovf); my_states += sv_states;
          solves += both ? 30 : 31;
          if (__any_sync(full, act && ovf)) { ovf_any = true; break; }
          eval_values(m, st, &y_t, &y_i, &pf);
          if (both) {
            spec_walk(sT, D, [&](int nd) { return __shfl_sync(full, y_t, nd - 1); });
            spec_walk(sI, D, [&](int nd) { return __shfl_sync(full, y_i, 16 + nd - 1); });
          } else if (sT.active) {
            spec_walk(sT, D, [&](int nd) { return __shfl_sync(full, y_t, nd - 1); });
          } else {
            spec_walk(sI, D, [&](int nd) { return __shfl_sync(full, y_i, nd - 1); });
          }
        }
      }
    }
    // ---- Size() tail + CreateAllocation (queueanalyzer.go:232-247, allocation.go:123-153) --------------
    Alloc a = alloc_none();
    float x;
    if (!failed && !ovf_any) {
      if (!size_lambda(z, x)) failed = true;
      else {
        warp_solve(m, tab, x, lane == 0, st, sv_states, ovf); my_states += sv_states;
        solves++;
        if (__shfl_sync(full, (int)ovf, 0)) ovf_any = true;
        else if (!alloc_replicas(z, __shfl_sync(full, st.throughput, 0), x)) failed = true;
        else {
          warp_solve(m, tab, x, lane == 0, st, sv_states, ovf); my_states += sv_states;
          solves++;
          if (__shfl_sync(full, (int)ovf, 0)) ovf_any = true;
          else if (lane == 0) {
            eval_values(m, st, &y_t, &y_i, &pf);
            a = alloc_final(z, s, st, y_i, pf);
          }
        }
      }
    }
    if (lane == 0) {
      if (ovf_any) {
        unsigned long long k = atomicAdd(&ctr->overflow_pairs, 1ull);
        if (overflow_list) overflow_list[k] = (int)idx;
      }
      store_candidate(out, idx, a, solves);   // nil when the pair is infeasible or overflowed
      my_solves += (unsigned long long)solves;
    }
    __syncwarp();
  }
  for (int o = 16; o; o >>= 1) my_states += __shfl_down_sync(full, my_states, o);
  if (lane == 0) { atomicAdd(&ctr->solves, my_solves); atomicAdd(&ctr->states, (unsigned long long)my_states); }
}
#endif  // __CUDACC__

}  // namespace wva
