// sizer_lane_kernel.cuh — System.Calculate for LARGE systems: one lane per (server,
// accelerator) candidate, persistent CTAs pulling pairs from a global counter, and the
// chain solves of the 32 pairs of a warp run in lock step (lockstep_solve.cuh) — each lane
// with its own head table (float32 column in shared memory, bank = lane) and its own
// arrival rate.  Between solves every lane advances its own bisection / Size / Analyze
// state machine (wva_core.cuh sizer_on_solve), idle lanes refill from the queue.
//
// Compared with sizer_kernel.cuh (one state per loop iteration, lanes in arbitrary
// phases) the lock-step rounds waste lanes whose chain ends early, but run ~10 instead
// of ~70 instructions per state.  Lanes of a warp must share N for the lock-step loops
// to be uniform; a round with mixed N falls back to the per-lane state machine.
#pragma once
#include "wva_core.cuh"
#include "sizer_kernel.cuh"
#include "lockstep_solve.cuh"

namespace wva {

// Split mode scratch: per pair two published results + a completion counter (zeroed before the launch).
struct SplitWs {
  float* res;     // [2 * n_pairs] lambda* of the TTFT / ITL item, < 0 = the search failed
  int* solves;    // [2 * n_pairs]
  int* cnt;       // [n_pairs]
};

// A split item finished its search: publish; the first finisher retires, the second merges and goes on.
template <bool DUAL>
__device__ __forceinline__ bool split_publish(SizerLane& z, const SysView& s, const CandView& out, const SplitWs& sw) {
  const size_t pair = (size_t)z.srv * s.n_acc + z.acc;
  const size_t me = pair * 2 + (size_t)z.split;
  sw.res[me] = z.failed ? -1.0f : (z.split == 0 ? z.sT.result : z.sI.result);
  sw.solves[me] = z.solves;
  __threadfence();
  const int old = atomicAdd(&sw.cnt[pair], 1);
  if (old == 0) return false;                          // partner still searching: it will finish the pair
  __threadfence();
  const float pr = *((volatile float*)&sw.res[me ^ 1]);
  z.solves += *((volatile int*)&sw.solves[me ^ 1]);
  z.merged = true;
  if (z.failed || pr < 0.0f) { lane_fail(z, s, out); return false; }
  if (z.split == 0) z.sI.result = pr; else z.sT.result = pr;
  return DUAL ? spec2_after_search(z, s, out) : sizer_after_search(z, s, out);   // -> the two Analyze solves
}

template <int THREADS, bool SMEM_TABLE, bool DUAL, bool SPLIT>
__device__ __forceinline__ void
sizer_lane_body(SysView s, CandView out, unsigned long long n_pairs, int nmax, float* gtab,
                  SizerCounters* ctr, int* overflow_list, SplitWs sw, const unsigned* order, int gang) {
  extern __shared__ float smem_tab[];
  const int lane = threadIdx.x & 31;
  const unsigned full = 0xffffffffu;
  float* tab;
  int stride;
  if (SMEM_TABLE) { tab = smem_tab + threadIdx.x; stride = THREADS; }
  else { tab = gtab + ((size_t)blockIdx.x * THREADS + threadIdx.x); stride = gridDim.x * THREADS; }

  SizerLane z;
  z.m.N = 1; z.m.K = 11; z.m.mono = 0; z.m.mu_last = 1.0; z.m.r_last = 1.0;
  SolveStats st;
  bool live = false, exhausted = false;
  unsigned long long my_solves = 0, my_states = 0, my_slots = 0;

  while (true) {
    // ---- refill ------------------------------------------------------------------------------
    bool need_table = false;
    // gang refill: the warp takes 32 new items only when all of its lanes are idle, so its lanes stay in the SAME
    // bisection step (a chain at the first midpoint is ~10x shorter than one at lambda_max: lanes in different
    // steps made every round as long as the longest step)
    const bool may_refill = !gang || !__any_sync(full, live);
    if (!live && !exhausted && may_refill) {
      while (true) {
        unsigned long long item = atomicAdd(&ctr->next_pair, 1ull);
        if (item >= (SPLIT ? 2 * n_pairs : n_pairs)) { exhausted = true; break; }
        if (order) item = order[item];                 // length-sorted queue (sizer_probe.cuh)
        const unsigned long long pair = SPLIT ? (item >> 1) : item;
        int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
        int lim = 0;
        int rc = sizer_setup(z, s, out, srv, acc, nmax, &lim, !SPLIT || (item & 1) == 0);
        if (lim) ctr->limit_hit = 1;
        if (rc == SETUP_NEEDS_TABLE) { need_table = true; if (SPLIT) z.split = (int)(item & 1); break; }
      }
    }
    unsigned need = __ballot_sync(full, need_table);
    while (need) {   // BuildModel, cooperatively (see sizer_kernel.cuh)
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
      model_fill_table(b, tab + (src - lane), stride, lane, 32);
    }
    __syncwarp();
    if (need_table) {
      model_finish(z.m, tab, stride);
      live = DUAL ? (SPLIT ? spec2_begin(z, s, out) : dual_begin(z, s, out)) : sizer_begin(z, s, out);
      if (SPLIT) { if (live && z.stage == SZ_PUBLISH) live = split_publish<DUAL>(z, s, out, sw); }
      if (!live) my_solves += z.solves;
    }
    const unsigned live_mask = __ballot_sync(full, live);
    if (!live_mask) {
      if (!__any_sync(full, !exhausted)) break;
      continue;
    }
    // ---- one round: every live lane solves its chain at z.cur_x -------------------------------
    const int nref = __shfl_sync(full, z.m.N, __ffs(live_mask) - 1);
    const bool uniform = __all_sync(full, !live || z.m.N == nref);
    bool bad = false;
    int sv = 0;
    if (uniform && !live) { z.m.N = nref; z.m.K = nref + nref * WVA_QUEUE_TO_BATCH; }   // idle lanes only keep the loops uniform
    LaneTable lt; lt.t = tab; lt.stride = stride;
    if (DUAL) {
      // TTFT and ITL searches advance together: two chains per lane share every table load
      SolveStats st2[2];
      float xs[2] = {z.x2[0], z.x2[1]};
      bool act[2] = {live && z.act2[0], live && z.act2[1]};
      if (uniform) {
        lockstep_solve_inl<2, LaneTable>(z.m, lt, xs, act, st2, sv, bad);   // single call site: inlined, own register budget
      } else if (live) {
        for (int c = 0; c < 2; c++) {
          if (!act[c]) continue;
          chain_start(z.c, xs[c]);
          z.c.tail_ok = d_bits(z.c.lamg) <= d_bits(z.m.mu_last);
          while (!chain_step(z.c, z.m, st2[c])) {}
          bad = bad || z.c.phase == CH_OVERFLOW;
          sv += z.c.states;
        }
      }
      if (live) {
        if (bad) {
          unsigned long long k = atomicAdd(&ctr->overflow_pairs, 1ull);
          if (overflow_list) overflow_list[k] = z.srv * s.n_acc + z.acc;
          z.states += sv;
          lane_fail(z, s, out);
          live = false;
        } else {
          live = SPLIT ? spec2_on_solve(z, s, out, st2, sv) : dual_on_solve(z, s, out, st2, sv);
          if (SPLIT) { if (live && z.stage == SZ_PUBLISH) live = split_publish<true>(z, s, out, sw); }
        }
        if (!live) { my_solves += z.solves; my_states += z.states; }
      }
    } else {
      if (uniform) {
        lockstep_solve(z.m, lt, z.cur_x, live, st, sv, bad);
        z.c.states = sv;
      } else if (live) {
        while (!chain_step(z.c, z.m, st)) {}
        bad = z.c.phase == CH_OVERFLOW;
      }
      if (live) {
        if (bad) {
          unsigned long long k = atomicAdd(&ctr->overflow_pairs, 1ull);
          if (overflow_list) overflow_list[k] = z.srv * s.n_acc + z.acc;
          z.states += z.c.states;
          lane_fail(z, s, out);
          live = false;
        } else {
          live = sizer_on_solve(z, s, out, st);
          if (SPLIT) { if (live && z.stage == SZ_PUBLISH) live = split_publish<false>(z, s, out, sw); }
        }
        if (!live) { my_solves += z.solves; my_states += z.states; }
      }
    }
    {
      int mxs = sv;
      for (int o = 16; o; o >>= 1) mxs = max(mxs, __shfl_xor_sync(full, mxs, o));
      if (lane == 0) my_slots += 32ull * (unsigned long long)mxs;
    }
  }
  for (int o = 16; o; o >>= 1) {
    my_solves += __shfl_down_sync(full, my_solves, o);
    my_states += __shfl_down_sync(full, my_states, o);
  }
  if (lane == 0) { atomicAdd(&ctr->solves, my_solves); atomicAdd(&ctr->states, my_states); atomicAdd(&ctr->lockstep_slots, my_slots); }
}

template <int THREADS, bool SMEM_TABLE, bool DUAL, bool SPLIT>
__global__ void __launch_bounds__(THREADS)
sizer_lane_kernel(SysView s, CandView out, unsigned long long n_pairs, int nmax, float* gtab,
                  SizerCounters* ctr, int* overflow_list, SplitWs sw, const unsigned* order, int gang) {
  sizer_lane_body<THREADS, SMEM_TABLE, DUAL, SPLIT>(s, out, n_pairs, nmax, gtab, ctr, overflow_list, sw, order, gang);
}

// The plain lane kernel with its table in global memory — large N on large systems (BASELINE config 3) — is launched
// two blocks per SM; left alone ptxas gives it 168 registers and the second block never becomes resident.  Capped at
// 128 registers (spills only around the solver call, none in the chunk loops) both blocks run: 4 warps per SMSP feed
// the FP64 pipe instead of 2.
__global__ void __launch_bounds__(256, 2)
sizer_lane_kernel_gtab_2blk(SysView s, CandView out, unsigned long long n_pairs, int nmax, float* gtab,
                            SizerCounters* ctr, int* overflow_list, SplitWs sw, const unsigned* order, int gang) {
  sizer_lane_body<256, false, false, false>(s, out, n_pairs, nmax, gtab, ctr, overflow_list, sw, order, gang);
}

}  // namespace wva
