// sizer_pool_kernel.cuh — System.Calculate for LARGE systems with the lock-step solver fed from a POOL of pairs.
//
// The lane sizer (sizer_lane_kernel.cuh) binds a pair to a lane for its whole life, so a lock-step round costs the
// longest of 32 chains that happen to sit in one warp: 49 % of the executed lane-steps do live work on BASELINE
// configs[2] (59-62 % with the probe-sorted queue).  Chain length is almost a function of lambda / mu_N alone (early exit
// E4), and it changes from one bisection step of a pair to the next — so here the binding is dropped:
//   * a CTA keeps a pool of P pairs whose state (the SizerLane of wva_core.cuh) lives in global memory (L2-resident:
//     368 bytes per pair); a pair has no head table (m.tab == nullptr): its service rates are computed where a solve
//     needs them (RateTable, model_rate);
//   * every solve a pair still needs is a REQUEST — the pair's slot — queued in shared memory by class: 28 fast classes
//     keyed by the head length N (the cost of the certified fast solve, E12) and 4 exact classes keyed by the exact
//     solver's chain-length estimate, which hold the solves the fast solve did not certify;
//   * a warp takes 32 requests from one class: an exact class as soon as it holds 32, else the fullest fast class
//     (filling up from its fast neighbours), and a partial exact batch only when no fast request is pending.  It loads
//     the 32 pairs' models and solves them in lock step (fast solve or exact lockstep_solve).  A lane the fast solve did
//     not certify re-queues its pair into an exact class at the same rate; every other lane advances its pair's
//     bisection / Size / Analyze state machine (sizer_on_solve, the same code as every other sizer), stores the state
//     back and queues the pair's next request — or retires the pair and frees its slot.
//   * Free slots are refilled with new pairs from the global work counter: setup runs lane by lane, then the warp scans
//     the service rates of the lanes that need a model together, 32 entries at a time.
// Which lanes solve which pairs together changes nothing in any pair's arithmetic: same solves, same order per pair,
// same state machine — candidates are bit-identical to the lane sizer's (and the oracle's).  tools/proto/lockstep_sim.py
// and the measured counters (WVA_SIZER_DEBUG) give 88-92 % live lane-steps.
//
// Head rates: each lane of a batch computes its own pair's rates from the model's coefficients (RateTable,
// lockstep_solve.cuh) on the FP32 pipe, which the FP64-bound solvers leave idle; nothing is read per state.
#pragma once
#include "wva_core.cuh"
#include "sizer_kernel.cuh"
#include "lockstep_solve.cuh"

namespace wva {

constexpr int POOL_THREADS = 512;
constexpr int POOL_NCLS = 32;
constexpr int POOL_PMAX = 1024;       // slots per CTA (power of two: queue rings index with & (PMAX - 1))

struct alignas(16) PoolEntry {
  SizerLane z;
};

struct PoolSmem {
  unsigned short q[POOL_NCLS][POOL_PMAX];   // per class: ring of slots with a pending solve
  unsigned short free_list[POOL_PMAX];
  int head[POOL_NCLS], tail[POOL_NCLS];
  int n_free, in_pool, exhausted, lock;
};

__device__ __forceinline__ void pool_lock(int* lock) {
  if ((threadIdx.x & 31) == 0) {
    while (atomicCAS(lock, 0, 1) != 0) __nanosleep(32);
  }
  __syncwarp();
  __threadfence_block();
}
__device__ __forceinline__ void pool_unlock(int* lock) {
  __threadfence_block();
  __syncwarp();
  if ((threadIdx.x & 31) == 0) atomicExch(lock, 0);
}

// state of a pair <-> the pool (through L2: a slot is rewritten by whichever warp solved it last)
static_assert(sizeof(PoolEntry) % 16 == 0 && offsetof(PoolEntry, z) == 0 && offsetof(SizerLane, m) == 0,
              "PoolEntry is copied in 16-byte words, the model first");
constexpr int POOL_MODEL_WORDS = (int)((sizeof(PairModel) + 15) / 16);
__device__ __forceinline__ void pool_load(PoolEntry& z, const PoolEntry* e) {
  int4* dst = reinterpret_cast<int4*>(&z);
  const int4* src = reinterpret_cast<const int4*>(e);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(PoolEntry) / 16); k++) dst[k] = __ldcg(src + k);
}
__device__ __forceinline__ void pool_store(PoolEntry* e, const PoolEntry& z) {
  const int4* src = reinterpret_cast<const int4*>(&z);
  int4* dst = reinterpret_cast<int4*>(e);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(PoolEntry) / 16); k++) __stcg(dst + k, src[k]);
}
// what a solve needs of the pair: its queue model and the arrival rate (the rest is re-read after the solve, so that the
// solver's registers are not shared with 300 bytes of bisection state)
struct alignas(16) PoolModel { PairModel m; };
__device__ __forceinline__ float pool_load_model(PoolModel& pm, const PoolEntry* e) {
  int4* dst = reinterpret_cast<int4*>(&pm);
  const int4* src = reinterpret_cast<const int4*>(e);
#pragma unroll
  for (int k = 0; k < (int)(sizeof(PoolModel) / 16); k++) dst[k] = __ldcg(src + k);
  return __ldcg(reinterpret_cast<const float*>(reinterpret_cast<const char*>(e) + offsetof(SizerLane, cur_x)));
}

// Request classes: rings 0 .. POOL_FAST_NCLS - 1 hold solves for the certified fast solve (E12), the last POOL_EXACT_NCLS
// rings hold the solves it did not certify, which go to the exact lockstep_solve.
constexpr int POOL_EXACT_NCLS = 4;
constexpr int POOL_FAST_NCLS = POOL_NCLS - POOL_EXACT_NCLS;

// fast class of a solve: the fast solve visits at most the N - 1 head states whatever the rate (the tail is closed-form),
// so the class is that of N (4 per octave, N >= 3444 share the last one); pairs of one N land in one class and their
// batches take the uniform-N path
__device__ __forceinline__ int pool_class(const PairModel& m) {
  int c = (int)(__log2f(fmaxf((float)m.N, 32.0f) * (1.0f / 32.0f)) * 4.0f);
  return c < 0 ? 0 : (c >= POOL_FAST_NCLS ? POOL_FAST_NCLS - 1 : c);
}
// exact class of a solve at arrival rate x: the exact solver leaves the chain (E4) ~37.4 / -ln(x / mu_N) states after
// the head, at most at K; one class per two octaves of that length from 32 to 2048 and one above
__device__ __forceinline__ int pool_exact_class(const PairModel& m, float x) {
  float ratio = x / (float)m.mu_last;
  if (!(ratio > 1e-6f)) ratio = 1e-6f;
  if (ratio > 0.999999f) ratio = 0.999999f;
  const float est = fminf((float)m.N + 37.4f / -__logf(ratio), (float)m.K);
  const int c = (int)(__log2f(fmaxf(est, 32.0f) * (1.0f / 32.0f)) * 0.5f);
  return POOL_FAST_NCLS + (c >= POOL_EXACT_NCLS ? POOL_EXACT_NCLS - 1 : c);
}

// Phase profile (tools/perf_pool_phases.py): built with -DWVA_POOL_PHASES, every warp adds the clock64() cycles of each
// phase of its loop and counts its batches in shared memory, and the sums land in g_pool_phase (read by
// wva_pool_phases).  The product build compiles none of it.
#ifdef WVA_POOL_PHASES
enum {
  PH_LOCK, PH_NEW, PH_FAST, PH_EXACT, PH_STATE, PH_TOTAL,          // cycles: critical section, new pairs + BuildModel,
                                                                  // fast solves, exact solves, state machine, whole loop
  PH_FAST_BATCHES, PH_FAST_STATES, PH_FAST_SLOTS,                 // batches, live lane-steps, 32 x longest solve
  PH_EXACT_BATCHES, PH_EXACT_STATES, PH_EXACT_SLOTS,
  PH_FAST_PARTIAL, PH_EXACT_PARTIAL,                              // batches of fewer than 32 requests
  PH_ROWS, PH_ITERS,
  PH_MODEL,                                                       // cycles of fast batches: model load (pool_load_model),
  PH_FAST_WAIT0, PH_FAST_CHUNKS, PH_FAST_FINISH,                  // first table preparation, head chunks, fast_solve_finish
  PH_N
};
__device__ unsigned long long g_pool_phase[PH_N];
#define POOL_PH(...) __VA_ARGS__
#define POOL_PH_ADD(k, v) do { if (lane == 0) ph_acc[warp][k] += (unsigned long long)(v); } while (0)
#else
#define POOL_PH(...)
#define POOL_PH_ADD(k, v) do {} while (0)
#endif

// A pair with a service rate outside the (E1) divisor range never enters the queues: its lane runs every solve of the
// pair through the per-lane chain (chain_step: IEEE divisions by such a rate), a float64 overflow to the slow path as
// below.  Out of line: it is rare, and inlined it costs the batch loop registers.  Returns false (the pair is done).
__device__ __noinline__ bool pool_pair_on_chain(PoolEntry& ze, const SysView& s, const CandView& out, SizerCounters* ctr,
                                                int* overflow_list, unsigned long long& my_states) {
  SizerLane& z = ze.z;
  SolveStats st;
  bool live = true;
  while (live) {
    while (!chain_step(z.c, z.m, st)) {}
    if (z.c.phase == CH_OVERFLOW) {
      retire_overflow(z, s, out, ctr, overflow_list, z.c.states);
      live = false;
    } else {
      live = sizer_on_solve(z, s, out, st);
    }
  }
  my_states += z.states;
  return false;
}

__global__ void __launch_bounds__(POOL_THREADS, 1)
sizer_pool_kernel(SysView s, CandView out, unsigned long long n_pairs, int nmax, int P, PoolEntry* pool_all,
                  SizerCounters* ctr, int* overflow_list) {
  extern __shared__ __align__(16) unsigned char pool_smem_raw[];
  PoolSmem& sm = *reinterpret_cast<PoolSmem*>(pool_smem_raw);
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
#ifdef WVA_POOL_PHASES
  const int warp = threadIdx.x >> 5;
  __shared__ unsigned long long ph_acc[POOL_THREADS / 32][PH_N];
  for (int k = lane; k < PH_N; k += 32) ph_acc[warp][k] = 0;
  const long long ph_start = clock64();
#endif
  const unsigned lt = (1u << lane) - 1u;
  PoolEntry* pool = pool_all + (size_t)blockIdx.x * P;

  for (int i = threadIdx.x; i < P; i += POOL_THREADS) sm.free_list[i] = (unsigned short)(P - 1 - i);
  if (threadIdx.x < POOL_NCLS) { sm.head[threadIdx.x] = 0; sm.tail[threadIdx.x] = 0; }
  if (threadIdx.x == 0) { sm.n_free = P; sm.in_pool = 0; sm.exhausted = 0; sm.lock = 0; }
  __syncthreads();

  // produced by the previous iteration, handed to the queues at the start of the next one (one critical section each)
  int pushA = -1, clsA = 0;      // solved pair that needs another solve
  int pushB = -1, clsB = 0;      // new pair's first solve
  int freeA = -1, freeB = -1;    // slots to release
  unsigned long long my_solves = 0, my_states = 0, my_slots = 0;

  while (true) {
    int my_slot = -1, new_slot = -1;
    bool finished = false, exact = false;
    POOL_PH(long long ph_t = clock64();)
    pool_lock(&sm.lock);
    {
      // ---- release slots
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int fs = k ? freeB : freeA;
        const unsigned fm = __ballot_sync(full, fs >= 0);
        if (fm) {
          const int base = sm.n_free;
          if (fs >= 0) sm.free_list[base + __popc(fm & lt)] = (unsigned short)fs;
          __syncwarp();
          if (lane == 0) { sm.n_free = base + __popc(fm); sm.in_pool -= __popc(fm); }
          __syncwarp();
        }
      }
      // ---- enqueue requests, aggregated per class
#pragma unroll
      for (int k = 0; k < 2; k++) {
        const int ps = k ? pushB : pushA, pc = k ? clsB : clsA;
        unsigned pm = __ballot_sync(full, ps >= 0);
        while (pm) {
          const int c = __shfl_sync(full, pc, __ffs(pm) - 1);
          const unsigned peers = __ballot_sync(full, ps >= 0 && pc == c);
          const int t0 = sm.tail[c];
          if (ps >= 0 && pc == c) sm.q[c][(t0 + __popc(peers & lt)) & (POOL_PMAX - 1)] = (unsigned short)ps;
          __syncwarp();
          if (lane == 0) sm.tail[c] = t0 + __popc(peers);
          __syncwarp();
          pm &= ~peers;
        }
      }
      // ---- dequeue up to 32 requests: an exact class that holds a full batch (its requests hold slots), else the
      //      fullest fast class, then its fast neighbours (similar lengths); a partial exact batch only when no fast
      //      request is pending (that drain also lets the pool empty)
      static_assert(POOL_NCLS == 32, "one lane per class");
      const int cnt = sm.tail[lane] - sm.head[lane];
      const bool xcls = lane >= POOL_FAST_NCLS;
      const unsigned xfull = __ballot_sync(full, xcls && cnt >= 32);
      const int bestf = __reduce_max_sync(full, xcls ? 0 : (cnt << 5) | lane);
      const int bestx = __reduce_max_sync(full, xcls ? (cnt << 5) | lane : 0);
      int c0 = -1;
      if (xfull) c0 = __ffs(xfull) - 1;
      else if ((bestf >> 5) > 0) c0 = bestf & 31;
      else if ((bestx >> 5) > 0) c0 = bestx & 31;
      exact = c0 >= POOL_FAST_NCLS;
      int got = 0;
      if (c0 >= 0) {
        const int cmin = exact ? c0 : 0, cmax = exact ? c0 : POOL_FAST_NCLS - 1;   // an exact batch comes from one class
        for (int d = 0; d < (exact ? 1 : 2 * POOL_FAST_NCLS) && got < 32; d++) {
          const int c = (d & 1) ? c0 + ((d + 1) >> 1) : c0 - (d >> 1);     // c0, c0+1, c0-1, c0+2, ...
          if (c < cmin || c > cmax) continue;
          const int avail = __shfl_sync(full, cnt, c);
          if (avail <= 0) continue;
          const int take = min(avail, 32 - got);
          const int h = sm.head[c];
          if (lane >= got && lane < got + take) my_slot = sm.q[c][(h + lane - got) & (POOL_PMAX - 1)];
          __syncwarp();
          if (lane == 0) sm.head[c] = h + take;
          __syncwarp();
          got += take;
        }
      }
      // ---- reserve free slots for new pairs
      if (!sm.exhausted) {
        const int nf = min(32, sm.n_free);
        if (lane < nf) new_slot = sm.free_list[sm.n_free - 1 - lane];
        __syncwarp();
        if (lane == 0) { sm.n_free -= nf; sm.in_pool += nf; }
        __syncwarp();
      }
      finished = got == 0 && sm.exhausted && sm.in_pool == 0;
    }
    pool_unlock(&sm.lock);
    POOL_PH(POOL_PH_ADD(PH_LOCK, clock64() - ph_t); POOL_PH_ADD(PH_ITERS, 1); ph_t = clock64();)
    pushA = pushB = freeA = freeB = -1;
    if (finished) break;

    // ---- new pairs into the reserved slots: setup lane by lane (nil and zero-load pairs need no model), then
    //      BuildModel (queueanalyzer.go:95-124) with the whole warp, one pair's rates after the other
    if (__any_sync(full, new_slot >= 0)) {
      POOL_PH(const unsigned ph_new = __ballot_sync(full, new_slot >= 0); POOL_PH_ADD(PH_ROWS, __popc(ph_new));)
      PoolEntry ze;
      SizerLane& z = ze.z;
      bool need_table = false;
      if (new_slot >= 0) {
        while (true) {
          const unsigned long long pair = atomicAdd(&ctr->next_pair, 1ull);
          if (pair >= n_pairs) { sm.exhausted = 1; break; }
          const int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
          int lim = 0;
          const int rc = sizer_setup(z, s, out, srv, acc, nmax, &lim, true);
          if (lim) ctr->limit_hit = 1;
          if (rc == SETUP_NEEDS_TABLE) { need_table = true; break; }
        }
      }
      // each pair's rates: lane l computes entries l, l + 32, ... and keeps none of them; the rate range needs the first
      // and last entry, the monotone region the LAST descent !(row[n-1] <= row[n]) (where model_finish's scan from the
      // top stops): a max over n, and e1_ok whether every entry is an (E1) divisor: an and over n (model_finish checks
      // the entries below mono and the two ends of the non-decreasing rest, which bound every entry between them)
      float r0 = 0.0f, rl = 0.0f;
      int mono = 0, e1_ok = 0;
      unsigned need = __ballot_sync(full, need_table);
      while (need) {
        const int src = __ffs(need) - 1;
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
        float cur = 0.0f, carry = 0.0f, first = 0.0f;
        int desc = 0;
        bool e1 = true;
        for (int n0 = 0; n0 < b.N; n0 += 32) {
          const int n = n0 + lane;
          if (n < b.N) { cur = serv_rate(b, n + 1); e1 = e1 && e1_divisor(cur); }
          float prev = __shfl_up_sync(full, cur, 1);
          if (lane == 0) prev = carry;
          if (n > 0 && n < b.N && !(prev <= cur)) desc = n;
          carry = __shfl_sync(full, cur, 31);
          if (n0 == 0) first = __shfl_sync(full, cur, 0);
        }
        const float last = __shfl_sync(full, cur, (b.N - 1) & 31);
        desc = __reduce_max_sync(full, desc);
        const bool all_e1 = __all_sync(full, e1);
        if (lane == src) { r0 = first; rl = last; mono = desc; e1_ok = all_e1; }
      }
      bool live = false;
      if (need_table) {
        PairModel& m = z.m;
        m.tab = nullptr; m.stride = 0;
        model_set_range(m, r0, rl);
        m.mono = mono;
        m.e1_ok = e1_ok;
        m.mu_last = (double)rl;
        m.r_last = rcp_f32den(rl, m.mu_last);
        live = sizer_begin(z, s, out);
        // a service rate outside the (E1) divisor range: the whole pair here, on the per-lane chain (rare)
        if (live && !m.e1_ok) live = pool_pair_on_chain(ze, s, out, ctr, overflow_list, my_states);
        if (!live) my_solves += z.solves;
      }
      if (live) { pool_store(pool + new_slot, ze); pushB = new_slot; clsB = pool_class(z.m); }
      else if (new_slot >= 0) freeB = new_slot;
      __syncwarp();
    }
    POOL_PH(POOL_PH_ADD(PH_NEW, clock64() - ph_t); ph_t = clock64();)

    // ---- solve the dequeued requests in lock step, advance their pairs
    const bool live = my_slot >= 0;
    const unsigned live_mask = __ballot_sync(full, live);
    if (!live_mask) {
      if (!__any_sync(full, pushB >= 0 || freeB >= 0)) __nanosleep(256);     // other warps hold all the work
      continue;
    }
    PoolModel pm;
    float x = 0.0f;
    if (live) x = pool_load_model(pm, pool + my_slot);
    const int nref = __shfl_sync(full, pm.m.N, __ffs(live_mask) - 1);
    const bool uniform = __all_sync(full, !live || pm.m.N == nref);
    POOL_PH(if (!exact) POOL_PH_ADD(PH_MODEL, clock64() - ph_t);)
    bool bad = false, requeue = false;
    int sv = 0;
    SolveStats st;
    if (uniform) {
      if (!live) { pm.m.N = nref; pm.m.K = nref + nref * WVA_QUEUE_TO_BATCH; pm.m.mono = 0; pm.m.mu_last = 1.0; pm.m.r_last = 1.0; }
      const RateTable tt = live ? RateTable{rate_coef(pm.m)} : RateTable::idle();
      if (exact) {
        lockstep_solve(pm.m, tt, x, live, st, sv, bad);
      } else {
        sv = lockstep_solve_fast_only(pm.m, tt, x, live, st POOL_PH(, &ph_acc[warp][PH_FAST_WAIT0]));
        requeue = live && sv < 0;
        if (sv < 0) sv = -1 - sv;
      }
    }
#ifdef WVA_POOL_PHASES
    {
      int ls = live ? sv : 0, mxs = ls;
      for (int o = 16; o; o >>= 1) { ls += __shfl_xor_sync(full, ls, o); mxs = max(mxs, __shfl_xor_sync(full, mxs, o)); }
      if (uniform) {
        POOL_PH_ADD(exact ? PH_EXACT : PH_FAST, clock64() - ph_t);
        POOL_PH_ADD(exact ? PH_EXACT_BATCHES : PH_FAST_BATCHES, 1);
        POOL_PH_ADD(exact ? PH_EXACT_STATES : PH_FAST_STATES, ls);
        POOL_PH_ADD(exact ? PH_EXACT_SLOTS : PH_FAST_SLOTS, 32ull * mxs);
        POOL_PH_ADD(exact ? PH_EXACT_PARTIAL : PH_FAST_PARTIAL, live_mask != full);
      }
      ph_t = clock64();
    }
#endif
    if (requeue) {
      // not certified: the same solve goes to an exact class; its head states are kept in the pair's chain counter,
      // where the exact solve adds its own
      atomicAdd(&ctr->certify_fallbacks, 1ull);
      __stcg(&pool[my_slot].z.c.states, sv);
      pushA = my_slot; clsA = pool_exact_class(pm.m, x);
    } else if (live) {
      PoolEntry ze;
      SizerLane& z = ze.z;
      pool_load(ze, pool + my_slot);
      if (!uniform) {                                  // mixed N in the batch: the per-lane state machine
        const int s0 = z.c.states;
        while (!chain_step(z.c, z.m, st)) {}
        bad = z.c.phase == CH_OVERFLOW;
        sv = z.c.states - s0;
      } else {
        z.c.states = exact ? z.c.states + sv : sv;
      }
      bool cont;
      if (bad) {
        retire_overflow(z, s, out, ctr, overflow_list, z.c.states);
        cont = false;
      } else {
        cont = sizer_on_solve(z, s, out, st);
      }
      if (cont) { pool_store(pool + my_slot, ze); pushA = my_slot; clsA = pool_class(z.m); }
      else { my_solves += z.solves; my_states += z.states; freeA = my_slot; }
    }
    {
      int mxs = sv;
      for (int o = 16; o; o >>= 1) mxs = max(mxs, __shfl_xor_sync(full, mxs, o));
      if (lane == 0) my_slots += 32ull * (unsigned long long)mxs;
    }
    POOL_PH(POOL_PH_ADD(PH_STATE, clock64() - ph_t);)
  }
  for (int o = 16; o; o >>= 1) {
    my_solves += __shfl_down_sync(full, my_solves, o);
    my_states += __shfl_down_sync(full, my_states, o);
  }
  if (lane == 0) { atomicAdd(&ctr->solves, my_solves); atomicAdd(&ctr->states, my_states); atomicAdd(&ctr->lockstep_slots, my_slots); }
#ifdef WVA_POOL_PHASES
  POOL_PH_ADD(PH_TOTAL, clock64() - ph_start);
  __syncwarp();
  for (int k = lane; k < PH_N; k += 32) atomicAdd(&g_pool_phase[k], ph_acc[warp][k]);
#endif
}

}  // namespace wva
