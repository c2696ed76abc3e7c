// sizer_pool_kernel.cuh — System.Calculate for LARGE systems with the lock-step solver fed from a POOL of pairs.
//
// The lane sizer (sizer_lane_kernel.cuh) binds a pair to a lane for its whole life, so a lock-step round costs the
// longest of 32 chains that happen to sit in one warp: 49 % of the executed lane-steps do live work on BASELINE
// configs[2] (59-62 % with the probe-sorted queue).  Chain length is almost a function of lambda / mu_N alone (early exit
// E4), and it changes from one bisection step of a pair to the next — so here the binding is dropped:
//   * a CTA keeps a pool of P pairs whose state (the SizerLane of wva_core.cuh) and head-table rows live in global
//     memory (L2-resident: ~1.4 KB per pair at N = 256);
//   * every solve a pair still needs is a REQUEST — the pair's slot — queued in shared memory by length class
//     (32 log-spaced classes of the solve's cost; with the certified fast solve (E12) that is the head length N);
//   * a warp takes 32 requests from the fullest class (filling up from its neighbours), loads the 32 pairs' models,
//     solves them in lock step, advances each pair's bisection / Size / Analyze state machine (sizer_on_solve, the same
//     code as every other sizer), stores the state back and queues the pair's next request — or retires the pair and
//     frees its slot.  Free slots are refilled with new pairs from the global work counter.
// Which lanes solve which pairs together changes nothing in any pair's arithmetic: same solves, same order per pair,
// same state machine — candidates are bit-identical to the lane sizer's (and the oracle's).  tools/proto/lockstep_sim.py
// and the measured counters (WVA_SIZER_DEBUG) give 88-92 % live lane-steps.
//
// Head tables: one row per slot in global memory; 32 arbitrary rows are read through TileTable (lockstep_solve.cuh): the
// warp stages 32 states of its 32 rows per step, each row a coalesced 128-byte load.
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
  float tiles[POOL_THREADS / 32][2 * 32 * 33];
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

// length class of the solve at arrival rate x: the certified fast solve (E12) visits at most the N - 1 head states
// whatever the rate (the tail is closed-form), so the class is that of N; pairs of one N land in one class and their
// batches take the uniform-N path
__device__ __forceinline__ int pool_class(const PairModel& m, float x) {
  (void)x;
  const float est = (float)m.N;
  int c = (int)(__log2f(fmaxf(est, 32.0f) * (1.0f / 32.0f)) * 4.0f);
  return c < 0 ? 0 : (c >= POOL_NCLS ? POOL_NCLS - 1 : c);
}

__global__ void __launch_bounds__(POOL_THREADS, 1)
sizer_pool_kernel(SysView s, CandView out, unsigned long long n_pairs, int nmax, int P, PoolEntry* pool_all, float* rows_all,
                  int row_stride, SizerCounters* ctr, int* overflow_list) {
  extern __shared__ __align__(16) unsigned char pool_smem_raw[];
  PoolSmem& sm = *reinterpret_cast<PoolSmem*>(pool_smem_raw);
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  PoolEntry* pool = pool_all + (size_t)blockIdx.x * P;
  float* rows = rows_all + (size_t)blockIdx.x * P * row_stride;
  float* tile = sm.tiles[warp];

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
    bool finished = false;
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
      // ---- dequeue up to 32 requests: the fullest class, then its neighbours (similar lengths)
      const int cnt = lane < POOL_NCLS ? sm.tail[lane] - sm.head[lane] : 0;
      const int best = __reduce_max_sync(full, (cnt << 5) | lane);
      const int c0 = best & 31;
      int got = 0;
      if ((best >> 5) > 0) {
        for (int d = 0; d < 2 * POOL_NCLS && got < 32; d++) {
          const int c = (d & 1) ? c0 + ((d + 1) >> 1) : c0 - (d >> 1);     // c0, c0+1, c0-1, c0+2, ...
          if (c < 0 || c >= POOL_NCLS) continue;
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
    pushA = pushB = freeA = freeB = -1;
    if (finished) break;

    // ---- new pairs into the reserved slots (BuildModel: the lane fills its own row)
    if (__any_sync(full, new_slot >= 0)) {
      if (new_slot >= 0) {
        PoolEntry ze;
        SizerLane& z = ze.z;
        bool need_table = false;
        while (true) {
          const unsigned long long pair = atomicAdd(&ctr->next_pair, 1ull);
          if (pair >= n_pairs) { sm.exhausted = 1; break; }
          const int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
          int lim = 0;
          const int rc = sizer_setup(z, s, out, srv, acc, nmax, &lim, true);
          if (lim) ctr->limit_hit = 1;
          if (rc == SETUP_NEEDS_TABLE) { need_table = true; break; }
        }
        bool live = false;
        if (need_table) {
          // BuildModel (queueanalyzer.go:95-124) into the slot's row; the monotone region and the rate range are taken
          // from the values as they are produced (model_finish's scan from the top stops at the LAST descent)
          float* row = rows + (size_t)new_slot * row_stride;
          PairModel& m = z.m;
          m.tab = row; m.stride = 1;
          float r0 = 0.0f, prev = 0.0f;
          int mono = 0;
          for (int n = 0; n < m.N; n++) {
            const float cur = serv_rate(m, n + 1);
            __stcg(row + n, cur);
            if (n == 0) r0 = cur;
            else if (!(prev <= cur)) mono = n;
            prev = cur;
          }
          const float rl = prev;
          const float lmin = f_mul(r0, WVA_EPSILON), lmax = f_mul(rl, f_sub(1.0f, WVA_EPSILON));   // queueanalyzer.go:107-108
          const float rmin = f_mul(lmin, 1000.0f);
          m.rate_max = f_mul(lmax, 1000.0f);
          m.lambda_min = f_div(rmin, 1000.0f);                                                       // :189-190
          m.lambda_max = f_div(m.rate_max, 1000.0f);
          m.mono = mono;
          m.mu_last = (double)rl;
          m.r_last = rcp_f32den(rl, m.mu_last);
          live = sizer_begin(z, s, out);
          if (!live) my_solves += z.solves;
        }
        if (live) { pool_store(pool + new_slot, ze); pushB = new_slot; clsB = pool_class(z.m, z.cur_x); }
        else freeB = new_slot;
      }
      __syncwarp();
    }

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
    bool bad = false;
    int sv = 0;
    SolveStats st;
    if (uniform) {
      if (!live) { pm.m.N = nref; pm.m.K = nref + nref * WVA_QUEUE_TO_BATCH; pm.m.mono = 0; pm.m.mu_last = 1.0; pm.m.r_last = 1.0; }
      TileTable tt; tt.rows = rows; tt.row_stride = row_stride; tt.slot = live ? my_slot : 0; tt.tile = tile; tt.n_head = nref - 1;
      sv = lockstep_solve_fast(pm.m, tt, x, live, st, &ctr->certify_fallbacks);
      bad = sv < 0;
      if (bad) sv = -1 - sv;
    }
    if (live) {
      PoolEntry ze;
      SizerLane& z = ze.z;
      pool_load(ze, pool + my_slot);
      if (!uniform) {                                  // mixed N in the batch: the per-lane state machine
        while (!chain_step(z.c, z.m, st)) {}
        bad = z.c.phase == CH_OVERFLOW;
        sv = z.c.states;
      } else {
        z.c.states = sv;
      }
      bool cont;
      if (bad) {
        const unsigned long long k = atomicAdd(&ctr->overflow_pairs, 1ull);
        if (overflow_list) overflow_list[k] = z.srv * s.n_acc + z.acc;
        z.states += z.c.states;
        lane_fail(z, s, out);
        cont = false;
      } else {
        cont = sizer_on_solve(z, s, out, st);
      }
      if (cont) { pool_store(pool + my_slot, ze); pushA = my_slot; clsA = pool_class(z.m, z.cur_x); }
      else { my_solves += z.solves; my_states += z.states; freeA = my_slot; }
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

}  // namespace wva
