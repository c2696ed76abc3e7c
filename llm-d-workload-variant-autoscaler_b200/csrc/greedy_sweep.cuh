// greedy_sweep.cuh — Solver.SolveGreedy's allocate() (pkg/solver/greedy.go:107-166) as ONE sweep over a statically
// ordered list of candidate events.  (The literal queue — sorted array + re-insertion heap — stays in greedy_solve.cuh
// and is still used for systems this formulation does not cover; both produce the oracle's result bit for bit.)
//
// allocate() is a priority queue over entries, keyed by the entry's CURRENT candidate j:
//     k(e, j) = (priority asc, delta_j desc, value_j desc),   re-inserted BEFORE equal elements (greedy.go:161-162).
// Event (e, j) — "entry e is tested at its j-th candidate" — can only happen after (e, j-1) failed, and then it is
// popped at queue position  tau(e, j) = max_{i <= j} k(e, i): a re-inserted key that is not after the queue head is popped
// at once, so the event inherits the position of its predecessor.  tau depends on the entry alone.  Therefore all
// S x A potential events are sorted ONCE by tau (radix sort, parallel); what remains sequential is a sweep that keeps
// one "alive" bit per entry and the available units per type: an event whose entry is no longer alive is skipped, an
// alive one is dropped (no accelerator), taken (fits) or fails (its entry stays alive for its next event; after the last
// candidate it joins the unallocated list, greedy.go:152-156).  No heap, no per-bump search: the sweep streams 16-byte
// event records through shared memory (cp.async ring) and spends its dependent instructions only on alive events.
//
// Ties in tau are where the queue's LIFO rule shows: among the events of one tau, the runs led by a RE-INSERTED
// candidate (key == tau > tau of its predecessor) come first, most recent insertion first; then the runs led by an
// original entry (j == 0) in canonical (server index) order; the events of one entry with the same tau form a run that is
// processed back to back (every later one is popped "at once").  The static order puts re-inserted runs first in entry
// order, which is exact whenever at most one of them is alive when its tau is reached; where a tie group statically
// holds two or more re-inserted leaders (flag MULTI) the sweep collects the alive ones and orders them by the stamp of
// their predecessors' failure — the insertion time.  tools/proto/greedy_static_order.py is the executable form of this
// argument (checked against the oracle's literal sorted-slice algorithm, duplicates and zero-load ties included).
#pragma once
#include "greedy_solve.cuh"

namespace wva {

struct __align__(16) GEvent { int srv; unsigned meta; long long cnt; };   // meta = type (8, 0xff = none) | flags (8) | rank (16)
enum { GE_TIE = 1, GE_LEADER = 2, GE_CLS1 = 4, GE_LAST = 8, GE_NEWPRIO = 16, GE_MULTI = 32 };
__device__ __forceinline__ int ge_type(unsigned meta) { const int t = (int)(meta & 0xffu); return t == 0xff ? -1 : t; }
__device__ __forceinline__ unsigned ge_flags(unsigned meta) { return (meta >> 8) & 0xffu; }
__device__ __forceinline__ int ge_rank(unsigned meta) { return (int)(meta >> 16); }

constexpr int GSW_BLOCK = 512;            // events per ring slot (8 KB)
constexpr int GSW_AVAIL = 64;             // capacity types (WVA_MAX_TYPES)

struct GSweepWs {
  // dense, indexed (server, rank): tau components and flags of every potential event
  unsigned* t_kd; unsigned* t_kv; unsigned char* fl; unsigned char* valid;
  // compaction + sort
  unsigned* idxA; unsigned* idxB; unsigned* keyA; unsigned* keyB; int* n_events;
  // sorted events
  GEvent* ev;
  int* stamp;        // [S] clock of the entry's last failure
  int* dyn_pos; int* dyn_stamp;   // [S] scratch of the tie-group procedure
  unsigned long long* blk_min;    // [n_blocks + 1][n_types] smallest unit count among the events of type t at or after the block
  // the head of the list (gsw_head_kernel): units of type t wanted by the first candidates (rank 0) in a block, then
  // the exclusive prefix of those sums over the blocks
  long long* blk_sum;             // [n_blocks + 1][n_types]
  long long* head_used;           // [n_types] units the committed head takes from each type
  unsigned* head_alive;           // [(S + 31) / 32] alive bits after the head
  // [0] first block some type runs out in, [1] first block the sweep's nothing-fits check stops at (both per type, then
  // min / max over the types), [2] P: first failure, [3] C: end of the head (events [0, C) are committed in parallel)
  int* head;
  unsigned long long* head_events;   // first candidates committed (the sweep's n_active at C)
};

// tau, run class and flags of every (server, rank); after greedy_prepare_kernel
__global__ void __launch_bounds__(128) gsw_events_kernel(SysView s, GreedyWs w, GSweepWs g) {
  const int srv = blockIdx.x * blockDim.x + threadIdx.x;
  if (srv >= s.n_servers) return;
  const int A = s.n_acc;
  const size_t p = (size_t)srv * A;
  const int n = w.ncand[srv];
  unsigned tkd = 0, tkv = 0;
  int cls = 1;
  for (int j = 0; j < n; j++) {
    const unsigned kd = w.r_kd[p + j], kv = w.r_kv[p + j];
    const bool leader = j == 0 || kd > tkd || (kd == tkd && kv > tkv);
    if (leader) { tkd = kd; tkv = kv; cls = j == 0 ? 1 : 0; }
    g.t_kd[p + j] = tkd; g.t_kv[p + j] = tkv;
    g.fl[p + j] = (unsigned char)((leader ? GE_LEADER : 0) | (cls ? GE_CLS1 : 0) | (j == n - 1 ? GE_LAST : 0));
    g.valid[p + j] = 1;
  }
  for (int j = n; j < A; j++) g.valid[p + j] = 0;
  g.stamp[srv] = 0;
  if ((srv & 31) == 0) g.head_alive[srv >> 5] = ~0u;
  if (srv == 0) {
    for (int t = 0; t < s.n_types; t++) g.head_used[t] = 0;
    g.head[0] = INT_MAX; g.head[1] = 0; g.head[2] = 0; g.head[3] = 0; *g.head_events = 0;
  }
}

// one LSD radix pass over the compacted events: which = 0 run class (re-inserted first), 1 tau value, 2 tau delta, 3 priority
__global__ void __launch_bounds__(256) gsw_keys_kernel(SysView s, GSweepWs g, const unsigned* idx, int n, int which, unsigned* keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned p = idx[i];
  if (which == 0) keys[i] = (g.fl[p] & GE_CLS1) ? 1u : 0u;
  else if (which == 1) keys[i] = g.t_kv[p];
  else if (which == 2) keys[i] = g.t_kd[p];
  else keys[i] = (unsigned)s.srv_priority[p / (unsigned)s.n_acc] ^ 0x80000000u;
}

// sorted order -> 16-byte event records with the tie / priority-boundary flags
__global__ void __launch_bounds__(256) gsw_gather_kernel(SysView s, GreedyWs w, GSweepWs g, const unsigned* idx, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned A = (unsigned)s.n_acc;
  const unsigned p = idx[i];
  const int srv = (int)(p / A), j = (int)(p % A);
  unsigned flags = g.fl[p];
  if (i == 0) flags |= GE_NEWPRIO;
  else {
    const unsigned q = idx[i - 1];
    const int psrv = (int)(q / A);
    const bool same_prio = s.srv_priority[psrv] == s.srv_priority[srv];
    if (!same_prio) flags |= GE_NEWPRIO;
    else if (g.t_kd[q] == g.t_kd[p] && g.t_kv[q] == g.t_kv[p]) flags |= GE_TIE;
  }
  const int ty = w.r_type[p];
  GEvent e;
  e.srv = srv;
  e.meta = (unsigned)(ty < 0 ? 0xff : ty) | (flags << 8) | ((unsigned)j << 16);
  e.cnt = (long long)w.r_nrep[p] * w.r_upr[p];
  g.ev[i] = e;
  if (ty >= 0) {
    const size_t r = (size_t)(i / GSW_BLOCK) * s.n_types + ty;
    atomicMin(&g.blk_min[r], (unsigned long long)e.cnt);
    if (j == 0) atomicAdd(reinterpret_cast<unsigned long long*>(&g.blk_sum[r]), (unsigned long long)e.cnt);
  }
}

// suffix minima over the blocks: one warp per type, 32 blocks per step (warp suffix scan + carry)
__global__ void __launch_bounds__(32) gsw_sufmin_kernel(GSweepWs g, int n_blocks, int n_types) {
  const int t = blockIdx.x, lane = threadIdx.x;
  if (t >= n_types) return;
  unsigned long long carry = ~0ull;
  for (int hi = n_blocks; hi > 0; hi -= 32) {
    const int b = hi - 1 - lane;                         // lane 0 holds the LAST block of the step
    unsigned long long v = b >= 0 ? g.blk_min[(size_t)b * n_types + t] : ~0ull;
    for (int o = 1; o < 32; o <<= 1) {                   // inclusive scan towards higher lanes = towards lower blocks
      const unsigned long long u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o && u < v) v = u;
    }
    if (carry < v) v = carry;
    if (b >= 0) g.blk_min[(size_t)b * n_types + t] = v;
    carry = __shfl_sync(0xffffffffu, v, 31);
  }
}

// The head of the list.  Event (e, j >= 1) can only be alive after (e, j-1) failed, and a failure needs avail[t] < cnt;
// so up to the first failure P every alive event is an entry's first candidate (rank 0), taken or — no accelerator —
// dropped, and every other event is dead.  Before P no stamp is drawn (the clock stays 0), no entry is unallocated and
// no MULTI leader is alive (MULTI marks re-inserted leaders only, rank >= 1), so a priority boundary runs bestEffort on
// an empty list.  The only state the head passes on is the units it takes from each type: P is the first event of rank 0
// and type t >= 0 at which the running sum of those units over the list's rank-0 events of type t exceeds the capacity.
// The sweep's nothing-fits check (per block, against the capacities at the block's first event) can also stop the
// sweep before P; the head ends at C = min(P, the first block start where that check stops it), the sweep starts at C
// with the state the sequential sweep had there, and checks the blocks from C's on as it always did.  (Unit counts
// are >= 0, as the check's unsigned block minima already assume: the running sums only grow.)

// per type, one warp, 32 blocks per step: blk_sum -> exclusive prefix over the blocks; the first block in which the type
// runs out (head[0], min over the types) and the first block whose nothing-fits check finds no event of the type that
// fits, assuming nothing failed before it (head[1], max over the types: the check stops where every type is past it;
// before P both terms only move one way, so "nothing fits at block b" is "b >= every type's block")
__global__ void __launch_bounds__(32) gsw_prefix_kernel(SysView s, GSweepWs g, int n_blocks) {
  const unsigned full = 0xffffffffu;
  const int t = blockIdx.x, lane = threadIdx.x, T = s.n_types;
  if (t >= T) return;
  const long long cap = s.type_count[t];
  long long carry = 0;
  int out = INT_MAX, stop = n_blocks;
  for (int b0 = 0; b0 < n_blocks; b0 += 32) {
    const int b = b0 + lane;
    const size_t r = (size_t)b * T + t;
    const long long v = b < n_blocks ? g.blk_sum[r] : 0;
    long long incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const long long u = __shfl_up_sync(full, incl, o);
      if (lane >= o) incl += u;
    }
    incl += carry;
    bool can = true;
    if (b < n_blocks) {
      const long long left = cap - (incl - v);      // the sweep's avail[t] at the block's first event
      const unsigned long long m = g.blk_min[r];
      can = m != ~0ull && left >= 0 && (unsigned long long)left >= m;
      g.blk_sum[r] = incl - v;
    }
    const unsigned runs = __ballot_sync(full, b < n_blocks && incl > cap), cant = __ballot_sync(full, !can);
    if (runs && out == INT_MAX) out = b0 + __ffs(runs) - 1;
    if (cant && stop == n_blocks) stop = b0 + __ffs(cant) - 1;
    carry = __shfl_sync(full, incl, 31);
  }
  if (lane == 0) {
    if (out != INT_MAX) atomicMin(&g.head[0], out);
    atomicMax(&g.head[1], stop);
  }
}

// adds the units of the rank-0 events in [i0, end) (one block at most) to used[type], in order, 32 per step; returns
// the first of them that does not fit (end if all do)
__device__ __forceinline__ int gsw_head_walk(const SysView& s, const GSweepWs& g, long long* used, int i0, int end) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  for (int b0 = i0; b0 < end; b0 += 32) {
    const int i = b0 + lane;
    int ty = -1;
    long long c = 0;
    if (i < end) {
      const GEvent e = g.ev[i];
      if (ge_rank(e.meta) == 0) { ty = ge_type(e.meta); c = e.cnt; }
    }
    long long acc = 0;                               // units of this type in the step, up to and including this lane
    for (int k = 0; k < 32; k++) {
      const int tk = __shfl_sync(full, ty, k);
      const long long ck = __shfl_sync(full, c, k);
      if (k <= lane && tk == ty) acc += ck;
    }
    const unsigned fm = __ballot_sync(full, ty >= 0 && used[ty] + acc > s.type_count[ty]);
    if (fm) return b0 + __ffs(fm) - 1;
    const unsigned later = __match_any_sync(full, ty) & ~((2u << lane) - 1u);
    __syncwarp();
    if (ty >= 0 && !later) used[ty] += acc;
    __syncwarp();
  }
  return end;
}

// P and C (head[2], head[3]) and the units the head takes from each type
__global__ void __launch_bounds__(32) gsw_head_kernel(SysView s, GSweepWs g, int n) {
  __shared__ long long used[GSW_AVAIL];
  const int lane = threadIdx.x, T = s.n_types;
  const int fb = g.head[0];
  int P = n;
  if (fb != INT_MAX) {
    for (int t = lane; t < T; t += 32) used[t] = g.blk_sum[(size_t)fb * T + t];
    __syncwarp();
    P = gsw_head_walk(s, g, used, fb * GSW_BLOCK, min(n, (fb + 1) * GSW_BLOCK));
    __syncwarp();
  }
  const int C = min(P, min(g.head[1] * GSW_BLOCK, n)), cb = C / GSW_BLOCK;
  for (int t = lane; t < T; t += 32) used[t] = g.blk_sum[(size_t)cb * T + t];
  __syncwarp();
  gsw_head_walk(s, g, used, cb * GSW_BLOCK, C);
  __syncwarp();
  for (int t = lane; t < T; t += 32) g.head_used[t] = used[t];
  if (lane == 0) { g.head[2] = P; g.head[3] = C; }
}

// the head, in parallel: every rank-0 event before C is taken (type >= 0) or dropped, and its entry leaves the queue
__global__ void __launch_bounds__(256) gsw_commit_kernel(GreedyWs w, GSweepWs g, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool first = false;
  if (i < n && i < g.head[3]) {
    const GEvent e = g.ev[i];
    if (ge_rank(e.meta) == 0) {
      first = true;
      if (ge_type(e.meta) >= 0) { w.kind[e.srv] = 1; w.sel_rank[e.srv] = 0; }   // greedy.go:143-145
      atomicAnd(&g.head_alive[e.srv >> 5], ~(1u << (e.srv & 31)));
    }
  }
  const int k = __syncthreads_count(first);
  if (threadIdx.x == 0 && k) atomicAdd(g.head_events, (unsigned long long)k);
}

// MULTI: the event leads a re-inserted run and its tie group holds another re-inserted leader.  Bounded walks; when a
// walk does not reach the end of the group's re-inserted part the flag is set (conservative: the sweep's tie-group
// procedure is exact for any number of alive leaders, including one).
__global__ void __launch_bounds__(256) gsw_multi_kernel(GSweepWs g, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned m = g.ev[i].meta;
  const unsigned f = ge_flags(m);
  if (!(f & GE_LEADER) || (f & GE_CLS1)) return;
  bool multi = false, open = false;
  // forward: the re-inserted part continues while TIE && !CLS1
  int k = i + 1, steps = 0;
  for (; k < n && steps < 64; k++, steps++) {
    const unsigned fk = ge_flags(g.ev[k].meta);
    if (!(fk & GE_TIE) || (fk & GE_CLS1)) break;
    if (fk & GE_LEADER) { multi = true; break; }
  }
  if (!multi && steps == 64) open = true;
  // backward: events before i belong to the same part while THIS side's TIE flag is set
  if (!multi) {
    int b = i; steps = 0;
    while (b > 0 && (ge_flags(g.ev[b].meta) & GE_TIE) && steps < 64) {
      b--; steps++;
      const unsigned fb = ge_flags(g.ev[b].meta);
      if (fb & GE_CLS1) break;                       // cannot happen (re-inserted runs come first), kept for safety
      if (fb & GE_LEADER) { multi = true; break; }
    }
    if (!multi && steps == 64) open = true;
  }
  if (multi || open) g.ev[i].meta = m | ((unsigned)GE_MULTI << 8);
}

// cycle counters of the sweep's phases (debug line of run_solve_greedy_sweep): compiled in with -DWVA_SWEEP_PROFILE only —
// the reads themselves cost ~10 % of the kernel
#ifdef WVA_SWEEP_PROFILE
#define GSW_CLK() clock64()
#else
#define GSW_CLK() 0ll
#endif
constexpr int GSW_SLOTS = 4;
constexpr int GSW_ALIVE_WORDS = 36 * 1024; // alive bits for up to 1 179 648 entries in shared memory (144 KB)
constexpr int GSW_TIE_CAP = 1024;          // events of a tie group staged in shared memory at a time
constexpr int GSW_DYN_CAP = 4096;          // alive leaders of a tie group ordered in shared memory (more: global-memory path)
constexpr int GSW_RUN_SLOTS = 8;           // runs of a tie group in flight (32 events each, in the staging area)
constexpr size_t GSW_SMEM = (size_t)GSW_BLOCK * GSW_SLOTS * sizeof(GEvent) + (size_t)GSW_ALIVE_WORDS * 4 + GSW_AVAIL * 8 +
                            (size_t)GSW_TIE_CAP * sizeof(GEvent) + (size_t)GSW_DYN_CAP * 8;

__device__ __forceinline__ void gsw_cp16(void* dst_smem, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void gsw_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void gsw_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Sweep state: plain values (kept in registers: nothing here has its address taken across a call)
struct GSweepState { int n_un, clock; long long n_active; long long d_fb, d_nact, d_maxact, d_fbev; };

__device__ __forceinline__ bool gsw_alive(const unsigned* alive, int srv) { return (alive[srv >> 5] >> (srv & 31)) & 1u; }
__device__ __forceinline__ void gsw_kill(unsigned* alive, int srv) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) alive[srv >> 5] &= ~(1u << (srv & 31));
  __syncwarp();
}
// one alive event, sequentially (greedy.go:120-165); every lane holds the same arguments.  True when the entry left the queue.
__device__ __forceinline__ bool gsw_process(const GreedyWs& w, const GSweepWs& g, long long* avail, unsigned* alive, GSweepState& z,
                                            int srv, unsigned meta, long long cnt) {
  const bool writer = (threadIdx.x & 31) == 0;
  z.n_active++;
  const int type = ge_type(meta);
  if (type < 0) { gsw_kill(alive, srv); return true; }                         // no accelerator: dropped (:126-136)
  if (avail[type] >= cnt) {                                                      // :143-145
    __syncwarp();
    if (writer) { avail[type] -= cnt; w.kind[srv] = 1; w.sel_rank[srv] = ge_rank(meta); }
    gsw_kill(alive, srv);
    return true;
  }
  z.clock++;
  if (writer) g.stamp[srv] = z.clock;                                            // when the next candidate is (re-)inserted
  if (ge_flags(meta) & GE_LAST) {                                                // :152-156
    if (writer) w.unalloc[z.n_un] = srv;
    z.n_un++;
    gsw_kill(alive, srv);
    return true;
  }
  return false;
}

// The re-inserted part of a tie group with several statically possible leaders, entered at its first ALIVE leader i0:
// collect the alive leaders, process their runs latest-insertion first.  Returns the position after the part, or -1 when
// i0 is the only alive leader (the caller then processes it in the normal flow).
__device__ __forceinline__ int gsw_tie_group(const GreedyWs& w, const GSweepWs& g, long long* avail, unsigned* alive,
                                             GSweepState& z, int i0, int n_ev) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  int n_act = 0, i = i0;
  __threadfence_block();           // the stamps written by other lanes of this warp are read below
  __syncwarp();
  while (true) {
    const int idx = i + lane;
    const bool v = idx < n_ev;
    unsigned m = 0; int sv = 0;
    if (v) { const GEvent e = g.ev[idx]; m = e.meta; sv = e.srv; }
    const unsigned f = ge_flags(m);
    const bool in_part = v && (idx == i0 || (f & GE_TIE)) && !(f & GE_CLS1);
    const unsigned stop = __ballot_sync(full, !in_part);
    const int nin = stop ? __ffs(stop) - 1 : 32;
    const bool is_cand = lane < nin && (f & GE_LEADER) && gsw_alive(alive, sv);
    const unsigned cm = __ballot_sync(full, is_cand);
    if (is_cand) {
      const int slot = n_act + __popc(cm & ((1u << lane) - 1u));
      g.dyn_pos[slot] = idx;
      g.dyn_stamp[slot] = *((volatile int*)&g.stamp[sv]);
    }
    n_act += __popc(cm);
    i += nin;
    if (nin < 32) break;
  }
  const int end_pos = i;
  z.d_nact += n_act; if (n_act > z.d_maxact) z.d_maxact = n_act;
  if (n_act <= 1) return -1;
  __syncwarp();
  __threadfence_block();
  for (int k = 0; k < n_act; k++) {
    // latest insertion first: arg-max of the remaining stamps (stamps are distinct clock values > 0)
    int best = -1, best_slot = -1;
    for (int q = lane; q < n_act; q += 32) {
      const int st = *((volatile int*)&g.dyn_stamp[q]);
      if (st > best) { best = st; best_slot = q; }
    }
    for (int o = 16; o; o >>= 1) {
      const int ob = __shfl_xor_sync(full, best, o), os = __shfl_xor_sync(full, best_slot, o);
      if (ob > best) { best = ob; best_slot = os; }
    }
    __syncwarp();
    if (lane == 0) g.dyn_stamp[best_slot] = -1;
    __threadfence_block();
    __syncwarp();
    int r = *((volatile int*)&g.dyn_pos[best_slot]);
    const int srv0 = g.ev[r].srv;
    for (int first = r; r < end_pos; r++) {
      const GEvent e = g.ev[r];
      if (r > first && (e.srv != srv0 || !(ge_flags(e.meta) & GE_TIE))) break;
      if (gsw_process(w, g, avail, alive, z, e.srv, e.meta, e.cnt)) break;
    }
    __syncwarp();
  }
  return end_pos;
}

// The same with the event list streamed through shared memory.  (1) The part is scanned in chunks of GSW_TIE_CAP events
// (cp.async, a whole chunk in flight) and its alive leaders collected; (2) their stamps are fetched lane-parallel and the
// leaders sorted latest insertion first (bitonic, shared memory); (3) the runs are processed in that order, 32 events per
// step, each run prefetched GSW_RUN_SLOTS - 1 runs ahead.  Returns -2 (nothing changed) when the part holds more than
// GSW_DYN_CAP alive leaders: the caller then takes the global-memory path above.
__device__ __forceinline__ int gsw_tie_group_staged(const GreedyWs& w, const GSweepWs& g, long long* avail, unsigned* alive,
                                                    GSweepState& z, int i0, int n_ev, GEvent* tev, int2* dyn) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  __threadfence_block();           // the stamps written by other lanes of this warp are read below
  __syncwarp();
  int scanned = 0, n_part = 0, n_act = 0, chunk = 256;
  bool ended = false;
  while (!ended) {
    const int cnt = min(chunk, n_ev - (i0 + scanned));
    if (cnt <= 0) break;
    for (int k = lane; k < cnt; k += 32) gsw_cp16(tev + k, g.ev + i0 + scanned + k);
    gsw_commit();
    gsw_wait<0>();
    __syncwarp();
    for (int base = 0; base < cnt && !ended; base += 32) {
      const int k = base + lane;
      const bool v = k < cnt;
      unsigned m = 0; int sv = 0;
      if (v) { m = tev[k].meta; sv = tev[k].srv; }
      const unsigned f = ge_flags(m);
      const bool in_part = v && (scanned + k == 0 || (f & GE_TIE)) && !(f & GE_CLS1);
      const unsigned stop = __ballot_sync(full, !in_part);
      const int nin = stop ? __ffs(stop) - 1 : 32;
      const bool is_cand = lane < nin && (f & GE_LEADER) && gsw_alive(alive, sv);
      const unsigned cm = __ballot_sync(full, is_cand);
      if (n_act + __popc(cm) > GSW_DYN_CAP) return -2;
      if (is_cand) dyn[n_act + __popc(cm & ((1u << lane) - 1u))] = make_int2(sv, i0 + scanned + k);
      n_act += __popc(cm);
      n_part = scanned + base + nin;
      if (nin < 32) ended = true;
    }
    __syncwarp();                  // the chunk is overwritten next
    scanned += cnt;
    chunk = GSW_TIE_CAP;
  }
  const int end_pos = i0 + n_part;
  z.d_nact += n_act; if (n_act > z.d_maxact) z.d_maxact = n_act;
  if (scanned > GSW_TIE_CAP) { z.d_fb++; z.d_fbev += n_part; }
  if (n_act <= 1) return -1;
  // (2) stamps (distinct clock values > 0), then descending order; the padding (-1) sorts last
  int n2 = 32;
  while (n2 < n_act) n2 <<= 1;
  __syncwarp();
#pragma unroll 4
  for (int q = lane; q < n2; q += 32) dyn[q].x = q < n_act ? *((volatile int*)&g.stamp[dyn[q].x]) : -1;
  __syncwarp();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n2; i += 32) {
        const int l = i ^ j;
        if (l > i) {
          const int2 a = dyn[i], b = dyn[l];
          if (((i & k) == 0) ? (a.x < b.x) : (a.x > b.x)) { dyn[i] = b; dyn[l] = a; }
        }
      }
      __syncwarp();
    }
  // (3) the runs.  Slot (it % GSW_RUN_SLOTS) of the staging area holds the first 32 events of run `it`.
  auto issue = [&](int it) {
    if (it < n_act) {
      const int p = dyn[it].y + lane;
      if (p < end_pos) gsw_cp16(tev + (it % GSW_RUN_SLOTS) * 32 + lane, g.ev + p);
    }
    gsw_commit();
  };
  for (int it = 0; it < GSW_RUN_SLOTS - 1; it++) issue(it);
  for (int it = 0; it < n_act; it++) {
    issue(it + GSW_RUN_SLOTS - 1);
    gsw_wait<GSW_RUN_SLOTS - 1>();
    __syncwarp();
    // the leader's run, 32 events per step: the events before the first one that fits (or has no accelerator) fail —
    // each failure re-inserts the entry in front of the queue (same tau, latest insertion) — and the run ends there, at
    // the entry's last candidate, or at the end of its events in this tie group (gsw_process, event by event)
    const int k0 = dyn[it].y;
    int srv0 = 0;
    bool done = false;
    for (int base = k0; base < end_pos && !done; base += 32) {
      const int k = base + lane;
      GEvent e; e.srv = -1; e.meta = 0; e.cnt = 0;
      if (k < end_pos) e = base == k0 ? tev[(it % GSW_RUN_SLOTS) * 32 + lane] : g.ev[k];
      if (base == k0) srv0 = __shfl_sync(full, e.srv, 0);
      const unsigned f = ge_flags(e.meta);
      const bool inrun = k < end_pos && (k == k0 || (e.srv == srv0 && (f & GE_TIE)));
      const unsigned stopm = __ballot_sync(full, !inrun);
      const int nrun = stopm ? __ffs(stopm) - 1 : 32;
      const int type = ge_type(e.meta);
      const bool mine = lane < nrun;
      const unsigned tm = __ballot_sync(full, mine && (type < 0 || avail[type < 0 ? 0 : type] >= e.cnt));
      const int F = tm ? __ffs(tm) - 1 : nrun;       // lanes below F fail
      const unsigned lastm = __ballot_sync(full, mine && lane < F && (f & GE_LAST));
      __syncwarp();
      z.n_active += F + (tm ? 1 : 0);
      z.clock += F;
      if (tm) {
        if (lane == F) {
          if (type >= 0) { avail[type] -= e.cnt; w.kind[srv0] = 1; w.sel_rank[srv0] = ge_rank(e.meta); }   // greedy.go:143-145
          alive[srv0 >> 5] &= ~(1u << (srv0 & 31));                                                           // (or dropped, :126-136)
        }
        done = true;
      } else if (lastm) {                            // :152-156
        if (lane == 0) { w.unalloc[z.n_un] = srv0; alive[srv0 >> 5] &= ~(1u << (srv0 & 31)); }
        z.n_un++;
        done = true;
      } else {
        if (lane == 0 && F > 0) g.stamp[srv0] = z.clock;
        if (nrun < 32) done = true;
      }
      __syncwarp();
    }
  }
  gsw_wait<0>();
  __syncwarp();
  return end_pos;
}

__global__ void __launch_bounds__(32, 1) gsw_sweep_kernel(SysView s, GreedyWs w, GSweepWs g, int delayed, int policy) {
  extern __shared__ __align__(16) unsigned char gsw_smem[];
  GEvent* ring = reinterpret_cast<GEvent*>(gsw_smem);
  unsigned* alive = reinterpret_cast<unsigned*>(gsw_smem + (size_t)GSW_BLOCK * GSW_SLOTS * sizeof(GEvent));
  long long* avail = reinterpret_cast<long long*>(alive + GSW_ALIVE_WORDS);
  GEvent* tie_ev = reinterpret_cast<GEvent*>(avail + GSW_AVAIL);
  int2* tie_dyn = reinterpret_cast<int2*>(tie_ev + GSW_TIE_CAP);
  // bestEffort never runs inside a tie group: its staging area is the tie group's (32 x G_STAGE_A x 16 B = GSW_TIE_CAP x 16 B)
  static_assert(32 * G_STAGE_A * 16 <= GSW_TIE_CAP * (int)sizeof(GEvent), "bestEffort staging");
  GStage be_stage;
  be_stage.upr = reinterpret_cast<long long*>(tie_ev);
  be_stage.type = reinterpret_cast<int*>(be_stage.upr + 32 * G_STAGE_A);
  be_stage.nrep = be_stage.type + 32 * G_STAGE_A;
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  const int n_ev = *g.n_events;
  const int S = s.n_servers;
  // the sweep starts where the head (gsw_commit_kernel) ends, in the state the sequential sweep had there
  const int head_end = g.head[3];
  for (int t = lane; t < GSW_AVAIL; t += 32) avail[t] = t < s.n_types ? s.type_count[t] - g.head_used[t] : 0;   // greedy.go:38-39
  for (int k = lane; k < (S + 31) / 32; k += 32) alive[k] = g.head_alive[k];
  __syncwarp();
  GSweepState z = {0, 0, (long long)*g.head_events, 0, 0, 0, 0};
  int group_un0 = 0;
  long long n_batches = 0, n_rounds = 0, n_seq = 0, n_tie = 0, cyc_be = 0, cyc_tie = 0, n_unalloc_be = 0;
  long long n_tie_global = 0, n_restart = 0;   // tie groups ordered in global memory; event streams restarted after a jump
  const long long cyc0 = GSW_CLK();

  // event stream: blocks of GSW_BLOCK records copied asynchronously into a ring of GSW_SLOTS slots; while block b is
  // read, blocks b+1 .. b+GSW_SLOTS-1 are in flight.  One commit group per block (empty past the end of the list).
  // The stream starts at the block of the head's end, so that the batches from the next block on (and the block checks)
  // fall where they fell in a sweep from event 0.  A head that ends inside a block stopped at P, after that block's
  // nothing-fits check had passed at its first event (gsw_head_kernel): the check is not repeated.
  int origin = head_end - head_end % GSW_BLOCK;   // event index of block 0 of the current stream (moves only after a far tie-group jump)
  int issued = 0;               // blocks of the current stream whose copies have been issued
  int cur_block = -1;
  int pos = head_end;
  int checked_blk = head_end % GSW_BLOCK ? head_end / GSW_BLOCK : -1;
  bool nothing_fits = false;
  int pf_blk = -1;
  unsigned long long pf0 = ~0ull, pf1 = ~0ull;
  long long n_survivors = -1, n_skip128 = 0;
  long long cyc_ring = 0, cyc_dead = 0, cyc_fast = 0, cyc_slow = 0, cyc_chk = 0;
  while (pos < n_ev) {
    const long long tc0 = GSW_CLK();
    // Once no remaining event of any type can fit (capacities only shrink, greedy.go:143-145; bestEffort only takes),
    // every entry still in the queue ends unallocated.  Policy None (bestEffort is a no-op): stop.  The other policies:
    // what is left of the sweep only fixes the ORDER of the unallocated list, and bestEffort gives nothing to an entry
    // none of whose candidates sits on a type with room for one replica of anything (g_live_types) whatever its place
    // in the list — those entries leave the queue here; the rest are swept on, in exactly the reference's order (the
    // relative order of insertion stamps does not depend on the entries removed; the unallocated list is sorted by
    // priority, so removing entries cannot merge two priority groups of makePriorityGroups, greedy.go:321-341).
    if (!nothing_fits && pos / GSW_BLOCK != checked_blk) {
      checked_blk = pos / GSW_BLOCK;
      // (the row of the NEXT block is fetched now and used at the next check: no load is consumed where it is issued;
      //  n_types <= GSW_AVAIL = 64: two values per lane)
      const int T = s.n_types;
      unsigned long long m0, m1;
      if (pf_blk == checked_blk) { m0 = pf0; m1 = pf1; }
      else {
        m0 = lane < T ? g.blk_min[(size_t)checked_blk * T + lane] : ~0ull;
        m1 = lane + 32 < T ? g.blk_min[(size_t)checked_blk * T + lane + 32] : ~0ull;
      }
      pf_blk = checked_blk + 1;
      if (pf_blk <= n_ev / GSW_BLOCK) {
        pf0 = lane < T ? g.blk_min[(size_t)pf_blk * T + lane] : ~0ull;
        pf1 = lane + 32 < T ? g.blk_min[(size_t)pf_blk * T + lane + 32] : ~0ull;
      } else pf_blk = -1;
      const bool can = (m0 != ~0ull && avail[lane] >= 0 && (unsigned long long)avail[lane] >= m0) ||
                       (m1 != ~0ull && avail[lane + 32] >= 0 && (unsigned long long)avail[lane + 32] >= m1);
      if (!__any_sync(full, can)) {
        if (policy == 0) break;
        nothing_fits = true;
        const long long mu_lo = lane < s.n_types ? w.min_upr[lane] : 0, mu_hi = (lane + 32 < s.n_types && lane + 32 < 64) ? w.min_upr[lane + 32] : 0;
        const g_u64 ltypes = g_live_types(avail, s.n_types, mu_lo, mu_hi);
        int survivors = 0;
        __syncwarp();
        for (int k0 = 0; k0 < (S + 31) / 32; k0 += 4) {              // 32 consecutive entries per step, 4 steps in flight
          unsigned wd[4]; g_u64 tm[4];
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const int k = k0 + q, srv = k * 32 + lane;
            wd[q] = k < (S + 31) / 32 ? alive[k] : 0u;
            tm[q] = (((wd[q] >> lane) & 1u) && srv < S && ltypes) ? w.tmask[srv] : 0ull;
          }
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const unsigned keep = __ballot_sync(full, (tm[q] & ltypes) != 0);
            if (wd[q] && lane == 0) alive[k0 + q] = keep;
            survivors += __popc(keep);
          }
        }
        __syncwarp();
        n_survivors = survivors;
        if (survivors == 0) break;
      }
    }
    const long long tc1 = GSW_CLK(); cyc_chk += tc1 - tc0;
    const int rel = pos - origin;
    const int b = rel / GSW_BLOCK;
    if (b != cur_block) {
      __syncwarp();                                 // every lane is done reading the slot that is refilled next
      while (issued < b + GSW_SLOTS) {
        const int base = origin + issued * GSW_BLOCK;
        GEvent* dst = ring + (size_t)(issued % GSW_SLOTS) * GSW_BLOCK;
        for (int k = lane; k < GSW_BLOCK; k += 32)
          if (base + k < n_ev) gsw_cp16(dst + k, g.ev + base + k);
        gsw_commit();
        issued++;
      }
      // block b is complete once at most (issued - b - 1) younger groups are pending
      const int younger = issued - b - 1;
      if (younger <= 0) gsw_wait<0>();
      else if (younger == 1) gsw_wait<1>();
      else if (younger == 2) gsw_wait<2>();
      else gsw_wait<3>();
      __syncwarp();
      cur_block = b;
    }
    const long long tc2 = GSW_CLK(); cyc_ring += tc2 - tc1;
    n_batches++;
    const GEvent* blk = ring + (size_t)(b % GSW_SLOTS) * GSW_BLOCK;
    const int in_blk = rel % GSW_BLOCK;
    // most events of the stream belong to entries that already left the queue: 128 of them are checked at once (their
    // entry's alive bit, a priority boundary), and skipped together when nothing is left of them
    if ((in_blk & 127) == 0 && in_blk + 128 <= GSW_BLOCK && pos + 128 <= n_ev) {
      bool any = false;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        const int2 hd = *reinterpret_cast<const int2*>(&blk[in_blk + 32 * q + lane]);        // srv, meta
        any = any || gsw_alive(alive, hd.x) || (!delayed && (ge_flags((unsigned)hd.y) & GE_NEWPRIO));
      }
      if (!__any_sync(full, any)) { pos += 128; n_batches += 3; n_skip128++; cyc_dead += GSW_CLK() - tc2; continue; }
    }
    const int nvalid = min(min(32, GSW_BLOCK - in_blk), n_ev - pos);
    const bool valid = lane < nvalid;
    GEvent me; me.srv = -1; me.meta = 0; me.cnt = 0;
    if (valid) me = blk[in_blk + lane];
    const unsigned fl = ge_flags(me.meta);
    const int type = ge_type(me.meta);
    unsigned npm = delayed ? 0u : __ballot_sync(full, valid && (fl & GE_NEWPRIO));
    // most events of the stream belong to entries that already left the queue: a batch without an alive event (and
    // without a priority boundary) costs one shared-memory look-up and a vote
    const bool al0 = valid && gsw_alive(alive, me.srv);
    const unsigned am0 = __ballot_sync(full, al0);
    if (!am0 && !npm) { pos += nvalid; cyc_dead += GSW_CLK() - tc2; continue; }
    // lanes of the same entry (only needed when two or more events of the batch are alive)
    const unsigned peers = (am0 & (am0 - 1)) ? __match_any_sync(full, me.srv) : (1u << lane);
    // ---- fast path: no alive leader of a multi-leader tie group and no priority boundary in the batch.
    // Only a lane that fits (or has no accelerator) under the capacities at the START of the batch can take (or be
    // dropped): capacities only shrink.  Those candidates are visited in lane order with the whole state in registers —
    // every lane keeps the capacity left for ITS type and its alive flag, a take is two shuffles and two predicated
    // updates — and everything else alive is a failure, processed once for the whole batch.  Exactly the sequential
    // semantics: lane L sees the takes of the lanes before it and nothing else.
    {
      bool al = al0;
      long long myavail = (al && type >= 0) ? avail[type] : 0;
      const unsigned multi_alive = __ballot_sync(full, al && (fl & GE_MULTI));
      if (!multi_alive && !npm) {
        unsigned cand = __ballot_sync(full, al && (type < 0 || myavail >= me.cnt));
        unsigned took = 0;
        // (taking all first candidates at once when their demands fit together — match.any + a segmented reduce.add — was
        //  measured slower than this pass: 3-4 candidates per batch, and the per-type groups serialise the reduction)
        while (cand) {
          const int F = __ffs(cand) - 1;
          cand &= cand - 1;
          const unsigned okm = __ballot_sync(full, lane == F && al && (type < 0 || myavail >= me.cnt));
          if (!okm) continue;                        // killed by an earlier lane of its entry, or no longer fits: it fails
          const int tF = __shfl_sync(full, type, F);
          const long long cF = __shfl_sync(full, me.cnt, F);
          if (tF >= 0 && type == tF) myavail -= cF;
          if (lane > F && ((peers >> F) & 1u)) al = false;   // later events of the same entry are dead ...
          cand &= ~__shfl_sync(full, peers, F);              // ... and no longer candidates
          took |= 1u << F;
          n_seq++;
        }
        const bool taker = (took >> lane) & 1u;
        if (taker) {                                 // greedy.go:143-145 (or dropped, :126-136): every taker writes its own decision
          if (type >= 0) {
            w.kind[me.srv] = 1; w.sel_rank[me.srv] = ge_rank(me.meta);
            atomicAdd(reinterpret_cast<unsigned long long*>(&avail[type]), (unsigned long long)(-me.cnt));
          }
          atomicAnd(&alive[me.srv >> 5], ~(1u << (me.srv & 31)));
        }
        const bool failing = al && !taker;
        const unsigned fm = __ballot_sync(full, failing);
        if (fm) {
          const int rank = __popc(fm & lt);
          if (failing && (fm & peers & ~lt & ~(1u << lane)) == 0) g.stamp[me.srv] = z.clock + rank + 1;   // the entry's latest failure
          const bool lastc = failing && (fl & GE_LAST);                                                     // :152-156
          const unsigned lm = __ballot_sync(full, lastc);
          if (lastc) {
            w.unalloc[z.n_un + __popc(lm & lt)] = me.srv;
            atomicAnd(&alive[me.srv >> 5], ~(1u << (me.srv & 31)));
          }
          z.n_un += __popc(lm);
          z.clock += __popc(fm);
        }
        z.n_active += __popc(fm) + __popc(took);
        n_rounds++;
        __syncwarp();
        pos += nvalid;
        cyc_fast += GSW_CLK() - tc2;
        continue;
      }
    }
    int cur = 0;                                   // lanes below `cur` are done
    int jump = -1;
    while (cur < nvalid) {
      n_rounds++;
      // Outcome of every remaining lane under the CURRENT capacities and alive bits.  Up to the first lane that takes,
      // is dropped, leads a multi-leader tie group or starts a priority group, every alive lane simply fails — and a
      // failure changes neither the capacities nor (unless it is the entry's last candidate) the alive bits, so all
      // of them are processed at once; then that one lane sequentially, then the outcomes are re-evaluated.
      const bool todo = valid && lane >= cur;
      const bool al = todo && gsw_alive(alive, me.srv);
      const bool stopper = al && (type < 0 || avail[type < 0 ? 0 : type] >= me.cnt || (fl & GE_MULTI));
      const unsigned stopm = __ballot_sync(full, stopper);
      const unsigned npm_todo = npm & ~((1u << cur) - 1u);
      const int ls = stopm ? __ffs(stopm) - 1 : 32, lp = npm_todo ? __ffs(npm_todo) - 1 : 32;
      const int first = min(min(ls, lp), nvalid);
      // ---- plain failures in [cur, first)
      const bool failing = al && lane < first;
      const unsigned fm = __ballot_sync(full, failing);
      if (fm) {
        const int rank = __popc(fm & lt);
        if (failing && (fm & peers & ~lt & ~(1u << lane)) == 0) g.stamp[me.srv] = z.clock + rank + 1;   // the entry's latest failure
        const bool lastc = failing && (fl & GE_LAST);                                                     // :152-156
        const unsigned lm = __ballot_sync(full, lastc);
        if (lastc) {
          w.unalloc[z.n_un + __popc(lm & lt)] = me.srv;
          atomicAnd(&alive[me.srv >> 5], ~(1u << (me.srv & 31)));
        }
        z.n_un += __popc(lm);
        z.clock += __popc(fm);
        z.n_active += __popc(fm);
        __syncwarp();
      }
      cur = first;
      if (first >= nvalid) break;
      if (lp <= ls) {
        // a new priority group starts at lane `first`: allocate() of the previous group is complete -> its bestEffort()
        // (greedy.go:96-103) on the entries it left unallocated, in the order they were exhausted
        npm &= ~(1u << first);
        if (z.n_un > group_un0) {
          const long long c0 = GSW_CLK();
          g_best_effort(s, w, avail, w.unalloc + group_un0, z.n_un - group_un0, policy, be_stage);
          cyc_be += GSW_CLK() - c0; n_unalloc_be += z.n_un - group_un0;
        }
        group_un0 = z.n_un;
        __syncwarp();
        continue;                                  // the lane itself is evaluated in the next round
      }
      const int e_srv = __shfl_sync(full, me.srv, first);
      const unsigned e_meta = __shfl_sync(full, me.meta, first);
      const long long e_cnt = __shfl_sync(full, me.cnt, first);
      if (ge_flags(e_meta) & GE_MULTI) {
        // Several re-inserted leaders share this tau statically.  Their order only matters when another one is ALIVE:
        // if the re-inserted part of the group ends inside this batch and holds no other alive leader, this one is
        // processed in place; otherwise the tie-group procedure orders the alive leaders by insertion time.
        const unsigned tm = __ballot_sync(full, valid && (fl & GE_TIE) && !(fl & GE_CLS1));
        const unsigned after = first >= 31 ? 0u : (tm >> (first + 1));
        const int run = __ffs(~after) - 1;                          // lanes of the part after `first` (contiguous)
        const bool ends_here = first + 1 + run < nvalid;
        const unsigned span = run >= 31 ? 0xffffffffu : (((1u << run) - 1u) << (first + 1));
        const unsigned others = __ballot_sync(full, al && (fl & GE_LEADER)) & span;
        if (!ends_here || others) {
          n_tie++;
          const long long c0 = GSW_CLK();
          int np = gsw_tie_group_staged(w, g, avail, alive, z, pos + first, n_ev, tie_ev, tie_dyn);
          if (np == -2) { n_tie_global++; np = gsw_tie_group(w, g, avail, alive, z, pos + first, n_ev); }
          cyc_tie += GSW_CLK() - c0;
          if (np >= 0) { jump = np; break; }
        }
      }
      n_seq++;
      gsw_process(w, g, avail, alive, z, e_srv, e_meta, e_cnt);
      cur = first + 1;
    }
    if (jump >= 0) {
      pos = jump;
      if (pos < n_ev && pos - origin >= issued * GSW_BLOCK) {        // jumped past everything in flight: restart the stream
        gsw_wait<0>();
        __syncwarp();
        origin = pos; issued = 0; cur_block = -1;
        n_restart++;
      }
    } else {
      pos += nvalid;
    }
    cyc_slow += GSW_CLK() - tc2;
  }
  __syncwarp();
  // the last group's (or, delayed, the whole list's) best effort
  if (z.n_un > group_un0) {
    const long long c0 = GSW_CLK();
    g_best_effort(s, w, avail, w.unalloc + group_un0, z.n_un - group_un0, policy, be_stage);
    cyc_be += GSW_CLK() - c0; n_unalloc_be += z.n_un - group_un0;
  }
  if (lane == 0) { w.stats[8] = cyc_be; w.stats[9] = cyc_tie; w.stats[10] = GSW_CLK() - cyc0; w.stats[11] = n_unalloc_be; w.stats[12] = z.d_fb; w.stats[13] = z.d_nact; w.stats[14] = z.d_maxact; w.stats[15] = z.d_fbev; w.stats[16] = cyc_chk; w.stats[17] = cyc_ring; w.stats[18] = cyc_dead; w.stats[19] = cyc_fast; w.stats[20] = cyc_slow; w.stats[21] = n_survivors; w.stats[22] = n_tie_global; w.stats[23] = n_skip128; w.stats[24] = n_restart; w.stats[25] = g.head[2]; w.stats[26] = (long long)*g.head_events; w.stats[27] = head_end; }
  if (lane == 0) { w.stats[0] = 0; w.stats[1] = z.n_active; w.stats[2] = n_batches; w.stats[3] = n_rounds; w.stats[4] = n_seq; w.stats[5] = n_tie; w.stats[6] = pos; w.stats[7] = n_ev; }
}

// host driver of the static-order sweep.  Returns WVA_ERR_LIMIT (nothing launched) when the system is outside what this
// formulation covers — the caller then runs the literal queue (run_solve_greedy).
static inline bool greedy_sweep_covers(const SysView& s) {
  return (size_t)s.n_servers <= (size_t)GSW_ALIVE_WORDS * 32 && s.n_types <= GSW_AVAIL && s.n_types < 255 && s.n_acc <= 65535 &&
         (size_t)s.n_servers * (size_t)s.n_acc < (size_t)0x7fffffff;
}
static inline int32_t run_solve_greedy_sweep(const SysView& s, const CandView& c, const SolView& o, int delayed, int policy,
                                             void** ws, size_t* ws_cap, cudaStream_t stream, long long* launches,
                                             long long* stats_out = nullptr) {
  static_assert(GSW_SLOTS <= 4, "cp.async.wait_group immediates cover up to 3 younger groups");
  const size_t S = (size_t)s.n_servers, A = (size_t)s.n_acc, P = S * A;
  size_t eo = 0;
  auto etake = [&](size_t b) { size_t o2 = eo; eo = (eo + b + 255) & ~(size_t)255; return o2; };
  const size_t e_tkd = etake(P * 4), e_tkv = etake(P * 4), e_fl = etake(P), e_va = etake(P), e_ia = etake(P * 4), e_ib = etake(P * 4),
               e_ka = etake(P * 4), e_kb = etake(P * 4), e_ne = etake(64), e_ev = etake(P * sizeof(GEvent) + 64), e_st = etake(S * 4),
               e_dp = etake(S * 4), e_ds = etake(S * 4);
  const size_t n_blocks_max = P / GSW_BLOCK + 2;
  const size_t row_bytes = (size_t)(s.n_types > 0 ? s.n_types : 1) * 8;
  const size_t e_bm = etake(n_blocks_max * row_bytes), e_bs = etake(n_blocks_max * row_bytes), e_hu = etake(GSW_AVAIL * 8),
               e_ha = etake((S + 31) / 32 * 4), e_hd = etake(4 * 4), e_he = etake(8);
  GreedyWs w;
  size_t tmp = 0;
  void* d_tmp = nullptr;
  char* ex = nullptr;
  {
    int32_t rc = greedy_layout(S, A, (size_t)s.n_types, eo + 256, ws, ws_cap, w, tmp, &d_tmp, &ex);
    if (rc != WVA_OK) return rc;
  }
  GSweepWs g;
  g.t_kd = (unsigned*)(ex + e_tkd); g.t_kv = (unsigned*)(ex + e_tkv); g.fl = (unsigned char*)(ex + e_fl); g.valid = (unsigned char*)(ex + e_va);
  g.idxA = (unsigned*)(ex + e_ia); g.idxB = (unsigned*)(ex + e_ib); g.keyA = (unsigned*)(ex + e_ka); g.keyB = (unsigned*)(ex + e_kb);
  g.n_events = (int*)(ex + e_ne); g.ev = (GEvent*)(ex + e_ev); g.stamp = (int*)(ex + e_st); g.dyn_pos = (int*)(ex + e_dp);
  g.dyn_stamp = (int*)(ex + e_ds);
  g.blk_min = (unsigned long long*)(ex + e_bm); g.blk_sum = (long long*)(ex + e_bs); g.head_used = (long long*)(ex + e_hu);
  g.head_alive = (unsigned*)(ex + e_ha); g.head = (int*)(ex + e_hd); g.head_events = (unsigned long long*)(ex + e_he);
  if (cudaFuncSetAttribute(gsw_sweep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)GSW_SMEM) != cudaSuccess) return WVA_ERR_CUDA;
  const unsigned sb = (unsigned)((S + 127) / 128);
  if (cudaMemsetAsync(w.min_upr, 0x7f, 64 * 8, stream) != cudaSuccess) return WVA_ERR_CUDA;
  greedy_prepare_kernel<<<sb, 128, 0, stream>>>(s, c, w);
  gsw_events_kernel<<<sb, 128, 0, stream>>>(s, w, g);
  cub::CountingInputIterator<unsigned> cnt(0u);
  size_t t2 = tmp;
  if (cub::DeviceSelect::Flagged(d_tmp, t2, cnt, g.valid, g.idxA, g.n_events, (int)P, stream) != cudaSuccess) return WVA_ERR_CUDA;
  int n = 0;
  if (cudaMemcpyAsync(&n, g.n_events, 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess) return WVA_ERR_CUDA;
  if (cudaStreamSynchronize(stream) != cudaSuccess) return WVA_ERR_CUDA;
  *launches += 3;
  unsigned* cur = g.idxA; unsigned* alt = g.idxB;
  if (n > 0) {
    const unsigned cb = (unsigned)((n + 255) / 256);
    for (int which = 0; which < 4; which++) {   // LSD: run class, tau value, tau delta, priority (each pass stable)
      gsw_keys_kernel<<<cb, 256, 0, stream>>>(s, g, cur, n, which, g.keyA);
      t2 = tmp;
      if (cub::DeviceRadixSort::SortPairs(d_tmp, t2, g.keyA, g.keyB, cur, alt, n, 0, which == 0 ? 1 : 32, stream) != cudaSuccess)
        return WVA_ERR_CUDA;
      unsigned* sw = cur; cur = alt; alt = sw;
      *launches += 2;
    }
    const int n_blocks = n / GSW_BLOCK + 1;
    if (cudaMemsetAsync(g.blk_min, 0xff, (size_t)n_blocks * row_bytes, stream) != cudaSuccess ||
        cudaMemsetAsync(g.blk_sum, 0, (size_t)n_blocks * row_bytes, stream) != cudaSuccess) return WVA_ERR_CUDA;
    gsw_gather_kernel<<<cb, 256, 0, stream>>>(s, w, g, cur, n);
    gsw_multi_kernel<<<cb, 256, 0, stream>>>(g, n);
    *launches += 2;
    if (s.n_types > 0) {
      gsw_sufmin_kernel<<<s.n_types, 32, 0, stream>>>(g, n_blocks, s.n_types);
      gsw_prefix_kernel<<<s.n_types, 32, 0, stream>>>(s, g, n_blocks);
      *launches += 2;
    }
    // the head: up to the first failure (or the first block the nothing-fits check stops at), committed in parallel
    gsw_head_kernel<<<1, 32, 0, stream>>>(s, g, n);
    gsw_commit_kernel<<<cb, 256, 0, stream>>>(w, g, n);
    *launches += 2;
  }
  gsw_sweep_kernel<<<1, 32, GSW_SMEM, stream>>>(s, w, g, delayed, policy);
  greedy_finalize_kernel<<<(unsigned)((S + 255) / 256), 256, 0, stream>>>(s, c, o, w);
  *launches += 2;
  if (stats_out) {
    long long h[28];
    if (cudaMemcpyAsync(h, w.stats, sizeof(h), cudaMemcpyDeviceToHost, stream) != cudaSuccess) return WVA_ERR_CUDA;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return WVA_ERR_CUDA;
    stats_out[0] = h[0]; stats_out[1] = h[1];
    if (getenv("WVA_SIZER_DEBUG"))
      fprintf(stderr, "greedy sweep: alive events %lld, batches %lld, rounds %lld, sequential events %lld, tie-group calls %lld, stopped at %lld of %lld; cycles: best effort %lld (%lld entries), tie groups %lld, kernel %lld; tie groups: %lld over the staging size (%lld events), %lld in global memory, alive leaders %lld (max %lld); loop cycles: early-exit check %lld, ring %lld, dead batches %lld, fast path %lld, slow path %lld; entries swept on after nothing fits: %lld; 128-event skips %lld; stream restarts %lld; head: first failure at %lld, %lld first candidates committed in parallel, swept from %lld to %lld\n",
              h[1], h[2], h[3], h[4], h[5], h[6], h[7], h[8], h[11], h[9], h[10], h[12], h[15], h[22], h[13], h[14], h[16], h[17], h[18], h[19], h[20], h[21], h[23], h[24],
              h[25], h[26], h[27], h[6]);
  }
  return cudaGetLastError() == cudaSuccess ? WVA_OK : WVA_ERR_CUDA;
}

}  // namespace wva
