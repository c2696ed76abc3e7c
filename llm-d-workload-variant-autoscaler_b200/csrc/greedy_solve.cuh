// greedy_solve.cuh — Solver.SolveGreedy (pkg/solver/greedy.go:35-341) on the device.
//
//   K1 greedy_prepare_kernel   (thread per server)  sort each server's candidates by value
//                              (slices.SortFunc greedy.go:61-63, stable = ascending accelerator
//                              index on ties) and pack one RECORD per (server, rank): the two sort keys
//                              of the entry while it points at that candidate (delta to the next
//                              candidate, greedy.go:64-70,157-160, and value), the capacity type, the
//                              replica count and the units per replica (greedy.go:139) — everything
//                              the sweep needs, so that it never chases model/accelerator tables
//   sort                       entries by (priority asc, delta desc, value desc), greedy.go:76-87:
//                              three stable LSD radix passes (CUB) carrying the server index, so ties
//                              keep ascending server index — the oracle's canonical order
//   K2 greedy_heads_kernel     rank-0 record of every entry in sorted order (coalesced for the sweep)
//   K3 greedy_allocate_kernel  allocate() + bestEffort() (greedy.go:107-316).  The reference keeps a
//                              sorted slice and re-inserts a bumped entry BEFORE equal elements
//                              (slices.BinarySearchFunc + slices.Insert, greedy.go:161-162).  That is
//                              the order (key asc; among equal keys re-inserted entries first, latest
//                              first; then the untouched entries in their sorted order), realised
//                              here as: the sorted array consumed from its head + a 32-ary heap of
//                              re-inserted entries keyed (key, insertion stamp desc); the next entry
//                              is the heap top when top <= head, else the head.
//   K4 greedy_finalize_kernel  (thread per server) expands the sweep's decision (rank, replicas, full or
//                              scaled) into the solution arrays
//
// K3 is inherently sequential (every fit test depends on all earlier takes of the type): ONE warp runs
// it, all lanes executing the same control flow, and everything on its critical path is either in shared
// memory (available units per type, the first 4096 heap slots) or arrives 32 items per global round trip
// (the head records; the remaining candidates of a bumped entry, tested by the lanes in parallel).
#pragma once
#include "wva_core.cuh"
#include "solve_kernels.cuh"
#include <cub/cub.cuh>

namespace wva {

// Go cmp.Compare on float32 (NaN sorts first)
__device__ __forceinline__ int cmp_f32(float x, float y) {
  bool xn = x != x, yn = y != y;
  if (xn) return yn ? 0 : -1;
  if (yn) return 1;
  return x < y ? -1 : (x > y ? 1 : 0);
}

// order-preserving float32 -> uint32 with NaN first and -0 == +0 (cmp.Compare's order); descending = bitwise not
__device__ __forceinline__ unsigned sortable_f32(float x) {
  if (x != x) return 0u;
  if (x == 0.0f) x = 0.0f;
  unsigned b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

typedef unsigned long long g_u64;

struct GreedyWs {   // device workspace views
  int* order;        // [S*A] accelerator index of the k-th cheapest candidate of a server
  int* ncand;        // [S]
  // records, [S*A] indexed (server, rank)
  unsigned* r_kd;    // ~sortable(delta to the next candidate | MaxFloat32 for the last)   (descending delta)
  unsigned* r_kv;    // ~sortable(value)                                                   (descending value)
  int* r_type;       // capacity type, -1 = no accelerator behind this candidate (nil / "" / unknown model)
  int* r_nrep;       // replicas wanted
  long long* r_upr;  // units per replica (instances x multiplicity)
  // entry sort
  unsigned* k_val; unsigned* k_val2; int* e_srv; int* e_srv2;
  unsigned char* flag;  // [S] server has candidates
  int* n_entries;    // [1]
  // rank-0 records in sorted entry order
  g_u64* hd_khi; unsigned* hd_kv; int* hd_type; long long* hd_cnt;
  // heap slots beyond the shared-memory part
  g_u64* h_khi; g_u64* h_klo; long long* h_cnt; int* h_srv; int* h_ci; int* h_type;
  int* unalloc;      // [S]
  // decision per server: kind 0 none, 1 full allocation of rank sel_rank, 2 sel_nrep replicas of it (scaled)
  unsigned char* kind; int* sel_rank; int* sel_nrep;
  // allocateEqually tickets, [S] indexed by ticket
  int* tk_srv; int* tk_type; int* tk_rank; int* tk_want; int* tk_nrep; long long* tk_upr;
  long long* avail;  // [T] (used when the types do not fit the shared-memory copy)
  // bestEffort filter: the capacity types (< 64) behind a server's candidates, and per type the smallest units per replica
  // of any candidate — a server none of whose types has that much left can get nothing (greedy.go:204-213, 262-272)
  g_u64* tmask; long long* min_upr;
  long long* stats;  // heap pushes, events (entries processed), largest heap of the last sweep (the event sweep: [25])
};

__global__ void __launch_bounds__(128) greedy_prepare_kernel(SysView s, CandView c, GreedyWs w) {
  int srv = blockIdx.x * blockDim.x + threadIdx.x;
  if (srv >= s.n_servers) return;
  const int A = s.n_acc;
  const size_t p = (size_t)srv * A;
  int* ord = w.order + p;
  int n = 0;
  // insertion sort, stable: ascending accelerator index among equal values
  for (int a = 0; a < A; a++) {
    if (c.state[p + a] == ALLOC_NONE) continue;
    float v = c.value[p + a];
    int k = n;
    while (k > 0 && cmp_f32(c.value[p + ord[k - 1]], v) > 0) { ord[k] = ord[k - 1]; k--; }
    ord[k] = a;
    n++;
  }
  const bool known = s.srv_model[srv] >= 0;                              // greedy.go:126-129
  g_u64 tmask = 0;
  for (int j = 0; j < n; j++) {
    const int a = ord[j];
    const float v = c.value[p + a];
    const float d = (j + 1 < n) ? f_sub(c.value[p + ord[j + 1]], v) : FLT_MAX;   // greedy.go:64-70,157-160
    w.r_kd[p + j] = ~sortable_f32(d);
    w.r_kv[p + j] = ~sortable_f32(v);
    const bool live = known && c.state[p + a] == ALLOC_ACC;              // greedy.go:133-136
    w.r_type[p + j] = live ? s.acc_type[a] : -1;
    w.r_nrep[p + j] = live ? c.num_replicas[p + a] : 0;
    const long long upr = live ? (long long)num_instances(s, s.srv_model[srv], a) * s.acc_multiplicity[a] : 0;   // greedy.go:139
    w.r_upr[p + j] = upr;
    if (live && upr > 0) {
      const int t = s.acc_type[a];
      if (t >= 64) tmask = ~0ull;
      else if (t >= 0) { if (upr < w.min_upr[t]) atomicMin(&w.min_upr[t], upr); tmask |= 1ull << t; }
    }
  }
  w.tmask[srv] = tmask;
  for (int j = n; j < A; j++) {   // ranks past the list are read (and masked) by the 32-wide record loads of the sweep
    w.r_kd[p + j] = 0; w.r_kv[p + j] = 0; w.r_type[p + j] = -1; w.r_nrep[p + j] = 0; w.r_upr[p + j] = 0;
  }
  w.ncand[srv] = n;
  w.kind[srv] = 0;
  w.flag[srv] = n > 0 ? 1 : 0;
}

// keys of the compacted entry list for one radix pass: which = 0 value (desc), 1 delta (desc), 2 priority (asc)
__global__ void __launch_bounds__(256) greedy_keys_kernel(SysView s, GreedyWs w, const int* e_srv, int n, int which,
                                                         unsigned* keys) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int srv = e_srv[i];
  const size_t p = (size_t)srv * s.n_acc;
  if (which == 0) keys[i] = w.r_kv[p];
  else if (which == 1) keys[i] = w.r_kd[p];
  else keys[i] = (unsigned)s.srv_priority[srv] ^ 0x80000000u;
}

__global__ void __launch_bounds__(256) greedy_heads_kernel(SysView s, GreedyWs w, const int* e_srv, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int srv = e_srv[i];
  const size_t p = (size_t)srv * s.n_acc;
  w.hd_khi[i] = ((g_u64)((unsigned)s.srv_priority[srv] ^ 0x80000000u) << 32) | w.r_kd[p];
  w.hd_kv[i] = w.r_kv[p];
  w.hd_type[i] = w.r_type[p];
  w.hd_cnt[i] = (long long)w.r_nrep[p] * w.r_upr[p];
}

// An entry of the queue.  serverEntriesOrder (greedy.go:76-87) = ascending (khi, kv):
//   khi = priority (biased) : ~sortable(delta),  kv = ~sortable(value);  klo = kv : ~stamp makes the heap
//   order total (latest insertion first among equal keys).
struct GEntry { g_u64 khi, klo; long long cnt; int srv, ci, type; };

__device__ __forceinline__ bool g_key_after(g_u64 khi_a, unsigned kv_a, g_u64 khi_b, unsigned kv_b) {   // order(a, b) > 0
  return khi_a > khi_b || (khi_a == khi_b && kv_a > kv_b);
}
__device__ __forceinline__ bool g_before(g_u64 khi_a, g_u64 klo_a, g_u64 khi_b, g_u64 klo_b) {
  return khi_a < khi_b || (khi_a == khi_b && klo_a < klo_b);
}

constexpr int G_HEAP_SM = 4096;   // heap slots held in shared memory (levels 0-2 and the start of level 3)
constexpr int G_AVAIL_SM = 2048;  // capacity types held in shared memory
constexpr int G_STAGE_A = 32;     // candidate ranks per server staged in shared memory for the 32 head entries in flight
constexpr size_t G_SMEM_BYTES = (size_t)G_HEAP_SM * (8 + 8 + 8 + 4 + 4 + 4) + (size_t)G_AVAIL_SM * 8 +
                                (size_t)32 * G_STAGE_A * (8 + 4 + 4 + 4 + 4) + 32 * 8;

// 32-ary min-heap of re-inserted entries, operated by the whole warp: every lane runs the same control
// flow on the same values, and a pop inspects the 32 children of a node with one load per field + a
// shuffle arg-min, so a heap of S entries is ~log32(S) <= 4 levels deep.
struct GHeap {
  g_u64* s_khi; g_u64* s_klo; long long* s_cnt; int* s_srv; int* s_ci; int* s_type;
  GreedyWs w; int n;
  __device__ GEntry get(int i) const {
    GEntry e;
    if (i < G_HEAP_SM) { e.khi = s_khi[i]; e.klo = s_klo[i]; e.cnt = s_cnt[i]; e.srv = s_srv[i]; e.ci = s_ci[i]; e.type = s_type[i]; }
    else { const int g = i - G_HEAP_SM; e.khi = w.h_khi[g]; e.klo = w.h_klo[g]; e.cnt = w.h_cnt[g]; e.srv = w.h_srv[g]; e.ci = w.h_ci[g]; e.type = w.h_type[g]; }
    return e;
  }
  __device__ void put(int i, const GEntry& e) {
    if ((threadIdx.x & 31) == 0) {
      if (i < G_HEAP_SM) { s_khi[i] = e.khi; s_klo[i] = e.klo; s_cnt[i] = e.cnt; s_srv[i] = e.srv; s_ci[i] = e.ci; s_type[i] = e.type; }
      else { const int g = i - G_HEAP_SM; w.h_khi[g] = e.khi; w.h_klo[g] = e.klo; w.h_cnt[g] = e.cnt; w.h_srv[g] = e.srv; w.h_ci[g] = e.ci; w.h_type[g] = e.type; }
    }
  }
  __device__ void push(const GEntry& e) {
    int i = n++;
    while (i > 0) {
      const int p = (i - 1) >> 5;
      const GEntry pe = get(p);
      if (!g_before(e.khi, e.klo, pe.khi, pe.klo)) break;
      __syncwarp();          // every lane has read slot i's previous content (as a parent, one level down) before lane 0 overwrites it
      put(i, pe);
      i = p;
    }
    __syncwarp();
    put(i, e);
    __syncwarp();
  }
  __device__ GEntry pop() {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const GEntry top = get(0);
    const GEntry last = get(--n);
    __syncwarp();
    int i = 0;
    while (true) {
      const int c0 = 32 * i + 1;
      if (c0 >= n) break;
      const int ci = c0 + lane;
      // the smallest child: arg-min over the 128-bit (khi, klo) in four 32-bit redux.sync rounds, most significant
      // word first; stamps make real keys distinct, and an absent child (all ones) loses to every real key
      g_u64 khi = ~0ull, klo = ~0ull;
      if (ci < n) {
        if (ci < G_HEAP_SM) { khi = s_khi[ci]; klo = s_klo[ci]; }
        else { khi = w.h_khi[ci - G_HEAP_SM]; klo = w.h_klo[ci - G_HEAP_SM]; }
      }
      const unsigned k3 = (unsigned)(khi >> 32), k2 = (unsigned)khi, k1 = (unsigned)(klo >> 32), k0 = (unsigned)klo;
      const unsigned m3 = __reduce_min_sync(full, k3);
      bool in = k3 == m3;
      const unsigned m2 = __reduce_min_sync(full, in ? k2 : 0xffffffffu);
      in = in && k2 == m2;
      const unsigned m1 = __reduce_min_sync(full, in ? k1 : 0xffffffffu);
      in = in && k1 == m1;
      const unsigned m0 = __reduce_min_sync(full, in ? k0 : 0xffffffffu);
      in = in && k0 == m0;
      const int who = __ffs(__ballot_sync(full, in)) - 1;
      khi = ((g_u64)m3 << 32) | m2; klo = ((g_u64)m1 << 32) | m0;
      if (!g_before(khi, klo, last.khi, last.klo)) break;
      const GEntry child = get(c0 + who);
      __syncwarp();          // slot i was read by every lane (as a child, one level up) before lane 0 overwrites it
      put(i, child);
      i = c0 + who;
    }
    __syncwarp();
    if (n > 0) put(i, last);
    __syncwarp();
    return top;
  }
};

__device__ __forceinline__ void g_prefetch(const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); }

// One chunk of a server's records, a candidate per lane (rank j0 + lane), loaded in one round trip
struct GRec { unsigned kd, kv; int type, nrep; long long upr; };
__device__ __forceinline__ GRec g_load_rec(const GreedyWs& w, size_t p, int j, int A) {
  GRec r; r.kd = 0; r.kv = 0; r.type = -1; r.nrep = 0; r.upr = 0;
  if (j < A) { r.kd = w.r_kd[p + j]; r.kv = w.r_kv[p + j]; r.type = w.r_type[p + j]; r.nrep = w.r_nrep[p + j]; r.upr = w.r_upr[p + j]; }
  return r;
}

// Optional shared-memory staging for bestEffort: the first G_STAGE_A records (type, replicas, units per replica) of 32
// servers of the list are fetched with all loads in flight, instead of one dependent round trip per server.
struct GStage { long long* upr; int* type; int* nrep; };
__device__ __forceinline__ void g_stage_fill(const GreedyWs& w, const GStage& st, int my_srv, int my_n, unsigned passm, int A) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  __syncwarp();
  for (int k0 = 0; k0 < 32; k0 += 8) {              // 8 servers' records in flight: loads first, stores after (the
    if (!((passm >> k0) & 0xffu)) continue;
    int t[8], nr[8]; long long u[8];                  // compiler cannot move a load above a store through generic pointers)
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int srv = __shfl_sync(full, my_srv, k0 + q);
      const int nc = __shfl_sync(full, my_n, k0 + q);
      t[q] = -1; nr[q] = 0; u[q] = 0;
      if (((passm >> (k0 + q)) & 1u) && lane < nc && lane < G_STAGE_A) {
        const size_t p = (size_t)srv * A + lane;
        t[q] = w.r_type[p]; nr[q] = w.r_nrep[p]; u[q] = w.r_upr[p];
      }
    }
#pragma unroll
    for (int q = 0; q < 8; q++)
      if (lane < G_STAGE_A) { st.type[(k0 + q) * G_STAGE_A + lane] = t[q]; st.nrep[(k0 + q) * G_STAGE_A + lane] = nr[q]; st.upr[(k0 + q) * G_STAGE_A + lane] = u[q]; }
  }
  __syncwarp();
}
__device__ __forceinline__ GRec g_staged_rec(const GreedyWs& w, const GStage& st, int k, size_t p, int j, int A) {
  if (st.upr && j < G_STAGE_A) {
    GRec r; r.kd = 0; r.kv = 0;
    r.type = st.type[k * G_STAGE_A + j]; r.nrep = st.nrep[k * G_STAGE_A + j]; r.upr = st.upr[k * G_STAGE_A + j];
    return r;
  }
  return g_load_rec(w, p, j, A);
}

// the capacity types that can still place one replica of SOME candidate (bit t: available[t] >= min_upr[t])
__device__ __forceinline__ g_u64 g_live_types(const long long* avail, int n_types, long long mu_lo, long long mu_hi) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  if (n_types > 64) return ~0ull;
  const unsigned lo = __ballot_sync(full, lane < n_types && avail[lane] >= mu_lo);
  const unsigned hi = __ballot_sync(full, lane + 32 < n_types && avail[(lane + 32) < n_types ? lane + 32 : 0] >= mu_hi);
  return (g_u64)lo | ((g_u64)hi << 32);
}

// allocateMaximally (greedy.go:194-223): servers in list order; the lanes test a server's candidates in parallel
__device__ void g_allocate_maximally(const SysView& s, const GreedyWs& w, long long* avail, const int* list, int n, const GStage& st) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int A = s.n_acc;
  const long long mu_lo = lane < s.n_types ? w.min_upr[lane] : 0, mu_hi = (lane + 32 < s.n_types && lane + 32 < 64) ? w.min_upr[lane + 32] : 0;
  int nxt_srv = lane < n ? list[lane] : -1;
  for (int k0 = 0; k0 < n; k0 += 32) {
    const int my_srv = nxt_srv;
    nxt_srv = (k0 + 32 + lane < n) ? list[k0 + 32 + lane] : -1;
    // only a server with a candidate on a type that still has room for one replica of something can get anything
    const g_u64 ltypes = g_live_types(avail, s.n_types, mu_lo, mu_hi);
    unsigned passm = __ballot_sync(full, my_srv >= 0 && ltypes != 0 && (w.tmask[my_srv] & ltypes) != 0);
    if (!passm) continue;
    const int my_n = ((passm >> lane) & 1u) ? w.ncand[my_srv] : 0;
    if (st.upr) g_stage_fill(w, st, my_srv, my_n, passm, A);
    while (passm) {
      const int k = __ffs(passm) - 1;
      passm &= passm - 1;
      const int srv = __shfl_sync(full, my_srv, k);
      const int nc = __shfl_sync(full, my_n, k);
      const size_t p = (size_t)srv * A;
      for (int j0 = 0; j0 < nc; j0 += 32) {
        const int j = j0 + lane;
        const GRec r = g_staged_rec(w, st, k, p, j, A);
        long long maxr = 0;
        if (j < nc && r.type >= 0 && r.upr > 0) {
          maxr = avail[r.type] / r.upr;
          if (maxr > r.nrep) maxr = r.nrep;
        }
        const unsigned m = __ballot_sync(full, maxr > 0);
        if (m) {
          if (lane == __ffs(m) - 1) {
            w.kind[srv] = 2; w.sel_rank[srv] = j; w.sel_nrep[srv] = (int)maxr;
            avail[r.type] -= maxr * r.upr;
          }
          __syncwarp();
          break;
        }
      }
    }
  }
}

// allocateEqually (greedy.go:239-316) over list[0..n): tickets take one replica per round in list order.
// Round 1 picks each server's accelerator (the first candidate with room for one replica AT THAT MOMENT) and is
// therefore sequential over the servers, with the candidates of a server tested by the lanes; the later rounds
// only touch the tickets, 32 per round trip.
__device__ void g_allocate_equally(const SysView& s, const GreedyWs& w, long long* avail, const int* list, int n, const GStage& st) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int A = s.n_acc;
  int n_tk = 0, live = 0;
  const long long mu_lo = lane < s.n_types ? w.min_upr[lane] : 0, mu_hi = (lane + 32 < s.n_types && lane + 32 < 64) ? w.min_upr[lane + 32] : 0;
  int nxt_srv = lane < n ? list[lane] : -1;
  for (int k0 = 0; k0 < n; k0 += 32) {
    const int my_srv = nxt_srv;
    nxt_srv = (k0 + 32 + lane < n) ? list[k0 + 32 + lane] : -1;
    // only a server with a candidate on a type that still has room for one replica of something can get anything
    const g_u64 ltypes = g_live_types(avail, s.n_types, mu_lo, mu_hi);
    unsigned passm = __ballot_sync(full, my_srv >= 0 && ltypes != 0 && (w.tmask[my_srv] & ltypes) != 0);
    if (!passm) continue;
    const int my_n = ((passm >> lane) & 1u) ? w.ncand[my_srv] : 0;
    if (st.upr) g_stage_fill(w, st, my_srv, my_n, passm, A);
    while (passm) {
      const int k = __ffs(passm) - 1;
      passm &= passm - 1;
      const int srv = __shfl_sync(full, my_srv, k);
      const int nc = __shfl_sync(full, my_n, k);
      const size_t p = (size_t)srv * A;
      for (int j0 = 0; j0 < nc; j0 += 32) {
        const int j = j0 + lane;
        const GRec r = g_staged_rec(w, st, k, p, j, A);
        const bool room = j < nc && r.type >= 0 && r.upr > 0 && avail[r.type] >= r.upr;
        const unsigned m = __ballot_sync(full, room);
        if (m) {
          const int src = __ffs(m) - 1;
          const bool takes = __shfl_sync(full, r.nrep, src) > 0;   // min(available / upr, wanted) > 0
          if (lane == src) {
            w.tk_srv[n_tk] = srv; w.tk_type[n_tk] = r.type; w.tk_rank[n_tk] = j; w.tk_want[n_tk] = takes ? r.nrep : 0;
            w.tk_upr[n_tk] = r.upr; w.tk_nrep[n_tk] = takes ? 1 : 0;
            if (takes) avail[r.type] -= r.upr;
          }
          n_tk++;
          if (takes) live++;
          __syncwarp();
          break;
        }
      }
    }
  }
  // rounds 2..: a ticket whose want is 0 has left the game (tk_want = 0 marks it)
  while (live > 0) {
    for (int t0 = 0; t0 < n_tk; t0 += 32) {
      const int t = t0 + lane;
      int ty = -1, want = 0, nrep = 0; long long upr = 1;
      if (t < n_tk) { ty = w.tk_type[t]; want = w.tk_want[t]; nrep = w.tk_nrep[t]; upr = w.tk_upr[t]; }
      unsigned alive = __ballot_sync(full, want > 0);
      if (!alive) continue;
      bool changed = false;
      while (alive) {
        const int src = __ffs(alive) - 1;
        alive &= alive - 1;
        const int sty = __shfl_sync(full, ty, src);
        const long long supr = __shfl_sync(full, upr, src);
        const bool ok = avail[sty] >= supr;
        __syncwarp();
        if (lane == src) {
          if (ok) { nrep++; avail[sty] -= supr; } else want = 0;
          changed = true;
        }
        if (!ok) live--;
        __syncwarp();
      }
      if (changed) { w.tk_nrep[t] = nrep; w.tk_want[t] = want; }
    }
    __syncwarp();
  }
  for (int t = lane; t < n_tk; t += 32) {
    const int nrep = w.tk_nrep[t];
    if (nrep > 0) { const int srv = w.tk_srv[t]; w.kind[srv] = 2; w.sel_rank[srv] = w.tk_rank[t]; w.sel_nrep[srv] = nrep; }
  }
  __syncwarp();
}

// bestEffort (greedy.go:169-192)
__device__ void g_best_effort(const SysView& s, const GreedyWs& w, long long* avail, const int* list, int n, int policy,
                              const GStage& st = GStage{nullptr, nullptr, nullptr}) {
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  __syncwarp();   // the list was written by lane 0
  if (policy == 1) g_allocate_maximally(s, w, avail, list, n, st);
  else if (policy == 2) {
    int i = 0;
    while (i < n) {   // makePriorityGroups (greedy.go:321-341): runs of equal priority in list order
      const int p0 = s.srv_priority[list[i]];
      int j = i + 1;
      while (j < n) {
        const int q = j + lane;
        const bool differs = q >= n || s.srv_priority[list[q]] != p0;
        const unsigned m = __ballot_sync(full, differs);
        if (m) { j += __ffs(m) - 1; break; }
        j += 32;
      }
      if (j > n) j = n;
      g_allocate_equally(s, w, avail, list + i, j - i, st);
      i = j;
    }
  } else if (policy == 3) g_allocate_equally(s, w, avail, list, n, st);
}

#ifdef WVA_GREEDY_PROFILE
static __device__ long long g_prof[16];
#define GP_T(x) const long long x = clock64()
#define GP_ADD(i, t0) prof[i] += clock64() - (t0)
#define GP_INC(i) prof[i]++
#else
#define GP_T(x)
#define GP_ADD(i, t0)
#define GP_INC(i)
#endif

__global__ void __launch_bounds__(32, 1) greedy_allocate_kernel(SysView s, GreedyWs w, int delayed, int policy) {
  extern __shared__ g_u64 g_smem[];
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const bool writer = lane == 0;
  const int A = s.n_acc;
  const int n0 = *w.n_entries;
  GHeap heap;
  heap.s_khi = g_smem; heap.s_klo = heap.s_khi + G_HEAP_SM; heap.s_cnt = (long long*)(heap.s_klo + G_HEAP_SM);
  long long* sm_avail = heap.s_cnt + G_HEAP_SM;
  heap.s_srv = (int*)(sm_avail + G_AVAIL_SM); heap.s_ci = heap.s_srv + G_HEAP_SM; heap.s_type = heap.s_ci + G_HEAP_SM;
  heap.w = w; heap.n = 0;
  // the records (rank >= 1) of the 32 head entries in flight: a head that does not fit scans its remaining candidates
  // from here instead of paying a dependent L2 round trip (~1 200 cycles) per failing entry
  long long* sb_upr = (long long*)(heap.s_type + G_HEAP_SM);
  unsigned* sb_kd = (unsigned*)(sb_upr + 32 * G_STAGE_A); unsigned* sb_kv = sb_kd + 32 * G_STAGE_A;
  int* sb_type = (int*)(sb_kv + 32 * G_STAGE_A); int* sb_nrep = sb_type + 32 * G_STAGE_A;
  int* sb_nc = sb_nrep + 32 * G_STAGE_A;
  const int AS = A < G_STAGE_A ? A : G_STAGE_A;
  long long* avail = s.n_types <= G_AVAIL_SM ? sm_avail : w.avail;
  for (int t = lane; t < s.n_types; t += 32) avail[t] = s.type_count[t];   // greedy.go:38-39
  __syncwarp();

#ifdef WVA_GREEDY_PROFILE
  long long prof[16] = {0};
#endif
  GP_T(t_all);
  unsigned tau = 0;
  long long n_events = 0;
  int head = 0, n_un = 0, group_un0 = 0, base = -32;
  int heap_max = 0;                                 // most entries the heap held at once (past G_HEAP_SM: the global tier)
  g_u64 l_khi = 0; unsigned l_kv = 0; int l_type = -1, l_srv = -1; long long l_cnt = 0;   // this lane's head record
  unsigned group_pw = 0;
  bool group_set = false, batch_staged = false;
  int fails_in_batch = 32;                          // the first batch is staged
  while (true) {
    GP_T(t_it);
    if (head < n0 && head >= base + 32) {
      base += 32;
      const int i = base + lane;
      if (i < n0) {
        l_khi = w.hd_khi[i]; l_kv = w.hd_kv[i]; l_type = w.hd_type[i]; l_cnt = w.hd_cnt[i]; l_srv = w.e_srv[i];
      }
      // an entry whose first candidate does not fit needs the rest of its records at once.  While heads keep failing
      // (4 or more of the last 32) all 32 entries' records come in together — 32 consecutive records per load
      // instruction, every load of the batch in flight at once; otherwise they are only started towards L1
      batch_staged = fails_in_batch >= 4;
      fails_in_batch = 0;
      if (!batch_staged && i < n0) {
        const size_t q = (size_t)l_srv * A + 1;
        if (A > 1) {
          g_prefetch(w.r_kd + q); g_prefetch(w.r_kv + q); g_prefetch(w.r_type + q); g_prefetch(w.r_nrep + q);
          g_prefetch(w.r_upr + q); g_prefetch(w.r_upr + q + (A > 17 ? 16 : 0));
        }
        g_prefetch(w.ncand + l_srv);
      }
      if (batch_staged) {
        const int my_srv = i < n0 ? l_srv : -1;
        const int my_nc = my_srv >= 0 ? w.ncand[my_srv] : 0;
        __syncwarp();
        // 8 loads of every field in flight per lane before the first store (the stores would otherwise fence the loads)
        for (int it0 = 0; it0 < AS; it0 += 8) {
          GRec r[8];
#pragma unroll
          for (int u = 0; u < 8; u++) {
            const int idx = (it0 + u) * 32 + lane;
            const int sv = (it0 + u < AS) ? idx / AS : 0, j = idx - sv * AS;
            const int ssrv = __shfl_sync(full, my_srv, sv);
            r[u].kd = 0; r[u].kv = 0; r[u].type = -1; r[u].nrep = 0; r[u].upr = 0;
            if (it0 + u < AS && ssrv >= 0 && j >= 1) r[u] = g_load_rec(w, (size_t)ssrv * A, j, A);
          }
#pragma unroll
          for (int u = 0; u < 8; u++) {
            const int idx = (it0 + u) * 32 + lane;
            if (it0 + u < AS) { sb_kd[idx] = r[u].kd; sb_kv[idx] = r[u].kv; sb_type[idx] = r[u].type; sb_nrep[idx] = r[u].nrep; sb_upr[idx] = r[u].upr; }
          }
        }
        sb_nc[lane] = my_nc;
        __syncwarp();
      }
    }
    const int hl = head < n0 ? head - base : 0;
    const g_u64 hkhi = __shfl_sync(full, l_khi, hl);
    if (!group_set && head < n0) { group_pw = (unsigned)(hkhi >> 32); group_set = true; }
    // non-delayed mode: allocate + bestEffort run per priority group (greedy.go:96-103); the array is
    // sorted by priority and a re-inserted entry keeps its priority, so a group ends when both the
    // heap and the group's stretch of the array are exhausted
    const bool head_ok = head < n0 && (delayed || (unsigned)(hkhi >> 32) == group_pw);
    if (!head_ok && heap.n == 0) {
      if (!delayed) {
        { GP_T(t_be); g_best_effort(s, w, avail, w.unalloc + group_un0, n_un - group_un0, policy); GP_ADD(6, t_be); }
        group_un0 = n_un;
        if (head < n0) { group_pw = (unsigned)(hkhi >> 32); continue; }
      }
      break;
    }
    GEntry e;
    bool from_heap = !head_ok;
    if (head_ok) {
      e.khi = hkhi; e.klo = (g_u64)__shfl_sync(full, l_kv, hl) << 32;
      e.type = __shfl_sync(full, l_type, hl); e.cnt = __shfl_sync(full, l_cnt, hl); e.srv = __shfl_sync(full, l_srv, hl);
      e.ci = 0;
      if (heap.n > 0) {
        const GEntry top = heap.get(0);
        if (!g_key_after(top.khi, (unsigned)(top.klo >> 32), e.khi, (unsigned)(e.klo >> 32))) from_heap = true;   // inserted BEFORE equal elements
      }
    }
    GP_ADD(0, t_it); GP_INC(8);
    n_events++;
    if (from_heap) { GP_T(t_pop); e = heap.pop(); GP_ADD(1, t_pop); GP_INC(9); } else head++;
    GP_T(t_fit);
    if (e.type < 0) continue;                       // no accelerator behind the candidate: dropped (greedy.go:126-136)
    const int srv = e.srv;
    if (avail[e.type] >= e.cnt) {                   // greedy.go:143-145
      __syncwarp();
      if (writer) { avail[e.type] -= e.cnt; w.kind[srv] = 1; w.sel_rank[srv] = e.ci; }
      __syncwarp();
      GP_ADD(2, t_fit);
      continue;
    }
    // The candidate does not fit: move down the server's list (greedy.go:146-163).  The reference re-inserts
    // the entry with the key of its next candidate and pops again; a re-inserted key that is not AFTER the
    // position just popped (order <= 0: "before equal elements") lands at the front and is popped at once.
    // Those immediate events are resolved here without touching the heap, all remaining candidates tested by
    // the lanes in parallel: the entry stops at the first candidate that (a) must WAIT in the queue (key after
    // the current position), (b) has no accelerator (the entry is dropped when it gets there), or (c) FITS now
    // (an immediate event is tested against the current capacity).  Exactly the reference's sequence; only
    // the immediate failures cost nothing.
    GP_ADD(2, t_fit); GP_INC(10);
    GP_T(t_scan);
    const size_t p = (size_t)srv * A;
    const bool staged = !from_heap && batch_staged; // a head entry of a staged batch: its records are in shared memory (row hl)
    if (!from_heap) fails_in_batch++;
    const int n = staged ? sb_nc[hl] : w.ncand[srv];
    const unsigned pos_kv = (unsigned)(e.klo >> 32);
    int stop_j = -1, stop_kind = 0, stop_type = -1;   // kind: 1 wait, 2 dead, 3 fit
    g_u64 stop_khi = 0; unsigned stop_kv = 0; long long stop_cnt = 0;
    bool any_fit = false;
    for (int j0 = e.ci + 1; j0 < A; j0 += 32) {
      const int j = j0 + lane;
      GRec r;
      if (staged && j < AS) {
        const int q = hl * AS + j;
        r.kd = sb_kd[q]; r.kv = sb_kv[q]; r.type = sb_type[q]; r.nrep = sb_nrep[q]; r.upr = sb_upr[q];
      } else {
        r = g_load_rec(w, p, j, A);
      }
      if (j0 >= n) break;
      const g_u64 khi_j = (e.khi & 0xffffffff00000000ull) | r.kd;
      const long long cnt_j = (long long)r.nrep * r.upr;
      const bool valid = j < n;
      const bool fit_j = valid && r.type >= 0 && avail[r.type] >= cnt_j;
      const int kind = !valid ? 0 : (g_key_after(khi_j, r.kv, e.khi, pos_kv) ? 1 : (r.type < 0 ? 2 : (fit_j ? 3 : 0)));
      if (__any_sync(full, fit_j)) any_fit = true;
      const unsigned m = __ballot_sync(full, kind != 0);
      if (m && stop_j < 0) {
        const int src = __ffs(m) - 1;
        stop_j = j0 + src;
        stop_kind = __shfl_sync(full, kind, src);
        stop_khi = __shfl_sync(full, khi_j, src);
        stop_kv = __shfl_sync(full, r.kv, src);
        stop_type = __shfl_sync(full, r.type, src);
        stop_cnt = __shfl_sync(full, cnt_j, src);
      }
      if (stop_j >= 0 && policy != 0) break;       // policy None also wants any_fit over the whole list
    }
    GP_ADD(3, t_scan);
    if (stop_j < 0 || (policy == 0 && !any_fit && stop_kind != 2)) {
      // every remaining candidate fails immediately — or, under policy None, can never be satisfied (`available`
      // only shrinks and bestEffort() is a no-op): the entry is exhausted (greedy.go:152-156)
      if (writer) w.unalloc[n_un] = srv;
      n_un++;
      continue;
    }
    if (stop_kind == 2) continue;                  // accelerator "": dropped when it gets there (greedy.go:133-136)
    if (stop_kind == 3) {                          // immediate event that fits (greedy.go:143-145)
      __syncwarp();
      if (writer) { avail[stop_type] -= stop_cnt; w.kind[srv] = 1; w.sel_rank[srv] = stop_j; }
      __syncwarp();
      continue;
    }
    GEntry ne;
    ne.khi = stop_khi; ne.klo = ((g_u64)stop_kv << 32) | (unsigned)~(++tau);
    ne.cnt = stop_cnt; ne.srv = srv; ne.ci = stop_j; ne.type = stop_type;
    { GP_T(t_push); heap.push(ne); GP_ADD(4, t_push); GP_INC(11); }
    if (heap.n > heap_max) heap_max = heap.n;
  }
  __syncwarp();
  { GP_T(t_be); if (delayed) g_best_effort(s, w, avail, w.unalloc, n_un, policy); GP_ADD(6, t_be); }
  GP_ADD(7, t_all);
  if (writer) { w.stats[0] = (long long)tau; w.stats[1] = n_events; w.stats[2] = heap_max; }
#ifdef WVA_GREEDY_PROFILE
  if (writer) for (int i = 0; i < 16; i++) g_prof[i] = prof[i];
#endif
}

// decision -> solution arrays (Allocation fields as greedy.go:143-145 / 206-211 / 301-308 leave them)
__global__ void __launch_bounds__(256) greedy_finalize_kernel(SysView s, CandView c, SolView o, GreedyWs w) {
  const int srv = blockIdx.x * blockDim.x + threadIdx.x;
  if (srv >= s.n_servers) return;
  const int kind = w.kind[srv];
  if (kind == 0) {                                                       // server.RemoveAllocation()
    o.state[srv] = ALLOC_NONE; o.acc[srv] = -1; o.num_replicas[srv] = 0; o.batch_size[srv] = 0;
    o.cost[srv] = o.value[srv] = o.itl[srv] = o.ttft[srv] = o.rho[srv] = o.max_arrv_rate[srv] = 0.0f;
    return;
  }
  const int acc = w.order[(size_t)srv * s.n_acc + w.sel_rank[srv]];
  const size_t i = (size_t)srv * s.n_acc + acc;
  int replicas = c.num_replicas[i];
  float cost = c.cost[i], value = c.value[i];
  if (kind == 2) {
    const int got = w.sel_nrep[srv];
    const float factor = f_div((float)got, (float)replicas);
    cost = f_mul(cost, factor); value = f_mul(value, factor);
    replicas = got;
  }
  o.state[srv] = ALLOC_ACC; o.acc[srv] = acc; o.num_replicas[srv] = replicas; o.batch_size[srv] = c.batch_size[i];
  o.cost[srv] = cost; o.value[srv] = value; o.itl[srv] = c.itl[i]; o.ttft[srv] = c.ttft[i]; o.rho[srv] = c.rho[i];
  o.max_arrv_rate[srv] = c.max_arrv_rate[i];
}

// workspace layout shared by the two formulations of the sweep; `extra` bytes are appended for the caller
// (ws/ws_cap: a growable device allocation owned by the ctx)
static inline int32_t greedy_layout(size_t S, size_t A, size_t T, size_t extra, void** ws, size_t* ws_cap, GreedyWs& w,
                                    size_t& tmp_bytes, void** d_tmp_out, char** extra_out) {
  size_t off = 0;
  auto take = [&](size_t b) { size_t o2 = off; off = (off + b + 255) & ~(size_t)255; return o2; };
  const size_t o_order = take(S * A * 4), o_ncand = take(S * 4), o_rkd = take(S * A * 4), o_rkv = take(S * A * 4),
               o_rty = take(S * A * 4), o_rnr = take(S * A * 4), o_rup = take(S * A * 8),
               o_k1 = take(S * 4), o_k2 = take(S * 4), o_e1 = take(S * 4), o_e2 = take(S * 4), o_flag = take(S), o_ne = take(64),
               o_dkh = take(S * 8), o_dkv = take(S * 4), o_dty = take(S * 4), o_dcn = take(S * 8),
               o_hkh = take(S * 8), o_hkl = take(S * 8), o_hcn = take(S * 8), o_hs = take(S * 4), o_hc = take(S * 4), o_ht = take(S * 4),
               o_un = take(S * 4), o_kind = take(S), o_sr = take(S * 4), o_sn = take(S * 4),
               o_ts = take(S * 4), o_tt = take(S * 4), o_tr = take(S * 4), o_tw = take(S * 4), o_tn = take(S * 4), o_tu = take(S * 8),
               o_av = take(T * 8 + 8), o_st = take(256), o_tm = take(S * 8), o_mu = take(64 * 8);
  size_t tmp = 0, tb = 0;
  cub::CountingInputIterator<int> cnt(0);
  const size_t n_sel = S * A > S ? S * A : S;
  cub::DeviceSelect::Flagged(nullptr, tb, cnt, (unsigned char*)nullptr, (int*)nullptr, (int*)nullptr, (int)n_sel, 0);
  tmp = tb;
  cub::DeviceRadixSort::SortPairs(nullptr, tb, (unsigned*)nullptr, (unsigned*)nullptr, (int*)nullptr, (int*)nullptr, (int)n_sel, 0, 32, 0);
  if (tb > tmp) tmp = tb;
  const size_t o_tmp = take(tmp + 256);
  const size_t o_extra = take(extra);
  if (off + 256 > *ws_cap) {
    if (*ws) cudaFree(*ws);
    *ws = nullptr; *ws_cap = 0;
    if (cudaMalloc(ws, off + 256) != cudaSuccess) return WVA_ERR_NOMEM;
    *ws_cap = off + 256;
  }
  char* d = (char*)*ws;
  w.order = (int*)(d + o_order); w.ncand = (int*)(d + o_ncand);
  w.r_kd = (unsigned*)(d + o_rkd); w.r_kv = (unsigned*)(d + o_rkv); w.r_type = (int*)(d + o_rty); w.r_nrep = (int*)(d + o_rnr);
  w.r_upr = (long long*)(d + o_rup);
  w.k_val = (unsigned*)(d + o_k1); w.k_val2 = (unsigned*)(d + o_k2); w.e_srv = (int*)(d + o_e1); w.e_srv2 = (int*)(d + o_e2);
  w.flag = (unsigned char*)(d + o_flag); w.n_entries = (int*)(d + o_ne);
  w.hd_khi = (g_u64*)(d + o_dkh); w.hd_kv = (unsigned*)(d + o_dkv); w.hd_type = (int*)(d + o_dty); w.hd_cnt = (long long*)(d + o_dcn);
  w.h_khi = (g_u64*)(d + o_hkh); w.h_klo = (g_u64*)(d + o_hkl); w.h_cnt = (long long*)(d + o_hcn);
  w.h_srv = (int*)(d + o_hs); w.h_ci = (int*)(d + o_hc); w.h_type = (int*)(d + o_ht);
  w.unalloc = (int*)(d + o_un); w.kind = (unsigned char*)(d + o_kind); w.sel_rank = (int*)(d + o_sr); w.sel_nrep = (int*)(d + o_sn);
  w.tk_srv = (int*)(d + o_ts); w.tk_type = (int*)(d + o_tt); w.tk_rank = (int*)(d + o_tr); w.tk_want = (int*)(d + o_tw);
  w.tk_nrep = (int*)(d + o_tn); w.tk_upr = (long long*)(d + o_tu);
  w.tmask = (g_u64*)(d + o_tm); w.min_upr = (long long*)(d + o_mu);
  w.avail = (long long*)(d + o_av);
  w.stats = (long long*)(d + o_st);
  tmp_bytes = tmp;
  *d_tmp_out = d + o_tmp;
  if (extra_out) *extra_out = d + o_extra;
  return WVA_OK;
}

// host driver of the literal queue (sorted array + re-insertion heap)
static inline int32_t run_solve_greedy(const SysView& s, const CandView& c, const SolView& o, int delayed, int policy,
                                       void** ws, size_t* ws_cap, cudaStream_t stream, long long* launches,
                                       long long* stats_out = nullptr) {
  const size_t S = (size_t)s.n_servers;
  GreedyWs w;
  size_t tmp = 0;
  void* d_tmp0 = nullptr;
  {
    int32_t rc = greedy_layout(S, (size_t)s.n_acc, (size_t)s.n_types, 0, ws, ws_cap, w, tmp, &d_tmp0, nullptr);
    if (rc != WVA_OK) return rc;
  }
  cub::CountingInputIterator<int> cnt(0);
  if (cudaFuncSetAttribute(greedy_allocate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G_SMEM_BYTES) != cudaSuccess)
    return WVA_ERR_CUDA;
  void* d_tmp = d_tmp0;
  const unsigned nb = (unsigned)((S + 255) / 256);
  if (cudaMemsetAsync(w.min_upr, 0x7f, 64 * 8, stream) != cudaSuccess) return WVA_ERR_CUDA;
  greedy_prepare_kernel<<<(unsigned)((S + 127) / 128), 128, 0, stream>>>(s, c, w);
  size_t t2 = tmp;
  if (cub::DeviceSelect::Flagged(d_tmp, t2, cnt, w.flag, w.e_srv, w.n_entries, (int)S, stream) != cudaSuccess) return WVA_ERR_CUDA;
  int n = 0;
  if (cudaMemcpyAsync(&n, w.n_entries, 4, cudaMemcpyDeviceToHost, stream) != cudaSuccess) return WVA_ERR_CUDA;
  if (cudaStreamSynchronize(stream) != cudaSuccess) return WVA_ERR_CUDA;
  *launches += 2;
  int* cur = w.e_srv; int* alt = w.e_srv2;
  if (n > 0) {
    const unsigned cb = (unsigned)((n + 255) / 256);
    for (int which = 0; which < 3; which++) {   // LSD: value, then delta, then priority
      greedy_keys_kernel<<<cb, 256, 0, stream>>>(s, w, cur, n, which, w.k_val);
      t2 = tmp;
      if (cub::DeviceRadixSort::SortPairs(d_tmp, t2, w.k_val, w.k_val2, cur, alt, n, 0, 32, stream) != cudaSuccess) return WVA_ERR_CUDA;
      int* sw = cur; cur = alt; alt = sw;
      *launches += 2;
    }
    greedy_heads_kernel<<<cb, 256, 0, stream>>>(s, w, cur, n);
    *launches += 1;
  }
  w.e_srv = cur;   // the sweep reads the sorted list
  greedy_allocate_kernel<<<1, 32, G_SMEM_BYTES, stream>>>(s, w, delayed, policy);
  greedy_finalize_kernel<<<nb, 256, 0, stream>>>(s, c, o, w);
  *launches += 2;
  if (stats_out) {
    long long h[3];
    if (cudaMemcpyAsync(h, w.stats, sizeof(h), cudaMemcpyDeviceToHost, stream) != cudaSuccess) return WVA_ERR_CUDA;
    if (cudaStreamSynchronize(stream) != cudaSuccess) return WVA_ERR_CUDA;
    stats_out[0] = h[0]; stats_out[1] = h[1];
    if (getenv("WVA_SIZER_DEBUG"))
      fprintf(stderr, "greedy queue: heap pushes %lld, events %lld, largest heap %lld (%d slots in shared memory)\n", h[0], h[1], h[2], G_HEAP_SM);
  }
#ifdef WVA_GREEDY_PROFILE
  {
    long long h[16];
    cudaStreamSynchronize(stream);
    cudaMemcpyFromSymbol(h, g_prof, sizeof(h));
    fprintf(stderr, "greedy profile pol=%d: cycles head=%lld pop=%lld fit=%lld scan=%lld push=%lld best_effort=%lld total=%lld | events=%lld heap_pops=%lld fails=%lld pushes=%lld\n",
            policy, h[0], h[1], h[2], h[3], h[4], h[6], h[7], h[8], h[9], h[10], h[11]);
  }
#endif
  return cudaGetLastError() == cudaSuccess ? WVA_OK : WVA_ERR_CUDA;
}

}  // namespace wva
