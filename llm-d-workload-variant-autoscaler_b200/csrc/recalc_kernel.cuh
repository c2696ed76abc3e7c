// recalc_kernel.cuh — device side of wva_update_servers / wva_recalculate: the per-cycle server columns (load and
// current allocation) compared with the resident ones and written over them, and the row moves and re-valuation
// around a sizer run on the servers whose sizing inputs changed.  The sizers themselves are the ones wva_calculate
// runs, handed a gathered view; wva_grid_update moves grid rows around a grid run on a gathered view the same way.
#pragma once
#include "wva_core.cuh"
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/discard_iterator.h>

namespace wva {

// marks[srv] bits, accumulated from update to update until the next wva_calculate / wva_recalculate
enum { MARK_RESIZE = 1,     // a sizing input changed (sizer_setup): the load, the model, a target or SLO, max batch,
                            // min replicas, keepAccelerator, or the current accelerator of a keepAccelerator server
       MARK_REVALUE = 2 };  // the current allocation changed: TransitionPenalty (every candidate's value) changed

__device__ __forceinline__ bool bits_differ(float a, float b) { return __float_as_uint(a) != __float_as_uint(b); }

// One pass over the servers of `nu`, the new values of every server column: new server i was server p = prev[i] of the
// resident columns `res` (prev NULL: p = i, the same set), or is new (p < 0).  The bitwise diff of each kept server's
// columns against row p, the write of `nu` into `out` (res itself for the same set), and the marks of the servers in
// [lo, hi) (the rank's block; every rank holds every column): the marks of row p (old_marks, NULL = none) carried over
// and this diff's added.  grid_marks[i] = 1 when a column grid_setup reads changed (the load, the model, a target or
// SLO, max batch); they accumulate until the next wva_grid_run / wva_grid_update, apart from the sizing marks.  A new
// server gets both.  srv_priority is written and marks nothing: only the allocators read it.
__global__ void classify_servers_kernel(SysView res, SysView nu, SysView out, const int* prev, int lo, int hi,
                                        const unsigned char* old_marks, const unsigned char* old_grid_marks,
                                        unsigned char* marks, unsigned char* grid_marks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nu.n_servers) return;
  const int p = prev ? prev[i] : i;
  const int model = nu.srv_model[i], prio = nu.srv_priority[i], minr = nu.srv_min_replicas[i], mb = nu.srv_max_batch[i];
  const unsigned char keep = nu.srv_keep_acc[i], tp = nu.srv_target_present[i];
  const float ttft = nu.srv_slo_ttft[i], itl = nu.srv_slo_itl[i], tps = nu.srv_slo_tps[i];
  const float arr = nu.srv_arrival[i], cost = nu.srv_cur_cost[i];
  const int in_tok = nu.srv_in_tokens[i], out_tok = nu.srv_out_tokens[i];
  const int acc = nu.srv_cur_acc[i], rep = nu.srv_cur_replicas[i];
  unsigned char mark = MARK_RESIZE, grid = 1;
  if (p >= 0) {
    const bool load = bits_differ(arr, res.srv_arrival[p]) || in_tok != res.srv_in_tokens[p] ||
                      out_tok != res.srv_out_tokens[p];
    const bool gridded = load || model != res.srv_model[p] || mb != res.srv_max_batch[p] ||
                         tp != res.srv_target_present[p] || bits_differ(ttft, res.srv_slo_ttft[p]) ||
                         bits_differ(itl, res.srv_slo_itl[p]) || bits_differ(tps, res.srv_slo_tps[p]);
    const bool acc_moved = acc != res.srv_cur_acc[p];
    const bool alloc = acc_moved || rep != res.srv_cur_replicas[p] || bits_differ(cost, res.srv_cur_cost[p]);
    // the candidate set depends on the current accelerator when keepAccelerator is set (server.go:70-82)
    const bool resize = gridded || minr != res.srv_min_replicas[p] || keep != res.srv_keep_acc[p] ||
                        (acc_moved && (keep || res.srv_keep_acc[p]));
    mark = (resize ? MARK_RESIZE : 0) | (alloc ? MARK_REVALUE : 0) | (old_marks ? old_marks[p] : 0);
    grid = (gridded ? 1 : 0) | (old_grid_marks ? old_grid_marks[p] : 0);
  }
  const_cast<int*>(out.srv_model)[i] = model;
  const_cast<int*>(out.srv_priority)[i] = prio;
  const_cast<int*>(out.srv_min_replicas)[i] = minr;
  const_cast<int*>(out.srv_max_batch)[i] = mb;
  const_cast<unsigned char*>(out.srv_keep_acc)[i] = keep;
  const_cast<unsigned char*>(out.srv_target_present)[i] = tp;
  const_cast<float*>(out.srv_slo_ttft)[i] = ttft;
  const_cast<float*>(out.srv_slo_itl)[i] = itl;
  const_cast<float*>(out.srv_slo_tps)[i] = tps;
  const_cast<float*>(out.srv_arrival)[i] = arr;
  const_cast<int*>(out.srv_in_tokens)[i] = in_tok;
  const_cast<int*>(out.srv_out_tokens)[i] = out_tok;
  const_cast<int*>(out.srv_cur_acc)[i] = acc;
  const_cast<int*>(out.srv_cur_replicas)[i] = rep;
  const_cast<float*>(out.srv_cur_cost)[i] = cost;
  if (i >= lo && i < hi) { marks[i] = mark; grid_marks[i] = grid; }
}

// the two lists wva_recalculate compacts from the marks (a re-sized server is re-valued by its sizing already)
struct MarkedResize {
  const unsigned char* marks;
  __device__ bool operator()(int i) const { return marks[i] & MARK_RESIZE; }
};
struct MarkedRevalueOnly {
  const unsigned char* marks;
  __device__ bool operator()(int i) const { return marks[i] == MARK_REVALUE; }
};

// The marks of wva_update_tables, keyed by table row so that a change of the server set leaves them valid.  size_row /
// size_acc accumulate until the next wva_calculate / wva_recalculate, grid_row until the next wva_grid_run /
// wva_grid_update; fresh holds the last call's own sizing diff ([M*A] rows, then [A] costs) for its count.
struct TableMarks {
  unsigned char *size_row, *size_acc, *grid_row, *fresh;
};

// One pass over the table entries of `nu` (thread t: perf row t of [M*A] and accelerator t of [A]): the bitwise diff
// against the resident tables `res`, the write of `nu` over them, and the marks.  A perf row is marked for sizing when
// a field sizer_setup / alloc_final reads changed (alpha, beta, gamma, max_batch, at_tokens, acc_count, present) and
// for the grid when one grid_setup reads changed (all of them but acc_count); an accelerator for sizing when its cost
// changed (every candidate's cost and value).  acc_multiplicity and acc_type are written and mark nothing: only the
// allocators read them.
__global__ void classify_tables_kernel(SysView res, SysView nu, int A, int M, TableMarks tm) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long MA = (long long)M * A;
  if (t < MA) {
    const float al = nu.perf_alpha[t], be = nu.perf_beta[t], ga = nu.perf_gamma[t];
    const int mb = nu.perf_max_batch[t], at = nu.perf_at_tokens[t], ac = nu.perf_acc_count[t];
    const unsigned char pr = nu.perf_present[t];
    const bool grid = bits_differ(al, res.perf_alpha[t]) || bits_differ(be, res.perf_beta[t]) ||
                      bits_differ(ga, res.perf_gamma[t]) || mb != res.perf_max_batch[t] || at != res.perf_at_tokens[t] ||
                      pr != res.perf_present[t];
    const bool size = grid || ac != res.perf_acc_count[t];
    const_cast<float*>(res.perf_alpha)[t] = al;
    const_cast<float*>(res.perf_beta)[t] = be;
    const_cast<float*>(res.perf_gamma)[t] = ga;
    const_cast<int*>(res.perf_max_batch)[t] = mb;
    const_cast<int*>(res.perf_at_tokens)[t] = at;
    const_cast<int*>(res.perf_acc_count)[t] = ac;
    const_cast<unsigned char*>(res.perf_present)[t] = pr;
    if (size) tm.size_row[t] = 1;
    if (grid) tm.grid_row[t] = 1;
    tm.fresh[t] = size;
  }
  if (t < A) {
    const float cost = nu.acc_cost[t];
    const bool changed = bits_differ(cost, res.acc_cost[t]);
    const_cast<float*>(res.acc_cost)[t] = cost;
    const_cast<int*>(res.acc_multiplicity)[t] = nu.acc_multiplicity[t];
    const_cast<int*>(res.acc_type)[t] = nu.acc_type[t];
    if (changed) tm.size_acc[t] = 1;
    tm.fresh[MA + t] = changed;
  }
}

// Pair t of a block view (server t / A, accelerator t % A) is listed when its server carries `bit` in srv_marks (the
// block's server marks, NULL = none pending), or when the server's model is known and its perf row (model, acc) is in
// `row` or its accelerator in `acc` (NULL = no accelerator marks).  Unknown-model servers read no table.
struct TablePair {
  const int* srv_model;
  const unsigned char* srv_marks;
  unsigned char bit;
  const unsigned char *row, *acc;
  int A;
  __device__ bool operator()(int t) const {
    const int srv = t / A, a = t % A;
    if (srv_marks && (srv_marks[srv] & bit)) return true;
    const int m = srv_model[srv];
    return m >= 0 && (row[(size_t)m * A + a] || (acc && acc[a]));
  }
};

// The pairs of the block view's n_pairs whose perf row or accelerator the last wva_update_tables changed (fresh), summed
// into *count.
__global__ void __launch_bounds__(256) count_table_pairs_kernel(const int* srv_model, int A, int M, unsigned long long n_pairs,
                                                                const unsigned char* fresh, unsigned long long* count) {
  const unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x;
  const TablePair marked{srv_model, nullptr, 0, fresh, fresh + (size_t)M * A, A};
  const unsigned hit = __ballot_sync(0xffffffffu, t < n_pairs && marked((int)t));
  if ((threadIdx.x & 31) == 0 && hit) atomicAdd(count, (unsigned long long)__popc(hit));
}

// Per-server rows of up to 32 columns moved between a resident arena and a compacted one: row rows[i] of the resident
// columns <-> row i of the compacted ones, `per` elements per row (1 for server columns, A for candidate rows).
struct RowMoves {
  enum { MAXC = 32 };
  int n = 0;
  const char* src[MAXC];
  char* dst[MAXC];
  int width[MAXC];
};

__global__ void move_rows_kernel(RowMoves m, const int* rows, unsigned long long n_items, int per, bool scatter) {
  for (unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; t < n_items;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long i = t / (unsigned)per, k = t % (unsigned)per;
    const unsigned long long resident = (unsigned long long)rows[i] * per + k;
    const unsigned long long from = scatter ? t : resident, to = scatter ? resident : t;
    for (int c = 0; c < m.n; c++) {
      switch (m.width[c]) {
        case 1: m.dst[c][to] = m.src[c][from]; break;
        case 2: ((short*)m.dst[c])[to] = ((const short*)m.src[c])[from]; break;
        case 4: ((int*)m.dst[c])[to] = ((const int*)m.src[c])[from]; break;
        default: ((long long*)m.dst[c])[to] = ((const long long*)m.src[c])[from]; break;
      }
    }
  }
}

// A run of a new server set: new rows [start, next run's start) are old rows prev[start].. in order, or new rows when
// prev[start] < 0.  A run starts where the set starts, where a kept row does not follow its predecessor's old row, and
// where kept and new rows alternate.
struct RunHead {
  const int* prev;
  __device__ bool operator()(int i) const {
    if (i == 0) return true;
    const int a = prev[i - 1], b = prev[i];
    return (a < 0) != (b < 0) || (b >= 0 && b != a + 1);
  }
};

// Every column of `m`, `per` elements per row, laid out for a new set of n_rows rows: each run of *n_runs (starts[]:
// their first new rows, ascending) copied from the old column as one contiguous range, new rows zero-filled (the nil
// candidate, a grid level that is not ok, frontier 0).  Column blockIdx.y; a warp takes 32 * CHUNKS consecutive 16-byte
// chunks of it at a time (16-byte loads and stores wherever source and destination are both aligned), looks up the run
// of its first chunk and walks forward.  Memory-bound: every destination byte is written once and every kept one read
// once, with streaming cache hints since neither side is touched again by this kernel.
template <int CHUNKS>
__global__ void __launch_bounds__(256) reindex_rows_kernel(RowMoves m, const int* prev, const int* starts,
                                                           const int* n_runs, int n_rows, int per) {
  const int c = blockIdx.y;
  if (c >= m.n) return;
  const int nr = *n_runs;
  const unsigned long long rb = (unsigned long long)per * m.width[c], total = (unsigned long long)n_rows * rb;
  const unsigned long long n_chunks = (total + 15) / 16, per_warp = 32ull * CHUNKS;
  const int lane = threadIdx.x & 31;
  const unsigned long long warps = (unsigned long long)gridDim.x * (blockDim.x / 32);
  const char* src = m.src[c];
  char* dst = m.dst[c];
  auto run_end = [&](int r) { return (unsigned long long)(r + 1 < nr ? starts[r + 1] : n_rows) * rb; };
  for (unsigned long long w = blockIdx.x * (unsigned long long)(blockDim.x / 32) + threadIdx.x / 32; w * per_warp < n_chunks;
       w += warps) {
    unsigned long long off = (w * per_warp + lane) * 16;
    if (off >= total) continue;
    int lo = 0, hi = nr;   // the run holding byte `off`: the last with start * rb <= off
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if ((unsigned long long)starts[mid] * rb <= off) lo = mid; else hi = mid;
    }
    int r = lo;
#pragma unroll 1
    for (int k = 0; k < CHUNKS && off < total; k++, off += 32 * 16) {
      while (off >= run_end(r)) r++;
      const unsigned long long end = run_end(r);
      const int from = prev[starts[r]];
      const unsigned long long s_off = (unsigned long long)from * rb + (off - (unsigned long long)starts[r] * rb);
      if (off + 16 <= end && (from < 0 || (s_off & 15) == 0)) {
        const uint4 v = from < 0 ? make_uint4(0, 0, 0, 0) : __ldcs((const uint4*)(src + s_off));
        __stcs((uint4*)(dst + off), v);
        continue;
      }
      // a chunk across a run boundary or off the source's alignment (rows of a width that is not a multiple of 16),
      // or the column's last bytes: byte by byte
      int rr = r;
      for (unsigned long long b = off; b < off + 16 && b < total; b++) {
        while (b >= run_end(rr)) rr++;
        const int f = prev[starts[rr]];
        dst[b] = f < 0 ? 0 : src[(unsigned long long)f * rb + (b - (unsigned long long)starts[rr] * rb)];
      }
    }
  }
}

// TransitionPenalty (allocation.go:283-292) of every candidate of the listed servers against their current allocation,
// the value CreateAllocation stores (wva_core.cuh alloc_final / sizer_setup); nil candidates keep value 0.  A candidate
// whose replica count was saturated to the int32 range compares as the saturated count.
__global__ void revalue_kernel(SysView s, CandView c, const int* rows, unsigned long long n_items) {
  const int A = s.n_acc;
  for (unsigned long long t = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; t < n_items;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    const int srv = rows[t / (unsigned)A], acc = (int)(t % (unsigned)A);
    const size_t idx = (size_t)srv * A + acc;
    const int st = c.state[idx];
    if (st == ALLOC_NONE) continue;
    Alloc b = alloc_none();
    b.state = st; b.num_replicas = c.num_replicas[idx]; b.cost = c.cost[idx];
    c.value[idx] = transition_penalty(s.srv_cur_acc[srv], s.srv_cur_replicas[srv], s.srv_cur_cost[srv], b, acc);
  }
}

}  // namespace wva
