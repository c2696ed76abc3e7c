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
enum { MARK_RESIZE = 1,     // a sizing input changed: the load, or the current accelerator of a keepAccelerator server
       MARK_REVALUE = 2 };  // the current allocation changed: TransitionPenalty (every candidate's value) changed

__device__ __forceinline__ bool bits_differ(float a, float b) { return __float_as_uint(a) != __float_as_uint(b); }

// One pass over the S servers: the bitwise diff of the six per-cycle columns of `nu` against the resident `res`, the
// write of `nu` over `res`, and the marks of the servers in [lo, hi) (the rank's block; every rank holds every column).
// grid_marks[srv] = 1 when the load changed: a server's grid rows read no other per-cycle column (grid_setup), and they
// accumulate until the next wva_grid_run / wva_grid_update, apart from the sizing marks.
__global__ void classify_servers_kernel(SysView res, SysView nu, int lo, int hi, unsigned char* marks,
                                        unsigned char* grid_marks) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= res.n_servers) return;
  const float arr = nu.srv_arrival[i], cost = nu.srv_cur_cost[i];
  const int in_tok = nu.srv_in_tokens[i], out_tok = nu.srv_out_tokens[i];
  const int acc = nu.srv_cur_acc[i], rep = nu.srv_cur_replicas[i];
  const bool load = bits_differ(arr, res.srv_arrival[i]) || in_tok != res.srv_in_tokens[i] ||
                    out_tok != res.srv_out_tokens[i];
  const bool acc_moved = acc != res.srv_cur_acc[i];
  const bool alloc = acc_moved || rep != res.srv_cur_replicas[i] || bits_differ(cost, res.srv_cur_cost[i]);
  // the candidate set depends on the current accelerator when keepAccelerator is set (server.go:70-82)
  const bool resize = load || (acc_moved && res.srv_keep_acc[i]);
  const_cast<float*>(res.srv_arrival)[i] = arr;
  const_cast<int*>(res.srv_in_tokens)[i] = in_tok;
  const_cast<int*>(res.srv_out_tokens)[i] = out_tok;
  const_cast<int*>(res.srv_cur_acc)[i] = acc;
  const_cast<int*>(res.srv_cur_replicas)[i] = rep;
  const_cast<float*>(res.srv_cur_cost)[i] = cost;
  if (i >= lo && i < hi && (resize || alloc)) marks[i] |= (resize ? MARK_RESIZE : 0) | (alloc ? MARK_REVALUE : 0);
  if (i >= lo && i < hi && load) grid_marks[i] = 1;
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
