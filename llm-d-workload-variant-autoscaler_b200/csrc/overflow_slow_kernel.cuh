// overflow_slow_kernel.cuh — device side of the slow exact path: CreateAllocation for the rare pairs whose chain
// overflows float64 (literal stored-p[] algorithm with the reference's rescale, one thread per pair).
#pragma once
#include "wva_core.cuh"
#include "solve_kernels.cuh"
#include "sizer_kernel.cuh"
#include <cuda_runtime.h>

namespace wva {

__global__ void __launch_bounds__(64) overflow_slow_kernel(SysView s, CandView out, const int* list, int n, int nmax,
                                                           double* pbuf, float* tabbuf, int* patho) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int pair = list[i];
  int srv = pair / s.n_acc, acc = pair % s.n_acc;
  SizerLane z;
  int lim = 0;
  if (sizer_setup(z, s, out, srv, acc, nmax, &lim) != SETUP_NEEDS_TABLE) return;
  float* tab = tabbuf + (size_t)i * nmax;
  double* p = pbuf + (size_t)i * ((size_t)nmax * (WVA_QUEUE_TO_BATCH + 1) + 1);
  model_fill_table(z.m, tab, 1, 0, 1);
  model_finish(z.m, tab, 1);
  bool live = sizer_begin(z, s, out);
  SolveStats st;
  bool bad = false;
  while (live) {
    literal_solve(z.m, z.cur_x, p, st, &bad);
    z.c.states = z.m.K + 1;
    live = sizer_on_solve(z, s, out, st);
  }
  if (bad) atomicAdd(patho, 1);
}

// Scratch for n literal solves of batch size <= nmax — p[0..K] (K + 1 doubles) and an N-entry float32 head table per
// item, item i at pbuf + i * (nmax * (WVA_QUEUE_TO_BATCH + 1) + 1) and tabbuf + i * nmax — handed out at most 1 GiB at a
// time: launch(first item, items, pbuf, tabbuf) enqueues one batch on `stream`.  0 on success.
template <class Launch>
static inline int32_t literal_scratch_batches(int n, int nmax, cudaStream_t stream, Launch launch) {
  const size_t p_len = (size_t)nmax * (WVA_QUEUE_TO_BATCH + 1) + 1;
  const size_t per_item = p_len * 8 + (size_t)nmax * 4;
  size_t batch = (size_t)(1ull << 30) / per_item;   // <= 1 GiB of scratch at a time
  if (batch < 1) batch = 1;
  if (batch > (size_t)n) batch = (size_t)n;
  double* pbuf = nullptr; float* tabbuf = nullptr;
  if (cudaMalloc(&pbuf, batch * p_len * 8) != cudaSuccess) return 1;
  if (cudaMalloc(&tabbuf, batch * (size_t)nmax * 4) != cudaSuccess) { cudaFree(pbuf); return 1; }
  int32_t rc = 0;
  for (size_t off = 0; off < (size_t)n; off += batch) {
    int cnt = (int)((size_t)n - off < batch ? (size_t)n - off : batch);
    launch((int)off, cnt, pbuf, tabbuf);
    if (cudaStreamSynchronize(stream) != cudaSuccess) { rc = 1; break; }
  }
  cudaFree(pbuf); cudaFree(tabbuf);
  return rc;
}

static inline int32_t run_overflow_slow_path(const SysView& s, const CandView& out, const int* d_list, int n,
                                             cudaStream_t stream, long long* launches) {
  // worst case N is not known here: re-derive it on the host side through a device reduction
  // would need another pass; the sizer already bounded N by its table limit (65536).
  int nmax_h = 0;
  int* d_nmax = nullptr;
  if (cudaMalloc(&d_nmax, 8) != cudaSuccess) return 1;
  cudaMemsetAsync(d_nmax, 0, 8, stream);
  unsigned long long n_pairs = (unsigned long long)s.n_servers * s.n_acc;
  max_batch_kernel<<<1024, 256, 0, stream>>>(s, n_pairs, d_nmax);
  (*launches)++;
  cudaMemcpyAsync(&nmax_h, d_nmax, 4, cudaMemcpyDeviceToHost, stream);
  cudaStreamSynchronize(stream);
  if (nmax_h < 1) nmax_h = 1;
  if (nmax_h > 65536) nmax_h = 65536;
  int32_t rc = literal_scratch_batches(n, nmax_h, stream, [&](int off, int cnt, double* pbuf, float* tabbuf) {
    overflow_slow_kernel<<<(cnt + 63) / 64, 64, 0, stream>>>(s, out, d_list + off, cnt, nmax_h, pbuf, tabbuf, d_nmax + 1);
    (*launches)++;
  });
  cudaFree(d_nmax);
  return rc;
}

}  // namespace wva
