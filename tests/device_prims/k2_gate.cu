// TEST INFRASTRUCTURE ONLY — the error-word gate of the k2 chain (csrc/k2_history_kernel.cuh): the product's
// k2_keys_kernel, then k2_resolve_kernel and k2_slot_kernel with in.gate pointing at the error word, as the
// wva_ingest_v2 analyze graph launches them.  Built by tests/test_k2_gate.py with the product's flags; never linked into
// the product.  One history group with one model group, one accelerator, one store slot; four replicas, three of which
// observe (queue >= threshold, tokens in use > 0).
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/k2_history_kernel.cuh"
#include <cuda_runtime.h>

using namespace wva;

// err_value: what the error word holds when the resolve and slot kernels run (the keys pass finds nothing wrong here;
// a set word stands for a cycle it rejected).  Outputs: count [3], values [30] of the three keys after the cycle, the
// slot's effective capacity and the replicas' k2.  Returns 0, or 1 on a CUDA error.
extern "C" int k2_gate(int err_value, int* count_out, double* values_out, long long* slot_eff_out, long long* rep_k2_out) {
  const int P = 4;
  const int h_mo[2] = {0, 1}, h_m[1] = {0}, h_ao[2] = {0, 1}, h_a[1] = {0}, h_mg[1] = {0}, h_off[2] = {0, P};
  const long long h_tk[P] = {1000, 1000, 1000, 1000}, h_used[P] = {500, 600, 0, 700}, h_q[P] = {10, 10, 10, 10};
  const double h_ai[P] = {100, 100, 100, 100}, h_ao_t[P] = {50, 50, 50, 50};
  const int h_acc[P] = {0, 0, 0, 0}, h_slot[P] = {0, 0, 0, 0};
  const long long h_B[1] = {0}, h_S[1] = {0};
  const double h_qthr[1] = {5.0}, h_kvthr[1] = {0.8};
  char* d = nullptr;
  if (cudaMalloc(&d, 1 << 16) != cudaSuccess) return 1;
  cudaMemset(d, 0, 1 << 16);
  size_t off = 0;
  auto put = [&](const void* src, size_t n) { char* p = d + off; cudaMemcpy(p, src, n, cudaMemcpyHostToDevice); off += (n + 255) & ~(size_t)255; return p; };
  auto take = [&](size_t n) { char* p = d + off; off += (n + 255) & ~(size_t)255; return p; };
  K2Reg reg{1, (const int*)put(h_mo, 8), (const int*)put(h_m, 4), (const int*)put(h_ao, 8), (const int*)put(h_a, 4),
            (const int*)put(h_mg, 4)};
  K2State st{(double*)take(3 * K2_WINDOW * 8), (int*)take(12), (int*)take(12)};
  K2In in = {};
  in.G = 1; in.n_slots = 1; in.n_out = 0; in.model_replica_off = (const int*)put(h_off, 8);
  in.tk = (const long long*)put(h_tk, 8 * P); in.used = (const long long*)put(h_used, 8 * P);
  in.queue = (const long long*)put(h_q, 8 * P); in.avg_in = (const double*)put(h_ai, 8 * P);
  in.avg_out = (const double*)put(h_ao_t, 8 * P); in.acc = (const int*)put(h_acc, 4 * P); in.slot = (const int*)put(h_slot, 4 * P);
  in.out_pos = nullptr; in.slot_B = (const long long*)put(h_B, 8); in.slot_S = (const long long*)put(h_S, 8);
  in.q_thr = (const double*)put(h_qthr, 8); in.kv_thr = (const double*)put(h_kvthr, 8);
  K2Out out{(long long*)take(8 * P), (long long*)take(8 * P), nullptr, (int*)take(4), (long long*)take(8), (int*)take(4 * P),
            (int*)take(4)};
  in.gate = out.err;
  cudaMemset(out.slot_last, 0xff, 4);
  k2_keys_kernel<<<1, 256>>>(reg, in, out.rep_key, out.err);
  cudaMemcpy(out.err, &err_value, 4, cudaMemcpyHostToDevice);
  k2_resolve_kernel<<<1, K2_WARPS * 32>>>(reg, in, st, out);
  k2_slot_kernel<<<1, 256>>>(1, out.slot_last, out.rep_eff, out.slot_eff, out.err);
  int rc = cudaDeviceSynchronize() != cudaSuccess || cudaGetLastError() != cudaSuccess;
  if (!rc) {
    cudaMemcpy(count_out, st.count, 12, cudaMemcpyDeviceToHost);
    cudaMemcpy(values_out, st.vals, 3 * K2_WINDOW * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(slot_eff_out, out.slot_eff, 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(rep_k2_out, out.rep_k2, 8 * P, cudaMemcpyDeviceToHost);
  }
  cudaFree(d);
  return rc;
}
