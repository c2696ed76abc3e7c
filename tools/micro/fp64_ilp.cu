// Microbenchmark: FP64 DFMA throughput per SM as a function of warps per SM and independent chains per thread.
// Answers: what is the dependent-issue latency of DFMA on H100, and how many chains x warps saturate the pipe?
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_ilp fp64_ilp.cu ; run: ./fp64_ilp
#include <cstdio>
#include <cuda_runtime.h>

template <int C>
__global__ void chains(double* out, int iters, double a, double b) {
  double x[C];
#pragma unroll
  for (int c = 0; c < C; c++) x[c] = 1.0 + threadIdx.x * 1e-9 + c;
  long long t0 = clock64();
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
#pragma unroll
      for (int c = 0; c < C; c++) x[c] = fma(x[c], a, b);
    }
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int c = 0; c < C; c++) s += x[c];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s + (double)(t1 - t0) * 1e-300;
  if (threadIdx.x == 0 && blockIdx.x == 0) ((long long*)out)[gridDim.x * blockDim.x] = t1 - t0;
}

template <int C>
void run(int warps_per_sm, int sms, double* d_out) {
  const int iters = 4096;
  chains<C><<<sms, warps_per_sm * 32>>>(d_out, iters, 0.999999, 1e-7);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  chains<C><<<sms, warps_per_sm * 32>>>(d_out, iters, 0.999999, 1e-7);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  long long cyc; cudaMemcpy(&cyc, (long long*)d_out + (size_t)sms * warps_per_sm * 32, 8, cudaMemcpyDeviceToHost);
  const double fmas = (double)iters * 8 * C;                 // per thread
  const double per_sm_per_clk = fmas * warps_per_sm * 32 / (double)cyc;
  printf("warps/SM %2d chains %d : %7.2f cycles per dependent DFMA step, %6.2f DFMA lanes/clk/SM, %6.2f TDFMA/s\n", warps_per_sm, C,
         (double)cyc / (iters * 8.0), per_sm_per_clk, fmas * warps_per_sm * 32 * sms / (ms * 1e-3) / 1e12);
}

int main() {
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double* d; cudaMalloc(&d, (size_t)sms * 1024 * 8 + 64);
  for (int w : {4, 8, 12, 16, 32}) {
    run<1>(w, sms, d); run<2>(w, sms, d); run<4>(w, sms, d); run<8>(w, sms, d);
  }
  return 0;
}
