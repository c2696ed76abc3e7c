// TEST INFRASTRUCTURE ONLY — div_rate, the branch-free service-rate division of csrc/wva_core.cuh, against the device's
// IEEE division __fdiv_rn.  Built by tests/test_rate_division.py with the product's flags; never linked into the product.
//
// Both checks reduce on the device to a RateRes: divisions compared, divisions left out, mismatches and the first 16
// mismatching operands.  The host entry points return 0, or 1 on a CUDA error.
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/wva_core.cuh"
#include <cuda_runtime.h>

using namespace wva;

struct RateRes {
  unsigned long long n, skipped, fail;
  unsigned long long first[16][2];   // (den bits << 32 | seed bits, nf) of the first mismatches
};

constexpr int NF_MAX = 1 << 16;      // the largest batch size (NLIMIT in capi.cu)

__device__ __forceinline__ void res_fail(RateRes* r, unsigned den, unsigned seed, float nf) {
  const unsigned long long k = atomicAdd(&r->fail, 1ull);
  if (k < 16) { r->first[k][0] = ((unsigned long long)den << 32) | seed; r->first[k][1] = (unsigned long long)nf; }
}

// Every den in [1, 2), every seed within seed_ulp ulps of RN(1/den) and every nf in [1, 2^16]: div_rate_seeded against
// __fdiv_rn.  No seed from rcp.approx enters, so the check covers whatever seed the device returns within that distance.
__global__ void seeded_kernel(RateRes* res, int seed_ulp) {
  unsigned long long n = 0;
  const unsigned long long items = (unsigned long long)(2 * seed_ulp + 1) << 23;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < items;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned db = 0x3F800000u | (unsigned)(i & 0x7FFFFFu);
    const int k = (int)(i >> 23) - seed_ulp;
    const float den = __uint_as_float(db);
    const unsigned sb = __float_as_uint(__frcp_rn(den)) + k;   // 1/den in (0.5, 1]: every neighbour is normal
    const float s = __uint_as_float(sb);
    float nf = 1.0f;
    for (int j = 0; j < NF_MAX; j++, nf += 1.0f) {
      const float q = div_rate_seeded(nf, den, s), ref = __fdiv_rn(nf, den);
      if (__float_as_uint(q) != __float_as_uint(ref)) res_fail(res, db, sb, nf);
    }
    n += NF_MAX;
  }
  atomicAdd(&res->n, n);
}

// Every den with the unbiased exponent e and every nf in [1, 2^16]: div_rate (the device's own seed) against __fdiv_rn
// where the quotient is an (E1) divisor; the other quotients are counted as skipped.  The quotient grows with nf, so the
// first nf past 2^126 ends a den's sweep.
__global__ void device_seed_kernel(RateRes* res, int e) {
  unsigned long long n = 0, skip = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < (1ull << 23);
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned db = ((unsigned)(e + 127) << 23) | (unsigned)i;
    const float den = __uint_as_float(db);
    float nf = 1.0f;
    int j = 0;
    for (; j < NF_MAX; j++, nf += 1.0f) {
      const float ref = __fdiv_rn(nf, den);
      if (!e1_divisor(ref)) break;
      const float q = div_rate(nf, den);
      if (__float_as_uint(q) != __float_as_uint(ref)) res_fail(res, db, __float_as_uint(f_rcp_approx(den)), nf);
    }
    n += j;
    skip += NF_MAX - j;
  }
  atomicAdd(&res->n, n);
  atomicAdd(&res->skipped, skip);
}

namespace {
constexpr int kBlocks = 132 * 8, kThreads = 256;

template <class Launch>
int run(RateRes* host, Launch launch) {
  RateRes* d = nullptr;
  if (cudaMalloc(&d, sizeof(RateRes)) != cudaSuccess) return 1;
  *host = RateRes{};
  int rc = 0;
  if (cudaMemcpy(d, host, sizeof(RateRes), cudaMemcpyHostToDevice) != cudaSuccess) rc = 1;
  if (!rc) {
    launch(d);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = 1;
  }
  if (!rc && cudaMemcpy(host, d, sizeof(RateRes), cudaMemcpyDeviceToHost) != cudaSuccess) rc = 1;
  cudaFree(d);
  return rc;
}
}  // namespace

extern "C" {
int rate_res_size() { return (int)sizeof(RateRes); }
int rate_div_seeded(RateRes* r, int seed_ulp) {
  return run(r, [&](RateRes* d) { seeded_kernel<<<kBlocks, kThreads>>>(d, seed_ulp); });
}
int rate_div_device_seed(RateRes* r, int e) {
  return run(r, [&](RateRes* d) { device_seed_kernel<<<kBlocks, kThreads>>>(d, e); });
}
}  // extern "C"
