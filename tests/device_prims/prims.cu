// TEST INFRASTRUCTURE ONLY — the chain solvers' division primitives (csrc/wva_core.cuh, lockstep_solve.cuh,
// saturation_kernel.cuh) run on the device over every float32 divisor and checked against the device's IEEE division.
// Built by tests/test_device_prims.py with the product's flags; never linked into the product.
//
// Every check is a grid-stride loop that reduces on the device to a PrimRes per divisor class: items checked, items
// failing, a maximum and the first 16 failing operands.  The host entry points return 0, or 1 on a CUDA error.
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/wva_core.cuh"
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/lockstep_solve.cuh"
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/saturation_kernel.cuh"
#include <cuda_runtime.h>

using namespace wva;

// divisor classes of a positive float32 mu
enum { CLS_SUB = 0, CLS_E1 = 1, CLS_HIGH = 2, CLS_INF = 3, NCLS = 4 };   // (0, 2^-126), [2^-126, 2^126], (2^126, 2^128), inf

struct PrimRes {
  unsigned long long n, fail, flagged;   // checked, failing, other events (check-specific)
  unsigned long long skipped;            // divisors the check leaves out (not E1 divisors)
  unsigned long long max_bits;           // maximum of a non-negative value, as its bit pattern
  unsigned long long first[16][2];       // operands of the first failures (bit patterns)
  unsigned lo, hi;                       // smallest / largest float32 bits with a flagged event
};

__device__ __forceinline__ int mu_class(unsigned b) {
  if (b < 0x00800000u) return CLS_SUB;
  if (b <= 0x7E800000u) return CLS_E1;
  if (b < 0x7F800000u) return CLS_HIGH;
  return CLS_INF;
}

__device__ __forceinline__ void res_fail(PrimRes* r, unsigned long long a, unsigned long long b) {
  const unsigned long long k = atomicAdd(&r->fail, 1ull);
  if (k < 16) { r->first[k][0] = a; r->first[k][1] = b; }
}

// positive float32 bit patterns [1, 0x7F800000] (subnormals, normals, +inf) in a grid-stride loop
#define FOR_ALL_MU(b) \
  for (unsigned long long i_ = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i_ < 0x7F800000ull; \
       i_ += (unsigned long long)gridDim.x * blockDim.x) \
    if (const unsigned b = (unsigned)(i_ + 1); true)

// ---- check 1: the seed f_rcp_approx against the correctly rounded float32 reciprocal ----------------------------------
// max_bits: largest ulp distance where both are normal; flagged: the seed is 0 or inf where 1/mu is a finite non-zero
// real (flushed), with lo/hi the range of such mu
__global__ void seed_kernel(PrimRes* res) {
  unsigned long long n[NCLS] = {}, fl[NCLS] = {}, mx[NCLS] = {};
  unsigned lo[NCLS], hi[NCLS];
  for (int c = 0; c < NCLS; c++) { lo[c] = 0xffffffffu; hi[c] = 0; }
  FOR_ALL_MU(b) {
    const float m = __uint_as_float(b);
    const float a = f_rcp_approx(m), ref = __frcp_rn(m);
    const unsigned ab = __float_as_uint(a), rb = __float_as_uint(ref);
    const int c = mu_class(b);
    n[c]++;
    const bool ref_real = c != CLS_INF;                               // 1/mu finite and non-zero
    if (ref_real && (ab == 0u || ab == 0x7F800000u)) { fl[c]++; lo[c] = min(lo[c], b); hi[c] = max(hi[c], b); }
    const bool normal = ab >= 0x00800000u && ab < 0x7F800000u && rb >= 0x00800000u && rb < 0x7F800000u;
    if (normal) {
      const unsigned long long d = ab > rb ? ab - rb : rb - ab;
      mx[c] = d > mx[c] ? d : mx[c];
    }
  }
  for (int c = 0; c < NCLS; c++) {
    atomicAdd(&res[c].n, n[c]);
    atomicAdd(&res[c].flagged, fl[c]);
    atomicMax(&res[c].max_bits, mx[c]);
    if (fl[c]) { atomicMin(&res[c].lo, lo[c]); atomicMax(&res[c].hi, hi[c]); }
  }
}

// ---- check 2: r = rcp_f32den(m, mu) and its exact residual 1 - mu r ---------------------------------------------------
// (mu has 24 significant bits and r 53, so fma(-mu, r, 1) is exact while |1 - mu r| < 2^-30.)
// fail: |residual| > 2^-40 (or not a number); flagged: |residual| + 3 u > 2^-39.99, the bound step_div's q0 relies on;
// max_bits: largest |residual|.  Only divisors the solvers use E1 for (e1_divisor) are checked; the others are skipped.
__global__ void rcp_kernel(PrimRes* res) {
  unsigned long long n[NCLS] = {}, fl[NCLS] = {}, mx[NCLS] = {}, skip[NCLS] = {};
  const double lim = 0x1p-40, lim_q0 = 0x1.fe4p-40 /* 2^-39.99 rounded down */, u3 = 3.0 * 0x1p-53;
  FOR_ALL_MU(b) {
    const float m = __uint_as_float(b);
    const int c = mu_class(b);
    if (!e1_divisor(m)) { skip[c]++; continue; }
    const double mu = (double)m;
    const double r = rcp_f32den(m, mu);
    const double e = fabs(__fma_rn(-mu, r, 1.0));
    n[c]++;
    if (!(e <= lim)) res_fail(&res[c], b, (unsigned long long)__double_as_longlong(r));
    if (!(e + u3 <= lim_q0)) fl[c]++;
    const unsigned long long eb = e == e ? (unsigned long long)__double_as_longlong(e) : 0x7FF0000000000000ull;
    mx[c] = eb > mx[c] ? eb : mx[c];
  }
  for (int c = 0; c < NCLS; c++) {
    atomicAdd(&res[c].n, n[c]);
    atomicAdd(&res[c].flagged, fl[c]);
    atomicMax(&res[c].max_bits, mx[c]);
    atomicAdd(&res[c].skipped, skip[c]);
  }
}

// ---- check 3: quotients against __ddiv_rn, bit for bit -----------------------------------------------------------------
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {   // splitmix64 finaliser
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// a double with exponent in [lo, hi] (unbiased) and a random significand
__device__ __forceinline__ double rand_double(unsigned long long h, int lo, int hi) {
  const int e = lo + (int)((h >> 52) % (unsigned long long)(hi - lo + 1));
  return __longlong_as_double((long long)(((unsigned long long)(e + 1023) << 52) | (h & 0xFFFFFFFFFFFFFull)));
}
// dividends over the E3 window [2^-500, 2^500): both edges, all-ones significands, two random ones
__device__ __forceinline__ double window_x(int k, unsigned b) {
  switch (k) {
    case 0: return 0x1p-500;                                   // lower edge
    case 1: return 0x1.fffffffffffffp-500;                     // lower binade, all-ones significand
    case 2: return 0x1.fffffffffffffp+499;                     // largest value below 2^500
    case 3: return 0x1.fffffffffffffp+0;
    default: return rand_double(mix64(((unsigned long long)b << 3) | (unsigned)k), -500, 499);
  }
}
constexpr int NX = 6;

// the solvers' quotient x / mu for one divisor: E1 where e1_divisor holds, else the IEEE division (chain_next)
__device__ __forceinline__ double solver_div(double x, float m) {
  const double mu = (double)m;
  return e1_divisor(m) ? div_f32den(x, mu, rcp_f32den(m, mu)) : d_div(x, mu);
}

// div_f32den: every positive float32 mu x NX dividends; flagged counts the quotients taken by E1
__global__ void div_kernel(PrimRes* res) {
  unsigned long long n[NCLS] = {}, fl[NCLS] = {};
  FOR_ALL_MU(b) {
    const float m = __uint_as_float(b);
    const int c = mu_class(b);
    const bool e1 = e1_divisor(m);
    for (int k = 0; k < NX; k++) {
      const double x = window_x(k, b);
      const double q = solver_div(x, m), ref = __ddiv_rn(x, (double)m);
      n[c]++;
      fl[c] += e1;
      if (__double_as_longlong(q) != __double_as_longlong(ref)) res_fail(&res[c], b, (unsigned long long)__double_as_longlong(x));
    }
  }
  for (int c = 0; c < NCLS; c++) { atomicAdd(&res[c].n, n[c]); atomicAdd(&res[c].flagged, fl[c]); }
}

// step_div (lockstep_solve.cuh): p and lambda with x = RN(p lambda) inside the window; lambda a float32 value.  Pairs of
// (p, lambda): all-ones significands, powers of two and random ones, x near both window edges and in the middle.
__device__ __forceinline__ void step_operands(int k, unsigned b, double& p, double& lam) {
  const unsigned long long h = mix64(((unsigned long long)b << 3) | (unsigned)k | 0x8000000000000000ull);
  const float l32 = __uint_as_float((0x3F800000u | (unsigned)(h & 0x7FFFFFu)) - (((unsigned)(h >> 40) % 40u) << 23));
  switch (k) {
    case 0: lam = (double)__uint_as_float(0x3FFFFFFFu); p = 0x1.fffffffffffffp-501; break;        // x just above 2^-500
    case 1: lam = (double)__uint_as_float(0x3F7FFFFFu); p = 0x1.fffffffffffffp+499; break;        // x just below 2^500
    case 2: lam = (double)__uint_as_float(0x3FFFFFFFu); p = 0x1.fffffffffffffp+0; break;
    case 3: lam = 1.0; p = 0x1p-500; break;
    default: lam = (double)l32; p = rand_double(h, -440, 440); break;
  }
}
__global__ void step_kernel(PrimRes* res) {
  unsigned long long n[NCLS] = {}, fl[NCLS] = {};
  FOR_ALL_MU(b) {
    const float m = __uint_as_float(b);
    const int c = mu_class(b);
    if (!e1_divisor(m)) { fl[c] += NX; continue; }   // step_div runs only for pairs whose every divisor is an E1 divisor
    const double mu = (double)m, r = rcp_f32den(m, mu);
    for (int k = 0; k < NX; k++) {
      double p, lam;
      step_operands(k, b, p, lam);
      const double x = __dmul_rn(p, lam);
      if (!in_window(x)) { res_fail(&res[c], b, (unsigned long long)__double_as_longlong(p)); continue; }   // operand bug
      int mn = 0x7fffffff, mx = 0;
      const double q = step_div(p, lam, d_mul(lam, r), mu, r, mn, mx), ref = __ddiv_rn(x, mu);
      n[c]++;
      if (__double_as_longlong(q) != __double_as_longlong(ref) || mn != d_hi(x) || mx != d_hi(x))
        res_fail(&res[c], b, (unsigned long long)__double_as_longlong(p));
    }
  }
  for (int c = 0; c < NCLS; c++) { atomicAdd(&res[c].n, n[c]); atomicAdd(&res[c].flagged, fl[c]); }
}

// div_markstein2 (E2) with y53 = __drcp_rn(y): n random pairs in the window
__global__ void markstein_kernel(PrimRes* res, unsigned long long n_pairs, unsigned long long seed) {
  unsigned long long n = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long h1 = mix64(seed ^ (2 * i)), h2 = mix64(seed ^ (2 * i + 1));
    const double x = rand_double(h1, -500, 499);
    double y = rand_double(h2, -500, 499);
    if ((i & 15) == 0) y = __longlong_as_double(__double_as_longlong(y) | 0xFFFFFFFFFFFFFll);   // all-ones significand
    if ((i & 15) == 1) y = __longlong_as_double(__double_as_longlong(y) & ~0xFFFFFFFFFFFFFll);  // power of two
    const double q = div_markstein2(x, y, __drcp_rn(y)), ref = __ddiv_rn(x, y);
    n++;
    if (__double_as_longlong(q) != __double_as_longlong(ref))
      res_fail(res, (unsigned long long)__double_as_longlong(x), (unsigned long long)__double_as_longlong(y));
  }
  atomicAdd(&res->n, n);
}

// div_small_int (saturation_kernel.cuh): every n in [1, 2^24) with a random x in the window, and with x = 0
__global__ void small_int_kernel(PrimRes* res, unsigned long long seed) {
  unsigned long long cnt = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < (1ull << 24) - 1;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const int n = (int)i + 1;
    const double xs[3] = {rand_double(mix64(seed ^ i), -500, 499), 0.0, (double)(n - 1)};
    for (int k = 0; k < 3; k++) {
      const double q = div_small_int(xs[k], n), ref = __ddiv_rn(xs[k], (double)n);
      cnt++;
      if (__double_as_longlong(q) != __double_as_longlong(ref)) res_fail(res, (unsigned long long)n, (unsigned long long)__double_as_longlong(xs[k]));
    }
  }
  atomicAdd(&res->n, cnt);
}

// ---- anchor: the device's __ddiv_rn results themselves, for comparison with IEEE division on the host ----------------
__global__ void anchor_kernel(const double* x, const double* y, double* q, unsigned long long n) {
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x)
    q[i] = __ddiv_rn(x[i], y[i]);
}

// ---- host entry points -------------------------------------------------------------------------------------------------
namespace {
constexpr int kBlocks = 132 * 8, kThreads = 256;

template <class Launch>
int run(PrimRes* host, int n_res, Launch launch) {
  PrimRes* d = nullptr;
  if (cudaMalloc(&d, sizeof(PrimRes) * n_res) != cudaSuccess) return 1;
  for (int c = 0; c < n_res; c++) { host[c] = PrimRes{}; host[c].lo = 0xffffffffu; }
  int rc = 0;
  if (cudaMemcpy(d, host, sizeof(PrimRes) * n_res, cudaMemcpyHostToDevice) != cudaSuccess) rc = 1;
  if (!rc) {
    launch(d);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = 1;
  }
  if (!rc && cudaMemcpy(host, d, sizeof(PrimRes) * n_res, cudaMemcpyDeviceToHost) != cudaSuccess) rc = 1;
  cudaFree(d);
  return rc;
}
}  // namespace

extern "C" {
int prims_res_size() { return (int)sizeof(PrimRes); }
int prims_seed(PrimRes* r) { return run(r, NCLS, [](PrimRes* d) { seed_kernel<<<kBlocks, kThreads>>>(d); }); }
int prims_rcp(PrimRes* r) { return run(r, NCLS, [](PrimRes* d) { rcp_kernel<<<kBlocks, kThreads>>>(d); }); }
int prims_div(PrimRes* r) { return run(r, NCLS, [](PrimRes* d) { div_kernel<<<kBlocks, kThreads>>>(d); }); }
int prims_step(PrimRes* r) { return run(r, NCLS, [](PrimRes* d) { step_kernel<<<kBlocks, kThreads>>>(d); }); }
int prims_markstein(PrimRes* r, unsigned long long n, unsigned long long seed) {
  return run(r, 1, [&](PrimRes* d) { markstein_kernel<<<kBlocks, kThreads>>>(d, n, seed); });
}
int prims_small_int(PrimRes* r, unsigned long long seed) {
  return run(r, 1, [&](PrimRes* d) { small_int_kernel<<<kBlocks, kThreads>>>(d, seed); });
}
int prims_anchor(const double* x, const double* y, double* q, unsigned long long n) {
  double *dx = nullptr, *dy = nullptr, *dq = nullptr;
  const size_t bytes = n * sizeof(double);
  int rc = 0;
  if (cudaMalloc(&dx, bytes) != cudaSuccess || cudaMalloc(&dy, bytes) != cudaSuccess || cudaMalloc(&dq, bytes) != cudaSuccess) rc = 1;
  if (!rc && (cudaMemcpy(dx, x, bytes, cudaMemcpyHostToDevice) != cudaSuccess ||
              cudaMemcpy(dy, y, bytes, cudaMemcpyHostToDevice) != cudaSuccess)) rc = 1;
  if (!rc) {
    anchor_kernel<<<kBlocks, kThreads>>>(dx, dy, dq, n);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = 1;
  }
  if (!rc && cudaMemcpy(q, dq, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) rc = 1;
  cudaFree(dx); cudaFree(dy); cudaFree(dq);
  return rc;
}
}  // extern "C"
