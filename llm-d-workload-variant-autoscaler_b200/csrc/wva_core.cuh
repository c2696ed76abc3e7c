// wva_core.cuh — device core of the H100 WVA hot path: service-time closed forms,
// the state-dependent birth-death chain solver, the float32 bisection sizer and
// CreateAllocation, written as per-lane state machines.
//
// The same source compiles for the device (nvcc, sm_90a) and — for logic tests
// only (tests/host_emul) — for the host, where every wrapper below maps to the
// IEEE operation it stands for.  The product never runs the host build.
//
// Reference (paths relative to /root/reference):
//   pkg/analyzer/queueanalyzer.go:95-308   BuildModel / Analyze / Size / *Time / Eval*
//   pkg/analyzer/mm1modelstatedependent.go:38-116  computeStatistics / computeProbabilities
//   pkg/analyzer/utils.go:12-70            WithinTolerance / BinarySearch
//   pkg/core/allocation.go:27-155,251-292  CreateAllocation / zeroLoadAllocation / TransitionPenalty
//
// Exactness contract (DESIGN.md §3): every float32/float64 operation the reference
// performs is performed here with the same operands, order and rounding.  What is
// changed is only HOW a correctly-rounded result is obtained and WHICH provably
// no-op operations are skipped:
//   (E1) x / mu, mu a float32-valued double in [2^-126, 2^126]: q0 = x*r, rem = fma(-q0,mu,x),
//        q = fma(rem,r,q0) with r within 2^-40 of 1/mu is the correctly rounded
//        quotient, because a quotient by a 24-bit divisor is never closer than
//        2^-25 ulp to a rounding boundary while the perturbation is < 2^-26 ulp.
//        A pair with any mu_n outside that range (e1_divisor, PairModel::e1_ok) is solved
//        by the per-lane chain, which divides by such a mu_n with the IEEE division.
//   (E2) p / sum: two Markstein correction steps with the correctly rounded
//        reciprocal (__drcp_rn) give the correctly rounded quotient.
//   (E3) outside the exponent window [2^-500, 2^500) the plain IEEE division is used.
//   (E4) the chain is left early once every remaining term provably cannot change
//        any accumulator (adding t to s with s + t == s, all later t' <= t).
//   (E5) p[] is not stored: pass 1 finds sum, pass 2 recomputes the recurrence and
//        accumulates on the normalised p[i] exactly like the reference (quirk Q4).
//   (E12) only float32 statistics leave a solve: a solve may take its float64 values from
//        one head pass and a closed-form tail (fast_solve_finish) when an error enclosure
//        of the reference's float64 values proves that their float32 roundings are the
//        reference's; otherwise the lane is re-solved by the exact solver.
#pragma once
#include <stdint.h>
#include <math.h>
#include <float.h>

#if defined(__CUDACC__)
#define WVA_HD __host__ __device__ __forceinline__
#define WVA_D __device__ __forceinline__
#else
#define WVA_HD inline
#define WVA_D inline
#include <cmath>
#include <cstring>
#endif

namespace wva {

// ------------------------------------------------------------------ IEEE wrappers
// Device: *_rn intrinsics are never contracted into FMAs by nvcc.
// Host (tests only): plain operators; the test build uses -ffp-contract=off.
#if defined(__CUDA_ARCH__)
WVA_HD float f_add(float a, float b) { return __fadd_rn(a, b); }
WVA_HD float f_sub(float a, float b) { return __fsub_rn(a, b); }
WVA_HD float f_mul(float a, float b) { return __fmul_rn(a, b); }
WVA_HD float f_div(float a, float b) { return __fdiv_rn(a, b); }
WVA_HD double d_add(double a, double b) { return __dadd_rn(a, b); }
WVA_HD double d_sub(double a, double b) { return __dsub_rn(a, b); }
WVA_HD double d_mul(double a, double b) { return __dmul_rn(a, b); }
WVA_HD double d_div(double a, double b) { return __ddiv_rn(a, b); }
WVA_HD double d_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
WVA_HD double d_rcp(double a) { return __drcp_rn(a); }
WVA_HD float f_rcp_approx(float a) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }
WVA_HD long long d_bits(double a) { return __double_as_longlong(a); }
WVA_HD int d_hi(double a) { return __double2hiint(a); }
#else
WVA_HD float f_add(float a, float b) { return a + b; }
WVA_HD float f_sub(float a, float b) { return a - b; }
WVA_HD float f_mul(float a, float b) { return a * b; }
WVA_HD float f_div(float a, float b) { return a / b; }
WVA_HD double d_add(double a, double b) { return a + b; }
WVA_HD double d_sub(double a, double b) { return a - b; }
WVA_HD double d_mul(double a, double b) { return a * b; }
WVA_HD double d_div(double a, double b) { return a / b; }
WVA_HD double d_fma(double a, double b, double c) { return fma(a, b, c); }
WVA_HD double d_rcp(double a) { return 1.0 / a; }
// rcp.approx.ftz: a subnormal input is read as 0 and a subnormal result is returned as 0
WVA_HD float f_rcp_approx(float a) {
  if (fabsf(a) < FLT_MIN) a = copysignf(0.0f, a);
  const float r = 1.0f / a;
  return fabsf(r) < FLT_MIN ? copysignf(0.0f, r) : r;
}
WVA_HD long long d_bits(double a) { long long b; memcpy(&b, &a, 8); return b; }
WVA_HD int d_hi(double a) { return (int)(d_bits(a) >> 32); }
#endif

// exponent window test (E3): 2^-500 <= |x| < 2^500, false for 0/inf/nan/subnormal
WVA_HD bool in_window(double x) {
  unsigned e = ((unsigned)d_hi(x) >> 20) & 0x7ffu;
  return (e - 523u) < 1000u;
}

// (E1) correctly rounded x / mu for float32-valued mu, r ~ 1/mu (rel. err <= 2^-40)
WVA_HD double div_f32den(double x, double mu, double r) {
  double q0 = d_mul(x, r);
  double rem = d_fma(-q0, mu, x);
  return d_fma(rem, r, q0);
}
// one Newton step on a float32 seed s of 1/mu
WVA_HD double rcp_refine(float s, double mu) {
  double r0 = (double)s;
  double e = d_fma(-mu, r0, 1.0);
  return d_fma(r0, e, r0);
}
// reciprocal of a float32-valued double, for mu in [2^-126, 2^126] only (e1_divisor).  There the seed rcp.approx.ftz.f32
// is within 1 ulp of RN(1/mu) and |1 - mu r| <= 2^-46.56 (H100, every float32 mu: tests/test_device_prims.py).  Outside,
// 1/mu is not a float32 normal number and the seed flushes: a subnormal mu reads as 0 (seed inf, r = NaN), mu > 2^126
// has a subnormal 1/mu (seed 0, r = 0), and mu = inf gives r = NaN.
WVA_HD double rcp_f32den(float m32, double mu) { return rcp_refine(f_rcp_approx(m32), mu); }
// (double)v for a positive normal float32 v, as every (E1) divisor and its rcp seed are (e1_divisor: [2^-126, 2^126]).  The
// exponent is rebiased and the significand shifted on the integer pipe — the same bits as the conversion, which on H100
// issues to the FP64 pipe at a quarter of the DFMA rate (CUDA C++ Programming Guide, arithmetic instruction throughput).
WVA_HD double f32pos_to_d(float v) {
#if defined(__CUDA_ARCH__)
  const unsigned b = __float_as_uint(v);
  return __hiloint2double((int)((b >> 3) + 0x38000000u), (int)(b << 29));
#else
  return (double)v;
#endif
}
// rcp_f32den of an (E1) divisor with both conversions on the integer pipe: the same bits as rcp_f32den(m32, (double)m32)
WVA_HD double rcp_f32den_e1(float m32, double mu) {
  const double r0 = f32pos_to_d(f_rcp_approx(m32));
  return d_fma(r0, d_fma(-mu, r0, 1.0), r0);
}
// mu in [2^-126, 2^126]: the divisors (E1) holds for
WVA_HD bool e1_divisor(float m32) {
#if defined(__CUDA_ARCH__)
  const unsigned b = __float_as_uint(m32);
#else
  unsigned b; memcpy(&b, &m32, 4);
#endif
  return b - 0x00800000u <= 0x7E800000u - 0x00800000u;
}
// (E2) correctly rounded x / y with y53 = RN(1/y)
WVA_HD double div_markstein2(double x, double y, double y53) {
  double q0 = d_mul(x, y53);
  double r0 = d_fma(-q0, y, x);
  double q1 = d_fma(r0, y53, q0);
  double r1 = d_fma(-q1, y, x);
  return d_fma(r1, y53, q1);
}

// ------------------------------------------------------------------ constants
// pkg/analyzer/queueanalyzer.go:8-14, utils.go:8-9, pkg/config/defaults.go:18,21
#define WVA_EPSILON 0.001f
#define WVA_STABILITY_SAFETY 0.1f
#define WVA_BS_EPSILON 1e-6f
#define WVA_MAX_ITER 100
#define WVA_QUEUE_TO_BATCH 10
#define WVA_ACCEL_PENALTY 0.1f

enum { ALLOC_NONE = 0, ALLOC_ACC = 1, ALLOC_EMPTY = 2 };

// ------------------------------------------------------------------ service model
// Per-(server, accelerator) queue model: the n-independent subexpressions of
// IterationTime/PrefillTime/DecodeTime are hoisted; each is the same float32 value
// the reference recomputes on every call, so results are bit-identical.
struct PairModel {
  float alpha, beta, gamma;
  float in_tok, out_tok;
  float slope;      // Beta*tokensCompute + Gamma*tokensMemory   (queueanalyzer.go:262-264)
  float pre_c;      // (Beta+Gamma)*AvgInputTokens               (queueanalyzer.go:272)
  float dec_c;      // Gamma*(AvgInputTokens+AvgOutputTokens/2)  (queueanalyzer.go:278)
  int N, K;
  float lambda_min, lambda_max;  // Size(): RateRange.Min/1000, RateRange.Max/1000
  float rate_max;                // RateRange.Max (req/s)
  int e1_ok;                     // every mu_n is an (E1) divisor; else the pair is solved by the per-lane chain (chain_step)
  // head table: mu_n as float32 at tab[n*stride], n in [0,N); nullptr: mu_n = serv_rate(n + 1) (model_rate)
  const float* tab;
  int stride;
  int mono;         // mu is non-decreasing on [mono, N-1]
  double mu_last, r_last;
};

WVA_HD void model_init(PairModel& m, float alpha, float beta, float gamma, int in_tok, int out_tok, int N) {
  m.alpha = alpha; m.beta = beta; m.gamma = gamma;
  m.in_tok = (float)in_tok; m.out_tok = (float)out_tok;
  float tc = f_div(f_add(m.in_tok, m.out_tok), f_add(m.out_tok, 1.0f));
  float tm = f_add(m.in_tok, f_div(m.out_tok, 2.0f));
  m.slope = f_add(f_mul(beta, tc), f_mul(gamma, tm));
  m.pre_c = f_mul(f_add(beta, gamma), m.in_tok);
  m.dec_c = f_mul(gamma, tm);
  m.N = N;
  m.K = N + N * WVA_QUEUE_TO_BATCH;
}
// queueanalyzer.go:261-265
WVA_HD float iteration_time(const PairModel& m, float n) { return f_add(m.alpha, f_mul(n, m.slope)); }
// queueanalyzer.go:268-273
WVA_HD float prefill_time(const PairModel& m, float n) {
  if (m.in_tok == 0.0f) return 0.0f;
  return f_add(iteration_time(m, n), m.pre_c);
}
// queueanalyzer.go:276-279
WVA_HD float decode_time(const PairModel& m, float n) {
  return f_add(f_add(iteration_time(m, n), m.beta), m.dec_c);
}
// What the service rate of a batch size needs of its model (RateTable in lockstep_solve.cuh holds it in registers)
struct RateCoef { float alpha, slope, beta, pre_c, dec_c, in_tok, out_tok; };
WVA_HD RateCoef rate_coef(const PairModel& m) { return {m.alpha, m.slope, m.beta, m.pre_c, m.dec_c, m.in_tok, m.out_tok}; }
// queueanalyzer.go:100-104: servRate[n-1] for the float32 batch size nf = n (prefill_time, decode_time spelled out)
WVA_HD float serv_rate_nf(const RateCoef& c, float nf) {
  const float it = f_add(c.alpha, f_mul(nf, c.slope));
  const float pre = c.in_tok == 0.0f ? 0.0f : f_add(it, c.pre_c);
  const float dec = f_mul(c.out_tok, f_add(f_add(it, c.beta), c.dec_c));
  return f_div(nf, f_add(pre, dec));
}
WVA_HD float serv_rate(const PairModel& m, int n) { return serv_rate_nf(rate_coef(m), (float)n); }
// mu_n (n in [0, N)) of a model: its head table, or serv_rate itself for a model without one (m.tab == nullptr: the pool
// sizer and the deferred grid pass compute their rates instead of storing them)
WVA_HD float model_rate(const PairModel& m, int n) { return m.tab ? m.tab[(size_t)n * m.stride] : serv_rate(m, n + 1); }

// BuildModel (queueanalyzer.go:95-124): fills the head table for entries
// [first, N) step `step` (so a warp can fill one table cooperatively).
WVA_HD void model_fill_table(const PairModel& m, float* tab, int stride, int first, int step) {
  for (int n = first; n < m.N; n += step) tab[(size_t)n * stride] = serv_rate(m, n + 1);
}
// RateRange of BuildModel from the first and last service rate r0, rl, and Size()'s lambda range
WVA_HD void model_set_range(PairModel& m, float r0, float rl) {
  float lmin = f_mul(r0, WVA_EPSILON);                       // queueanalyzer.go:107
  float lmax = f_mul(rl, f_sub(1.0f, WVA_EPSILON));          // queueanalyzer.go:108
  float rmin = f_mul(lmin, 1000.0f);                         // :109 RateRange{Min,Max}
  m.rate_max = f_mul(lmax, 1000.0f);
  m.lambda_min = f_div(rmin, 1000.0f);                       // Size(): queueanalyzer.go:189-190
  m.lambda_max = f_div(m.rate_max, 1000.0f);
}
// finish the model once the table is complete
WVA_HD void model_finish(PairModel& m, const float* tab, int stride) {
  m.tab = tab; m.stride = stride;
  float rl = tab[(size_t)(m.N - 1) * stride];
  model_set_range(m, tab[0], rl);
  int mono = 0;
  float nxt = rl;
  for (int n = m.N - 2; n >= 0; n--) {
    float cur = tab[(size_t)n * stride];
    if (!(cur <= nxt)) { mono = n + 1; break; }
    nxt = cur;
  }
  m.mono = mono;
  // mu is non-decreasing on [mono, N-1]: its ends bound it there, only the entries below mono are checked one by one
  int e1 = e1_divisor(tab[(size_t)mono * stride]) && e1_divisor(rl);
  for (int n = 0; n < mono; n++) e1 &= (int)e1_divisor(tab[(size_t)n * stride]);
  m.e1_ok = e1;
  m.mu_last = (double)rl;
  m.r_last = rcp_f32den(rl, m.mu_last);
}

// ------------------------------------------------------------------ chain solver
// One MM1ModelStateDependent.Solve(lambda, 1) (mm1modelstatedependent.go:28-116),
// advanced one birth-death state per step() so that the lanes of a warp can sit in
// different solves / passes / states (flattened SIMT loop).
struct SolveStats {  // float32 results of computeStatistics (mm1modelstatedependent.go:57-66)
  float avgNumInServers, avgNumInSystem, throughput, avgRespTime, avgServTime, avgWaitTime;
};

enum { CH_IDLE = 0, CH_PASS1 = 1, CH_PASS2 = 2, CH_DONE = 3, CH_OVERFLOW = 4 };

struct Chain {
  double lam, lamg;        // float64(lambda); lambda*(1+1e-6) guard for the monotone test
  double p;                // unnormalised p~[n]
  double sum, rsum;        // pass-1 total and its correctly rounded reciprocal
  double L, sumP, Lserv;   // pass-2 accumulators (avgNumInSystem, sumP, avgNumInServers)
  double pK;               // normalised p[K]
  float lambda;
  int n;                   // index of the state held in p
  int phase;
  bool tail_ok;            // lambda guard <= mu_last: terms are non-increasing on the tail
  bool sum_ok;             // sum inside the exponent window
  int states;              // states visited (instrumentation)
};

WVA_HD void chain_start(Chain& c, float lambda) {
  c.lambda = lambda;
  c.lam = (double)lambda;
  c.lamg = d_mul(c.lam, 1.000001);
  c.p = 1.0;
  c.sum = 1.0;  // sum += p[0]
  c.n = 0;
  c.phase = CH_PASS1;
  c.states = 0;
}

// p~[n+1] = p~[n]*lambda / mu_min(n,N-1)   (mm1modelstatedependent.go:77-83)
WVA_HD double chain_next(const Chain& c, const PairModel& m, bool* exit_ok) {
  double x = d_mul(c.p, c.lam);
  double mu, r;
  bool mono_ok;
  if (c.n < m.N - 1) {
    float m32 = model_rate(m, c.n);
    mu = (double)m32;
    r = rcp_f32den(m32, mu);
    mono_ok = (c.n >= m.mono) && (d_bits(c.lamg) <= d_bits(mu));
  } else {
    mu = m.mu_last; r = m.r_last;
    mono_ok = c.tail_ok;
  }
  *exit_ok = mono_ok;
  // (E1) only for an E1 divisor: for any other float32 mu the seed flushes and r is 0 or NaN, whose high word fails the
  // test (integer ops: this loop is FP64-bound)
  if (in_window(x) && (unsigned)d_hi(r) - 1u < 0x7FEFFFFFu) return div_f32den(x, mu, r);
  return d_div(x, mu);
}

// Advance one state.  Returns true when the solve has just completed (stats valid).
WVA_HD bool chain_step(Chain& c, const PairModel& m, SolveStats& st) {
  bool exit_ok;
  double pn1 = chain_next(c, m, &exit_ok);
  c.n++;
  c.states++;
  if (c.phase == CH_PASS1) {
    // overflow rescale branch of the reference (mm1modelstatedependent.go:84-89,96-104)
    // is taken by the slow-path kernel; here it is only detected.
    if (!(pn1 >= 0.0) || pn1 > DBL_MAX) { c.phase = CH_OVERFLOW; return true; }
    double s2 = d_add(c.sum, pn1);
    if (s2 > DBL_MAX) { c.phase = CH_OVERFLOW; return true; }
    bool done = (c.n == m.K) || (d_bits(pn1) == 0) || (exit_ok && d_bits(s2) == d_bits(c.sum));
    c.sum = s2;
    c.p = pn1;
    if (done) {
      // normalisation starts: p[0] = 1/sum; sumP = p[0]; L = 0
      c.sum_ok = in_window(c.sum);
      c.rsum = d_rcp(c.sum);
      double p0 = d_div(1.0, c.sum);
      c.sumP = p0;
      c.L = 0.0;
      c.Lserv = 0.0;
      c.p = 1.0;
      c.n = 0;
      c.phase = CH_PASS2;
    }
    return false;
  }
  // pass 2: p[i] = p~[i]/sum; avgNumInSystem += i*p[i]; sumP += p[i]   (:108-112, :47-55)
  int i = c.n;
  double pi;
  if (c.sum_ok && in_window(pn1)) pi = div_markstein2(pn1, c.sum, c.rsum);
  else pi = d_div(pn1, c.sum);
  double L2 = d_add(c.L, d_mul((double)i, pi));
  double sP2 = d_add(c.sumP, pi);
  if (i == m.N) c.Lserv = d_add(L2, d_mul(d_sub(1.0, sP2), (double)m.N));
  bool done = (i == m.K) || (d_bits(pn1) == 0);
  if (!done && exit_ok) {
    double tmax = d_mul((double)m.K, pi);
    done = (d_bits(d_add(L2, tmax)) == d_bits(L2)) && (d_bits(d_add(sP2, pi)) == d_bits(sP2));
  }
  c.L = L2; c.sumP = sP2; c.p = pn1;
  if (!done) return false;
  c.pK = (i == m.K) ? pi : 0.0;   // (E4) an early exit implies p[K] < 2^-53
  if (i < m.N) c.Lserv = d_add(c.L, d_mul(d_sub(1.0, c.sumP), (double)m.N));
  st.avgNumInServers = (float)c.Lserv;
  st.avgNumInSystem = (float)c.L;
  st.throughput = f_mul(c.lambda, f_sub(1.0f, (float)c.pK));
  st.avgRespTime = f_div(st.avgNumInSystem, st.throughput);
  st.avgServTime = f_div(st.avgNumInServers, st.throughput);
  float w = f_sub(st.avgRespTime, st.avgServTime);
  st.avgWaitTime = (w < 0.0f) ? 0.0f : w;
  c.phase = CH_DONE;
  return true;
}

// Literal MM1ModelStateDependent.Solve with stored p[] — the float64 overflow-rescale
// branches of computeProbabilities (mm1modelstatedependent.go:84-89,96-104) need every
// earlier p[i], so pairs that hit them (CH_OVERFLOW) are redone through this path.
// p must hold K+1 doubles.  `pathological` is set where the reference would never
// terminate (NaN / zero service rate); the oracle carries the same guard.
WVA_HD void literal_solve(const PairModel& m, float lambda, double* p, SolveStats& st, bool* pathological) {
  const int K = m.K, num = m.N;
  const double lam = (double)lambda;
  p[0] = 1.0;
  const double scale = DBL_MAX / (double)K;
  double sRate = 0.0;
  for (int n = 0; n < K; n++) {
    sRate = (double)model_rate(m, n < num ? n : num - 1);
    p[n + 1] = d_div(d_mul(p[n], lam), sRate);
    int guard = 0;
    while (p[n + 1] < 0.0 || p[n + 1] > DBL_MAX || p[n + 1] != p[n + 1]) {
      for (int i = 0; i <= n; i++) p[i] = d_div(p[i], scale);
      p[n + 1] = d_div(d_mul(p[n], lam), sRate);
      if (++guard > 64) { *pathological = true; break; }
    }
  }
  double sum = 0.0;
  for (int n = 0; n <= K; n++) {
    sum = d_add(sum, p[n]);
    if (sum < 0.0 || sum > DBL_MAX) {
      sum = 0.0;
      for (int i = 0; i <= K; i++) {
        p[i] = d_div(p[i], scale);
        if (i <= n) sum = d_add(sum, p[i]);
      }
    }
  }
  for (int n = 0; n <= K; n++) p[n] = d_div(p[n], sum);
  double L = 0.0, Lserv = 0.0, sumP = p[0];
  for (int i = 1; i <= K; i++) {
    L = d_add(L, d_mul((double)i, p[i]));
    sumP = d_add(sumP, p[i]);
    if (i == num) Lserv = d_add(L, d_mul(d_sub(1.0, sumP), (double)num));
  }
  st.avgNumInServers = (float)Lserv;
  st.avgNumInSystem = (float)L;
  st.throughput = f_mul(lambda, f_sub(1.0f, (float)p[K]));
  st.avgRespTime = f_div(st.avgNumInSystem, st.throughput);
  st.avgServTime = f_div(st.avgNumInServers, st.throughput);
  float w = f_sub(st.avgRespTime, st.avgServTime);
  st.avgWaitTime = (w < 0.0f) ? 0.0f : w;
}

// ------------------------------------------------------------------ (E12) certified fast solve
// The reference evaluates ~3K roundings per solve, but its consumers only read three float32 values:
// (float)Lserv, (float)L and f_sub(1, (float)p[K]).  The fast solve runs ONE pass over the head (n < N-1, the same
// E1 step as the exact solver, so p~[0..N-1] and their sequential sum are the reference's bits), then forms the tail
// n >= N-1, where mu is the constant mu_last and p~[N-1+k] = p~[N-1] rho^k, in closed form.  It also bounds
//   (a) the distance of the reference's float64 values from the exact real values, and
//   (b) the distance of its own values from the exact real values,
// and accepts a lane only if every float32 value the consumers read is the same at both ends of
// [v - 4(a+b), v + 4(a+b)] (the factor 4 covers second-order terms and the rounding of the bound itself).
// Proof sketch (DESIGN.md §3, E12).  u = 2^-53; all terms are non-negative.  Write p_n for the exact chain,
// S = sum p_n, T = sum n p_n, L = T/S, and R = the rounding error of a sequential sum of non-negative terms:
// adding t to s errs by at most min(u (s+t), t).
//   (a) reference: p~_n = p_n (1+th), |th| <= 2n u; its sum errs by <= 2u T + sum_n min(u S, p~_n) =: 2u T + Aref with
//       Aref <= A_head + u T + A_tail, where A_head accumulates min(u * partial sum, p~_n) in the head pass (the partial
//       sum falls short of S by the remaining mass; summed over n that is <= T) and A_tail = min(M u S, S_tail).  Hence
//       the normalising sum has relative error eta <= 2u L + Aref/S + u, and
//         L:      |L_ref - L|  <= L ((3K + 2) u + eta)                 (i^2 p_i <= K i p_i; K accumulations)
//         Lserv:  Lserv_ref = L_N + (1 - sumP_N) N; the N-weighted error of sumP_N gives the absolute term:
//                 |Ls_ref - Ls| <= Ls ((5N + 4) u + eta) + N (eta + 3u + Aref/S)
//         p[K]:   |pK_ref - pK| <= pK ((2K + 1) u + eta) + 2^-1000     (underflowed terms: K 2^-1074 each, at most)
//                 evaluated at the upper end pK + epK of (b): after a head exit the fast p[K] is 0 and only epK bounds it
//   (b) fast path: running error analysis of the closed form below (first order; every quantity carries its bound).
//       rho^M by binary powering is within (M - 1) u of rho_hat^M and rho_hat = RN(lambda/mu) is conditioned M times
//       through the power: 2M u relative, plus 2^-1000 absolute for underflow (all factors <= 1).
//       1 - rho = (mu - lambda)/mu is formed without cancellation (mu - lambda of two float32 values is exact).
//       p[K] = q rho^M / S carries 2^-1000 absolute of its own: q rho^M and the quotient may be subnormal (1 ulp =
//       2^-1074 each), and the 2^-1000 inside the error of rho^M is scaled by q / S <= 1, so it can underflow with them.
// Preconditions (otherwise not certified): every head x = p~*lambda inside the E3 window, p~[N-1] and S inside it,
// N >= 2 and 1 - rho >= 2^-12.  The last one keeps rho < 1 (the closed form needs a convergent tail) with margin;
// rates the sizer and the grid evaluate stay below lambda_max = 0.999 mu_{N-1}, so it never rejects an admitted rate.
// Light loads leave the head early (fast_head_exit) once lambda <= mu_n/2 on the whole rest of the chain: the
// remainder is then below a geometric series of ratio 1/2, sum_{j>n} p~_j <= p~_n and sum_{j>n} j p~_j <= (n+2) p~_n,
// and those bounds are added to the error of every value.
#ifndef WVA_TILE_CHUNK
#define WVA_TILE_CHUNK 16
#endif
#define WVA_FAST_OMEGA_MIN 0x1p-12
// Test hook: fast_solve_finish hands its values (L, Lserv, p[K]), their bounds (b) eL, eLs, epK and (a) fL, fLs, fpK and
// whether the head pass left early to WVA_FAST_PROBE right before certification.  Empty in the product; the host tests
// define it to check every bound against exact arithmetic.
#ifndef WVA_FAST_PROBE
#define WVA_FAST_PROBE(...)
#endif

struct FastHead {  // what the head pass leaves for fast_solve_finish
  double p;        // p~[n] of the last state visited
  double sum;      // sequential sum of p~[0..n] (the reference's partial sum, bit for bit)
  double T;        // sum of j p~[j], j <= n (fma accumulation)
  double A;        // sum of min(2^-53 * partial sum, p~[j]): the reference's rounding error of the head sum
  int n;           // index of the last state visited (N - 1 unless the pass left early)
  bool ok;         // every x = p~ lambda of the pass was inside the exponent window
  bool exited;     // left the head early (light load): the rest of the chain is the bounded remainder
};

WVA_HD double d_min(double a, double b) { return a < b ? a : b; }

// chunk-boundary early exit of the head pass; mu0 = mu at the chunk's first state n0 (mu is non-decreasing from
// n0 >= mono on, the tail rate included), p = p~[n], sum = partial sum at n
WVA_HD bool fast_head_exit(const PairModel& m, double lam, double mu0, int n0, int n, double p, double sum) {
  return n0 >= m.mono && d_mul(lam, 2.0) <= mu0 && d_mul(p, (double)(n + 2 + m.N)) <= d_mul(sum, 0x1p-64);
}

// does v +- r round to one float32 (and to what)?
WVA_HD bool f32_certain(double v, double r) { return (float)d_sub(v, r) == (float)d_add(v, r); }

// closed-form tail, error enclosure and certification.  true: st holds the reference's statistics
WVA_HD bool fast_solve_finish(const PairModel& m, float lambda, const FastHead& h, SolveStats& st) {
  const double u = 0x1p-53, tiny = 0x1p-1000;
  const int N = m.N, K = m.K;
  if (!h.ok || N < 2 || !(h.T > 0.0)) return false;
  const double hn = (double)h.n;
  // head, against exact arithmetic: sum errs by 2u T + A (recurrence, accumulation), T by 3 n u T (and fma)
  const double eH = d_add(d_mul(d_mul(2.0, u), h.T), h.A), eTH = d_mul(d_mul(d_mul(3.0, hn), u), h.T);
  double S, T, num, pKn, eS, eT, eN, epKn, Atail;
  if (h.exited) {
    const double RS = h.p, RT = d_mul(h.p, hn + 2.0);     // remainder bounds (ratio <= 1/2 from n on)
    S = h.sum; T = h.T; num = h.T; pKn = 0.0;
    eS = d_add(eH, RS); eT = d_add(eTH, RT); eN = d_add(eTH, d_add(RT, d_mul((double)N, RS))); epKn = RS;
    Atail = RS;
  } else {
    const double q = h.p;
    if (!in_window(q)) return false;
    const double lam = (double)lambda, mu = m.mu_last;
    const double om = d_div(d_sub(mu, lam), mu);          // 1 - rho, rel. error <= 2u
    if (!(om >= WVA_FAST_OMEGA_MIN)) return false;
    const double rho = d_div(lam, mu);                     // rel. error <= u
    const int M = K - N + 1;                               // tail states N .. K: p~[N-1+k] = q rho^k, k = 1..M
    const double dM = (double)M;
    double a = 1.0, b = rho;                               // a = rho^M
    for (int e = M; e; e >>= 1) { if (e & 1) a = d_mul(a, b); b = d_mul(b, b); }
    const double ea = d_add(d_mul(a, d_mul(d_mul(2.0, dM), u)), tiny);              // absolute
    const double c1 = d_sub(1.0, a), ec1 = d_add(ea, d_mul(u, c1));                 // 1 - rho^M, absolute
    if (!(c1 > 0.0)) return false;
    const double G1 = d_div(d_mul(rho, c1), om);                                    // sum rho^k
    const double rG1 = d_add(d_div(ec1, c1), d_mul(5.0, u));                        // relative
    const double bM = d_mul(d_mul(dM, a), rho);                                     // M rho^(M+1)
    const double ebM = d_add(d_mul(bM, d_mul(3.0, u)), d_mul(dM, ea));
    const double dd = d_sub(G1, bM);
    if (!(dd > 0.0)) return false;
    const double G2 = d_div(dd, om);                                                // sum k rho^k
    const double rG2 = d_add(d_div(d_add(d_add(d_mul(G1, rG1), ebM), d_mul(u, dd)), dd), d_mul(3.0, u));
    const double rq = d_mul(d_mul(2.0, hn), u);                                     // p~[N-1] vs exact
    const double St = d_mul(q, G1), rSt = d_add(d_add(rq, rG1), u);
    const double in = d_add(d_mul(hn, G1), G2);
    const double rin = d_add(d_add(rG1, u) > rG2 ? d_add(rG1, u) : rG2, u);
    const double Tt = d_mul(q, in), rTt = d_add(d_add(rq, rin), u);
    S = d_add(h.sum, St);
    if (!in_window(S)) return false;
    T = d_add(h.T, Tt);
    num = d_add(h.T, d_mul((double)N, St));                // Lserv = (T_head + N S_tail) / S
    pKn = d_mul(q, a);                                      // p~[K]
    eS = d_add(d_add(eH, d_mul(St, rSt)), d_mul(u, S));
    eT = d_add(d_add(eTH, d_mul(Tt, rTt)), d_mul(u, T));
    eN = d_add(d_add(eTH, d_mul(d_mul((double)N, St), d_add(rSt, u))), d_mul(u, num));
    epKn = d_add(d_mul(q, ea), d_mul(pKn, d_add(rq, u)));
    Atail = d_min(d_mul(d_mul(dM, u), S), St);
  }
  const double L = d_div(T, S), Ls = d_div(num, S), pK = d_div(pKn, S);
  const double rS = d_div(eS, S);
  // (b) fast values against exact arithmetic
  const double eL = d_mul(L, d_add(d_add(d_div(eT, T), rS), u));
  const double eLs = d_mul(Ls, d_add(d_add(d_div(eN, num), rS), u));
  const double epK = d_add(d_add(d_div(epKn, S), d_mul(pK, d_add(rS, u))), tiny);
  // (a) the reference against exact arithmetic
  const double Aref = d_add(d_add(h.A, d_mul(u, T)), Atail), rA = d_div(Aref, S);
  const double eta = d_add(d_add(d_mul(d_mul(2.0, u), L), rA), u);
  const double fL = d_mul(L, d_add(d_mul((double)(3 * K + 2), u), eta));
  const double fLs = d_add(d_mul(Ls, d_add(d_mul((double)(5 * N + 4), u), eta)),
                           d_mul((double)N, d_add(d_add(eta, d_mul(3.0, u)), rA)));
  const double fpK = d_add(d_mul(d_add(pK, epK), d_add(d_mul((double)(2 * K + 1), u), eta)), tiny);
  const double radL = d_mul(4.0, d_add(eL, fL)), radLs = d_mul(4.0, d_add(eLs, fLs)), radpK = d_mul(4.0, d_add(epK, fpK));
  WVA_FAST_PROBE(L, Ls, pK, eL, fL, eLs, fLs, epK, fpK, h.exited);
  if (!f32_certain(L, radL) || !f32_certain(Ls, radLs)) return false;
  const double pK_hi = d_add(pK, radpK);
  if (!(pK_hi < 0x1p-26) && f_sub(1.0f, (float)d_sub(pK, radpK)) != f_sub(1.0f, (float)pK_hi)) return false;
  st.avgNumInServers = (float)Ls;
  st.avgNumInSystem = (float)L;
  st.throughput = f_mul(lambda, f_sub(1.0f, (float)pK));
  st.avgRespTime = f_div(st.avgNumInSystem, st.throughput);
  st.avgServTime = f_div(st.avgNumInServers, st.throughput);
  float w = f_sub(st.avgRespTime, st.avgServTime);
  st.avgWaitTime = (w < 0.0f) ? 0.0f : w;
  return true;
}

// One fast solve on a single lane (the host replay of lockstep_solve_fast; the device runs the same steps, chunks
// and exit tests with each lane's rates in registers).  Returns whether it is certified.
WVA_HD bool fast_solve(const PairModel& m, float lambda, SolveStats& st, int* states) {
  *states = 0;
  if (!m.e1_ok) return false;   // the device never gives such a pair to the fast solve
  FastHead h;
  h.p = 1.0; h.sum = 1.0; h.T = 0.0; h.A = 0.0; h.n = 0; h.ok = true; h.exited = false;
  const double lam = (double)lambda;
  const int NH = m.N - 1;
  int n = 0;
  while (n < NH) {
    const int cnt = NH - n < WVA_TILE_CHUNK ? NH - n : WVA_TILE_CHUNK;
    const double mu0 = (double)model_rate(m, n);
    for (int j = 0; j < cnt; j++) {
      const float m32 = model_rate(m, n + j);
      const double mu = (double)m32, r = rcp_f32den(m32, mu);
      const double x = d_mul(h.p, lam);
      if (!in_window(x)) h.ok = false;
      h.p = div_f32den(x, mu, r);
      h.sum = d_add(h.sum, h.p);
      h.T = d_fma((double)(n + j + 1), h.p, h.T);
      h.A = d_add(h.A, d_min(d_mul(h.sum, 0x1p-53), h.p));
    }
    n += cnt;
    if (!h.ok) break;
    if (n < NH && fast_head_exit(m, lam, mu0, n - cnt, n, h.p, h.sum)) { h.exited = true; break; }
  }
  h.n = n;
  *states = n;
  return fast_solve_finish(m, lambda, h, st);
}

// utils.go:12-23
WVA_HD bool within_tolerance(float x, float value, float tolerance) {
  if (x == value) return true;
  if (value == 0.0f || tolerance < 0.0f) return false;
  return fabs((double)f_div(f_sub(x, value), value)) <= (double)tolerance;
}

// ------------------------------------------------------------------ device views
struct SysView {  // device image of wva_system (include/wva_b200.h)
  int n_acc, n_types, n_models, n_servers;
  const float* acc_cost; const int* acc_multiplicity; const int* acc_type; const int* type_count;
  const float *perf_alpha, *perf_beta, *perf_gamma;
  const int *perf_max_batch, *perf_at_tokens, *perf_acc_count;
  const unsigned char* perf_present;
  const int *srv_model, *srv_priority, *srv_min_replicas, *srv_max_batch;
  const unsigned char *srv_keep_acc, *srv_target_present;
  const float *srv_slo_ttft, *srv_slo_itl, *srv_slo_tps, *srv_arrival;
  const int *srv_in_tokens, *srv_out_tokens, *srv_cur_acc, *srv_cur_replicas;
  const float* srv_cur_cost;
};

struct CandView {  // device image of wva_candidates, row-major [S][A]
  unsigned char* state;
  int *num_replicas, *batch_size;
  float *cost, *value, *itl, *ttft, *rho, *max_arrv_rate;
  int* n_solves;
};

struct Alloc {  // core.Allocation (pkg/core/allocation.go:13-24)
  int state; long long num_replicas; int batch_size;
  float cost, value, itl, ttft, rho, max_arrv;
};

// the nil allocation: no candidate on this accelerator
WVA_HD Alloc alloc_none() {
  Alloc a; a.state = ALLOC_NONE; a.num_replicas = 0; a.batch_size = 0;
  a.cost = a.value = a.itl = a.ttft = a.rho = a.max_arrv = 0.0f;
  return a;
}

WVA_HD int sat_i32(long long v) {
  return v > 2147483647LL ? 2147483647 : (v < -2147483647LL - 1 ? (-2147483647 - 1) : (int)v);
}

// model.go:40-42,52-55
WVA_HD int num_instances(const SysView& s, int model, int acc) {
  int c = s.perf_acc_count[(size_t)model * s.n_acc + acc];
  return c <= 0 ? 1 : c;
}

// allocation.go:283-292 with a = the server's current allocation
WVA_HD float transition_penalty(int cur_acc, int cur_rep, float cur_cost, const Alloc& b, int b_acc) {
  bool same = (b.state == ALLOC_EMPTY) ? (cur_acc == -1) : (cur_acc == b_acc);
  if (same) {
    if ((long long)cur_rep == b.num_replicas) return 0.0f;
    return f_sub(b.cost, cur_cost);
  }
  return f_add(f_mul(WVA_ACCEL_PENALTY, f_add(cur_cost, b.cost)), f_sub(b.cost, cur_cost));
}

WVA_HD void store_candidate(const CandView& o, size_t idx, const Alloc& a, int solves) {
  o.state[idx] = (unsigned char)a.state;
  o.num_replicas[idx] = sat_i32(a.num_replicas);
  o.batch_size[idx] = a.batch_size;
  o.cost[idx] = a.cost;
  o.value[idx] = a.value;
  o.itl[idx] = a.itl;
  o.ttft[idx] = a.ttft;
  o.rho[idx] = a.rho;
  o.max_arrv_rate[idx] = a.max_arrv;
  if (o.n_solves) o.n_solves[idx] = solves;
}

// Go int(math.Ceil(x)) on amd64 (CVTTSD2SQ): out-of-range / NaN -> MinInt64
WVA_HD long long go_int_ceil(double x) {
  double c = ceil(x);
  if (!(c < 9223372036854775808.0) || !(c >= -9223372036854775808.0)) return (long long)0x8000000000000000ULL;
  return (long long)c;
}

// ------------------------------------------------------------------ sizer lane
// CreateAllocation for one (server, accelerator) as a resumable state machine:
// setup() classifies the pair (nil / zero-load / needs sizing); step() advances the
// current chain solve by one state and, when a solve completes, the bisection /
// Size / Analyze control flow (queueanalyzer.go:181-258, utils.go:26-70).
enum { SZ_LO = 0, SZ_HI = 1, SZ_SEARCH = 2, SZ_FINAL1 = 3, SZ_FINAL2 = 4, SZ_PUBLISH = 5 };

struct Search {   // one BinarySearch (utils.go:26-70)
  float lo, hi, target, x, result, y_lo;
  float y_hi;       // speculative split driver: f(hi) (y_lo = f(lo)), the evaluations at the current bounds
  int iter;
  bool active;      // still bisecting
  bool enabled;     // target > 0
  bool increasing;
};

struct SizerLane {
  PairModel m;
  Chain c;
  Search sT, sI;          // TTFT and ITL searches
  float slo_tps, total_rate, rate_star, acc_cost;
  float cur_x;
  float x2[2];           // dual driver: the (up to) two arrival rates of the coming round
  bool act2[2];
  int i_chain;           // dual driver: chain that carries the ITL search's point
  int stage;
  int srv, acc, model;
  int min_replicas, n_inst;
  int solves;
  // split mode (lane sizer on mid-size systems): a pair is two work items, one per search; the item that
  // finishes second merges the partner's result and runs the two Analyze solves
  int split;             // -1 whole pair, 0 TTFT item, 1 ITL item
  bool merged, failed;
  long long states;
  long long num_replicas;
  float cost;
};

// result of setup()
enum { SETUP_DONE = 0, SETUP_NEEDS_TABLE = 1 };

// allocation.go:27-99: everything before the queue analyzer exists.  When the pair
// is decided without any chain solve the candidate is written and SETUP_DONE returned.
WVA_HD int sizer_setup(SizerLane& z, const SysView& s, const CandView& out, int srv, int acc, int n_limit,
                       int* limit_hit, bool write = true) {
  z.srv = srv; z.acc = acc; z.solves = 0; z.states = 0;
  z.split = -1; z.merged = false; z.failed = false;
  size_t idx = (size_t)srv * s.n_acc + acc;
  Alloc a = alloc_none();
  int cur_acc = s.srv_cur_acc[srv];
  // Server.GetCandidateAccelerators (server.go:70-82)
  bool restricted = s.srv_keep_acc[srv] && cur_acc != -1;
  float arrival = s.srv_arrival[srv];
  int in_tok = s.srv_in_tokens[srv], out_tok = s.srv_out_tokens[srv];
  int model = s.srv_model[srv];
  z.model = model;
  bool nil = (restricted && acc != cur_acc) || arrival < 0.0f || in_tok < 0 || out_tok < 0 || model < 0 ||
             model >= s.n_models || !s.srv_target_present[srv];
  size_t pi = nil ? 0 : (size_t)model * s.n_acc + acc;
  if (!nil && !s.perf_present[pi]) nil = true;
  if (nil) { if (write) store_candidate(out, idx, a, 0); return SETUP_DONE; }
  z.min_replicas = s.srv_min_replicas[srv];
  z.n_inst = num_instances(s, model, acc);
  z.acc_cost = s.acc_cost[acc];
  if (arrival == 0.0f || out_tok == 0) {
    // zeroLoadAllocation (allocation.go:251-280)
    if (z.min_replicas == 0) {
      a.state = ALLOC_EMPTY;
    } else {
      int mb = s.perf_max_batch[pi];
      if (s.srv_max_batch[srv] > 0) mb = s.srv_max_batch[srv];
      long long tot = (long long)z.n_inst * z.min_replicas;
      float alpha = s.perf_alpha[pi], beta = s.perf_beta[pi];
      float decode = f_add(alpha, beta);
      float max_decode = f_add(alpha, f_mul(beta, (float)mb));
      float prefill = f_add(alpha, beta);
      float max_serv = f_add(prefill, max_decode);
      a.state = ALLOC_ACC;
      a.num_replicas = z.min_replicas;
      a.batch_size = mb;
      a.cost = f_mul(z.acc_cost, (float)tot);
      a.itl = decode; a.ttft = prefill; a.rho = 0.0f;
      a.max_arrv = f_div((float)mb, max_serv);
    }
    a.value = transition_penalty(cur_acc, s.srv_cur_replicas[srv], s.srv_cur_cost[srv], a, acc);
    if (write) store_candidate(out, idx, a, 0);
    return SETUP_DONE;
  }
  // allocation.go:78-87
  long long Nll;
  if (s.srv_max_batch[srv] > 0) Nll = s.srv_max_batch[srv];
  else {
    Nll = (long long)s.perf_max_batch[pi] * s.perf_at_tokens[pi] / out_tok;
    if (Nll < 1) Nll = 1;
  }
  if (Nll > n_limit) {  // larger than the kernels are built for: reported, never silently clipped
    if (limit_hit) *limit_hit = 1;
    if (write) store_candidate(out, idx, a, 0);
    return SETUP_DONE;
  }
  // Configuration.check / RequestSize.check (utils.go:95-118): N>0 holds; AvgOutputTokens >= 1 holds
  model_init(z.m, s.perf_alpha[pi], s.perf_beta[pi], s.perf_gamma[pi], in_tok, out_tok, (int)Nll);
  float ttft = s.srv_slo_ttft[srv], itl = s.srv_slo_itl[srv];
  z.slo_tps = s.srv_slo_tps[srv];
  z.sT.target = ttft; z.sI.target = itl;
  // TargetPerf.check (utils.go:121-128)
  if (itl < 0.0f || ttft < 0.0f || z.slo_tps < 0.0f) { if (write) store_candidate(out, idx, a, 0); return SETUP_DONE; }
  // allocation.go:126-131
  z.total_rate = (z.slo_tps == 0.0f) ? f_div(arrival, 60.0f) : f_div(z.slo_tps, (float)out_tok);
  return SETUP_NEEDS_TABLE;
}

WVA_HD void lane_start_solve(SizerLane& z, float lambda) {
  chain_start(z.c, lambda);
  z.c.tail_ok = d_bits(z.c.lamg) <= d_bits(z.m.mu_last);
  z.cur_x = lambda;
  z.solves++;
}

WVA_HD void lane_fail(SizerLane& z, const SysView& s, const CandView& out) {
  store_candidate(out, (size_t)z.srv * s.n_acc + z.acc, alloc_none(), z.solves);
}

// a failure during the search phase: in split mode it is published for the partner item instead of written
WVA_HD bool search_fail(SizerLane& z, const SysView& s, const CandView& out) {
  if (z.split >= 0 && !z.merged) { z.failed = true; z.stage = SZ_PUBLISH; return true; }
  lane_fail(z, s, out);
  return false;
}

// Analyze() pre-checks (queueanalyzer.go:128-136)
WVA_HD bool analyze_admits(const PairModel& m, float rate) { return rate > 0.0f && !(rate > m.rate_max); }

// ---- the steps of Size() and CreateAllocation, shared by every sizer driver -------------------------------------

// EvalTTFT / EvalITL of a finished solve, and the prefill time Analyze adds to the waiting time
// (queueanalyzer.go:143-149,283-308)
WVA_HD void eval_values(const PairModel& m, const SolveStats& st, float* ttft, float* itl, float* pf) {
  *pf = prefill_time(m, st.avgNumInServers);
  *itl = f_div(f_sub(st.avgServTime, *pf), m.out_tok);
  *ttft = f_add(f_add(st.avgWaitTime, *pf), *itl);
}

// Size()'s two BinarySearch calls (queueanalyzer.go:197-230): a search runs when its target is positive, and a split
// item runs only its own.  Returns false when neither runs.
WVA_HD bool searches_begin(SizerLane& z) {
  z.sT.enabled = z.sT.target > 0.0f && z.split != 1;
  z.sI.enabled = z.sI.target > 0.0f && z.split != 0;
  z.sT.active = z.sT.enabled; z.sI.active = z.sI.enabled;
  z.sT.result = z.m.lambda_max; z.sI.result = z.m.lambda_max;
  z.sT.iter = z.sI.iter = 0;
  return z.sT.enabled || z.sI.enabled;
}

// BinarySearch's end points (utils.go:33-57), xMin first: when f(xMin) is within tolerance the search ends at xMin and
// the reference never evaluates xMax.
WVA_HD void search_lo(Search& q, const PairModel& m, float y_lo) {
  q.y_lo = y_lo;
  if (within_tolerance(y_lo, q.target, WVA_BS_EPSILON)) { q.result = m.lambda_min; q.active = false; }
}
// xMax, for a search search_lo left active: within tolerance or a target above the bounded region ends it at xMax; a
// target below the region fails it (returns false); else the bisection starts on [xMin, xMax].
WVA_HD bool search_hi(Search& q, const PairModel& m, float y_hi) {
  if (within_tolerance(y_hi, q.target, WVA_BS_EPSILON)) { q.result = m.lambda_max; q.active = false; return true; }
  q.increasing = q.y_lo < y_hi;
  if ((q.increasing && q.target < q.y_lo) || (!q.increasing && q.target > q.y_lo)) { q.active = false; return false; }  // ind = -1
  if ((q.increasing && q.target > y_hi) || (!q.increasing && q.target < y_hi)) { q.result = m.lambda_max; q.active = false; return true; }  // ind = +1
  q.lo = m.lambda_min; q.hi = m.lambda_max; q.iter = 0; q.y_hi = y_hi;
  q.x = f_mul(0.5f, f_add(q.lo, q.hi));
  return true;
}
// both end points, evaluated in the same round; false when the search fails
WVA_HD bool search_bracket(Search& q, const PairModel& m, float y_lo, float y_hi) {
  search_lo(q, m, y_lo);
  return !q.active || search_hi(q, m, y_hi);
}

// one search consumes the evaluation y = f(x) of the solve just finished
WVA_HD void search_consume(Search& q, float x, float y) {
  if (within_tolerance(y, q.target, WVA_BS_EPSILON)) { q.result = x; q.active = false; return; }
  if ((q.increasing && q.target < y) || (!q.increasing && q.target > y)) q.hi = x; else q.lo = x;
  q.iter++;
  if (q.iter >= WVA_MAX_ITER) { q.result = x; q.active = false; return; }
  q.x = f_mul(0.5f, f_add(q.lo, q.hi));
  // (E6) fixpoint: once the next midpoint equals the point just evaluated, eval() returns
  // the same y, the same branch is taken and (lo, hi) no longer change, so every remaining
  // iteration up to maxIterations repeats this one and BinarySearch returns x.  (The 1e-6
  // relative tolerance sits at float32 resolution, so ~1 in 5 searches ends this way.)
  if (q.x == x) { q.result = x; q.active = false; }
}

// Size()'s tail (queueanalyzer.go:232-239) and Analyze's admission of its rate (:128-136): false when the rate is not
// admitted, else x = the arrival rate of the first Analyze solve (:139)
WVA_HD bool size_lambda(const SizerLane& z, float& x) {
  float l_tps = z.m.lambda_max;
  if (z.slo_tps > 0.0f) l_tps = f_mul(z.m.lambda_max, f_sub(1.0f, WVA_STABILITY_SAFETY));  // :232-235
  float lambda = fminf(fminf(z.sT.result, z.sI.result), l_tps);                             // :238
  float request_rate = f_mul(lambda, 1000.0f);                                               // :239
  if (!analyze_admits(z.m, request_rate)) return false;
  x = f_div(request_rate, 1000.0f);
  return true;
}

// CreateAllocation's replica count from the first Analyze solve (allocation.go:123-145): false when the rate per
// replica is not admitted, else x = the arrival rate of the second Analyze solve
WVA_HD bool alloc_replicas(SizerLane& z, float throughput, float& x) {
  z.rate_star = f_mul(throughput, 1000.0f);                                           // allocation.go:123
  long long nr = go_int_ceil(d_div((double)z.total_rate, (double)z.rate_star));       // :132
  if (nr < (long long)z.min_replicas) nr = z.min_replicas;
  z.num_replicas = nr;
  long long tot = (long long)((unsigned long long)z.n_inst * (unsigned long long)nr);
  z.cost = f_mul(z.acc_cost, (float)tot);
  float rate = f_div(z.total_rate, (float)nr);
  if (!analyze_admits(z.m, rate)) return false;
  x = f_div(rate, 1000.0f);
  return true;
}

// the allocation CreateAllocation returns, from the second Analyze solve st and its eval_values itl, pf
// (allocation.go:146-153)
WVA_HD Alloc alloc_final(const SizerLane& z, const SysView& s, const SolveStats& st, float itl, float pf) {
  Alloc a;
  a.state = ALLOC_ACC;
  a.num_replicas = z.num_replicas;
  a.batch_size = z.m.N;
  a.cost = z.cost;
  a.itl = itl;
  a.ttft = f_add(st.avgWaitTime, pf);
  float rho = f_div(st.avgNumInServers, (float)z.m.N);
  a.rho = fminf(fmaxf(rho, 0.0f), 1.0f);
  a.max_arrv = f_div(z.rate_star, 1000.0f);
  a.value = transition_penalty(s.srv_cur_acc[z.srv], s.srv_cur_replicas[z.srv], s.srv_cur_cost[z.srv], a, z.acc);
  return a;
}

// ---- sequential driver: one chain per lane, the solves of the two searches one after the other ----------------
WVA_HD bool sizer_after_search(SizerLane& z, const SysView& s, const CandView& out) {
  if (z.split >= 0 && !z.merged) { z.stage = SZ_PUBLISH; return true; }   // publish; the second finisher goes on
  float x;
  if (!size_lambda(z, x)) { lane_fail(z, s, out); return false; }
  z.stage = SZ_FINAL1;
  lane_start_solve(z, x);
  return true;
}

// After the table is built: start Size() (queueanalyzer.go:181-258).  Returns false
// if the pair finished without needing a solve.
WVA_HD bool sizer_begin(SizerLane& z, const SysView& s, const CandView& out) {
  if (!searches_begin(z)) return sizer_after_search(z, s, out);
  // BinarySearch: xMin > xMax -> error (utils.go:29-31)
  if (z.m.lambda_min > z.m.lambda_max) return search_fail(z, s, out);
  z.stage = SZ_LO;
  lane_start_solve(z, z.m.lambda_min);
  return true;
}

// ---- two-chain drivers: the lane solves the arrival rates z.x2[c] where z.act2[c] in one round -----------------
WVA_HD void dual_start1(SizerLane& z, float x) {   // one solve in the coming round
  z.x2[0] = x; z.act2[0] = true; z.act2[1] = false;
  z.solves++;
}

WVA_HD bool dual_after_search(SizerLane& z, const SysView& s, const CandView& out) {
  float x;
  if (!size_lambda(z, x)) { lane_fail(z, s, out); return false; }
  z.stage = SZ_FINAL1;
  dual_start1(z, x);
  return true;
}

// a split item publishes its search's result first (split_publish); the item that finishes second goes on
WVA_HD bool spec2_after_search(SizerLane& z, const SysView& s, const CandView& out) {
  if (z.split >= 0 && !z.merged) { z.stage = SZ_PUBLISH; return true; }
  return dual_after_search(z, s, out);
}

// round 0 evaluates both end points of every search the split item (or the whole pair) runs
WVA_HD bool spec2_begin(SizerLane& z, const SysView& s, const CandView& out) {
  if (!searches_begin(z)) return spec2_after_search(z, s, out);
  if (z.m.lambda_min > z.m.lambda_max) return search_fail(z, s, out);   // utils.go:29-31
  z.stage = SZ_LO;
  z.x2[0] = z.m.lambda_min; z.x2[1] = z.m.lambda_max; z.act2[0] = z.act2[1] = true;
  z.solves += 2;
  return true;
}
// a whole pair starts as a split item does: the split steps do nothing for it
WVA_HD bool dual_begin(SizerLane& z, const SysView& s, const CandView& out) { return spec2_begin(z, s, out); }

// the two Analyze solves (stages SZ_FINAL1, SZ_FINAL2), on chain 0
WVA_HD bool dual_final(SizerLane& z, const SysView& s, const CandView& out, const SolveStats& st) {
  if (z.stage == SZ_FINAL1) {
    float x;
    if (!alloc_replicas(z, st.throughput, x)) { lane_fail(z, s, out); return false; }
    z.stage = SZ_FINAL2;
    dual_start1(z, x);
    return true;
  }
  float ttft, itl, pf;
  eval_values(z.m, st, &ttft, &itl, &pf);
  const Alloc a = alloc_final(z, s, st, itl, pf);
  store_candidate(out, (size_t)z.srv * s.n_acc + z.acc, a, z.solves);
  return false;
}

// ---- dual-chain driver: TTFT and ITL searches advance in the SAME round (two chains per lane) -----
// Used by the lock-step lane sizer.  Same decisions as sizer_on_solve (which runs the two searches one
// after the other): both end points in round 0, then one bisection step of each search per round,
// then the two Analyze solves.  ~30 rounds per pair instead of ~58 solves in sequence.
WVA_HD bool dual_schedule(SizerLane& z, const SysView& s, const CandView& out) {
  if (!z.sT.active && !z.sI.active) return dual_after_search(z, s, out);
  z.stage = SZ_SEARCH;
  z.act2[0] = true; z.act2[1] = false; z.i_chain = 0;
  if (z.sT.active) {
    z.x2[0] = z.sT.x;
    if (z.sI.active && z.sI.x != z.sT.x) { z.x2[1] = z.sI.x; z.act2[1] = true; z.i_chain = 1; }
  } else {
    z.x2[0] = z.sI.x;
  }
  z.solves += z.act2[1] ? 2 : 1;
  return true;
}

// st[c] = statistics of the solve at z.x2[c] (valid where z.act2[c]); n_states = states visited by the round
WVA_HD bool dual_on_solve(SizerLane& z, const SysView& s, const CandView& out, const SolveStats* st, int n_states) {
  z.states += n_states;
  if (z.stage == SZ_FINAL1 || z.stage == SZ_FINAL2) return dual_final(z, s, out, st[0]);
  const PairModel& m = z.m;
  float ttft[2], itl[2], pf;
  for (int c = 0; c < 2; c++) eval_values(m, st[c], &ttft[c], &itl[c], &pf);
  if (z.stage == SZ_LO) {
    if ((z.sT.active && !search_bracket(z.sT, m, ttft[0], ttft[1])) || (z.sI.active && !search_bracket(z.sI, m, itl[0], itl[1]))) {
      lane_fail(z, s, out);
      return false;
    }
  } else {
    if (z.sT.active) search_consume(z.sT, z.x2[0], ttft[0]);
    if (z.sI.active) search_consume(z.sI, z.x2[z.i_chain], itl[z.i_chain]);
  }
  return dual_schedule(z, s, out);
}

// ---- speculative split driver: ONE search per lane, two chains per round -------------------------------
// Mid-size systems have fewer (pair, search) items than the GPU has lanes x latency-hiding depth, so the lane's
// second chain is spent on the bisection step AFTER the current one: chain 0 evaluates the midpoint x, chain 1
// the midpoint of the half the search is predicted to keep (the prediction compares the target with the value
// interpolated between the evaluations at the two bounds).  The midpoints are pure float32 arithmetic on
// (lo, hi), so chain 1's point is exactly what BinarySearch would evaluate next if the prediction holds; the
// walk consumes y0 as the reference does and consumes y1 only if the next x is bit-identical to the point
// chain 1 evaluated.  A wrong guess wastes one chain, never changes a decision.  Results are bit-identical to
// the sequential search; a correct guess halves the rounds on the critical path (E7 with a 2-leaf tree).
// Items end with dual_final, as whole pairs do.

// the half BinarySearch keeps if f(x) equals the interpolated value: true = [lo, x]
WVA_HD bool spec2_predict_left(const Search& q) {
  // harmonic interpolation (exact for the hyperbolic growth of waiting time towards saturation) when both
  // evaluations are positive, arithmetic otherwise; any rule is correct, a better one only saves rounds
  float y = (q.y_lo > 0.0f && q.y_hi > 0.0f) ? f_div(f_mul(2.0f, f_mul(q.y_lo, q.y_hi)), f_add(q.y_lo, q.y_hi))
                                             : f_mul(0.5f, f_add(q.y_lo, q.y_hi));
  return (q.increasing && q.target < y) || (!q.increasing && q.target > y);
}

WVA_HD bool spec2_schedule(SizerLane& z, const SysView& s, const CandView& out) {
  Search& q = z.split == 1 ? z.sI : z.sT;
  if (!q.active) return spec2_after_search(z, s, out);
  z.stage = SZ_SEARCH;
  z.x2[0] = q.x; z.act2[0] = true;
  z.x2[1] = spec2_predict_left(q) ? f_mul(0.5f, f_add(q.lo, q.x)) : f_mul(0.5f, f_add(q.x, q.hi));
  z.act2[1] = q.iter + 1 < WVA_MAX_ITER && z.x2[1] != q.x;
  z.solves += z.act2[1] ? 2 : 1;
  return true;
}

// one consumed evaluation; keeps (y_lo, y_hi) = f at the bounds
WVA_HD void spec2_consume(Search& q, float x, float y) {
  const bool left = (q.increasing && q.target < y) || (!q.increasing && q.target > y);
  search_consume(q, x, y);
  if (q.active) { if (left) q.y_hi = y; else q.y_lo = y; }
}

// st[c] = statistics of the solve at z.x2[c] (valid where z.act2[c])
WVA_HD bool spec2_on_solve(SizerLane& z, const SysView& s, const CandView& out, const SolveStats* st, int n_states) {
  z.states += n_states;
  if (z.stage == SZ_FINAL1 || z.stage == SZ_FINAL2) return dual_final(z, s, out, st[0]);
  const PairModel& m = z.m;
  Search& q = z.split == 1 ? z.sI : z.sT;
  float y[2];
  for (int c = 0; c < 2; c++) {
    float ttft, itl, pf;
    eval_values(m, st[c], &ttft, &itl, &pf);
    y[c] = z.split == 1 ? itl : ttft;
  }
  if (z.stage == SZ_LO) {
    if (q.active && !search_bracket(q, m, y[0], y[1])) return search_fail(z, s, out);
  } else {
    spec2_consume(q, z.x2[0], y[0]);
    if (q.active && z.act2[1] && q.x == z.x2[1]) spec2_consume(q, z.x2[1], y[1]);
  }
  return spec2_schedule(z, s, out);
}

// ---- speculative bisection (used by the warp-per-pair sizer; see sizer_warp_kernel.cuh) ----
// x of heap node `node` (1-based; children 2j, 2j+1) of the bisection tree rooted at (lo, hi):
// left child = the branch that sets hi = x, right child = the branch that sets lo = x.
WVA_HD float spec_node_x(float lo, float hi, int node, int depth_of_node) {
  float x = f_mul(0.5f, f_add(lo, hi));
  for (int b = depth_of_node - 2; b >= 0; b--) {
    if ((node >> b) & 1) lo = x; else hi = x;
    x = f_mul(0.5f, f_add(lo, hi));
  }
  return x;
}
WVA_HD int spec_depth_of(int node) {  // 1 for the root
  int d = 0;
  while (node) { d++; node >>= 1; }
  return d;
}

// Walk one search through an evaluated tree of `depth` levels.  get_y(node) returns f(x_node).
// On return either the search finished (q.active == false, q.result set) or (q.lo, q.hi, q.iter,
// q.x) describe the interval for the next round.
template <typename GetY>
WVA_HD void spec_walk(Search& q, int depth, GetY get_y) {
  int node = 1;
  for (int lvl = 0; lvl < depth && q.active; lvl++) {
    float x = q.x;
    float y = get_y(node);
    bool right;
    if (within_tolerance(y, q.target, WVA_BS_EPSILON)) { q.result = x; q.active = false; break; }
    if ((q.increasing && q.target < y) || (!q.increasing && q.target > y)) { q.hi = x; right = false; }
    else { q.lo = x; right = true; }
    q.iter++;
    if (q.iter >= WVA_MAX_ITER) { q.result = x; q.active = false; break; }
    q.x = f_mul(0.5f, f_add(q.lo, q.hi));
    if (q.x == x) { q.result = x; q.active = false; break; }   // (E6) fixpoint
    node = 2 * node + (right ? 1 : 0);
  }
}

// The solve at z.cur_x completed with stats st.  Returns false when the pair is finished.
WVA_HD bool sizer_on_solve(SizerLane& z, const SysView& s, const CandView& out, const SolveStats& st) {
  z.states += z.c.states;
  const PairModel& m = z.m;
  float ttft, itl, pf;
  eval_values(m, st, &ttft, &itl, &pf);
  if (z.stage == SZ_LO) {
    if (z.sT.active) search_lo(z.sT, m, ttft);
    if (z.sI.active) search_lo(z.sI, m, itl);
    if (z.sT.active || z.sI.active) { z.stage = SZ_HI; lane_start_solve(z, m.lambda_max); return true; }
    return sizer_after_search(z, s, out);
  }
  if (z.stage == SZ_HI) {
    if ((z.sT.active && !search_hi(z.sT, m, ttft)) || (z.sI.active && !search_hi(z.sI, m, itl)))
      return search_fail(z, s, out);   // "target is below the bounded region"
    z.stage = SZ_SEARCH;
  } else if (z.stage == SZ_SEARCH) {
    float x = z.cur_x;
    if (z.sT.active && z.sT.x == x) search_consume(z.sT, x, ttft);
    if (z.sI.active && z.sI.x == x) search_consume(z.sI, x, itl);
  }
  if (z.stage == SZ_SEARCH) {
    if (z.sT.active) { lane_start_solve(z, z.sT.x); return true; }
    if (z.sI.active) { lane_start_solve(z, z.sI.x); return true; }
    return sizer_after_search(z, s, out);
  }
  if (z.stage == SZ_FINAL1) {
    float x;
    if (!alloc_replicas(z, st.throughput, x)) { lane_fail(z, s, out); return false; }
    z.stage = SZ_FINAL2;
    lane_start_solve(z, x);
    return true;
  }
  const Alloc a = alloc_final(z, s, st, itl, pf);   // SZ_FINAL2
  store_candidate(out, (size_t)z.srv * s.n_acc + z.acc, a, z.solves);
  return false;
}

}  // namespace wva
