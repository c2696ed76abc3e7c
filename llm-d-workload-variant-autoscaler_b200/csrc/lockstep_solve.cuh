// lockstep_solve.cuh — MM1ModelStateDependent.Solve (pkg/analyzer/mm1modelstatedependent.go:28-116)
// for NC independent arrival rates per lane, all 32 lanes of a warp advancing the state index
// together: pass 1 (sum of p~) for every lane and chain, then pass 2 (normalise + accumulate).
// The loops are unrolled in chunks of 16/NC states and carry NO per-state control flow:
//   - the early exit (E4) is decided once per chunk: a chain is `done` when its current term is
//     below 2^-54 of every accumulator (compared on the high words — conservative) and the
//     remaining terms are non-increasing; a done chain keeps executing the same instructions,
//     which by that very criterion are exact no-ops on its accumulators;
//   - the exponent window (E3) is tracked with one integer min and one max per state and checked
//     per chunk; a violation (float64 overflow / underflow regime, never seen on sane inputs)
//     marks the solve `bad` and the pair is redone by the literal slow path;
//   - the warp leaves a loop when every chain of every lane is done.
// With NC = 2 the two chains of a lane share the table load (and, for per-lane float32 tables,
// the reciprocal refinement) and give the FP64 pipe two independent dependency chains per lane.
// Per state and chain: pass 1 = 5 FP64-pipe ops, pass 2 = 13 FP64-pipe ops (DESIGN.md §4).
#pragma once
#include "wva_core.cuh"

namespace wva {

#if defined(__CUDACC__)

#define WVA_HI_LO 0x20B00000   // high word of 2^-500
#define WVA_HI_HI 0x5F300000   // high word of 2^500

// head-table accessors -----------------------------------------------------------------------------
// Every table also loads a whole chunk of CH states starting at n (load_chunk; n a multiple of CH).
struct WarpTable {   // one table per warp in shared memory: (mu_n, ~1/mu_n) as float64 pairs, broadcast reads
  static constexpr int kChunk = 16;
  const double2* t;
  __device__ __forceinline__ void load(int n, double& mu, double& r) const { double2 v = t[n]; mu = v.x; r = v.y; }
  template <int CH> __device__ __forceinline__ void load_chunk(int n, double (&mu)[CH], double (&r)[CH]) const {
#pragma unroll
    for (int j = 0; j < CH; j++) load(n + j, mu[j], r[j]);
  }
  __device__ __forceinline__ double mu_at(int n) const { return t[n].x; }
  __device__ __forceinline__ void prepare(int) const {}
};
struct LaneTable {   // one float32 column per lane ([n][thread], bank = lane); 1/mu refined on the fly
  static constexpr int kChunk = 16;
  const float* t;
  int stride;
  __device__ __forceinline__ void load(int n, double& mu, double& r) const {
    float m32 = t[(size_t)n * stride]; mu = (double)m32; r = rcp_f32den(m32, mu);
  }
  template <int CH> __device__ __forceinline__ void load_chunk(int n, double (&mu)[CH], double (&r)[CH]) const {
#pragma unroll
    for (int j = 0; j < CH; j++) load(n + j, mu[j], r[j]);
  }
  __device__ __forceinline__ double mu_at(int n) const { return (double)t[(size_t)n * stride]; }
  __device__ __forceinline__ void prepare(int) const {}
};
// Each lane's own rates, computed where they are used (sizer_pool_kernel.cuh, grid_deferred_kernel): any 32 pairs solve
// together with no table in memory.  Entry n is serv_rate(n + 1) — the function BuildModel's table is filled with, so
// the same bits — from the model's coefficients, held by value so that a __noinline__ solver keeps them in registers.
// The float32 batch size is counted up by 1.0f (exact below 2^24).  A chunk's CH rates are formed before the
// recurrence that uses them and do not depend on it: their float32 divisions run on the FP32 pipe, which the
// FP64-bound head pass leaves idle.  Only models with e1_ok are solved through it (the pool queues and the deferred grid
// pass take no other pair): every rate is an (E1) divisor, so the conversions run on the integer pipe (f32pos_to_d,
// rcp_f32den_e1), and every denominator passed rate_den_ok, so the divisions are div_rate's branch-free sequence
// (serv_rate_e1) and a chunk's rates are straight-line code the scheduler interleaves.
struct RateTable {
  static constexpr int kChunk = WVA_TILE_CHUNK;   // states per unrolled chunk of the solver (code size vs loop overhead)
  RateCoef c;
  // a lane with no pair: mu_n = n + 1, every entry an (E1) divisor with den = 1
  static __device__ __forceinline__ RateTable idle() { return RateTable{{1.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 1.0f}}; }
  __device__ __forceinline__ void prepare(int) const {}
  __device__ __forceinline__ void load(int n, double& mu, double& r) const {
    const float m32 = serv_rate_e1(c, (float)(n + 1)); mu = f32pos_to_d(m32); r = rcp_f32den_e1(m32, mu);
  }
  template <int CH> __device__ __forceinline__ void load_chunk(int n, double (&mu)[CH], double (&r)[CH]) const {
    float m32[CH], nf = (float)(n + 1);
#pragma unroll
    for (int j = 0; j < CH; j++) { m32[j] = serv_rate_e1(c, nf); nf = f_add(nf, 1.0f); }
#pragma unroll
    for (int j = 0; j < CH; j++) { mu[j] = f32pos_to_d(m32[j]); r[j] = rcp_f32den_e1(m32[j], mu[j]); }
  }
  __device__ __forceinline__ double mu_at(int n) const { return f32pos_to_d(serv_rate_e1(c, (float)(n + 1))); }
};

// high word of v * 2^-54 for a normal v >= 2^-900: the exponent field moves, nothing rounds
__device__ __forceinline__ int hi_scale_m54(double v) { return d_hi(v) - (54 << 20); }

struct P1 { double p, sum; int mn, mx; };
struct P2 { double p, L, sumP, pi; int mn, mx; };

// (E1) with a 3-deep dependency chain: the approximation q0 of x/mu = RN(p*lambda)/mu is formed as
// p * RN(lambda*r) next to x = p*lambda instead of after it.  q0 only has to be within 2^-39.99 of the
// quotient (it is within ~2^-45.9: r's 2^-46.56 plus three roundings); the remainder and the final fma use the
// exact x, so the result is still the correctly rounded RN(x/mu).  Only for mu in [2^-126, 2^126] (e1_divisor): the
// callers never give this solver a pair with another service rate (PairModel::e1_ok).
__device__ __forceinline__ double step_div(double p, double lam, double lamr, double mu, double r, int& mn, int& mx) {
  double x = d_mul(p, lam);
  double q0 = d_mul(p, lamr);
  int h = d_hi(x);
  mn = min(mn, h); mx = max(mx, h);
  double rem = d_fma(-q0, mu, x);
  return d_fma(rem, r, q0);
}
__device__ __forceinline__ void p1_step(P1& s, double lam, double mu, double r) {
  s.p = step_div(s.p, lam, d_mul(lam, r), mu, r, s.mn, s.mx);
  s.sum = d_add(s.sum, s.p);
}
__device__ __forceinline__ void p1_step_c(P1& s, double lam, double lamr, double mu, double r) {   // constant rate (tail)
  s.p = step_div(s.p, lam, lamr, mu, r, s.mn, s.mx);
  s.sum = d_add(s.sum, s.p);
}
__device__ __forceinline__ void p2_step_c(P2& s, double lam, double lamr, double mu, double r, double sum, double rsum, double di) {
  s.p = step_div(s.p, lam, lamr, mu, r, s.mn, s.mx);
  s.pi = div_markstein2(s.p, sum, rsum);
  s.L = d_add(s.L, d_mul(di, s.pi));
  s.sumP = d_add(s.sumP, s.pi);
}
__device__ __forceinline__ void p2_step(P2& s, double lam, double mu, double r, double sum, double rsum, double di) {
  s.p = step_div(s.p, lam, d_mul(lam, r), mu, r, s.mn, s.mx);
  s.pi = div_markstein2(s.p, sum, rsum);
  s.L = d_add(s.L, d_mul(di, s.pi));
  s.sumP = d_add(s.sumP, s.pi);
}

// ---- software-pipelined chunks --------------------------------------------------------------------------
// ptxas keeps the FP64 ops of an unrolled chunk in source order (measured: ncu source page, r1), and a warp issues
// in order, so a chunk written state after state stalls ~8 cycles on every dependent op: the 5-deep normalising
// division and the two accumulations of state j sit between the recurrence steps of states j and j+1 although
// they are off the recurrence.  Here the ops are EMITTED in pipeline order instead: stage s of state j at slot
// 3*j + s (the recurrence p -> p' is 3 ops deep), so every slot holds ops of different states (and chains) that
// are independent of each other and only consume results of earlier slots.  Same ops, same operands, same
// rounding — only the order in the instruction stream changes.
//   stage 0: x = p*lam, q0 = p*lamr (+ exponent window)   1: rem = fma(-q0, mu, x)   2: p' = fma(rem, r, q0)
//   pass 1   3: sum += p'
//   pass 2   3..7: pi = RN(p'/sum) (two-step Markstein)   8: t = i*pi, sumP += pi   9: L += t
template <int NC, int CH, bool HEAD>
__device__ __forceinline__ void p1_chunk(P1 (&a)[NC], const double (&lam)[NC], const double (&lamr_c)[NC],
                                         const double (&mu)[HEAD ? CH : 1], const double (&r)[HEAD ? CH : 1]) {
  double x[NC][CH], q0[NC][CH], rem[NC][CH], pn[NC][CH + 1], lamr[NC][HEAD ? CH : 1];
#pragma unroll
  for (int c = 0; c < NC; c++) {
    pn[c][0] = a[c].p;
#pragma unroll
    for (int j = 0; j < (HEAD ? CH : 1); j++) lamr[c][j] = HEAD ? d_mul(lam[c], r[j]) : lamr_c[c];
  }
#pragma unroll
  for (int slot = 0; slot < 3 * CH + 1; slot++) {
#pragma unroll
    for (int j = 0; j < CH; j++) {
      const int st = slot - 3 * j;
      const int k = HEAD ? j : 0;
#pragma unroll
      for (int c = 0; c < NC; c++) {
        if (st == 0) {
          x[c][j] = d_mul(pn[c][j], lam[c]);
          q0[c][j] = d_mul(pn[c][j], lamr[c][k]);
          const int h = d_hi(x[c][j]);
          a[c].mn = min(a[c].mn, h); a[c].mx = max(a[c].mx, h);
        }
        if (st == 1) rem[c][j] = d_fma(-q0[c][j], mu[k], x[c][j]);
        if (st == 2) pn[c][j + 1] = d_fma(rem[c][j], r[k], q0[c][j]);
        if (st == 3) a[c].sum = d_add(a[c].sum, pn[c][j + 1]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < NC; c++) a[c].p = pn[c][CH];
}

template <int NC, int CH, bool HEAD>
__device__ __forceinline__ void p2_chunk(P2 (&b)[NC], const double (&lam)[NC], const double (&lamr_c)[NC],
                                         const double (&mu)[HEAD ? CH : 1], const double (&r)[HEAD ? CH : 1],
                                         const double (&sum)[NC], const double (&rsum)[NC], double& di) {
  double x[NC][CH], q0[NC][CH], rem[NC][CH], pn[NC][CH + 1], q[NC][CH], r1[NC][CH], q1[NC][CH], r2[NC][CH], pi[NC][CH],
      t[NC][CH], dj[CH], lamr[NC][HEAD ? CH : 1];
#pragma unroll
  for (int j = 0; j < CH; j++) dj[j] = d_add(di, (double)(j + 1));   // float64(i): exact integers
#pragma unroll
  for (int c = 0; c < NC; c++) {
    pn[c][0] = b[c].p;
#pragma unroll
    for (int j = 0; j < (HEAD ? CH : 1); j++) lamr[c][j] = HEAD ? d_mul(lam[c], r[j]) : lamr_c[c];
  }
#pragma unroll
  for (int slot = 0; slot < 3 * CH + 7; slot++) {
#pragma unroll
    for (int j = 0; j < CH; j++) {
      const int st = slot - 3 * j;
      const int k = HEAD ? j : 0;
#pragma unroll
      for (int c = 0; c < NC; c++) {
        if (st == 0) {
          x[c][j] = d_mul(pn[c][j], lam[c]);
          q0[c][j] = d_mul(pn[c][j], lamr[c][k]);
          const int h = d_hi(x[c][j]);
          b[c].mn = min(b[c].mn, h); b[c].mx = max(b[c].mx, h);
        }
        if (st == 1) rem[c][j] = d_fma(-q0[c][j], mu[k], x[c][j]);
        if (st == 2) pn[c][j + 1] = d_fma(rem[c][j], r[k], q0[c][j]);
        if (st == 3) q[c][j] = d_mul(pn[c][j + 1], rsum[c]);                       // div_markstein2, step by step
        if (st == 4) r1[c][j] = d_fma(-q[c][j], sum[c], pn[c][j + 1]);
        if (st == 5) q1[c][j] = d_fma(r1[c][j], rsum[c], q[c][j]);
        if (st == 6) r2[c][j] = d_fma(-q1[c][j], sum[c], pn[c][j + 1]);
        if (st == 7) pi[c][j] = d_fma(r2[c][j], rsum[c], q1[c][j]);
        if (st == 8) { t[c][j] = d_mul(dj[j], pi[c][j]); b[c].sumP = d_add(b[c].sumP, pi[c][j]); }
        if (st == 9) b[c].L = d_add(b[c].L, t[c][j]);
      }
    }
  }
#pragma unroll
  for (int c = 0; c < NC; c++) { b[c].p = pn[c][CH]; b[c].pi = pi[c][CH - 1]; }
  di = dj[CH - 1];
}

// Chains c with active[c] solve at lambda[c]; the others ride along (lambda 0).  On return `bad`
// is set for a lane when one of its solves left the exponent window (caller: redo the pair on the
// slow path).  Forced inline: the NC = 2 instantiation has a single call site and needs its own register
// budget (as a .func ptxas re-serialised the pipelined chunks); NC = 1 callers go through the
// __noinline__ wrapper below so that one copy of the unrolled loops stays in the instruction cache.
template <int NC, class Tab>
__device__ __forceinline__ void lockstep_solve_inl(const PairModel& m, const Tab& tab, const float* lambda,
                                                   const bool* active, SolveStats* st, int& states_out, bool& bad_out) {
  // (kept in registers here: the reference parameters live in the caller's local memory when this is not inlined, and a
  //  load-add-store per chunk on them was 10 % of the pool sizer's stall samples)
  int states;
  bool bad;
  constexpr int CH = Tab::kChunk / NC;                 // states per unrolled chunk (per chain)
  const unsigned full = 0xffffffffu;
  const int K = m.K, N = m.N, NH = N - 1;
  const double mu_l = m.mu_last, r_l = m.r_last;
  const double mu_c[1] = {mu_l}, r_c[1] = {r_l};
  double lam[NC], lamg[NC], lamr_l[NC];
  bool tail_ok[NC], done[NC];
#pragma unroll
  for (int c = 0; c < NC; c++) {
    lam[c] = active[c] ? (double)lambda[c] : 0.0;
    lamg[c] = d_mul((double)lambda[c], 1.000001);
    lamr_l[c] = d_mul(lam[c], r_l);
    tail_ok[c] = d_bits(lamg[c]) <= d_bits(mu_l);
    done[c] = !active[c];
  }
  bad = false;
  states = 0;
  // ------------------------------------------------------------------ pass 1
  P1 a[NC];
#pragma unroll
  for (int c = 0; c < NC; c++) { a[c].p = 1.0; a[c].sum = 1.0; }
  int n = 0;
  bool all_done = false;
  while (n < NH && !all_done) {                       // head: table entries n .. n+cnt-1
    const int cnt = min(CH, NH - n);
    tab.prepare(n);
    double mu0;
#pragma unroll
    for (int c = 0; c < NC; c++) { a[c].mn = 0x7fffffff; a[c].mx = 0; }
    if (cnt == CH) {
      double mu[CH], r[CH];
      tab.template load_chunk<CH>(n, mu, r);
      mu0 = mu[0];
      p1_chunk<NC, CH, true>(a, lam, lamr_l, mu, r);
    } else {
      mu0 = tab.mu_at(n);
      for (int j = 0; j < cnt; j++) {
        double mu, r; tab.load(n + j, mu, r);
#pragma unroll
        for (int c = 0; c < NC; c++) p1_step(a[c], lam[c], mu, r);
      }
    }
    bool any = false;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      // branch-free chunk epilogue (the lanes of a warp are in different situations: a branchy one runs twice)
      const bool live = !done[c];
      states += live ? cnt : 0;
      const bool eok = (n >= m.mono) & (d_bits(lamg[c]) <= d_bits(mu0));
      const bool oob = (a[c].mn < WVA_HI_LO) | (a[c].mx >= WVA_HI_HI);
      const bool tiny = eok & (d_hi(a[c].p) < hi_scale_m54(a[c].sum));
      bad = bad | (live & oob);
      done[c] = done[c] | oob | tiny;
      any = any | !done[c];
    }
    n += cnt;
    all_done = !__any_sync(full, any);
  }
  while (n < K && !all_done) {                        // tail: constant service rate
    const int cnt = min(CH, K - n);
#pragma unroll
    for (int c = 0; c < NC; c++) { a[c].mn = 0x7fffffff; a[c].mx = 0; }
    if (cnt == CH) {
      p1_chunk<NC, CH, false>(a, lam, lamr_l, mu_c, r_c);
    } else {
      for (int j = 0; j < cnt; j++) {
#pragma unroll
        for (int c = 0; c < NC; c++) p1_step_c(a[c], lam[c], lamr_l[c], mu_l, r_l);
      }
    }
    bool any = false;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      const bool live = !done[c];
      states += live ? cnt : 0;
      const bool oob = (a[c].mn < WVA_HI_LO) | (a[c].mx >= WVA_HI_HI);
      const bool tiny = tail_ok[c] & (d_hi(a[c].p) < hi_scale_m54(a[c].sum));
      bad = bad | (live & oob);
      done[c] = done[c] | oob | tiny;
      any = any | !done[c];
    }
    n += cnt;
    all_done = !__any_sync(full, any);
  }
  // ------------------------------------------------------------------ pass 2
  const double cK = 0x1p-55 / (double)K;              // 2x margin covers the rounding of cK itself
  double sum[NC], rsum[NC], Lserv[NC];
  bool reached_K[NC];
  P2 b[NC];
  bool any0 = false;
#pragma unroll
  for (int c = 0; c < NC; c++) {
    sum[c] = a[c].sum;
    if (active[c] && !in_window(sum[c])) bad = true;
    rsum[c] = d_rcp(sum[c]);
    b[c].p = 1.0; b[c].L = 0.0; b[c].pi = 0.0;
    b[c].sumP = d_div(1.0, sum[c]);                   // p[0] = 1/sum
    reached_K[c] = false;
    Lserv[c] = 0.0;
  }
#pragma unroll
  for (int c = 0; c < NC; c++) { done[c] = !active[c] || bad; any0 = any0 || !done[c]; }
  all_done = !__any_sync(full, any0);
  double di = 0.0;                                    // float64(i), shared by the chains
  n = 0;
  while (n < NH && !all_done) {                       // head (i = n+1 <= N-1)
    const int cnt = min(CH, NH - n);
    tab.prepare(n);
    double mu0;
#pragma unroll
    for (int c = 0; c < NC; c++) { b[c].mn = 0x7fffffff; b[c].mx = 0; }
    if (cnt == CH) {
      double mu[CH], r[CH];
      tab.template load_chunk<CH>(n, mu, r);
      mu0 = mu[0];
      p2_chunk<NC, CH, true>(b, lam, lamr_l, mu, r, sum, rsum, di);
    } else {
      mu0 = tab.mu_at(n);
      for (int j = 0; j < cnt; j++) {
        double mu, r; tab.load(n + j, mu, r);
        di = d_add(di, 1.0);
#pragma unroll
        for (int c = 0; c < NC; c++) p2_step(b[c], lam[c], mu, r, sum[c], rsum[c], di);
      }
    }
    bool any = false;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      const bool live = !done[c];
      states += live ? cnt : 0;
      const bool eok = (n >= m.mono) & (d_bits(lamg[c]) <= d_bits(mu0));
      const bool oob = (b[c].mn < WVA_HI_LO) | (b[c].mx >= WVA_HI_HI);
      const int thr = min(d_hi(d_mul(b[c].L, cK)), hi_scale_m54(b[c].sumP));
      const bool tiny = eok & (d_hi(b[c].pi) < thr);
      bad = bad | (live & oob);
      done[c] = done[c] | oob | tiny;
      any = any | !done[c];
    }
    n += cnt;
    all_done = !__any_sync(full, any);
  }
  if (all_done) {
    // every chain left before state N: the accumulators no longer change, so the value the
    // reference computes at i == N (mm1modelstatedependent.go:52-54) is the current one
#pragma unroll
    for (int c = 0; c < NC; c++) Lserv[c] = d_add(b[c].L, d_mul(d_sub(1.0, b[c].sumP), (double)N));
  } else {
    di = d_add(di, 1.0);                              // state i == N uses servRate[N-1]
    bool any = false;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      b[c].mn = 0x7fffffff; b[c].mx = 0;
      p2_step_c(b[c], lam[c], lamr_l[c], mu_l, r_l, sum[c], rsum[c], di);
      {
        const bool live = !done[c];
        states += live ? 1 : 0;
        const bool oob = (b[c].mn < WVA_HI_LO) | (b[c].mx >= WVA_HI_HI);
        Lserv[c] = d_add(b[c].L, d_mul(d_sub(1.0, b[c].sumP), (double)N));
        const int thr = min(d_hi(d_mul(b[c].L, cK)), hi_scale_m54(b[c].sumP));
        const bool tiny = tail_ok[c] & (d_hi(b[c].pi) < thr);
        bad = bad | (live & oob);
        done[c] = done[c] | oob | tiny;
      }
      any = any | !done[c];
    }
    n = N;
    all_done = !__any_sync(full, any);
  }
  while (n < K && !all_done) {                        // tail (i = n+1 in N+1 .. K)
    const int cnt = min(CH, K - n);
#pragma unroll
    for (int c = 0; c < NC; c++) { b[c].mn = 0x7fffffff; b[c].mx = 0; }
    if (cnt == CH) {
      p2_chunk<NC, CH, false>(b, lam, lamr_l, mu_c, r_c, sum, rsum, di);
    } else {
      for (int j = 0; j < cnt; j++) {
        di = d_add(di, 1.0);
#pragma unroll
        for (int c = 0; c < NC; c++) p2_step_c(b[c], lam[c], lamr_l[c], mu_l, r_l, sum[c], rsum[c], di);
      }
    }
    n += cnt;
    bool any = false;
#pragma unroll
    for (int c = 0; c < NC; c++) {
      const bool live = !done[c];
      states += live ? cnt : 0;
      const bool oob = (b[c].mn < WVA_HI_LO) | (b[c].mx >= WVA_HI_HI);
      const bool at_K = n == K;
      const int thr = min(d_hi(d_mul(b[c].L, cK)), hi_scale_m54(b[c].sumP));
      const bool tiny = tail_ok[c] & (d_hi(b[c].pi) < thr);
      bad = bad | (live & oob);
      reached_K[c] = reached_K[c] | (live & !oob & at_K);
      done[c] = done[c] | oob | at_K | tiny;
      any = any | !done[c];
    }
    all_done = !__any_sync(full, any);
  }
#pragma unroll
  for (int c = 0; c < NC; c++) {
    const double pK = reached_K[c] ? b[c].pi : 0.0;   // (E4): an early exit implies p[K] < 2^-53
    SolveStats& s = st[c];
    s.avgNumInServers = (float)Lserv[c];
    s.avgNumInSystem = (float)b[c].L;
    s.throughput = f_mul(lambda[c], f_sub(1.0f, (float)pK));
    s.avgRespTime = f_div(s.avgNumInSystem, s.throughput);
    s.avgServTime = f_div(s.avgNumInServers, s.throughput);
    float w = f_sub(s.avgRespTime, s.avgServTime);
    s.avgWaitTime = (w < 0.0f) ? 0.0f : w;
  }
  states_out = states;
  bad_out = bad;
}

template <int NC, class Tab>
__device__ __noinline__ void lockstep_solve_n(const PairModel& m, const Tab tab, const float* lambda,
                                              const bool* active, SolveStats* st, int& states, bool& bad) {
  lockstep_solve_inl<NC, Tab>(m, tab, lambda, active, st, states, bad);
}

template <class Tab>
__device__ __forceinline__ void lockstep_solve(const PairModel& m, const Tab tab, float lambda, bool active,
                                               SolveStats& st, int& states, bool& bad) {
  lockstep_solve_n<1, Tab>(m, tab, &lambda, &active, &st, states, bad);
}

// ---- (E12) certified fast solve: one head pass per lane, closed-form tail, exact solver for the rest --------------
// Head chunk, software-pipelined like p1_chunk (stage s of state j at slot 3j + s):
//   0: x = p*lam, q0 = p*lamr (+ exponent window)   1: rem   2: p'   3: sum += p', T = fma(j, p', T)
//   4: m = min(2^-53 sum, p')   5: A += m
template <int CH>
__device__ __forceinline__ void fast_chunk(FastHead& h, double lam, const double (&mu)[CH], const double (&r)[CH], double dn,
                                           int& mn, int& mx) {
  double x[CH], q0[CH], rem[CH], pn[CH + 1], sm[CH + 1], mm[CH], lamr[CH];
  pn[0] = h.p; sm[0] = h.sum;
#pragma unroll
  for (int j = 0; j < CH; j++) lamr[j] = d_mul(lam, r[j]);
#pragma unroll
  for (int slot = 0; slot < 3 * CH + 3; slot++) {
#pragma unroll
    for (int j = 0; j < CH; j++) {
      const int st = slot - 3 * j;
      if (st == 0) {
        x[j] = d_mul(pn[j], lam);
        q0[j] = d_mul(pn[j], lamr[j]);
        const int hw = d_hi(x[j]);
        mn = min(mn, hw); mx = max(mx, hw);
      }
      if (st == 1) rem[j] = d_fma(-q0[j], mu[j], x[j]);
      if (st == 2) pn[j + 1] = d_fma(rem[j], r[j], q0[j]);
      if (st == 3) { sm[j + 1] = d_add(sm[j], pn[j + 1]); h.T = d_fma(d_add(dn, (double)(j + 1)), pn[j + 1], h.T); }
      if (st == 4) mm[j] = d_min(d_mul(sm[j + 1], 0x1p-53), pn[j + 1]);
      if (st == 5) h.A = d_add(h.A, mm[j]);
    }
  }
  h.p = pn[CH]; h.sum = sm[CH];
}

// Phase profile of the fast solve (tools/perf_pool_phases.py): built with -DWVA_POOL_PHASES, lockstep_solve_fast_only
// adds lane 0's clock64() cycles of the first chunk's table preparation (nothing for RateTable), the head chunks and
// fast_solve_finish to ph[0..2].  The product build compiles none of it.
#ifdef WVA_POOL_PHASES
#define FAST_PH(...) __VA_ARGS__
#else
#define FAST_PH(...)
#endif
struct FastPhases { long long wait0, chunks, finish; };

// One solve per lane at `lambda` (inactive lanes ride along): the fast head pass for every active lane, then the
// closed-form tail and certification (fast_solve_finish).  Sets `cert` where st holds the reference's statistics and
// returns the head states visited.
template <class Tab>
__device__ __forceinline__ int lockstep_fast_head(const PairModel& m, const Tab tab, float lambda, bool active,
                                                  SolveStats& st, bool& cert, FastPhases& ph) {
  constexpr int CH = Tab::kChunk;
  static_assert(CH == WVA_TILE_CHUNK, "the head pass exits at the chunk boundaries the host replay (fast_solve) uses");
  const unsigned full = 0xffffffffu;
  const int NH = m.N - 1;
  double lam = active ? (double)lambda : 0.0;
  FastHead h;
  h.p = 1.0; h.sum = 1.0; h.T = 0.0; h.A = 0.0; h.n = 0; h.ok = true; h.exited = false;
  bool live = active;
  int states = 0, n = 0;
  double p_exit = 0.0;
  FAST_PH(const long long ph_t0 = clock64();)
  while (n < NH && __any_sync(full, live)) {
    const int cnt = min(CH, NH - n);
    FAST_PH(const long long ph_w = clock64();)
    tab.prepare(n);
    FAST_PH(if (n == 0) ph.wait0 += clock64() - ph_w;)
    double mu0;
    int mn = 0x7fffffff, mx = 0;
    if (cnt == CH) {
      double mu[CH], r[CH];
      tab.template load_chunk<CH>(n, mu, r);
      mu0 = mu[0];
      fast_chunk<CH>(h, lam, mu, r, (double)n, mn, mx);
    } else {
      mu0 = tab.mu_at(n);
      for (int j = 0; j < cnt; j++) {
        double mu, r; tab.load(n + j, mu, r);
        h.p = step_div(h.p, lam, d_mul(lam, r), mu, r, mn, mx);
        h.sum = d_add(h.sum, h.p);
        h.T = d_fma((double)(n + j + 1), h.p, h.T);
        h.A = d_add(h.A, d_min(d_mul(h.sum, 0x1p-53), h.p));
      }
    }
    states += live ? cnt : 0;
    const int n0 = n;
    n += cnt;
    // a lane that leaves keeps running with lambda = 0: its terms are 0 and its accumulators stay as they are
    const bool oob = live & ((mn < WVA_HI_LO) | (mx >= WVA_HI_HI));
    const bool leave = live & !oob & (n < NH) & fast_head_exit(m, lam, mu0, n0, n, h.p, h.sum);
    h.ok = h.ok & !oob;
    if (leave) { h.exited = true; h.n = n; p_exit = h.p; }
    if (oob | leave) { live = false; lam = 0.0; }
  }
  if (h.exited) h.p = p_exit;
  else h.n = n;
  FAST_PH(const long long ph_t1 = clock64(); ph.chunks += ph_t1 - ph_t0;)
  cert = active && fast_solve_finish(m, lambda, h, st);
  FAST_PH(__syncwarp(); ph.finish += clock64() - ph_t1;)
  return states;
}

// The fast solve, then the exact lockstep_solve for the lanes that were not certified (in the same batch: for callers
// whose fallbacks are too rare to queue).  Returns the states visited (the fallback's included), or -1 - states when the
// solve is `bad` as for lockstep_solve (by value: out-parameters cost the callers stack and spills).  Every lane that
// takes the exact solver adds 1 to *fallbacks (rare: a counter in registers would be live across the caller's whole loop).
template <class Tab>
__device__ __noinline__ int lockstep_solve_fast(const PairModel& m, const Tab tab, float lambda, bool active, SolveStats& st,
                                                unsigned long long* fallbacks) {
  const unsigned full = 0xffffffffu;
  bool cert;
  FastPhases ph{};
  int states = lockstep_fast_head(m, tab, lambda, active, st, cert, ph);
  const bool redo = active && !cert;
  bool bad = false;
  if (__any_sync(full, redo)) {
    SolveStats st2;
    int sv = 0;
    lockstep_solve(m, tab, lambda, redo, st2, sv, bad);
    if (redo) { st = st2; states += sv; atomicAdd(fallbacks, 1ull); }
  }
  return bad ? -1 - states : states;
}

// The fast solve alone, for callers that queue the lanes it does not certify for an exact batch of their own: returns
// the head states visited, or -1 - states when the lane's solve is not certified.
template <class Tab>
__device__ __noinline__ int lockstep_solve_fast_only(const PairModel& m, const Tab tab, float lambda, bool active,
                                                     SolveStats& st FAST_PH(, unsigned long long* ph_out)) {
  bool cert;
  FastPhases ph{};
  const int states = lockstep_fast_head(m, tab, lambda, active, st, cert, ph);
  FAST_PH(if ((threadIdx.x & 31) == 0) { ph_out[0] += ph.wait0; ph_out[1] += ph.chunks; ph_out[2] += ph.finish; })
  return cert || !active ? states : -1 - states;
}

#endif  // __CUDACC__
}  // namespace wva
