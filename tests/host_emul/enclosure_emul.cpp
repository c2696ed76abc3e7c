// TEST INFRASTRUCTURE ONLY — the error bounds of the certified fast solve (E12, csrc/wva_core.cuh fast_solve_finish)
// against exact arithmetic.  fast_solve_finish hands its values and bounds to WVA_FAST_PROBE (empty in the product);
// this build records them, and compares them with
//   - a binary128 (__float128) term-by-term chain over all K + 1 states on the same float32 lambda and mu values
//     ("exact": no closed form, nothing shared with the code under test), and
//   - a literal float64 chain in the reference's loop order (stored p[], normalise, then accumulate): the reference's
//     float64 values, whose float32 statistics are checked against literal_solve and the exact lane solver.
// Never linked into the product.
#include <cstdint>

namespace {
struct ProbeRec {
  bool hit;
  double L, Ls, pK, eL, fL, eLs, fLs, epK, fpK;
  bool exited;
};
thread_local ProbeRec g_probe;
}  // namespace
#define WVA_FAST_PROBE(L_, Ls_, pK_, eL_, fL_, eLs_, fLs_, epK_, fpK_, exited_) \
  (g_probe = ProbeRec{true, L_, Ls_, pK_, eL_, fL_, eLs_, fLs_, epK_, fpK_, exited_})

#include "fast_emul.cpp"
#include <algorithm>

namespace {

typedef __float128 q128;

struct Vals { q128 L, Ls, pK; };

// exact chain: p_0 = 1, p_{n+1} = p_n lambda / mu_min(n, N-1); L = sum n p_n / S, Lserv = sum min(n, N) p_n / S,
// p[K] = p_K / S.  113-bit significand: the relative error is below 4 (K + 1) 2^-113.
Vals exact_chain(const float* tab, int N, int K, float lambda) {
  const q128 lam = (q128)lambda;
  q128 p = 1, S = 1, T = 0, U = 0;
  for (int n = 0; n < K; n++) {
    p = p * lam / (q128)tab[n < N ? n : N - 1];
    S += p;
    T += (q128)(n + 1) * p;
    U += (q128)(n + 1 < N ? n + 1 : N) * p;
  }
  return Vals{T / S, U / S, p / S};
}

// the reference's float64 chain (MM1ModelStateDependent.Solve without its overflow rescaling; false when that would be
// needed).  Plain IEEE operators (the test build uses -ffp-contract=off).
bool ref64_chain(const float* tab, int N, int K, float lambda, std::vector<double>& p, double* L_out, double* Ls_out,
                 double* pK_out, SolveStats& st) {
  const double lam = (double)lambda;
  p.assign((size_t)K + 1, 0.0);
  p[0] = 1.0;
  for (int n = 0; n < K; n++) p[n + 1] = p[n] * lam / (double)tab[n < N ? n : N - 1];
  double sum = 0.0;
  for (int n = 0; n <= K; n++) sum += p[n];
  if (!(sum <= DBL_MAX)) return false;
  for (int n = 0; n <= K; n++) p[n] = p[n] / sum;
  double L = 0.0, Ls = 0.0, sumP = p[0];
  for (int i = 1; i <= K; i++) {
    L += (double)i * p[i];
    sumP += p[i];
    if (i == N) Ls = L + (1.0 - sumP) * (double)N;
  }
  *L_out = L; *Ls_out = Ls; *pK_out = p[K];
  st.avgNumInServers = (float)Ls;
  st.avgNumInSystem = (float)L;
  st.throughput = lambda * (1.0f - (float)p[K]);
  st.avgRespTime = st.avgNumInSystem / st.throughput;
  st.avgServTime = st.avgNumInServers / st.throughput;
  const float w = st.avgRespTime - st.avgServTime;
  st.avgWaitTime = w < 0.0f ? 0.0f : w;
  return true;
}

double q_abs_diff(double v, q128 x) {
  q128 d = (q128)v - x;
  return (double)(d < 0 ? -d : d);
}
double ratio(double err, double bound) {
  if (err == 0.0) return 0.0;
  return bound > 0.0 ? err / bound : INFINITY;
}

enum { RG_RANDOM = 0, RG_LMAX = 1, RG_FLOOR = 2, RG_LIGHT = 3, RG_NONMONO = 4, RG_HEAVY_PK = 5 };

// 1 - rho as fast_solve_finish forms it
double one_minus_rho(const PairModel& m, float lambda) { return d_div(d_sub(m.mu_last, (double)lambda), m.mu_last); }

// lambda with 1 - rho >= 2^-12 where p[K] is likely to land in [2^-26, 2^-8]
float heavy_lambda(std::mt19937_64& g, const PairModel& m) {
  std::uniform_real_distribution<double> u01(0.0, 1.0);
  const double M = (double)(m.K - m.N + 1);
  const double lo = std::max(0x1p-12, 0.2 / M), hi = std::min(0.5, 20.0 / M);
  float x = (float)(m.mu_last * (1.0 - exp(log(lo) + (log(hi) - log(lo)) * u01(g))));
  while (!(one_minus_rho(m, x) >= WVA_FAST_OMEGA_MIN)) x = nextafterf(x, 0.0f);
  return x;
}

// one draw of regime `rg`; false: no usable draw (the caller skips it)
bool draw(int rg, std::mt19937_64& g, int N, int64_t i, RandModel& r, float* lambda) {
  std::uniform_real_distribution<double> u01(0.0, 1.0);
  auto log_uniform = [&](double lo, double hi) { return exp(log(lo) + (log(hi) - log(lo)) * u01(g)); };
  switch (rg) {
    case RG_RANDOM:
      if (i % 64 == 0) rand_model(g, N, r);
      *lambda = rand_lambda(g, r.m);
      return true;
    case RG_LMAX:
      rand_model(g, N, r);
      *lambda = r.m.lambda_max;
      return true;
    case RG_FLOOR: {  // 1 - rho in [2^-12, 2^-10]: above lambda_max, never admitted by the sizer, still claimed by the guard
      rand_model(g, N, r);
      float x = (float)(r.m.mu_last * (1.0 - log_uniform(0x1p-12, 0x1p-10)));
      while (!(one_minus_rho(r.m, x) >= WVA_FAST_OMEGA_MIN)) x = nextafterf(x, 0.0f);
      *lambda = x;
      return true;
    }
    case RG_LIGHT: {  // lambda <= mu_0 / 64: from N = 18 on the head pass leaves after its first chunk
      rand_model(g, N, r);
      const double mu0 = (double)r.m.tab[0];
      *lambda = (float)log_uniform((double)r.m.lambda_min, mu0 / 64.0);
      return true;
    }
    case RG_NONMONO: {  // arbitrary positive table with at least one descent (mono > 0)
      rand_model(g, N, r);
      const double base = (double)r.tab[(size_t)N - 1];
      for (int n = 0; n < N; n++) r.tab[n] = (float)(base * (0.9 + 0.7 * u01(g)));
      model_finish(r.m, r.tab.data(), 1);
      if (r.m.mono == 0) { r.tab[0] = 1.25f * r.tab[1]; model_finish(r.m, r.tab.data(), 1); }
      if (r.m.mono == 0) return false;
      *lambda = (float)(r.m.mu_last * (0.05 + 0.949 * u01(g)));
      return true;
    }
    case RG_HEAVY_PK:  // p[K] in [2^-26, 2^-8] (the f_sub(1, .) rule); the caller filters on p[K]
      rand_model(g, N, r);
      *lambda = heavy_lambda(g, r.m);
      return true;
  }
  return false;
}

}  // namespace

extern "C" {

// The bounds of fast_solve_finish against exact arithmetic for n draws of regime rg at max batch N.
// out[0] draws, [1] probed (the enclosure was formed), [2] certified, [3] probed lanes that left the head early,
// [4..6] largest |ref64 - exact| / (a) for L, Lserv, p[K], [7..9] largest |fast - exact| / (b) for L, Lserv, p[K],
// [10..15] the number of ratios above 1 in the same order, [16] probed solves whose literal float64 chain's float32
// statistics differ from literal_solve or from the exact lane solver, [17] certified lanes whose statistics differ from
// the literal chain's, [18] probed solves skipped (the reference would rescale on float64 overflow),
// [19] probed solves with a subnormal fast p[K], [20] probed solves with p[K] in [2^-26, 2^-8]
int enc_cell(int rg, int N, int64_t n, uint64_t seed, double* out) {
  std::mt19937_64 g(seed);
  for (int k = 0; k < 21; k++) out[k] = 0.0;
  RandModel r;
  std::vector<double> p, p2;
  for (int64_t i = 0; i < n; i++) {
    float x = 0.0f;
    if (!draw(rg, g, N, i, r, &x)) continue;
    out[0]++;
    SolveStats st{};
    int sv = 0;
    g_probe.hit = false;
    const bool cert = fast_solve(r.m, x, st, &sv);
    if (!g_probe.hit) continue;
    const ProbeRec pr = g_probe;
    if (rg == RG_HEAVY_PK && !(pr.pK >= 0x1p-26 && pr.pK <= 0x1p-8)) continue;
    out[1]++;
    if (cert) out[2]++;
    if (pr.exited) out[3]++;
    if (pr.pK > 0.0 && pr.pK < DBL_MIN) out[19]++;
    if (pr.pK >= 0x1p-26 && pr.pK <= 0x1p-8) out[20]++;
    double L64, Ls64, pK64;
    SolveStats st64{};
    if (!ref64_chain(r.m.tab, N, r.m.K, x, p, &L64, &Ls64, &pK64, st64)) { out[18]++; continue; }
    SolveStats lit{};
    bool patho = false;
    p2.assign((size_t)r.m.K + 1, 0.0);
    literal_solve(r.m, x, p2.data(), lit, &patho);
    bool ovf = false;
    const SolveStats lane = host_solve(r.m, x, &ovf);
    if (patho || ovf || !same_bits(st64, lit) || !same_bits(st64, lane)) out[16]++;
    if (cert && !same_bits(st, st64)) out[17]++;
    const Vals ex = exact_chain(r.m.tab, N, r.m.K, x);
    const double ra[3] = {ratio(q_abs_diff(L64, ex.L), pr.fL), ratio(q_abs_diff(Ls64, ex.Ls), pr.fLs),
                          ratio(q_abs_diff(pK64, ex.pK), pr.fpK)};
    const double rb[3] = {ratio(q_abs_diff(pr.L, ex.L), pr.eL), ratio(q_abs_diff(pr.Ls, ex.Ls), pr.eLs),
                          ratio(q_abs_diff(pr.pK, ex.pK), pr.epK)};
    for (int k = 0; k < 3; k++) {
      out[4 + k] = std::max(out[4 + k], ra[k]);
      out[7 + k] = std::max(out[7 + k], rb[k]);
      if (ra[k] > 1.0) out[10 + k]++;
      if (rb[k] > 1.0) out[13 + k]++;
    }
  }
  return 0;
}

// The binary128 chain on caller-given values: L, Lserv, p[K] each as (hi, lo, e) with value (hi + lo) 2^e, hi in
// [1/2, 1) (hi + lo carries 106 bits; p[K] may lie far below the float64 range).
int enc_exact(const float* tab, int N, int K, float lambda, double* out) {
  const Vals v = exact_chain(tab, N, K, lambda);
  const q128 a[3] = {v.L, v.Ls, v.pK};
  for (int k = 0; k < 3; k++) {
    q128 x = a[k];
    int e = 0;
    while (x > 0 && x < (q128)0.5) { x *= (q128)2; e--; }
    while (x >= (q128)1) { x /= (q128)2; e++; }
    const double hi = (double)x;
    out[3 * k] = hi;
    out[3 * k + 1] = (double)(x - (q128)hi);
    out[3 * k + 2] = (double)e;
  }
  return 0;
}

// Boundary search: per configs[2]-shaped model, `steps` consecutive float32 lambda (nextafterf, downward from a
// rand_lambda draw, or for every other model from a lambda with p[K] likely in [2^-26, 2^-8]).  A solve whose enclosure
// is formed is solved again by the exact lane solver when its fast L or Lserv lies within 10^-9 of a float32 midpoint;
// both lambda next to a step where the fast f_sub(1, (float)p[K]) changes are solved again as well (with float32
// lambda, p[K] moves by ~10^-7 relative per step, so those two are as close to that boundary as any lambda gets).
// stats: [0] solves whose reference L or Lserv lies within `band` (relative) of a float32 midpoint, or that sit next to
// a change of f_sub(1, (float)p[K]); [1] of those certified; [2] of those certified with statistics that differ from the
// reference; [3] solves within the a-priori floor of the enclosure (4 (3K+2) u for L, 4 (5N+4) u for Lserv); [4] of
// those certified; [5] solves whose enclosure was formed; [6] of [0] next to a change of f_sub(1, (float)p[K])
int enc_boundary(int N, int64_t n_models, int steps, uint64_t seed, double band, int64_t* stats) {
  std::mt19937_64 g(seed);
  for (int k = 0; k < 7; k++) stats[k] = 0;
  const double pre = 1e-9, u = 0x1p-53;
  RandModel r;
  auto check = [&](float x, bool pk_edge) {
    SolveStats st{};
    int sv = 0;
    const bool cert = fast_solve(r.m, x, st, &sv);
    Chain c; SolveStats ref{};
    chain_start(c, x);
    c.tail_ok = d_bits(c.lamg) <= d_bits(r.m.mu_last);
    while (!chain_step(c, r.m, ref)) {}
    if (c.phase == CH_OVERFLOW) return;
    const double dL = f32_boundary_dist(c.L), dLs = f32_boundary_dist(c.Lserv);
    const bool near = dL < band || dLs < band || pk_edge;
    const bool floor_hit = dL < 4.0 * (3.0 * r.m.K + 2.0) * u || dLs < 4.0 * (5.0 * N + 4.0) * u;
    if (near) {
      stats[0]++;
      if (pk_edge) stats[6]++;
      if (cert) { stats[1]++; if (!same_bits(st, ref)) stats[2]++; }
    }
    if (floor_hit) { stats[3]++; if (cert) stats[4]++; }
  };
  for (int64_t mi = 0; mi < n_models; mi++) {
    rand_model(g, N, r);
    float x = (mi & 1) ? heavy_lambda(g, r.m) : rand_lambda(g, r.m);
    bool prev_hit = false;
    float prev_x = 0.0f, prev_om = 0.0f;
    for (int s = 0; s < steps; s++, x = nextafterf(x, 0.0f)) {
      SolveStats st{};
      int sv = 0;
      g_probe.hit = false;
      fast_solve(r.m, x, st, &sv);
      if (!g_probe.hit) { prev_hit = false; continue; }
      stats[5]++;
      const ProbeRec pr = g_probe;
      const float om = f_sub(1.0f, (float)pr.pK);
      if (prev_hit && om != prev_om) {
        check(prev_x, true);
        check(x, true);
      } else if (f32_boundary_dist(pr.L) < pre || f32_boundary_dist(pr.Ls) < pre) {
        check(x, false);
      }
      prev_hit = true; prev_x = x; prev_om = om;
    }
  }
  return 0;
}

}  // extern "C"
