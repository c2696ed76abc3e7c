// TEST INFRASTRUCTURE ONLY — host replay of the certified fast solve (E12, csrc/wva_core.cuh fast_solve) next to the
// literal chain solver of emul.cpp.  Never linked into the product.
#include "emul.cpp"
#include <cmath>

namespace {

// a configs[2]-shaped queue model (synth.queue_system's parameter ranges) with max batch N
struct RandModel {
  PairModel m;
  std::vector<float> tab;
};
void rand_model(std::mt19937_64& g, int N, RandModel& r) {
  std::uniform_real_distribution<float> ua(4.0f, 20.0f), ub(0.01f, 0.3f), ug(5e-4f, 2e-2f), sp(0.5f, 2.0f);
  std::uniform_int_distribution<int> ui(16, 4096), uo(8, 1024);
  const float speed = sp(g);
  model_init(r.m, ua(g) * speed, ub(g) * speed, ug(g) * speed, ui(g), uo(g), N);
  r.tab.assign((size_t)N, 0.0f);
  model_fill_table(r.m, r.tab.data(), 1, 0, 1);
  model_finish(r.m, r.tab.data(), 1);
}
// lambda over [lambda_min, lambda_max], half of the draws with lambda / lambda_max in [0.95, 1]
float rand_lambda(std::mt19937_64& g, const PairModel& m) {
  std::uniform_real_distribution<double> u01(0.0, 1.0);
  const double lo = m.lambda_min, hi = m.lambda_max;
  const double x = (g() & 1) ? lo + (hi - lo) * u01(g) : hi * (0.95 + 0.05 * u01(g));
  float f = (float)x;
  if (f < m.lambda_min) f = m.lambda_min;
  if (f > m.lambda_max) f = m.lambda_max;
  return f;
}
bool same_bits(const SolveStats& a, const SolveStats& b) { return memcmp(&a, &b, sizeof(SolveStats)) == 0; }
// does a head term p~[n] lambda leave the exponent window (E3)?  The exact lock-step solver marks such solves `bad`
// and sends the pair to the literal slow path as well.
bool head_leaves_window(const PairModel& m, float lambda) {
  double p = 1.0;
  const double lam = (double)lambda;
  for (int n = 0; n < m.N - 1; n++) {
    const double x = d_mul(p, lam);
    if (!in_window(x)) return true;
    p = d_div(x, (double)m.tab[n]);
  }
  return false;
}

// relative distance of v from the nearest float32 rounding boundary
double f32_boundary_dist(double v) {
  const float f = (float)v;
  const float nb = nextafterf(f, (double)f < v ? INFINITY : -INFINITY);
  const double mid = 0.5 * ((double)f + (double)nb);
  return fabs(v - mid) / v;
}

}  // namespace

extern "C" {

// n random solves at max batch N: the fast solve against the literal chain solver.
// stats[0] certified, [1] not certified, [2] certified lanes whose SolveStats differ in any bit, [3] overflow (skipped),
// [4] not certified because a head term left the exponent window
int emul_check_fast_solve(int64_t n, uint64_t seed, int N, int64_t* stats) {
  std::mt19937_64 g(seed);
  for (int i = 0; i < 5; i++) stats[i] = 0;
  RandModel r;
  for (int64_t i = 0; i < n; i++) {
    if (i % 64 == 0) rand_model(g, N, r);
    const float x = rand_lambda(g, r.m);
    bool ovf = false;
    const SolveStats ref = host_solve(r.m, x, &ovf);
    if (ovf) { stats[3]++; continue; }
    SolveStats st{};
    int sv = 0;
    if (fast_solve(r.m, x, st, &sv)) {
      stats[0]++;
      if (!same_bits(st, ref)) stats[2]++;
    } else {
      stats[1]++;
      if (head_leaves_window(r.m, x)) stats[4]++;
    }
  }
  return 0;
}

// Solves whose reference float64 L or Lserv lies near a float32 rounding boundary.
// stats[0] values within `band` (relative) of a boundary, [1] of those certified, [2] of those certified with SolveStats
// that differ from the reference, [3] values within the a-priori floor of the enclosure (4 (3K+2) u for L,
// 4 (5N+4) u for Lserv), [4] of those certified
int emul_fast_boundary(int64_t n, uint64_t seed, int N, double band, int64_t* stats) {
  std::mt19937_64 g(seed);
  for (int i = 0; i < 5; i++) stats[i] = 0;
  RandModel r;
  for (int64_t i = 0; i < n; i++) {
    if (i % 64 == 0) rand_model(g, N, r);
    const float x = rand_lambda(g, r.m);
    Chain c; SolveStats ref{};
    chain_start(c, x);
    c.tail_ok = d_bits(c.lamg) <= d_bits(r.m.mu_last);
    while (!chain_step(c, r.m, ref)) {}
    if (c.phase == CH_OVERFLOW) continue;
    const double dL = f32_boundary_dist(c.L), dLs = f32_boundary_dist(c.Lserv);
    const double u = 0x1p-53;
    const bool floor_hit = dL < 4.0 * (3.0 * r.m.K + 2.0) * u || dLs < 4.0 * (5.0 * N + 4.0) * u;
    if (!(dL < band || dLs < band) && !floor_hit) continue;
    SolveStats st{};
    int sv = 0;
    const bool cert = fast_solve(r.m, x, st, &sv);
    if (dL < band || dLs < band) {
      stats[0]++;
      if (cert) { stats[1]++; if (!same_bits(st, ref)) stats[2]++; }
    }
    if (floor_hit) { stats[3]++; if (cert) stats[4]++; }
  }
  return 0;
}

// System.Calculate through the lane state machine with every chain solve taken by the fast solve, the literal
// chain solver where it is not certified.  counts: [0] solves, [1] not certified, [2] overflow redos
int emul_calculate_fast(const wva_system* sys, wva_candidates* out, int64_t* counts) {
  SysView s = make_view(sys);
  CandView o;
  o.state = out->state; o.num_replicas = out->num_replicas; o.batch_size = out->batch_size; o.cost = out->cost;
  o.value = out->value; o.itl = out->itl; o.ttft = out->ttft; o.rho = out->rho; o.max_arrv_rate = out->max_arrv_rate;
  o.n_solves = out->n_solves;
  counts[0] = counts[1] = counts[2] = 0;
  std::vector<float> tab;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++) {
      SizerLane z;
      int lim = 0;
      if (sizer_setup(z, s, o, srv, acc, 1 << 20, &lim) == SETUP_DONE) continue;
      tab.assign((size_t)z.m.N, 0.0f);
      model_fill_table(z.m, tab.data(), 1, 0, 1);
      model_finish(z.m, tab.data(), 1);
      bool live = sizer_begin(z, s, o);
      while (live) {
        SolveStats st{};
        int sv = 0;
        counts[0]++;
        if (fast_solve(z.m, z.c.lambda, st, &sv)) {
          z.c.states = sv;
        } else {
          counts[1]++;
          while (!chain_step(z.c, z.m, st)) {}
          if (z.c.phase == CH_OVERFLOW) {
            // the literal stored-p[] algorithm from the start of the pair (overflow_slow_kernel)
            counts[2]++;
            SizerLane y;
            int lim2 = 0;
            sizer_setup(y, s, o, srv, acc, 1 << 20, &lim2);
            model_finish(y.m, tab.data(), 1);
            std::vector<double> p((size_t)y.m.K + 1);
            bool bad = false;
            bool l2 = sizer_begin(y, s, o);
            while (l2) {
              literal_solve(y.m, y.cur_x, p.data(), st, &bad);
              y.c.states = y.m.K + 1;
              l2 = sizer_on_solve(y, s, o, st);
            }
            break;
          }
        }
        live = sizer_on_solve(z, s, o, st);
      }
    }
  return 0;
}

}  // extern "C"
