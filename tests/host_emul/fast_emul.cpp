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

// does a head term p~[n] lambda reach 2^500?  (Terms that fall below 2^-500 come after the exact lock-step solver's
// early exit on sane inputs; these are the ones it marks `bad`.)
bool head_grows_past_window(const PairModel& m, float lambda) {
  double p = 1.0;
  const double lam = (double)lambda;
  for (int n = 0; n < m.N - 1; n++) {
    const double x = d_mul(p, lam);
    if (!(x < 0x1p500)) return true;
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
// chain solver where it is not certified.  counts: [0] solves, [1] not certified, [2] overflow redos, [3] pairs redone
// like an overflow because a solve that was not certified grows past the exponent window (a head term or the sum at
// 2^500 or above: the device's exact lock-step solver marks it `bad`, and the pair goes to the literal slow path)
int emul_calculate_fast(const wva_system* sys, wva_candidates* out, int64_t* counts) {
  SysView s = make_view(sys);
  CandView o;
  o.state = out->state; o.num_replicas = out->num_replicas; o.batch_size = out->batch_size; o.cost = out->cost;
  o.value = out->value; o.itl = out->itl; o.ttft = out->ttft; o.rho = out->rho; o.max_arrv_rate = out->max_arrv_rate;
  o.n_solves = out->n_solves;
  counts[0] = counts[1] = counts[2] = counts[3] = 0;
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
        if (!z.m.e1_ok) {
          // a service rate outside the (E1) divisor range: the device solves every chain of the pair with the per-lane
          // chain (IEEE divisions), neither the fast solve nor the lock-step solver
          while (!chain_step(z.c, z.m, st)) {}
          if (z.c.phase == CH_OVERFLOW) {
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
        } else if (fast_solve(z.m, z.c.lambda, st, &sv)) {
          z.c.states = sv;
        } else {
          counts[1]++;
          const float x = z.c.lambda;
          while (!chain_step(z.c, z.m, st)) {}
          const bool ovf = z.c.phase == CH_OVERFLOW;
          if (ovf || head_grows_past_window(z.m, x) || !z.c.sum_ok) {
            // the literal stored-p[] algorithm from the start of the pair (overflow_slow_kernel)
            counts[ovf ? 2 : 3]++;
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

// ---- replica grid with deferral (grid_kernel.cuh grid_kernel + grid_deferred_kernel), replayed level by level

// grid_setup with the pair's arrival rate given; false: every level of the pair is "not ok"
static bool grid_pair(const SysView& s, int srv, int acc, float arrival, PairModel& m, std::vector<float>& tab,
                      float* total_rate, float* slo_ttft, float* slo_itl, float* slo_tps) {
  const int in_tok = s.srv_in_tokens[srv], out_tok = s.srv_out_tokens[srv], model = s.srv_model[srv];
  if (arrival < 0.0f || in_tok < 0 || out_tok < 0 || model < 0 || model >= s.n_models) return false;
  const size_t pi = (size_t)model * s.n_acc + acc;
  if (!s.perf_present[pi] || !s.srv_target_present[srv] || arrival == 0.0f || out_tok == 0) return false;
  long long N;
  if (s.srv_max_batch[srv] > 0) N = s.srv_max_batch[srv];
  else { N = (long long)s.perf_max_batch[pi] * s.perf_at_tokens[pi] / out_tok; if (N < 1) N = 1; }
  model_init(m, s.perf_alpha[pi], s.perf_beta[pi], s.perf_gamma[pi], in_tok, out_tok, (int)N);
  tab.assign((size_t)N, 0.0f);
  model_fill_table(m, tab.data(), 1, 0, 1);
  model_finish(m, tab.data(), 1);
  *slo_ttft = s.srv_slo_ttft[srv]; *slo_itl = s.srv_slo_itl[srv]; *slo_tps = s.srv_slo_tps[srv];
  *total_rate = (*slo_tps == 0.0f) ? f_div(arrival, 60.0f) : f_div(*slo_tps, (float)out_tok);
  return true;
}
// the level's arrival rate and whether grid_kernel defers it (its ratio lambda / mu_{N-1} above thr)
static bool grid_level(const PairModel& m, float total_rate, int r, float thr, float* lambda, bool* deferred) {
  const float rate = f_div(total_rate, (float)r);
  *lambda = f_div(rate, 1000.0f);
  const bool admitted = analyze_admits(m, rate);
  *deferred = admitted && *lambda / (float)m.mu_last > thr;
  return admitted;
}

extern "C" {

// wva_analyze_grid with deferral at threshold thr (thr <= 0: none): the levels grid_kernel keeps are solved by the
// exact chain solver, the deferred ones by the fast solve and, where it is not certified, the exact chain solver, as
// grid_deferred_kernel does for a batch of one N.  Outputs [S, A, R] and frontier [S, A] as wva_analyze_grid.
// counts: [0] levels solved, [1] deferred levels, [2] deferred levels not certified by the fast solve, [3] overflow
int emul_grid_deferred(const wva_system* sys, int R, float thr, uint8_t* ok, float* ttft, float* itl, float* rho,
                       float* tput, int32_t* frontier, int64_t* counts) {
  SysView s = make_view(sys);
  for (int k = 0; k < 4; k++) counts[k] = 0;
  std::vector<float> tab;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++) {
      const size_t pair = (size_t)srv * s.n_acc + acc;
      PairModel m;
      float total_rate = 0, slo_ttft = 0, slo_itl = 0, slo_tps = 0;
      const bool valid = grid_pair(s, srv, acc, s.srv_arrival[srv], m, tab, &total_rate, &slo_ttft, &slo_itl, &slo_tps);
      const float lambda_tps = valid ? f_mul(m.lambda_max, f_sub(1.0f, WVA_STABILITY_SAFETY)) : 0.0f;
      int front = 0;
      for (int r = 1; r <= R; r++) {
        const size_t o = pair * (size_t)R + (size_t)(r - 1);
        ok[o] = 0; ttft[o] = itl[o] = rho[o] = tput[o] = 0.0f;
        float lambda;
        bool deferred;
        if (!valid || !grid_level(m, total_rate, r, thr, &lambda, &deferred)) continue;
        deferred = deferred && thr > 0.0f;
        counts[0]++;
        SolveStats st{};
        bool solved = false;
        if (deferred) counts[1]++;
        if (deferred && m.e1_ok) {                     // grid_deferred_kernel: per-lane chain for the other pairs
          int sv = 0;
          solved = fast_solve(m, lambda, st, &sv);
          if (!solved) counts[2]++;
        }
        if (!solved) {
          bool ovf = false;
          st = host_solve(m, lambda, &ovf);
          if (ovf) { counts[3]++; continue; }
        }
        float pf, dec, avg_ttft;
        eval_values(m, st, &avg_ttft, &dec, &pf);
        float rh = f_div(st.avgNumInServers, (float)m.N);
        rh = fminf(fmaxf(rh, 0.0f), 1.0f);
        ok[o] = 1;
        ttft[o] = f_add(st.avgWaitTime, pf);
        itl[o] = dec;
        rho[o] = rh;
        tput[o] = f_mul(st.throughput, 1000.0f);
        const bool meets = (slo_ttft <= 0.0f || avg_ttft <= slo_ttft) && (slo_itl <= 0.0f || dec <= slo_itl) &&
                           (slo_tps <= 0.0f || lambda <= lambda_tps);
        if (meets && front == 0) front = r;
      }
      frontier[pair] = front;
    }
  return 0;
}

// Arrival-rate search for server srv: from the arrival at which acc 0's level r = 1 has lambda / mu_{N-1} = ratio0,
// consecutive float32 arrival rates (nextafterf, upward) until a level deferred at threshold thr, of any accelerator,
// is not certified by the fast solve (its enclosure straddles a float32 rounding boundary).  Returns that arrival rate,
// or -1 when none is found within max_steps.
float emul_grid_boundary_arrival(const wva_system* sys, int srv, int R, float thr, float ratio0, int max_steps) {
  SysView s = make_view(sys);
  std::vector<float> tab;
  PairModel m;
  float total_rate, a, b, c;
  if (s.srv_slo_tps[srv] != 0.0f || !grid_pair(s, srv, 0, 1.0f, m, tab, &total_rate, &a, &b, &c)) return -1.0f;
  float arrival = (float)(m.mu_last * ratio0 * 1000.0 * 60.0);
  for (int step = 0; step < max_steps; step++, arrival = nextafterf(arrival, INFINITY)) {
    for (int acc = 0; acc < s.n_acc; acc++) {
      if (!grid_pair(s, srv, acc, arrival, m, tab, &total_rate, &a, &b, &c)) continue;
      for (int r = 1; r <= R; r++) {
        float lambda;
        bool deferred;
        if (!grid_level(m, total_rate, r, thr, &lambda, &deferred) || !deferred) {
          if (lambda / (float)m.mu_last <= thr) break;    // lower levels only
          continue;
        }
        SolveStats st{};
        int sv = 0;
        if (!fast_solve(m, lambda, st, &sv)) return arrival;
      }
    }
  }
  return -1.0f;
}

}  // extern "C"
