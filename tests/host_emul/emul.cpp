// TEST INFRASTRUCTURE ONLY — host build of the device core (csrc/wva_core.cuh) so
// the lane state machines and the exact-division / early-exit logic can be checked
// against the oracle on a machine without a GPU.  Never linked into the product.
#include "../../include/wva_b200.h"
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/wva_core.cuh"
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/sizer_probe.cuh"
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/ingest_scatter.hpp"
#include <vector>
#include <cstdio>
#include <cstdlib>
#include <random>

using namespace wva;

static SysView make_view(const wva_system* s) {
  SysView v;
  v.n_acc = s->n_acc; v.n_types = s->n_types; v.n_models = s->n_models; v.n_servers = s->n_servers;
  v.acc_cost = s->acc_cost; v.acc_multiplicity = s->acc_multiplicity; v.acc_type = s->acc_type; v.type_count = s->type_count;
  v.perf_alpha = s->perf_alpha; v.perf_beta = s->perf_beta; v.perf_gamma = s->perf_gamma;
  v.perf_max_batch = s->perf_max_batch; v.perf_at_tokens = s->perf_at_tokens; v.perf_acc_count = s->perf_acc_count;
  v.perf_present = s->perf_present;
  v.srv_model = s->srv_model; v.srv_priority = s->srv_priority; v.srv_min_replicas = s->srv_min_replicas;
  v.srv_max_batch = s->srv_max_batch; v.srv_keep_acc = s->srv_keep_acc; v.srv_target_present = s->srv_target_present;
  v.srv_slo_ttft = s->srv_slo_ttft; v.srv_slo_itl = s->srv_slo_itl; v.srv_slo_tps = s->srv_slo_tps;
  v.srv_arrival = s->srv_arrival; v.srv_in_tokens = s->srv_in_tokens; v.srv_out_tokens = s->srv_out_tokens;
  v.srv_cur_acc = s->srv_cur_acc; v.srv_cur_replicas = s->srv_cur_replicas; v.srv_cur_cost = s->srv_cur_cost;
  return v;
}


// host replay of one chain solve through the lane state machine
static SolveStats host_solve(const PairModel& m, float x, bool* ovf) {
  Chain c; SolveStats st{};
  chain_start(c, x);
  c.tail_ok = d_bits(c.lamg) <= d_bits(m.mu_last);
  while (!chain_step(c, m, st)) {}
  *ovf = c.phase == CH_OVERFLOW;
  return st;
}

// System.Calculate through the SPECULATIVE bisection of sizer_warp_kernel.cuh, replayed lane by lane
// (tests spec_node_x / spec_walk and the round structure against the oracle).
extern "C" int emul_calculate_spec(const wva_system* sys, wva_candidates* out) {
  SysView s = make_view(sys);
  CandView o;
  o.state = out->state; o.num_replicas = out->num_replicas; o.batch_size = out->batch_size; o.cost = out->cost;
  o.value = out->value; o.itl = out->itl; o.ttft = out->ttft; o.rho = out->rho; o.max_arrv_rate = out->max_arrv_rate;
  o.n_solves = out->n_solves;
  std::vector<float> tab;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++) {
      SizerLane z; int lim = 0;
      if (sizer_setup(z, s, o, srv, acc, 1 << 20, &lim) == SETUP_DONE) continue;
      tab.assign((size_t)z.m.N, 0.0f);
      model_fill_table(z.m, tab.data(), 1, 0, 1);
      model_finish(z.m, tab.data(), 1);
      PairModel& m = z.m;
      size_t idx = (size_t)srv * s.n_acc + acc;
      bool failed = false, ovf = false;
      Search& sT = z.sT;
      Search& sI = z.sI;
      float yt[32], yi[32], pf;
      if (searches_begin(z)) {
        if (m.lambda_min > m.lambda_max) failed = true;
        else {
          for (int lane = 0; lane < 17; lane++) {
            float x = lane == 0 ? m.lambda_min : lane == 1 ? m.lambda_max
                      : spec_node_x(m.lambda_min, m.lambda_max, lane - 1, spec_depth_of(lane - 1));
            SolveStats st = host_solve(m, x, &ovf);
            eval_values(m, st, &yt[lane], &yi[lane], &pf);
          }
          for (int k = 0; k < 2; k++) {
            Search& q = k ? sI : sT;
            if (!q.active) continue;
            float* y = k ? yi : yt;
            if (!search_bracket(q, m, y[0], y[1])) failed = true;
            else if (q.active) spec_walk(q, 4, [&](int node) { return y[node + 1]; });
          }
          while (!failed && (sT.active || sI.active)) {
            bool both = sT.active && sI.active;
            int D = both ? 4 : 5;
            for (int lane = 0; lane < 32; lane++) {
              int half = lane >> 4, hl = lane & 15, node; bool isI, act;
              if (both) { node = hl + 1; isI = half == 1; act = hl < 15; } else { node = lane + 1; isI = sI.active; act = lane < 31; }
              if (!act) continue;
              const Search& mq = isI ? sI : sT;
              float x = spec_node_x(mq.lo, mq.hi, node, spec_depth_of(node));
              SolveStats st = host_solve(m, x, &ovf);
              eval_values(m, st, &yt[lane], &yi[lane], &pf);
            }
            if (both) { spec_walk(sT, D, [&](int nd) { return yt[nd - 1]; }); spec_walk(sI, D, [&](int nd) { return yi[16 + nd - 1]; }); }
            else if (sT.active) spec_walk(sT, D, [&](int nd) { return yt[nd - 1]; });
            else spec_walk(sI, D, [&](int nd) { return yi[nd - 1]; });
          }
        }
      }
      Alloc a = alloc_none();
      float x;
      if (!failed && size_lambda(z, x)) {
        SolveStats st = host_solve(m, x, &ovf);
        if (alloc_replicas(z, st.throughput, x)) {
          st = host_solve(m, x, &ovf);
          float t, i2;
          eval_values(m, st, &t, &i2, &pf);
          a = alloc_final(z, s, st, i2, pf);
        }
      }
      store_candidate(o, idx, a, 0);
    }
  return 0;
}

// System.Calculate through the DUAL-chain driver (dual_begin / dual_on_solve) of the lock-step lane sizer.
extern "C" int emul_calculate_dual(const wva_system* sys, wva_candidates* out) {
  SysView s = make_view(sys);
  CandView o;
  o.state = out->state; o.num_replicas = out->num_replicas; o.batch_size = out->batch_size; o.cost = out->cost;
  o.value = out->value; o.itl = out->itl; o.ttft = out->ttft; o.rho = out->rho; o.max_arrv_rate = out->max_arrv_rate;
  o.n_solves = out->n_solves;
  std::vector<float> tab;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++) {
      SizerLane z; int lim = 0;
      if (sizer_setup(z, s, o, srv, acc, 1 << 20, &lim) == SETUP_DONE) continue;
      tab.assign((size_t)z.m.N, 0.0f);
      model_fill_table(z.m, tab.data(), 1, 0, 1);
      model_finish(z.m, tab.data(), 1);
      bool live = dual_begin(z, s, o);
      while (live) {
        SolveStats st2[2] = {};
        bool ovf = false;
        for (int c = 0; c < 2; c++)
          if (z.act2[c]) st2[c] = host_solve(z.m, z.x2[c], &ovf);
        live = dual_on_solve(z, s, o, st2, 0);
      }
    }
  return 0;
}

// System.Calculate through the SPECULATIVE SPLIT driver (spec2_*): every pair is two items (TTFT search, ITL
// search), each advancing with two chains per round; the item that finishes second merges and runs the two
// Analyze solves — the host replay of sizer_lane_kernel<.., DUAL = true, SPLIT = true> incl. split_publish.
// stats: [0] search rounds, [1] bisection steps consumed, [2] rounds with a speculative chain, [3] guesses used
extern "C" int emul_calculate_spec2(const wva_system* sys, wva_candidates* out, int64_t* stats) {
  SysView s = make_view(sys);
  CandView o;
  o.state = out->state; o.num_replicas = out->num_replicas; o.batch_size = out->batch_size; o.cost = out->cost;
  o.value = out->value; o.itl = out->itl; o.ttft = out->ttft; o.rho = out->rho; o.max_arrv_rate = out->max_arrv_rate;
  o.n_solves = out->n_solves;
  std::vector<float> tab;
  for (int i = 0; i < 4; i++) stats[i] = 0;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++) {
      SizerLane item[2];
      bool dead = false;   // a lane failed the pair outright
      int lim = 0, n_pub = 0;
      if (sizer_setup(item[0], s, o, srv, acc, 1 << 20, &lim, true) == SETUP_DONE) continue;
      sizer_setup(item[1], s, o, srv, acc, 1 << 20, &lim, false);
      tab.assign((size_t)item[0].m.N, 0.0f);
      model_fill_table(item[0].m, tab.data(), 1, 0, 1);
      for (int k = 0; k < 2 && !dead; k++) {
        SizerLane& z = item[k];
        z.split = k;
        model_finish(z.m, tab.data(), 1);
        bool live = spec2_begin(z, s, o);
        while (live && z.stage != SZ_PUBLISH) {
          SolveStats st2[2] = {};
          bool ovf = false;
          const bool searching = z.stage == SZ_SEARCH;
          Search& q = k ? z.sI : z.sT;
          const int it0 = q.iter; const bool spec = z.act2[1];
          for (int c = 0; c < 2; c++)
            if (z.act2[c]) st2[c] = host_solve(z.m, z.x2[c], &ovf);
          live = spec2_on_solve(z, s, o, st2, 0);
          if (searching) {
            const int used = q.iter - it0;
            stats[0]++; if (spec) stats[2]++;
            stats[1] += used > 0 ? used : 1;
            if (spec && used >= 2) stats[3]++;
          }
        }
        if (live) n_pub++; else dead = true;
      }
      if (dead || n_pub < 2) continue;
      // split_publish: the second finisher (here: item 1) merges
      SizerLane& z = item[1];
      SizerLane& p = item[0];
      z.solves += p.solves;
      z.merged = true;
      if (z.failed || p.failed) { lane_fail(z, s, o); continue; }
      z.sT.result = p.sT.result;
      bool live = spec2_after_search(z, s, o);
      while (live) {
        SolveStats st2[2] = {};
        bool ovf = false;
        for (int c = 0; c < 2; c++)
          if (z.act2[c]) st2[c] = host_solve(z.m, z.x2[c], &ovf);
        live = spec2_on_solve(z, s, o, st2, 0);
      }
    }
  return 0;
}

// The float32 probe keys of sizer_probe.cuh for every split item (analysis: how well do they predict the chain length)
extern "C" int emul_probe_keys(const wva_system* sys, uint32_t* keys) {
  SysView s = make_view(sys);
  const unsigned long long n = 2ull * s.n_servers * s.n_acc;
  for (unsigned long long i = 0; i < n; i++) keys[i] = probe_item_key(s, i, true, 1 << 20);
  return 0;
}

extern "C" int emul_probe_debug(const wva_system* sys, int item) {
  SysView s = make_view(sys);
  const int pair = item >> 1, srv = pair / s.n_acc, acc = pair % s.n_acc;
  SizerLane z; CandView none = {}; int lim = 0;
  int rc = sizer_setup(z, s, none, srv, acc, 1 << 20, &lim, false);
  PairModel& m = z.m;
  m.lambda_min = serv_rate(m, 1) * WVA_EPSILON; m.lambda_max = serv_rate(m, m.N) * (1.0f - WVA_EPSILON);
  printf("rc %d N %d K %d lmin %g lmax %g tT %g tI %g mu1 %g muN %g\n", rc, m.N, m.K, m.lambda_min, m.lambda_max, z.sT.target, z.sI.target, serv_rate(m,1), serv_rate(m,m.N));
  for (float f : {0.0f, 0.25f, 0.5f, 0.75f, 0.9f, 1.0f}) {
    float x = m.lambda_min + f * (m.lambda_max - m.lambda_min);
    ProbeEval e = probe_eval(m, nullptr, x), e2 = e;
    bool ovf; SolveStats st; float t, i, pf; 
    std::vector<float> tab(m.N); model_fill_table(m, tab.data(), 1, 0, 1); PairModel mm = m; model_finish(mm, tab.data(), 1);
    st = host_solve(mm, x, &ovf); eval_values(mm, st, &t, &i, &pf);
    printf("  x %g probe ttft %g itl %g len %d len54 %d | exact ttft %g itl %g\n", x, e.ttft, e.itl, e.len, e2.len, t, i);
  }
  return 0;
}

// Analysis helper: per split item (2 * pair + kind), the number of states of each chain solve of its search, in
// order (trace[item * W] = count, then the lengths) — used to study how the lock-step rounds of a warp line up.
extern "C" int emul_trace_split(const wva_system* sys, int32_t* trace, int W) {
  SysView s = make_view(sys);
  CandView o = {};
  std::vector<float> tab;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++)
      for (int k = 0; k < 2; k++) {
        int32_t* t = trace + ((size_t)(srv * s.n_acc + acc) * 2 + k) * W;
        t[0] = 0;
        SizerLane z; int lim = 0;
        if (sizer_setup(z, s, o, srv, acc, 1 << 20, &lim, false) == SETUP_DONE) continue;
        tab.assign((size_t)z.m.N, 0.0f);
        model_fill_table(z.m, tab.data(), 1, 0, 1);
        model_finish(z.m, tab.data(), 1);
        z.split = k;
        bool live = sizer_begin(z, s, o);
        while (live && z.stage != SZ_PUBLISH) {
          SolveStats st{};
          while (!chain_step(z.c, z.m, st)) {}
          if (z.c.phase == CH_OVERFLOW) break;
          if (t[0] + 1 < W) t[++t[0]] = z.c.states;
          live = sizer_on_solve(z, s, o, st);
        }
      }
  return 0;
}

// Analysis helper: per WHOLE pair, the number of states of each chain solve of Size() + the two Analyze solves, in order
// (trace[pair * W] = count, then the lengths) — input of tools/proto/lockstep_sim.py.
extern "C" int emul_trace_pair(const wva_system* sys, int32_t* trace, int W, float* ratio) {
  SysView s = make_view(sys);
  CandView o = {};
  std::vector<float> tab;
  for (int srv = 0; srv < s.n_servers; srv++)
    for (int acc = 0; acc < s.n_acc; acc++) {
      int32_t* t = trace + (size_t)(srv * s.n_acc + acc) * W;
      t[0] = 0;
      SizerLane z; int lim = 0;
      if (sizer_setup(z, s, o, srv, acc, 1 << 20, &lim, false) == SETUP_DONE) continue;
      tab.assign((size_t)z.m.N, 0.0f);
      model_fill_table(z.m, tab.data(), 1, 0, 1);
      model_finish(z.m, tab.data(), 1);
      std::vector<unsigned char> st_none(1);
      o.state = nullptr;
      // candidates are not written: a scratch view
      static thread_local std::vector<unsigned char> b1; static thread_local std::vector<int> b4; static thread_local std::vector<float> bf;
      b1.assign((size_t)s.n_servers * s.n_acc, 0); b4.assign((size_t)s.n_servers * s.n_acc, 0); bf.assign((size_t)s.n_servers * s.n_acc, 0.f);
      o.state = b1.data(); o.num_replicas = b4.data(); o.batch_size = b4.data(); o.cost = bf.data(); o.value = bf.data();
      o.itl = bf.data(); o.ttft = bf.data(); o.rho = bf.data(); o.max_arrv_rate = bf.data(); o.n_solves = nullptr;
      bool live = sizer_begin(z, s, o);
      while (live) {
        SolveStats st{};
        while (!chain_step(z.c, z.m, st)) {}
        if (z.c.phase == CH_OVERFLOW) break;
        if (t[0] + 1 < W) {
          t[++t[0]] = z.c.states;
          if (ratio) ratio[(size_t)(srv * s.n_acc + acc) * W + t[0]] = (float)((double)z.cur_x / z.m.mu_last);
        }
        live = sizer_on_solve(z, s, o, st);
      }
    }
  return 0;
}

extern "C" {

// the host side of wva_ingest_write (csrc/ingest_scatter.hpp) on caller-provided columns
int emul_ingest_scatter(double* col, uint8_t* has, int64_t S, int bit, int64_t n, const int32_t* slot, const double* value, int threads) {
  static IngestScratch sc;
  return ingest_scatter(col, has, (long long)S, (uint8_t)bit, n, slot, value, sc, threads) ? 0 : 1;
}

// System.Calculate through the lane state machine, one lane at a time.
int emul_calculate(const wva_system* sys, wva_candidates* out, int64_t* solves, int64_t* states, int64_t* overflow) {
  SysView s = make_view(sys);
  CandView o;
  o.state = out->state; o.num_replicas = out->num_replicas; o.batch_size = out->batch_size; o.cost = out->cost;
  o.value = out->value; o.itl = out->itl; o.ttft = out->ttft; o.rho = out->rho; o.max_arrv_rate = out->max_arrv_rate;
  o.n_solves = out->n_solves;
  int64_t ns = 0, nst = 0, nov = 0;
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
      SolveStats st;
      while (live) {
        if (chain_step(z.c, z.m, st)) {
          if (z.c.phase == CH_OVERFLOW) {
            // same redo as overflow_slow_kernel: literal stored-p[] algorithm from the start of the pair
            nov++;
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
            z = y;
            break;
          }
          live = sizer_on_solve(z, s, o, st);
        }
      }
      ns += z.solves; nst += z.states;
    }
  if (solves) *solves = ns;
  if (states) *states = nst;
  if (overflow) *overflow = nov;
  return 0;
}

}  // extern "C"

// exact-division self-checks against the IEEE operator; return the number of mismatches.
// (E1) divisor of the checks: every exponent of [2^-126, 2^126] (e1_divisor), all-ones significands and powers of two
// included, 2^126 itself now and then
static float e1_test_divisor(uint64_t b, int64_t i) {
  uint32_t mm = (uint32_t)(b & 0x7FFFFF);
  const int me = 1 + (int)((b >> 23) % 252);                          // biased exponent 1 .. 252: 2^-126 .. 2^125
  if ((i & 7) == 0) mm = 0x7FFFFFu;                                   // all-ones significand
  if ((i & 7) == 1) mm = 0;                                           // power of two
  uint32_t mb = ((uint32_t)me << 23) | mm;
  if ((i & 255) == 2) mb = 0x7E800000u;                               // 2^126, the largest E1 divisor
  float m32; memcpy(&m32, &mb, 4);
  return m32;
}
// the seeds the device can produce: f_rcp_approx(m) is within seed_ulp ulps of RN(1/m) for every E1 divisor
// (tests/test_device_prims.py), so every seed within that distance is checked; seeds that leave the normal range are
// left to the device check (the device flushes them)
template <class Check>
static bool for_each_seed(float m32, int seed_ulp, Check check) {
  const float s0 = 1.0f / m32;
  bool ok = true;
  for (int k = -seed_ulp; k <= seed_ulp; k++) {
    float s = s0;
    for (int j = 0; j < (k < 0 ? -k : k); j++) s = nextafterf(s, k < 0 ? 0.0f : INFINITY);
    if (!(s >= FLT_MIN && s <= FLT_MAX)) continue;
    ok = ok && check(rcp_refine(s, (double)m32));
  }
  return ok;
}

extern "C" {

int64_t emul_check_div_f32den(int64_t n, uint64_t seed, int seed_ulp) {
  std::mt19937_64 g(seed);
  int64_t bad = 0;
  for (int64_t i = 0; i < n; i++) {
    uint64_t a = g(), b = g();
    // random double with exponent in the E3 window, random E1 divisor
    uint64_t xm = a & 0xFFFFFFFFFFFFFull; int xe = 1023 + (int)((a >> 52) % 1000) - 500;
    uint64_t xb = ((uint64_t)xe << 52) | xm; double x; memcpy(&x, &xb, 8);
    const float m32 = e1_test_divisor(b, i);
    const double mu = (double)m32;
    if (!e1_divisor(m32) || rcp_f32den(m32, mu) != rcp_refine(1.0f / m32, mu)) { bad++; continue; }
    if (!for_each_seed(m32, seed_ulp, [&](double r) { return div_f32den(x, mu, r) == x / mu; })) bad++;
  }
  return bad;
}
// the 3-deep variant of (E1) used by lockstep_solve.cuh step_div: q0 = p * RN(lambda*r) formed beside x = p*lambda
int64_t emul_check_step_div(int64_t n, uint64_t seed, int seed_ulp) {
  std::mt19937_64 g(seed);
  int64_t bad = 0;
  for (int64_t i = 0; i < n; i++) {
    uint64_t a = g(), b = g(), c = g();
    uint32_t lm = (uint32_t)(c & 0x7FFFFF); int le = 127 + (int)((c >> 23) % 40) - 20;
    uint32_t lb = ((uint32_t)le << 23) | lm; float l32; memcpy(&l32, &lb, 4);
    const double lam = (double)l32;
    // p such that x = p lambda lies in the E3 window
    uint64_t pm = a & 0xFFFFFFFFFFFFFull; int pe = 1023 + (int)((a >> 52) % 960) - 480;
    uint64_t pb = ((uint64_t)pe << 52) | pm; double p; memcpy(&p, &pb, 8);
    const float m32 = e1_test_divisor(b, i);
    const double mu = (double)m32;
    const double x = d_mul(p, lam);
    if (!in_window(x)) continue;
    if (!for_each_seed(m32, seed_ulp, [&](double r) {
          double lamr = d_mul(lam, r);
          double q0 = d_mul(p, lamr);
          double rem = d_fma(-q0, mu, x);
          return d_fma(rem, r, q0) == x / mu;
        }))
      bad++;
  }
  return bad;
}
// e1_divisor over every float32 bit pattern: true exactly on [2^-126, 2^126]; returns the number of wrong answers
int64_t emul_check_e1_range() {
  int64_t bad = 0;
  for (uint64_t b = 0; b <= 0xFFFFFFFFull; b++) {
    float m; const uint32_t b32 = (uint32_t)b; memcpy(&m, &b32, 4);
    const bool want = m >= 0x1p-126f && m <= 0x1p126f;
    if (e1_divisor(m) != want) bad++;
  }
  return bad;
}
// the host f_rcp_approx flushes as rcp.approx.ftz.f32 does: subnormal inputs read as 0, subnormal results are 0
int64_t emul_check_seed_ftz() {
  int64_t bad = 0;
  for (uint32_t b = 1; b < 0x7F800000u; b++) {
    float m; memcpy(&m, &b, 4);
    const float s = f_rcp_approx(m);
    const float want = m < FLT_MIN ? INFINITY : (1.0f / m < FLT_MIN ? 0.0f : 1.0f / m);
    if (memcmp(&s, &want, 4) != 0) bad++;
  }
  return bad;
}
int64_t emul_check_div_markstein2(int64_t n, uint64_t seed) {
  std::mt19937_64 g(seed);
  int64_t bad = 0;
  for (int64_t i = 0; i < n; i++) {
    uint64_t a = g(), b = g();
    uint64_t xm = a & 0xFFFFFFFFFFFFFull; int xe = 1023 + (int)((a >> 52) % 400) - 200;
    uint64_t xb = ((uint64_t)xe << 52) | xm; double x; memcpy(&x, &xb, 8);
    uint64_t ym = b & 0xFFFFFFFFFFFFFull; int ye = 1023 + (int)((b >> 52) % 400) - 200;
    if ((i & 15) == 0) ym = 0xFFFFFFFFFFFFFull;
    if ((i & 15) == 1) ym = 0;
    if ((i & 15) == 2) ym = 0xFFFFFFFFFFFFEull;
    uint64_t yb = ((uint64_t)ye << 52) | ym; double y; memcpy(&y, &yb, 8);
    double q = div_markstein2(x, y, 1.0 / y);
    if (q != x / y) bad++;
  }
  return bad;
}

}  // extern "C"
