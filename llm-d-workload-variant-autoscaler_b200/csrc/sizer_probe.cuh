// sizer_probe.cuh — length-sorted work queue for the lock-step lane sizer.
//
// The lanes of a warp solve their chains in lock step, so a round costs the LONGEST chain among the 32 work items of
// the warp.  Chain length (early exit E4) varies 10x between the bisection steps of an item and between items, and in
// natural (server, accelerator) order only 40-52 % of the executed lane-steps did live work
// (SizerCounters.lockstep_slots).  This pass makes the queue order a function of the expected work: a throw-away
// float32 PROBE sizes every item (6 bisection steps on a float32 birth-death chain whose constant-rate tail is summed in
// closed form, < 5 % of the real work), estimates where the exact chain's 2^-54 early exit fires at the probed rate,
// and the item ids are radix-sorted by (N, bisects?, length) descending — longest first, equal N together (mixed N in a
// warp forces the slow per-lane path), items whose search ends at an end point (2 solves instead of ~22) last.  With gang
// refill (a warp takes 32 new items only when all its lanes are idle) 81-83 % of the lane-steps are live.
// wva_calculate uses it where it was measured to pay (130-1500 pairs per SM, capi.cu launch_sizer); see DESIGN.md §4.
//
// NOTHING computed here reaches a result: the probe only chooses the ORDER in which the exact, bit-reproducible
// sizer visits the items (each item's arithmetic is independent of every other item's), so a bad probe can
// cost time, never parity.  A probe needs no reference counterpart — it replaces the random map iteration order
// of System.Calculate (pkg/core/system.go:258-268).
#pragma once
#include "wva_core.cuh"

namespace wva {

struct ProbeEval { float ttft, itl; int len; };
#define WVA_PROBE_TAB 256   // head states kept per thread (local memory); larger N recompute mu_i

// float32 state-dependent M/M/1/K at arrival rate x (req/ms): the N head states one by one (mu_i from mu[], or
// from serv_rate when mu == nullptr), the K - N tail states — constant service rate, a geometric series — in
// closed form.  len = the state at which the exact chain's early exit (E4: term < 2^-54 of the sums) would fire.
WVA_HD ProbeEval probe_eval(const PairModel& m, const float* mu, float x) {
  const int N = m.N, M = m.K - m.N;
  float p = 1.0f, sum = 1.0f, L = 0.0f, muN = 1.0f;
  for (int i = 1; i <= N; i++) {
    muN = mu ? mu[i - 1] : serv_rate(m, i);
    p = p * (x / muN);
    sum += p; L += (float)i * p;
  }
  float Ls = L;                                        // sum min(i, N) p_i so far
  const float r = x / muN;                             // < 1 on the whole search range (lambda_max < mu_N)
  const float rM = powf(r, (float)M);
  const float g = r * (1.0f - rM) / (1.0f - r);        // sum_{j=1..M} r^j
  const float h = r * (1.0f - (float)(M + 1) * rM + (float)M * rM * r) / ((1.0f - r) * (1.0f - r));   // sum j r^j
  sum += p * g; L += p * ((float)N * g + h); Ls += p * (float)N * g;
  const float pK = p * rM / sum;
  const float thr = x * (1.0f - pK);
  const float in_sys = L / sum, in_srv = Ls / sum;
  const float resp = in_sys / thr, serv = in_srv / thr;
  const float wait = fmaxf(resp - serv, 0.0f);
  const float pf = prefill_time(m, in_srv);
  ProbeEval e;
  e.itl = (serv - pf) / m.out_tok;
  e.ttft = wait + pf + e.itl;
  // p_N r^j < 2^-54 sum  <=>  j > log(2^-54 sum / p_N) / log r
  float j = (float)M;
  if (!(p > 0x1p-54f * sum)) j = 1.0f;                 // already negligible at state N
  else if (r < 1.0f) j = logf(0x1p-54f * sum / p) / logf(r);
  if (!(j < (float)M)) j = (float)M;
  if (j < 1.0f) j = 1.0f;
  e.len = N + (int)j;
  return e;
}

// item = pair (SPLIT == false: key from the longer of the two searches) or 2*pair + kind (SPLIT: kind 0 TTFT, 1 ITL)
WVA_HD unsigned probe_item_key(const SysView& s, unsigned long long item, bool split, int nmax) {
  const unsigned long long pair = split ? (item >> 1) : item;
  const int srv = (int)(pair / (unsigned)s.n_acc), acc = (int)(pair % (unsigned)s.n_acc);
  SizerLane z;
  CandView none = {};
  int lim = 0;
  if (sizer_setup(z, s, none, srv, acc, nmax, &lim, false) != SETUP_NEEDS_TABLE) return 0;
  PairModel& m = z.m;
  // the rate range model_finish() derives from the head table (queueanalyzer.go:107-109, 189-190), approximately
  m.lambda_min = serv_rate(m, 1) * WVA_EPSILON;
  m.lambda_max = serv_rate(m, m.N) * (1.0f - WVA_EPSILON);
  if (m.lambda_min > m.lambda_max) return 0;
  int len = 0;
  bool bisects = false;   // some search of the item runs its ~20 bisection steps (otherwise: the two end points only)
  float mu_tab[WVA_PROBE_TAB];
  const float* mu = nullptr;
  if (m.N <= WVA_PROBE_TAB) {                          // head table once per item (else: recomputed per evaluation)
    for (int i = 0; i < m.N; i++) mu_tab[i] = serv_rate(m, i + 1);
    mu = mu_tab;
  }
  for (int kind = 0; kind < 2; kind++) {
    if (split && kind != (int)(item & 1)) continue;
    const float target = kind ? z.sI.target : z.sT.target;
    if (!(target > 0.0f)) continue;
    float lo = m.lambda_min, hi = m.lambda_max;
    const ProbeEval e_lo = probe_eval(m, mu, lo), e_hi = probe_eval(m, mu, hi);
    const float y_lo = kind ? e_lo.itl : e_lo.ttft, y_hi = kind ? e_hi.itl : e_hi.ttft;
    const bool inc = y_lo < y_hi;
    int l = e_hi.len;
    if ((inc && target < y_lo) || (!inc && target > y_lo)) l = e_lo.len;           // the search fails at once
    else if (!((inc && target > y_hi) || (!inc && target < y_hi))) {
      bisects = true;
      for (int it = 0; it < 6; it++) {
        const float xs = 0.5f * (lo + hi);
        const ProbeEval e = probe_eval(m, mu, xs);
        const float y = kind ? e.itl : e.ttft;
        if ((inc && target < y) || (!inc && target > y)) hi = xs; else lo = xs;
      }
      l = probe_eval(m, mu, 0.5f * (lo + hi)).len;
    }
    len = l > len ? l : len;
  }
  // items whose searches end at an end point do 2 solves instead of ~22: with gang refill they must not share a
  // warp with bisecting items (their lanes would idle for 20 rounds), so they sort below every bisecting item
  unsigned long long l16 = (unsigned long long)len * 65535ull / (unsigned long long)(m.K > 0 ? m.K : 1);
  if (l16 > 65535ull) l16 = 65535ull;
  if (l16 < 2ull) l16 = 2ull;
  const unsigned nn = (unsigned)(m.N < 65535 ? m.N : 65535);
  return (nn << 16) | (bisects ? (unsigned)l16 : 1u);
}

#if defined(__CUDACC__)
// keys[item] for every item of the launch; with a pair list the items are list positions (ids stay positions, which is
// what the lane sizer's queue holds) and each is probed as the item of its listed pair
template <bool SPLIT>
__global__ void __launch_bounds__(128) sizer_probe_kernel(SysView s, const int* list, unsigned long long n_items, int nmax,
                                                          unsigned* keys, unsigned* ids) {
  const unsigned long long item = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= n_items) return;
  const unsigned long long probed = SPLIT ? 2 * list_pair(list, item >> 1) + (item & 1) : list_pair(list, item);
  keys[item] = probe_item_key(s, probed, SPLIT, nmax);
  ids[item] = (unsigned)item;
}

#endif  // __CUDACC__

}  // namespace wva
