// TEST INFRASTRUCTURE ONLY — the host build of csrc/wva_core.cuh's service-rate pieces (model_init, rate_den, div_rate)
// for the CPU tests of tests/test_rate_division.py.  The host div_rate uses the correctly rounded seed; the host build
// of the core maps every wrapper to the IEEE operation it stands for.
#include "../../llm-d-workload-variant-autoscaler_b200/csrc/wva_core.cuh"
#include <cstdint>

using namespace wva;

extern "C" {
// den(1) .. den(N) of the pair model_init builds from the given coefficients
void host_rate_den(float alpha, float beta, float gamma, int in_tok, int out_tok, int N, float* den) {
  PairModel m;
  model_init(m, alpha, beta, gamma, in_tok, out_tok, N);
  const RateCoef c = rate_coef(m);
  float nf = 1.0f;
  for (int n = 0; n < N; n++, nf = f_add(nf, 1.0f)) den[n] = rate_den(c, nf);
}
void host_div_rate(const float* nf, const float* den, float* q, int64_t n) {
  for (int64_t i = 0; i < n; i++) q[i] = div_rate(nf[i], den[i]);
}
}  // extern "C"
