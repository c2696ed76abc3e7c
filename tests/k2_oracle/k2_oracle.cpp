// TEST INFRASTRUCTURE ONLY — CPU restatement of SaturationAnalyzer.computeK2
// (internal/engines/analyzers/saturation_v2/analyzer.go:218-262) and its rolling history (history.go), over the same
// integer registry and inputs as wva_k2_resolve (include/wva_b200.h), one replica after another as Analyze calls it:
//   - history groups (modelIDs) in order; their model groups in registry order (one of the orders Go's map iteration
//     over GroupVariantAutoscalingByModel can produce); each group's replicas in ReplicaMetrics slice order;
//   - a replica with TotalKvCapacityTokens <= 0 is skipped (:148-150): k2 = -1, effective = 0, no history access;
//   - priority 1 observed (queueLen >= int(QueueLengthThreshold) && tokensInUse > 0): k2 = tokensInUse, appended to the
//     key's window, which drops its oldest value at 10 (rollingAverage.Add);
//   - priority 2: rollingAverage.Average, the float64 sum oldest to newest / float64(len); > 0 -> int64(avg);
//   - priority 3: estimateCapacityFromParams (oracle/pipeline_v2.hpp) with the slot's params; priority 4: k1;
//   - effective = min(k1, k2); per store slot the last data replica in that order and its effective capacity.
// The window is a plain vector with erase-at-front, as the Go slice is.  Built with -ffp-contract=off like the oracle.
#include "../../oracle/pipeline_v2.hpp"

#include <cstdint>
#include <vector>

namespace {
struct Hist {
  int H, G, S;
  std::vector<int> hg_model_off, hg_models, hg_acc_off, hg_acc, mg_hg;
  std::vector<std::vector<double>> win;    // per key (hg_acc_off[h] + k) * 3 + bucket
};
int bucket_of(double avg_out) { return avg_out < 100 ? 0 : (avg_out < 500 ? 1 : 2); }   // types.go:28-37
long long key_of(const Hist& h, int hg, int acc, double avg_out) {
  for (int j = h.hg_acc_off[hg]; j < h.hg_acc_off[hg + 1]; j++)
    if (h.hg_acc[j] == acc) return (long long)j * 3 + bucket_of(avg_out);
  return -1;
}
}  // namespace

extern "C" {

void* k2o_create(int H, int G, int S, const int32_t* hg_model_off, const int32_t* hg_models, const int32_t* hg_acc_off,
                 const int32_t* hg_acc) {
  Hist* h = new Hist();
  h->H = H; h->G = G; h->S = S;
  h->hg_model_off.assign(hg_model_off, hg_model_off + H + 1);
  h->hg_models.assign(hg_models, hg_models + G);
  h->hg_acc_off.assign(hg_acc_off, hg_acc_off + H + 1);
  h->hg_acc.assign(hg_acc, hg_acc + hg_acc_off[H]);
  h->mg_hg.assign(G, -1);
  for (int g = 0; g < H; g++)
    for (int i = hg_model_off[g]; i < hg_model_off[g + 1]; i++) h->mg_hg[hg_models[i]] = g;
  h->win.assign((size_t)hg_acc_off[H] * 3, {});
  return h;
}

void k2o_destroy(void* p) { delete (Hist*)p; }

// 0 = ok, 1 = a data replica's accelerator is not registered for its history group or its slot is out of range
// (nothing changes then)
int k2o_resolve(void* p, const int32_t* model_replica_off, const int64_t* tk, const int64_t* used, const int64_t* queue,
                const double* avg_in, const double* avg_out, const int32_t* acc, const int32_t* slot,
                const double* q_thr, const double* kv_thr, const int64_t* slot_B, const int64_t* slot_S,
                int64_t* rep_k2, int64_t* rep_eff, int32_t* slot_last, int64_t* slot_eff) {
  Hist& h = *(Hist*)p;
  for (int g = 0; g < h.G; g++)
    for (int r = model_replica_off[g]; r < model_replica_off[g + 1]; r++)
      if (tk[r] > 0 && (key_of(h, h.mg_hg[g], acc[r], avg_out[r]) < 0 || slot[r] < 0 || slot[r] >= h.S)) return 1;
  for (int s = 0; s < h.S; s++) { slot_last[s] = -1; slot_eff[s] = 0; }
  for (int hg = 0; hg < h.H; hg++)
    for (int mi = h.hg_model_off[hg]; mi < h.hg_model_off[hg + 1]; mi++) {
      const int g = h.hg_models[mi];
      for (int r = model_replica_off[g]; r < model_replica_off[g + 1]; r++) {
        rep_k2[r] = -1; rep_eff[r] = 0;
        if (tk[r] <= 0) continue;
        const long long k1 = oracle_v2::go_int((double)tk[r] * kv_thr[g]);
        std::vector<double>& w = h.win[key_of(h, hg, acc[r], avg_out[r])];
        long long k2;
        if (queue[r] >= oracle_v2::go_int(q_thr[g]) && used[r] > 0) {
          if ((int)w.size() >= 10) w.erase(w.begin());
          w.push_back((double)used[r]);
          k2 = used[r];
        } else {
          double avg = 0;
          if (!w.empty()) {
            double sum = 0;
            for (double v : w) sum += v;
            avg = sum / (double)w.size();
          }
          if (avg > 0) {
            k2 = oracle_v2::go_int(avg);
          } else {
            const long long d = oracle_v2::estimate_capacity_from_params(slot_B[slot[r]], slot_S[slot[r]], avg_in[r], avg_out[r]);
            k2 = d > 0 ? d : k1;
          }
        }
        rep_k2[r] = k2;
        rep_eff[r] = k2 < k1 ? k2 : k1;
        if (r > slot_last[slot[r]]) { slot_last[slot[r]] = r; slot_eff[slot[r]] = rep_eff[r]; }
      }
    }
  return 0;
}

// every key in key order: count and values oldest first (zeros past count)
void k2o_export(void* p, int32_t* count, double* values) {
  Hist& h = *(Hist*)p;
  for (size_t k = 0; k < h.win.size(); k++) {
    count[k] = (int32_t)h.win[k].size();
    for (int t = 0; t < 10; t++) values[k * 10 + t] = t < count[k] ? h.win[k][t] : 0.0;
  }
}

void k2o_import(void* p, const int32_t* count, const double* values) {
  Hist& h = *(Hist*)p;
  for (size_t k = 0; k < h.win.size(); k++) h.win[k].assign(values + k * 10, values + k * 10 + count[k]);
}

}  // extern "C"
