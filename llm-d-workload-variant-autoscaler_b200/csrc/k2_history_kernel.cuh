// k2_history_kernel.cuh — SaturationAnalyzer.computeK2 (internal/engines/analyzers/saturation_v2/analyzer.go:218-262)
// for a whole cycle, with the rolling k2 history (history.go, window 10) resident in HBM.  The semantics are stated
// with wva_k2_resolve in include/wva_b200.h.
//
//   k2_keys_kernel      per replica: the history key (accelerator slot x output bucket) or -1 without capacity data,
//                       and the input checks (unregistered accelerator, store slot or output position out of range).
//                       It writes only scratch: wva_k2_resolve reads the error word back before the history changes.
//   k2_resolve_kernel   one warp per history group (one modelID): its model groups in registry order, each group's
//                       replicas in slice order, 32 per step.  A lane finds its window with a ballot: the newest
//                       10 - c values of the stored ring, then the c observations of its key by earlier lanes of the step
//                       (only the last 10 of them when c >= 10), and adds it oldest to newest (at most 10 dependent
//                       float64 adds) before it resolves priorities 2-4.  After the step the last observing lane of each
//                       key appends the step's observations of that key to the ring.  The rings of a history group with
//                       at most K2_SMEM_KEYS keys are staged in shared memory for the walk; larger groups work on them in
//                       place in global memory.  Both run the same code on different pointers.
//   k2_slot_kernel      per store slot: EffectiveCapacity of the slot's last data replica (atomicMax of its index).
//   A caller that cannot read the error word back before the next launch (wva_ingest_v2's graph) passes it as `gate`:
//   the resolve and slot kernels then return at once when it is set.
//
// Rings: per key `count` (0..10), `head` (index of the oldest value) and 10 float64 values; key index =
// (hg_acc_off[h] + accelerator slot) * 3 + bucket.  A history group's keys are touched by its warp only.
#pragma once
#include "pipeline_v2_kernel.cuh"

namespace wva {

#define K2_WINDOW 10        // RollingAverageWindowSize (constants.go)
#define K2_SMEM_KEYS 24     // keys a warp stages in shared memory: 8 accelerators x 3 buckets
#define K2_WARPS 8

struct K2Reg {              // the registry, on the device
  int H;
  const int *hg_model_off, *hg_models, *hg_acc_off, *hg_acc, *mg_hg;
};
struct K2State { double* vals; int* count; int* head; };   // [K*10], [K], [K]
struct K2In {
  int G, n_slots;
  long long n_out;
  const int* model_replica_off;
  const long long *tk, *used, *queue;
  const double *avg_in, *avg_out;
  const int *acc, *slot, *out_pos;
  const long long *slot_B, *slot_S;
  const double *q_thr, *kv_thr;
  const int* gate;          // NULL, or the keys pass's error word: set = the resolve and slot kernels change nothing
};
struct K2Out { long long *rep_k2, *rep_eff, *out_k2; int* slot_last; long long* slot_eff; int* rep_key; int* err; };

// classifyOutputLength (types.go:28-37): NaN compares false twice and lands in "long", as in Go
__device__ __forceinline__ int k2_bucket(double avg_out) { return avg_out < 100.0 ? 0 : (avg_out < 500.0 ? 1 : 2); }

// estimateCapacityFromParams (analyzer.go:418-437); B <= 0 also stands for "no VLLMParams"
__device__ __forceinline__ long long k2_estimate(long long B, long long S, double ai, double ao) {
  if (B <= 0 || ao <= 0) return 0;
  double n = __ddiv_rn(__dmul_rn((double)B, ao), __dadd_rn(ai, ao));
  if (n > (double)S) n = (double)S;
  const long long k2 = go_int64(__dmul_rn(n, __dadd_rn(ai, __ddiv_rn(ao, 2.0))));
  return k2 > 0 ? k2 : 0;
}

__global__ void __launch_bounds__(256) k2_keys_kernel(K2Reg reg, K2In in, int* rep_key, int* err) {
  const int lane = threadIdx.x & 31;
  const long long nw = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long g = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < in.G; g += nw) {
    const int h = reg.mg_hg[g], a0 = reg.hg_acc_off[h], na = reg.hg_acc_off[h + 1] - a0;
    int bad = 0;
    for (int r = in.model_replica_off[g] + lane; r < in.model_replica_off[g + 1]; r += 32) {
      int key = -1;
      if (in.tk[r] > 0) {                                                    // analyzer.go:148-150
        const int a = in.acc[r], s = in.slot[r];
        int k = -1;
        for (int j = 0; j < na; j++)
          if (reg.hg_acc[a0 + j] == a) { k = j; break; }
        if (k < 0 || s < 0 || s >= in.n_slots) bad |= 1;
        else key = k * 3 + k2_bucket(in.avg_out[r]);
      }
      if (in.out_pos && (in.out_pos[r] < -1 || in.out_pos[r] >= in.n_out)) bad |= 2;
      rep_key[r] = key;
    }
    if (bad) atomicOr(err, bad);
  }
}

__global__ void __launch_bounds__(K2_WARPS * 32) k2_resolve_kernel(K2Reg reg, K2In in, K2State st, K2Out out) {
  __shared__ double s_vals[K2_WARPS][K2_SMEM_KEYS * K2_WINDOW];
  __shared__ int s_cnt[K2_WARPS][K2_SMEM_KEYS], s_head[K2_WARPS][K2_SMEM_KEYS];
  __shared__ double s_obs[K2_WARPS][32];
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned before = (1u << lane) - 1u;
  double* obs_v = s_obs[wid];
  if (in.gate && *in.gate) return;                                           // a rejected cycle leaves the history as it was
  for (int h = blockIdx.x * K2_WARPS + wid; h < reg.H; h += gridDim.x * K2_WARPS) {
    const int key0 = reg.hg_acc_off[h] * 3, nk = reg.hg_acc_off[h + 1] * 3 - key0;
    const bool staged = nk <= K2_SMEM_KEYS;
    double* vals;
    int *cnt, *head;
    if (staged) {
      vals = s_vals[wid]; cnt = s_cnt[wid]; head = s_head[wid];
      for (int i = lane; i < nk * K2_WINDOW; i += 32) vals[i] = st.vals[(size_t)key0 * K2_WINDOW + i];
      for (int i = lane; i < nk; i += 32) { cnt[i] = st.count[key0 + i]; head[i] = st.head[key0 + i]; }
    } else {
      vals = st.vals + (size_t)key0 * K2_WINDOW; cnt = st.count + key0; head = st.head + key0;
    }
    __syncwarp();
    bool appended = false;                                                   // warp-uniform
    for (int mi = reg.hg_model_off[h]; mi < reg.hg_model_off[h + 1]; mi++) {
      const int g = reg.hg_models[mi];
      const long long q_thr = go_int64(in.q_thr[g]);                         // int(QueueLengthThreshold), :235
      const double kv_thr = in.kv_thr[g];
      const int r1 = in.model_replica_off[g + 1];
      for (int r = in.model_replica_off[g] + lane; r - lane < r1; r += 32) {
        const bool live = r < r1;
        const int key = live ? out.rep_key[r] : -1;
        long long used = 0, k2 = -1, eff = 0;
        bool obs = false;
        if (key >= 0) {
          used = in.used[r];
          obs = in.queue[r] >= q_thr && used > 0;                            // priority 1
        }
        const unsigned obs_mask = __ballot_sync(FULL, obs);
        const unsigned mine = __match_any_sync(FULL, key) & obs_mask;       // this key's observing lanes
        if (obs) obs_v[lane] = (double)used;
        __syncwarp();
        if (key >= 0) {
          const long long k1 = go_int64(__dmul_rn((double)in.tk[r], kv_thr));   // :159
          if (obs) {
            k2 = used;
          } else {                                                           // priority 2: window = ring tail + earlier obs
            unsigned m = mine & before;
            const int c = __popc(m), c_win = c < K2_WINDOW ? c : K2_WINDOW;
            const int n_ring = cnt[key], from_ring = n_ring < K2_WINDOW - c_win ? n_ring : K2_WINDOW - c_win;
            const int hd = head[key];
            const double* ring = vals + key * K2_WINDOW;
            double s = 0.0;
            for (int t = n_ring - from_ring; t < n_ring; t++) {
              const int p = hd + t;
              s = __dadd_rn(s, ring[p >= K2_WINDOW ? p - K2_WINDOW : p]);
            }
            for (int skip = c - c_win; skip > 0; skip--) m &= m - 1;
            while (m) {
              const int j = __ffs(m) - 1;
              m &= m - 1;
              s = __dadd_rn(s, obs_v[j]);
            }
            const int n = from_ring + c_win;
            bool hist = false;
            if (n > 0) {
              const double avg = __ddiv_rn(s, (double)n);
              if (avg > 0) { k2 = go_int64(avg); hist = true; }
            }
            if (!hist) {                                                     // priority 3, else 4
              const int sl = in.slot[r];
              const long long d = k2_estimate(in.slot_B[sl], in.slot_S[sl], in.avg_in[r], in.avg_out[r]);
              k2 = d > 0 ? d : k1;
            }
          }
          eff = k2 < k1 ? k2 : k1;                                           // :175-178
          atomicMax(out.slot_last + in.slot[r], r);
        }
        if (live) {
          out.rep_k2[r] = k2;
          out.rep_eff[r] = eff;
          if (out.out_k2) {
            const int p = in.out_pos[r];
            if (p >= 0) out.out_k2[p] = k2;
          }
        }
        __syncwarp();                                                        // every window is read before a ring moves
        if (obs && (mine >> lane) == 1u) {                                   // the key's last observing lane appends
          double* ring = vals + key * K2_WINDOW;
          int n_ring = cnt[key], hd = head[key];
          unsigned m = mine;
          for (int skip = __popc(m) - K2_WINDOW; skip > 0; skip--) m &= m - 1;
          while (m) {
            const int j = __ffs(m) - 1;
            m &= m - 1;
            if (n_ring < K2_WINDOW) {
              const int p = hd + n_ring;
              ring[p >= K2_WINDOW ? p - K2_WINDOW : p] = obs_v[j];
              n_ring++;
            } else {                                                         // history.go Add: drop the oldest
              ring[hd] = obs_v[j];
              hd = hd + 1 == K2_WINDOW ? 0 : hd + 1;
            }
          }
          cnt[key] = n_ring; head[key] = hd;
        }
        appended |= obs_mask != 0;
        __syncwarp();
      }
    }
    if (staged && appended) {
      for (int i = lane; i < nk * K2_WINDOW; i += 32) st.vals[(size_t)key0 * K2_WINDOW + i] = vals[i];
      for (int i = lane; i < nk; i += 32) { st.count[key0 + i] = cnt[i]; st.head[key0 + i] = head[i]; }
    }
    __syncwarp();
  }
}

__global__ void k2_slot_kernel(int n_slots, const int* slot_last, const long long* rep_eff, long long* slot_eff, const int* gate) {
  if (gate && *gate) return;
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < n_slots; s += gridDim.x * blockDim.x) {
    const int r = slot_last[s];
    slot_eff[s] = r >= 0 ? rep_eff[r] : 0;
  }
}

}  // namespace wva
