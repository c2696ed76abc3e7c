// Microbenchmark: the certified fast solve's head pass (lockstep_fast_head over a TileTable) as the pool sizer runs it,
// and variants that each remove one cost, to find where a head chunk's cycles go.
//
// Every warp of a 512-thread CTA (__launch_bounds__(512, 1), as sizer_pool_kernel) takes batches of 32 rows drawn at
// random from its CTA's pool of 1024 rows in global memory (N = 256, rows built by serv_rate as BuildModel does, so μ is
// monotone from `mono` on), one arrival rate per lane spread over (0, 0.999 μ_{N-1}) so that light lanes leave the head
// early and heavy ones do not.  Reported: clock64() cycles of the head pass per warp-state (one state index of a 32-lane
// batch), first tile wait included, as tools/perf_pool_phases.py counts them; with 16 and with 4 working warps per SM
// (4 and 1 per scheduler: the pipe-bound and the latency-bound figure).
//
//   product  lockstep_solve_fast_only itself over the rows (its head-pass counter, built with -DWVA_POOL_PHASES)
//   base     the same head loop written out here: TileTable::load_chunk + fast_chunk + the chunk-boundary exit
//   computed the same head loop over RateTable (lockstep_solve.cuh): each lane computes its rates from its model's
//            coefficients, no row is read (what the pool sizer and the deferred grid pass run)
//   ieee     computed with every rate divided by __fdiv_rn (IeeeRateTable, kept here): RateTable before div_rate
//   (a) reg  the tile read replaced by values in registers: no ld.shared, conversion, rcp seed, refinement or λ·r per state
//   (b) nof  the tile fetch hoisted out: both tiles fetched once at the start of a pass, no shfl / cp.async after it
//   (d) noTA fast_chunk without the T / A accumulations (p1_chunk: the recurrence and the sum only)
//   (c) CH = 8 is the same program built with -DWVA_TILE_CHUNK=8 (head_chunk_ch8).
// The variants (a), (b), (d) are measurements only: (a) and (b) read wrong table values and (d) drops what
// certification needs.  TileTable, which streamed the pool's rows before RateTable replaced them, and IeeeRateTable,
// RateTable before its divisions became div_rate, are kept here.
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 --fmad=false -DWVA_POOL_PHASES \
//          -I../../llm-d-workload-variant-autoscaler_b200/csrc -o head_chunk head_chunk.cu        (add -DWVA_TILE_CHUNK=8 for (c))
// run:   ./head_chunk [batches per warp]
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include "wva_core.cuh"
#include "lockstep_solve.cuh"

using namespace wva;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int THREADS = 512, P = 1024, N = 256, STRIDE = 256;
enum { V_PRODUCT, V_BASE, V_COMPUTED, V_IEEE, V_REG, V_NOFETCH, V_NOTA, V_COUNT };
static const char* kNames[V_COUNT] = {"product", "base", "computed", "ieee", "(a) reg", "(b) nof", "(d) noTA"};

// Rows in global memory, one per pool slot, and any 32 of them solved together: the warp keeps two shared tiles of 32
// head states x 32 lanes.  Tile k+1 is fetched with cp.async while the lanes work on tile k, so the only exposed
// latency is the first tile of a pass.  A tile is lane-major: lane l's 32 states are 8 chunks of 4 states (16 bytes) at
// l * 128 bytes, chunk c stored in place c ^ (l & 7) (conflict-free 16-byte reads); a chunk of 16 states is 4 loads.
struct TileTable {
  static constexpr int kChunk = WVA_TILE_CHUNK;
  static constexpr int kWarpFloats = 2 * 32 * 32; // shared floats per warp (two tiles)
  static_assert(32 % kChunk == 0 && kChunk % 4 == 0, "a chunk lies inside one tile and is whole 16-byte groups");
  const float* rows;      // base of the CTA's rows (16-byte aligned)
  int row_stride;         // floats per row (a multiple of 32, >= N)
  int slot;               // this lane's row
  unsigned tile;          // shared-space address of the warp's two tiles (kWarpFloats, 16-byte aligned)
  int n_head;             // head entries (N - 1): tiles beyond are never fetched
  __device__ __forceinline__ unsigned group_addr(unsigned l, int n) const {
    return tile + (((unsigned)n >> 5) & 1u) * 4096u + l * 128u + (((((unsigned)n >> 2) & 7u) ^ (l & 7u)) << 4);
  }
  __device__ __forceinline__ void fetch(int n0) const {
    const unsigned lane = threadIdx.x & 31, c = lane & 7;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const unsigned l = 4 * k + (lane >> 3);
      const int sr = __shfl_sync(0xffffffffu, slot, l);
      const float* src = rows + (size_t)sr * row_stride + n0 + 4 * c;
      asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(group_addr(l, n0 + 4 * c)), "l"(src) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  __device__ __forceinline__ unsigned addr(int n) const { return group_addr(threadIdx.x & 31, n & ~3) + 4u * (n & 3); }
  static __device__ __forceinline__ float lds(unsigned a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
  }
  static __device__ __forceinline__ float4 lds4(unsigned a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
  }
  __device__ __forceinline__ void prepare(int n) const {
    if (n & 31) return;
    if (n == 0) {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncwarp();
      fetch(0);
    }
    if (n + 32 < n_head) {
      __syncwarp();
      fetch(n + 32);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncwarp();
  }
  __device__ __forceinline__ void load(int n, double& mu, double& r) const {
    float m32 = lds(addr(n)); mu = f32pos_to_d(m32); r = rcp_f32den_e1(m32, mu);
  }
  template <int CH> __device__ __forceinline__ void load_chunk(int n, double (&mu)[CH], double (&r)[CH]) const {
    const unsigned l = threadIdx.x & 31;
#pragma unroll
    for (int g = 0; g < CH / 4; g++) {
      const float4 v = lds4(group_addr(l, n + 4 * g));
      const float m32[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; e++) { mu[4 * g + e] = f32pos_to_d(m32[e]); r[4 * g + e] = rcp_f32den_e1(m32[e], mu[4 * g + e]); }
    }
  }
  __device__ __forceinline__ double mu_at(int n) const { return f32pos_to_d(lds(addr(n))); }
};

__device__ __forceinline__ unsigned hash32(unsigned x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

// the synthetic model of row i
__device__ __forceinline__ PairModel row_model(int i) {
  const unsigned h = hash32(i * 2654435761u + 7u);
  PairModel m;
  model_init(m, 4.0f + (float)(h & 1023) * (8.0f / 1024.0f), 0.02f + (float)((h >> 10) & 255) * 1e-4f, 5e-4f,
             256 + (int)((h >> 18) & 1023), 64 + (int)((h >> 24) & 255), N);
  return m;
}

// one row per slot, BuildModel's service rates of a synthetic model; mono = the last descent
__global__ void build_rows(float* rows, int* mono, int n_rows) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  const PairModel m = row_model(i);
  float* row = rows + (size_t)i * STRIDE;
  int desc = 0;
  float prev = 0.0f;
  for (int n = 0; n < N; n++) {
    const float v = serv_rate(m, n + 1);
    row[n] = v;
    if (n > 0 && !(prev <= v)) desc = n;
    prev = v;
  }
  mono[i] = desc;
}

// table variants ----------------------------------------------------------------------------------------------------
struct RegTable {             // (a): every state reads the same per-lane (mu, r), held in registers
  static constexpr int kChunk = WVA_TILE_CHUNK;
  double mu, r;
  __device__ __forceinline__ void prepare(int) const {}
  template <int CH> __device__ __forceinline__ void load_chunk(int, double (&m)[CH], double (&rr)[CH]) const {
#pragma unroll
    for (int j = 0; j < CH; j++) { m[j] = mu; rr[j] = r; }
  }
  __device__ __forceinline__ void load(int, double& m, double& rr) const { m = mu; rr = r; }
  __device__ __forceinline__ double mu_at(int) const { return mu; }
};
struct IeeeRateTable {        // ieee: RateTable with the IEEE division (serv_rate_nf), one slow-path branch per rate
  static constexpr int kChunk = WVA_TILE_CHUNK;
  RateCoef c;
  __device__ __forceinline__ void prepare(int) const {}
  __device__ __forceinline__ void load(int n, double& mu, double& r) const {
    const float m32 = serv_rate_nf(c, (float)(n + 1)); mu = f32pos_to_d(m32); r = rcp_f32den_e1(m32, mu);
  }
  template <int CH> __device__ __forceinline__ void load_chunk(int n, double (&mu)[CH], double (&r)[CH]) const {
    float m32[CH], nf = (float)(n + 1);
#pragma unroll
    for (int j = 0; j < CH; j++) { m32[j] = serv_rate_nf(c, nf); nf = f_add(nf, 1.0f); }
#pragma unroll
    for (int j = 0; j < CH; j++) { mu[j] = f32pos_to_d(m32[j]); r[j] = rcp_f32den_e1(m32[j], mu[j]); }
  }
  __device__ __forceinline__ double mu_at(int n) const { return f32pos_to_d(serv_rate_nf(c, (float)(n + 1))); }
};
struct NoFetchTable : TileTable {   // (b): tiles 0 and 1 fetched once per pass; later states read them again
  __device__ __forceinline__ void prepare(int n) const {
    if (n) return;
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    fetch(0);
    if (32 < n_head) fetch(32);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
  }
};

// the head loop of lockstep_fast_head, spelled out so that the chunk can be swapped (TA = false: p1_chunk)
template <bool TA, class Tab>
__device__ __noinline__ int head_loop(const PairModel& m, const Tab tab, float lambda, bool active, double* keep) {
  constexpr int CH = Tab::kChunk;
  const unsigned full = 0xffffffffu;
  const int NH = m.N - 1;
  double lam = active ? (double)lambda : 0.0;
  FastHead h;
  h.p = 1.0; h.sum = 1.0; h.T = 0.0; h.A = 0.0; h.n = 0; h.ok = true; h.exited = false;
  bool live = active;
  int states = 0, n = 0;
  while (n < NH && __any_sync(full, live)) {
    const int cnt = min(CH, NH - n);
    tab.prepare(n);
    double mu0;
    int mn = 0x7fffffff, mx = 0;
    if (cnt == CH) {
      double mu[CH], r[CH];
      tab.template load_chunk<CH>(n, mu, r);
      mu0 = mu[0];
      if (TA) {
        fast_chunk<CH>(h, lam, mu, r, (double)n, mn, mx);
      } else {
        P1 a[1]; a[0].p = h.p; a[0].sum = h.sum; a[0].mn = mn; a[0].mx = mx;
        const double lamv[1] = {lam}, lamr_c[1] = {0.0};
        p1_chunk<1, CH, true>(a, lamv, lamr_c, mu, r);
        h.p = a[0].p; h.sum = a[0].sum; mn = a[0].mn; mx = a[0].mx;
      }
    } else {
      mu0 = tab.mu_at(n);
      for (int j = 0; j < cnt; j++) {
        double mu, r; tab.load(n + j, mu, r);
        h.p = step_div(h.p, lam, d_mul(lam, r), mu, r, mn, mx);
        h.sum = d_add(h.sum, h.p);
        if (TA) {
          h.T = d_fma((double)(n + j + 1), h.p, h.T);
          h.A = d_add(h.A, d_min(d_mul(h.sum, 0x1p-53), h.p));
        }
      }
    }
    states += live ? cnt : 0;
    const int n0 = n;
    n += cnt;
    const bool oob = live & ((mn < WVA_HI_LO) | (mx >= WVA_HI_HI));
    const bool leave = live & !oob & (n < NH) & fast_head_exit(m, lam, mu0, n0, n, h.p, h.sum);
    h.ok = h.ok & !oob;
    if (leave) { h.exited = true; h.n = n; }
    if (oob | leave) { live = false; lam = 0.0; }
  }
  *keep = d_add(*keep, d_add(d_add(h.sum, h.T), h.A));
  return states;
}

struct Acc { unsigned long long cycles, warp_states, lane_states, batches; };

template <int V>
__global__ void __launch_bounds__(THREADS, 1)
head_kernel(const float* rows_all, const int* mono_all, int batches, int warps_on, Acc* acc, double* sink) {
  extern __shared__ __align__(16) float tiles[];      // [THREADS / 32][TileTable::kWarpFloats]
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp >= warps_on) return;
  const float* rows = rows_all + (size_t)blockIdx.x * P * STRIDE;
  const int* mono = mono_all + (size_t)blockIdx.x * P;
  const unsigned tile = (unsigned)__cvta_generic_to_shared(tiles + warp * TileTable::kWarpFloats);
  unsigned long long cyc = 0, ws = 0, ls = 0;
  double keep = 0.0;
  for (int b = 0; b < batches; b++) {
    const unsigned hh = hash32((blockIdx.x * 64u + warp) * 65599u + b * 2246822519u + lane);
    const int slot = (int)(hh & (P - 1));
    PairModel m;
    m.N = N; m.K = N + N * WVA_QUEUE_TO_BATCH; m.mono = __ldg(mono + slot); m.e1_ok = 1; m.tab = nullptr; m.stride = 1;
    const float rl = __ldg(rows + (size_t)slot * STRIDE + N - 1);
    m.mu_last = (double)rl; m.r_last = rcp_f32den(rl, m.mu_last);
    const float lambda = f_mul(f_mul(0.999f, rl), (float)((hh >> 10) + 1) * (1.0f / 4194305.0f));
    TileTable tt; tt.rows = rows; tt.row_stride = STRIDE; tt.slot = slot; tt.tile = tile; tt.n_head = N - 1;
    int sv = 0;
    long long t = 0;
    __syncwarp();
    if (V == V_PRODUCT) {
      SolveStats st;
      unsigned long long ph[3] = {0, 0, 0};
      sv = lockstep_solve_fast_only(m, tt, lambda, true, st, ph);
      if (sv < 0) sv = -1 - sv;
      t = __shfl_sync(full, (long long)ph[1], 0);
      keep = d_add(keep, (double)st.avgNumInSystem);
    } else {
      const long long t0 = clock64();
      if (V == V_BASE) sv = head_loop<true>(m, tt, lambda, true, &keep);
      if (V == V_COMPUTED) sv = head_loop<true>(m, RateTable{rate_coef(row_model(blockIdx.x * P + slot))}, lambda, true, &keep);
      if (V == V_IEEE) sv = head_loop<true>(m, IeeeRateTable{rate_coef(row_model(blockIdx.x * P + slot))}, lambda, true, &keep);
      if (V == V_NOFETCH) { NoFetchTable nf; static_cast<TileTable&>(nf) = tt; sv = head_loop<true>(m, nf, lambda, true, &keep); }
      if (V == V_NOTA) sv = head_loop<false>(m, tt, lambda, true, &keep);
      if (V == V_REG) {
        RegTable rt;
        const float m32 = __ldg(rows + (size_t)slot * STRIDE + N / 2);
        rt.mu = (double)m32; rt.r = rcp_f32den(m32, rt.mu);
        sv = head_loop<true>(m, rt, lambda, true, &keep);
      }
      __syncwarp();
      t = clock64() - t0;
    }
    const int mx = __reduce_max_sync(full, sv);
    const int sum = __reduce_add_sync(full, sv);
    cyc += t; ws += mx; ls += sum;
  }
  if (lane == 0) {
    atomicAdd(&acc->cycles, cyc); atomicAdd(&acc->warp_states, ws); atomicAdd(&acc->lane_states, ls);
    atomicAdd(&acc->batches, (unsigned long long)batches);
  }
  sink[blockIdx.x * THREADS + threadIdx.x] = keep;
}

template <int V>
void run(int sms, int warps, int batches, const float* rows, const int* mono, Acc* d_acc, double* sink) {
  const int smem = THREADS / 32 * TileTable::kWarpFloats * (int)sizeof(float);
  CK(cudaFuncSetAttribute(head_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  head_kernel<V><<<sms, THREADS, smem>>>(rows, mono, batches / 4 + 1, warps, d_acc, sink);     // warm-up
  CK(cudaGetLastError());
  CK(cudaMemset(d_acc, 0, sizeof(Acc)));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  CK(cudaEventRecord(e0));
  head_kernel<V><<<sms, THREADS, smem>>>(rows, mono, batches, warps, d_acc, sink);
  CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
  CK(cudaGetLastError());
  float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
  Acc a; CK(cudaMemcpy(&a, d_acc, sizeof(Acc), cudaMemcpyDeviceToHost));
  printf("CH %2d  %-9s warps/SM %2d : %7.1f cycles per warp-state, %5.1f %% live lane-states, %8.3f ms, %.3g warp-states/s\n",
         WVA_TILE_CHUNK, kNames[V], warps, (double)a.cycles / (double)a.warp_states,
         100.0 * (double)a.lane_states / (32.0 * (double)a.warp_states), ms, (double)a.warp_states / (ms * 1e-3));
}

int main(int argc, char** argv) {
  const int batches = argc > 1 ? atoi(argv[1]) : 64;
  int sms; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const int n_rows = sms * P;
  float* rows; int* mono; Acc* acc; double* sink;
  CK(cudaMalloc(&rows, (size_t)n_rows * STRIDE * sizeof(float)));
  CK(cudaMalloc(&mono, (size_t)n_rows * sizeof(int)));
  CK(cudaMalloc(&acc, sizeof(Acc)));
  CK(cudaMalloc(&sink, (size_t)sms * THREADS * sizeof(double)));
  build_rows<<<(n_rows + 255) / 256, 256>>>(rows, mono, n_rows);
  CK(cudaDeviceSynchronize());
  for (int w : {16, 4}) {
    run<V_PRODUCT>(sms, w, batches, rows, mono, acc, sink);
    run<V_BASE>(sms, w, batches, rows, mono, acc, sink);
    run<V_COMPUTED>(sms, w, batches, rows, mono, acc, sink);
    run<V_IEEE>(sms, w, batches, rows, mono, acc, sink);
    run<V_REG>(sms, w, batches, rows, mono, acc, sink);
    run<V_NOFETCH>(sms, w, batches, rows, mono, acc, sink);
    run<V_NOTA>(sms, w, batches, rows, mono, acc, sink);
  }
  return 0;
}
