// ingest_scatter.hpp — host side of wva_ingest_write: one Prometheus-shaped vector (slot, value) in result order into the
// page-locked per-slot columns (plain C++, no CUDA: also compiled into tests/host_emul for the CPU tests).
//
// Semantics (internal/collector/replica_metrics.go:133-160: the reference assigns into a map keyed by pod): a LATER sample
// of a pod overwrites an earlier one; a sample with slot < 0 (no pod label / unknown pod) is skipped; slot >= S is an
// argument error.
//
// A response in registry order is written by the plain serial loop.  A response in arbitrary pod order costs that loop a
// cache miss per sample, so it goes through a two-pass radix partition over T host threads:
//   pass 1  thread t takes the t-th contiguous chunk of the samples and bins them by slot range (B ranges of 2^shift
//           <= 64 K slots) into its own segment of a scratch array — sequential reads, B sequential write streams;
//   pass 2  range b is owned by ONE thread, which replays the bins (0, b), (1, b), … (T-1, b) in that order — i.e. in
//           sample order, so duplicates resolve exactly as in the serial loop — and scatters into a range that fits its
//           L2.  No two threads write the same slot (or the same 64-byte line of `has`: shift >= 6).
// The price: the columns are the page-locked arena the cycle's H2D copy reads, and lines left dirty in the caches of
// cores all over the host slow that DMA down; doing pass 2 on the calling thread alone avoids that but is much slower
// per vector, so the threads win (tools/cfg5_ingest.py compares the two).
#pragma once
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <thread>
#include <vector>

namespace wva {

struct IngestScratch {                 // reused from call to call (owned by the wva_ingest object)
  std::vector<int32_t> slot;
  std::vector<double> value;
  std::vector<int64_t> off;            // [T][B + 1] bin offsets inside a thread's segment
};

// host threads for large vectors: min(8, hardware threads, cgroup v2 CPU quota) — a container that exposes 128 hardware
// threads under a 16-CPU quota must not be oversubscribed
inline int ingest_host_threads() {
  static const int cached = [] {
    unsigned hw = std::thread::hardware_concurrency();
    int t = (int)(hw >= 8 ? 8 : (hw ? hw : 1));
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
      long long quota = 0, period = 0;
      if (fscanf(f, "%lld %lld", &quota, &period) == 2 && quota > 0 && period > 0) {
        const int q = (int)(quota / period);
        if (q < t) t = q < 1 ? 1 : q;
      }
      fclose(f);
    }
    return t;
  }();
  return cached;
}

// the serial loop; returns false if a slot is >= S (the columns then hold the samples before it)
inline bool ingest_scatter_serial(double* col, uint8_t* has, long long S, uint8_t bit, int64_t n, const int32_t* slot,
                                  const double* value) {
  for (int64_t i = 0; i < n; i++) {
    const long long k = slot[i];
    if (k < 0) continue;
    if (k >= S) return false;
    col[k] = value[i];
    has[k] |= bit;
  }
  return true;
}

// threads: 0 = choose (serial below 64 K samples and for responses in registry order, else up to 8 binning threads —
// WVA_INGEST_THREADS overrides the count), > 0 = the partition with that many binning threads whatever the input
inline bool ingest_scatter(double* col, uint8_t* has, long long S, uint8_t bit, int64_t n, const int32_t* slot,
                           const double* value, IngestScratch& sc, int threads_arg = 0) {
  int threads = threads_arg;
  if (threads <= 0) {
    const char* e = getenv("WVA_INGEST_THREADS");
    threads = e ? atoi(e) : 0;
    if (threads <= 0) threads = n < 65536 ? 1 : ingest_host_threads();
  }
  if (threads > 64) threads = 64;
  if (threads <= 1 || n < 2 || S < 128) return ingest_scatter_serial(col, has, S, bit, n, slot, value);
  if (threads_arg <= 0) {
    // mostly ascending slots (a response in registry order): the serial loop already streams
    int64_t asc = 0;
    const int64_t probes = 4096, step = (n - 1) / probes;
    if (step >= 1) {
      for (int64_t j = 0; j < probes; j++) asc += slot[j * step] < slot[j * step + 1];
      if (asc * 100 >= probes * 95) return ingest_scatter_serial(col, has, S, bit, n, slot, value);
    }
  }
  const int T = threads;
  int shift = 16;                                       // ranges of 2^shift slots: 64 K slots (0.6 MB of columns) ...
  while (shift > 6 && ((S - 1) >> shift) + 1 < 8) shift--;      // ... at least 8 ranges on a small registry ...
  while (((S - 1) >> shift) + 1 > 256) shift++;                 // ... and at most 256 write streams on a huge one
  const int B = (int)(((S - 1) >> shift) + 1);
  sc.slot.resize((size_t)n); sc.value.resize((size_t)n); sc.off.assign((size_t)T * (B + 1), 0);
  std::atomic<bool> ok{true};
  auto chunk = [&](int t, int64_t& lo, int64_t& hi) { lo = n * t / T; hi = n * (t + 1) / T; };
  auto run = [&](auto&& fn) {
    std::vector<std::thread> pool;
    pool.reserve(T - 1);
    for (int t = 1; t < T; t++) pool.emplace_back(fn, t);
    fn(0);
    for (auto& th : pool) th.join();
  };
  // ---- pass 1 (T threads): count, then place (the thread's segment of the scratch arrays is [lo, hi) of the samples)
  run([&](int t) {
    int64_t lo, hi; chunk(t, lo, hi);
    int64_t* off = sc.off.data() + (size_t)t * (B + 1);
    for (int64_t i = lo; i < hi; i++) {
      const long long k = slot[i];
      if (k < 0) continue;
      if (k >= S) { ok.store(false); continue; }
      off[(k >> shift) + 1]++;
    }
    for (int b = 0; b < B; b++) off[b + 1] += off[b];
    std::vector<int64_t> cur(off, off + B);
    for (int64_t i = lo; i < hi; i++) {
      const long long k = slot[i];
      if (k < 0 || k >= S) continue;
      const int64_t p = lo + cur[k >> shift]++;
      sc.slot[(size_t)p] = (int32_t)k; sc.value[(size_t)p] = value[i];
    }
  });
  if (!ok.load()) return false;                         // (nothing written: stricter than the serial loop, same status)
  // ---- pass 2 (T threads): range b belongs to thread b % T; bins replayed in thread (= sample) order
  run([&](int t) {
    for (int b = t; b < B; b += T) {
      for (int u = 0; u < T; u++) {
        int64_t lo, hi; chunk(u, lo, hi);
        const int64_t* off = sc.off.data() + (size_t)u * (B + 1);
        for (int64_t p = lo + off[b]; p < lo + off[b + 1]; p++) {
          const int32_t k = sc.slot[(size_t)p];
          col[k] = sc.value[(size_t)p];
          has[k] |= bit;
        }
      }
    }
  });
  return true;
}

}  // namespace wva
