// Error reporting, version string, launch accounting and launch sizing for libqrec.so.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <mutex>
#include <utility>

#include "common.h"

namespace {
thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};
}  // namespace

namespace qrec {
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  static std::atomic<int> cached[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  int v = cached[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    cached[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}

int capped_grid(long long blocks, int ctas_per_sm) {
  const long long cap = (long long)sm_count() * ctas_per_sm;
  return (int)(blocks < 1 ? 1 : (blocks < cap ? blocks : cap));
}

// 2 CTAs of 8 warps per SM: enough warps to cover the dependency DAG's width at the synthetic scale (~25 independent
// triples per level of K1 in user-major order) without drowning the LSU in pollers.
// n_warps > 0: the caller knows the width of the dependency DAG (e.g. qrec_bpr_order_depth) and asks for about that
// many pollers -- thousands of idle warps hammering the version counters slow the few that can make progress
// (1.4 independent triples per level on FilmTrust, ~25 at SYN scale)
int ordered_grid(int n_warps) { return n_warps > 0 ? capped_grid((n_warps + 7) / 8, 2) : sm_count() * 2; }

cudaError_t allow_dynamic_smem(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> granted;   // (kernel, device) -> limit set
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  int& have = granted[{kernel, dev}];
  if (bytes <= have) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess) have = bytes;
  return e;
}
}  // namespace qrec

extern "C" {
const char* qrec_last_error(void) { return g_err; }
const char* qrec_version(void) { return "qrec-b200 0.1.0 sm_90a"; }
int64_t qrec_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
}
