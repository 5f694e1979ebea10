// Error reporting, version string and launch accounting for libqrec.so.
#include <atomic>
#include <cstdarg>
#include <cstdio>

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
}  // namespace qrec

extern "C" {
const char* qrec_last_error(void) { return g_err; }
const char* qrec_version(void) { return "qrec-b200 0.1.0 sm_90a"; }
int64_t qrec_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
}
