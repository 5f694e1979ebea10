// Internal helpers shared by the translation units of libqrec.so.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#include "qrec.h"

namespace qrec {

void set_error(const char* fmt, ...);
void count_launch(int n = 1);

// Launch sizing (core.cpp).  sm_count(): SMs of the current device, queried once per device (132, an H100 SXM's,
// if the query fails).  capped_grid(): `blocks` CTAs, but at most ctas_per_sm per SM and at least one (the
// kernels are grid-stride loops).
int sm_count();
int capped_grid(long long blocks, int ctas_per_sm);
// Raises `kernel`'s dynamic shared-memory limit to at least `bytes` on the current device.  The limit belongs to
// the kernel as loaded on each device, so it is set once per (kernel, device); safe to call from several threads.
cudaError_t allow_dynamic_smem(const void* kernel, int bytes);

inline int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("%s failed at %s:%d: %s", what, file, line, cudaGetErrorString(e));
  return QREC_ERR_CUDA;
}

}  // namespace qrec

#define QREC_CUDA(call)                                                     \
  do {                                                                      \
    cudaError_t e__ = (call);                                               \
    if (e__ != cudaSuccess) return qrec::cuda_fail(e__, #call, __FILE__, __LINE__); \
  } while (0)

#define QREC_REQUIRE(cond, ...)      \
  do {                               \
    if (!(cond)) {                   \
      qrec::set_error(__VA_ARGS__);  \
      return QREC_ERR_ARG;           \
    }                                \
  } while (0)

// Launch-error check that does not synchronise.
#define QREC_LAUNCH_CHECK()                                                        \
  do {                                                                             \
    cudaError_t e__ = cudaGetLastError();                                          \
    if (e__ != cudaSuccess) return qrec::cuda_fail(e__, "kernel launch", __FILE__, __LINE__); \
    qrec::count_launch();                                                          \
  } while (0)
