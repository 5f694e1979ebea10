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
// kernels are grid-stride loops).  ordered_grid(): the grid of 8-warp CTAs for a warp-per-position in-order kernel
// (device.cuh) asked for about n_warps pollers, 0 for the default.
int sm_count();
int capped_grid(long long blocks, int ctas_per_sm);
int ordered_grid(int n_warps);
// Raises `kernel`'s dynamic shared-memory limit to at least `bytes` on the current device.  The limit belongs to
// the kernel as loaded on each device, so it is set once per (kernel, device); safe to call from several threads.
cudaError_t allow_dynamic_smem(const void* kernel, int bytes);

// K1 launchers (bpr_kernels.cu), also driven chunk by chunk by the host-buffer pipeline (runtime.cu).
// launch_bpr_batch: the order-agnostic fused SGD step over n triples (u, i, j).
int launch_bpr_batch(float* P, float* Q, int d, long long n, const int* u, const int* i, const int* j, float lr,
                     float reg_u, float reg_i, double* loss, cudaStream_t st);
// launch_usermajor: the user-major epoch over a CSR of whole users.  rowptr holds global triple offsets, i / j are
// indexed from trip_off.  sample: draw the negatives in the kernel (FusedSampler) instead of reading j; rated_sig
// (may be null) adds the signature pre-test.
int launch_usermajor(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, const int64_t* rowptr,
                     const int32_t* i, const int32_t* j, float lr, float reg_u, float reg_i, double* loss,
                     bool sample, const int64_t* rated_rowptr, const int32_t* rated_cols, int32_t num_items,
                     uint64_t seed, uint32_t epoch, int32_t* j_out, long long trip_off, cudaStream_t st,
                     const uint32_t* rated_sig);

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
