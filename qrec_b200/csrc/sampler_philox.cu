// K0 (fast): device negative sampler.  Same job as the rejection loop at
// base/deepRecommender.py:47-49 / model/ranking/BPR.py:35-37, but drawn from a counter-based
// Philox4x32-10 stream so that every triple is independent (the reference's MT19937 stream is
// inherently serial; the bit-exact clone lives in host_sampler.cpp).
//
//   j = (philox(key=(seed_lo, seed_hi); ctr=(k_lo, k_hi, attempt, epoch)).x * num_items) >> 32
// attempt = 0, 1, ... until j is not in user u[k]'s sorted rated-item row (binary search).
#include "common.h"
#include "philox.cuh"

namespace {

__global__ void __launch_bounds__(256)
sample_neg_philox_kernel(long long n, int num_items, const int* __restrict__ u,
                         const long long* __restrict__ rowptr, const int* __restrict__ cols,
                         uint32_t seed_lo, uint32_t seed_hi, uint32_t epoch, int* __restrict__ out_j) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) {
    const int uu = __ldg(u + k);
    out_j[k] = qrec::sample_negative(k, epoch, seed_lo, seed_hi, num_items, cols, __ldg(rowptr + uu),
                                     __ldg(rowptr + uu + 1));
  }
}

}  // namespace

extern "C" int qrec_sample_neg_philox(int64_t n, int32_t num_items, const int32_t* u,
                                      const int64_t* rowptr, const int32_t* cols, uint64_t seed,
                                      uint32_t epoch, int32_t* out_j, void* stream) {
  QREC_REQUIRE(n >= 0 && num_items >= 1, "qrec_sample_neg_philox: bad sizes");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && rowptr && cols && out_j, "qrec_sample_neg_philox: null pointer");
  const long long blocks = (n + 255) / 256;
  const long long cap = 132LL * 16;
  sample_neg_philox_kernel<<<(int)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(
      n, num_items, u, reinterpret_cast<const long long*>(rowptr), cols, (uint32_t)seed,
      (uint32_t)(seed >> 32), epoch, out_j);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
