// Pieces of the top-N selection shared by the two K8 kernels (topn_kernels.cu, topn_tc.cu).  A candidate is the
// 64-bit key (ord_of(score) << 32) | (0xffffffff - item): descending keys are (score descending, item ascending).
#pragma once
#include <cstdint>

namespace qrec {

// monotone float -> uint; -0.0 and +0.0 are one score (the reference compares them equal), both map to +0.0's key
__device__ __forceinline__ uint32_t ord_of(float s) {
  const uint32_t u = __float_as_uint(s) == 0x80000000u ? 0u : __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float score_of(uint32_t o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// item in the sorted rated row cols[lo, hi)?  (bisection)
__device__ __forceinline__ bool is_rated(const int* __restrict__ cols, long long lo, long long hi, int item) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    const int c = __ldg(cols + mid);
    if (c == item) return true;
    if (c < item) lo = mid + 1; else hi = mid;
  }
  return false;
}

// one warp sorts SZ keys, descending (bitonic network in shared memory)
template <int SZ>
__device__ __forceinline__ void warp_sort_desc(unsigned long long* k, int lane) {
#pragma unroll 1
  for (int size = 2; size <= SZ; size <<= 1) {
#pragma unroll 1
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncwarp();
      for (int t = lane; t < SZ / 2; t += 32) {
        const int lo = 2 * t - (t & (stride - 1));           // index of the lower partner
        const int hi = lo + stride;
        const bool desc = (lo & size) == 0;
        const unsigned long long a = k[lo], b = k[hi];
        if ((a < b) == desc) { k[lo] = b; k[hi] = a; }
      }
    }
  }
  __syncwarp();
}

}  // namespace qrec
