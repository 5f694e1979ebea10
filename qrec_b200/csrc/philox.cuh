// Philox4x32-10 (Salmon et al., SC'11; Random123 constants), shared by the device sampler, the
// fused user-major kernel, the SimGCL noise and the NGCF dropout masks.
#pragma once
#include <cstdint>

namespace qrec {

__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t out[4]) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// Negative item for triple k of epoch `epoch`: j = (philox(seed; k, attempt, epoch).x * num_items) >> 32,
// attempt = 0,1,... until j is not in the sorted row cols[lo, hi) (binary search).
__device__ __forceinline__ int sample_negative(long long k, uint32_t epoch, uint32_t seed_lo, uint32_t seed_hi,
                                               int num_items, const int* __restrict__ cols, long long lo0,
                                               long long hi0) {
  // a user whose (deduplicated) row already holds every item has no negative: take the first draw
  // instead of spinning forever (the host sampler reports this case as an error; a kernel cannot)
  const bool saturated = (hi0 - lo0) >= (long long)num_items;
  uint32_t attempt = 0;
  while (true) {
    uint32_t w[4];
    philox4x32_10((uint32_t)k, (uint32_t)((unsigned long long)k >> 32), attempt, epoch, seed_lo, seed_hi, w);
    const int j = (int)(((unsigned long long)w[0] * (unsigned long long)(uint32_t)num_items) >> 32);
    if (saturated) return j;
    long long lo = lo0, hi = hi0;
    bool hit = false;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      const int c = __ldg(cols + mid);
      if (c < j) lo = mid + 1;
      else if (c > j) hi = mid;
      else { hit = true; break; }
    }
    if (!hit) return j;
    ++attempt;
  }
}

// The same draw with a pre-test: `sig` points at the user's 512-bit signature (16 words, bit c & 511
// set for every rated column c, built by rated_signature_kernel).  A clear bit proves j is not rated,
// so ~1 - deg/512 of the draws skip the dependent-load bisection; a set bit falls through to it.  The
// signature has no false negatives, hence the result is identical to sample_negative().
constexpr int RATED_SIG_WORDS = 16;
__device__ __forceinline__ int sample_negative_sig(long long k, uint32_t epoch, uint32_t seed_lo, uint32_t seed_hi,
                                                   int num_items, const int* __restrict__ cols, long long lo0,
                                                   long long hi0, const uint32_t* __restrict__ sig) {
  const bool saturated = (hi0 - lo0) >= (long long)num_items;
  uint32_t attempt = 0;
  while (true) {
    uint32_t w[4];
    philox4x32_10((uint32_t)k, (uint32_t)((unsigned long long)k >> 32), attempt, epoch, seed_lo, seed_hi, w);
    const int j = (int)(((unsigned long long)w[0] * (unsigned long long)(uint32_t)num_items) >> 32);
    if (saturated) return j;
    const uint32_t word = __ldg(sig + ((j >> 5) & (RATED_SIG_WORDS - 1)));
    if (((word >> (j & 31)) & 1u) == 0u) return j;
    long long lo = lo0, hi = hi0;
    bool hit = false;
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      const int c = __ldg(cols + mid);
      if (c < j) lo = mid + 1;
      else if (c > j) hi = mid;
      else { hit = true; break; }
    }
    if (!hit) return j;
    ++attempt;
  }
}

// Arguments of the negatives drawn inside the fused user-major kernels (bpr_kernels.cu): the rejection
// sets, the Philox key and epoch of sample_negative(), and where to write the drawn j (may be null).
struct FusedSampler {
  const long long* rated_rowptr;   // rejection sets: CSR over users, sorted columns
  const int* rated_cols;
  int num_items;
  uint32_t seed_lo, seed_hi, epoch;
  int* j_out;
};

}  // namespace qrec
