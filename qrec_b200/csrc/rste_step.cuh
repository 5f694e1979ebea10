// Scalar pieces of RSTE's rating pass (rste_kernels.cu), kept apart so that the CPU suite can compile and run the
// very same source (tests/host_shims/rste_step_host.cpp).  numpy's evaluation order, every product, sum and
// quotient rounded separately (the mf_* helpers of mf_step.cuh never contract into an FMA).
//
//   predictForRating  RSTE.py:41-64
//     s    = sum_f w_f * (P[f].Q[i])                  followees f of u in the cleaned followee dict's order
//     pred = alpha*(P[u].Q[i]) + ((1-alpha)*s) / denom[u]     when denom[u] != 0
//     pred = P[u].Q[i]                                         when denom[u] == 0 (also: no followees)
//   update  RSTE.py:31-34: K9 kind 1's step (mf_update_parity<T, 1>) with the error scaled to alpha*e;
//   loss += e^2, unscaled.
#pragma once

#include "mf_step.cuh"

namespace qrec {

__device__ __forceinline__ float mf_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double mf_div(double a, double b) { return __ddiv_rn(a, b); }

// s + w*dot: one followee's term of the social sum, in the followee order
template <typename T>
__device__ __forceinline__ T rste_social_add(T s, T w, T dot) {
  return mf_add(s, mf_mul(w, dot));
}

template <typename T>
__device__ __forceinline__ T rste_prediction(T dot, T social, T alpha, T denom) {
  if (denom == T(0)) return dot;
  return mf_add(mf_mul(alpha, dot), mf_div(mf_mul(mf_sub(T(1), alpha), social), denom));
}

}  // namespace qrec
