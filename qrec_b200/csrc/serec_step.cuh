// Per-pair arithmetic of the SERec row solve (als_kernels.cu) that expomf_step.cuh does not already hold: the social
// exposure prior.  Kept apart so that the CPU suite can compile and run the very same source
// (tests/host_shims/serec_step_host.cpp).
//
//   reference: model/ranking/SERec.py (_update_expo).  The reference holds the prior as a dense U x I matrix:
//     A_sum = tile(sum_u A_u., [U, 1]),   S_sum = T.dot(A_sum),   T the 0/1 (user, followee) matrix
//     mu = (a + A_sum + (s-1)*S_sum - 1) / (a + b + (s-1)*S_sum + U - 2)
//   Every row of A_sum is the same vector A (A_i = sum_u A_ui), so S_sum[u, i] = deg(u) * A_i with deg(u) the number
//   of u's followees, and
//     mu(u, i) = (a + A_i + (s-1)*deg_u*A_i - 1) / (a + b + (s-1)*deg_u*A_i + U - 2)
//   is all the state the prior needs: one float64 A per item and one degree per user.  The operand order is the
//   reference's.  T.dot adds A_i to itself deg_u times; here S = deg_u * A_i is one product, which differs from the
//   repeated sum by a few ulps once deg_u >= 7 (oracle/serec_oracle.py offers both).
#pragma once

namespace qrec {

// the prior of the pair (u, i) from u's followee count and item i's summed posterior
__host__ __device__ __forceinline__ double serec_prior(double A, int deg, double a, double b, double s, double n_users) {
#ifdef __CUDA_ARCH__
  // separate roundings, as numpy does: no multiply-add contraction
  const double sS = __dmul_rn(s - 1.0, __dmul_rn((double)deg, A));
  return __dadd_rn(__dadd_rn(__dadd_rn(a, A), sS), -1.0) /
         __dadd_rn(__dadd_rn(__dadd_rn(a + b, sS), n_users), -2.0);
#else
  const double sS = (s - 1.0) * ((double)deg * A);
  return (a + A + sS - 1.0) / (a + b + sS + n_users - 2.0);
#endif
}

}  // namespace qrec
