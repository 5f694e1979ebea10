// Per-entry arithmetic of the ExpoMF row solve (als_kernels.cu) that als_step.cuh does not already hold: the exposure
// posterior, the weight that lifts an observed entry's posterior to 1, and the exposure prior.  Kept apart so that the
// CPU suite can compile and run the very same source (tests/host_shims/expomf_step_host.cpp).
//
//   reference: model/ranking/ExpoMF.py (a_row_batch, _solve, _update_expo).  For row r against the other table Z:
//     s = x_old.z_k,   p = sqrt(lam_y/2/pi) * exp(-lam_y * s^2 / 2),   A_k = (p + EPS) / (p + EPS + (1 - mu) / mu)
//     A_k = 1 on the row's observed entries
//     B = sum_k A_k z_k z_k^T + lambda*I,   x_r = B^-1 sum_{observed k} z_k
//     prior (item rows, new tables):  mu_i = (a + sum_u A_ui - 1) / (a + b + U - 2)
//   The operand order of every expression is the reference's.
#pragma once
#include <math.h>

namespace qrec {

constexpr double kExpoEps = 1e-8;                    // ExpoMF.py: EPS
constexpr double kExpoPi = 3.141592653589793;        // np.pi

// posterior of exposure of one entry: s = x.z, mu its prior
__host__ __device__ __forceinline__ double expomf_exposure(double s, double mu, double lam_y) {
  const double p = sqrt(lam_y / 2.0 / kExpoPi) * exp(-lam_y * (s * s) / 2.0);
  return (p + kExpoEps) / (p + kExpoEps + (1.0 - mu) / mu);
}

// weight of the sparse correction that lifts an observed entry's posterior A to 1 (A[Y.nonzero()] = 1)
__host__ __device__ __forceinline__ double expomf_lift(double A) { return 1.0 - A; }

// the exposure prior from the sum of one item's posteriors over all n users
__host__ __device__ __forceinline__ double expomf_prior(double asum, double a, double b, long long n) {
  return (a + asum - 1.0) / (a + b + (double)n - 2.0);
}

}  // namespace qrec
