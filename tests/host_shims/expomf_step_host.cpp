// Host build of qrec_b200/csrc/expomf_step.cuh (with als_step.cuh): one ExpoMF row solve and one row's exposure
// prior on the CPU with the headers' own posterior, lift, prior, factorization and substitution functions, in the
// order exposure_solve_rows_kernel applies them (every row of Z weighted by its posterior, then the observed entries
// lifted to 1) -- so the CPU suite pins the device source to the float64 oracle.  (The kernel spreads the sums over
// threads; only the grouping of the float64 sums differs.)
#include <cstddef>
#include <cstdint>
#include <vector>
#define __host__
#define __device__
#define __forceinline__ inline
#include "als_step.cuh"
#include "expomf_step.cuh"

namespace {

double dot(const double* x, const float* z, int d) {
  double s = 0.0;
  for (int c = 0; c < d; ++c) s += x[c] * (double)z[c];
  return s;
}

double mu_of(const float* mu, int mu_by_row, double mu_r, int64_t k) { return mu_by_row ? mu_r : (double)mu[k]; }

}  // namespace

// x_out = (sum_k A_k z_k z_k^T + lambda*I)^-1 sum_{observed k} z_k for the row x_old (float64, d) against Z
// (float32 [n_z][d]); observed columns cols[0..n_cols); mu by row (mu_r) or by Z's row (mu[k]).  Returns 1 on
// success, 0 when the system is not positive definite (x_out untouched).
extern "C" int32_t host_expomf_solve_row(const double* x_old, const float* Z, int d, int64_t n_z, const int32_t* cols,
                                         int64_t n_cols, const float* mu, int mu_by_row, double mu_r, double lambda,
                                         double lam_y, double* x_out) {
  std::vector<double> A((size_t)d * d, 0.0), b(d, 0.0), s(d);
  auto add = [&](const float* z, double w) {
    for (int a = 0; a < d; ++a)
      for (int e = a; e < d; ++e) A[(size_t)a * d + e] += (w * (double)z[a]) * (double)z[e];
  };
  for (int64_t k = 0; k < n_z; ++k) {
    const float* z = Z + (size_t)k * d;
    add(z, qrec::expomf_exposure(dot(x_old, z, d), mu_of(mu, mu_by_row, mu_r, k), lam_y));
  }
  for (int64_t k = 0; k < n_cols; ++k) {
    const float* z = Z + (size_t)cols[k] * d;
    add(z, qrec::expomf_lift(qrec::expomf_exposure(dot(x_old, z, d), mu_of(mu, mu_by_row, mu_r, cols[k]), lam_y)));
    for (int a = 0; a < d; ++a) b[a] += (double)z[a];
  }
  for (int a = 0; a < d; ++a) A[(size_t)a * d + a] += lambda;
  if (!qrec::als_cholesky(A.data(), d, d, s.data())) return 0;
  qrec::als_solve(A.data(), d, d, s.data(), b.data());
  for (int a = 0; a < d; ++a) x_out[a] = b[a];
  return 1;
}

// The exposure prior of one row x (its new value) against Z with its own mu_r: (a + sum_k A_k - 1) / (a + b + n_z - 2),
// A_k = 1 on the observed columns.
extern "C" double host_expomf_prior(const double* x, const float* Z, int d, int64_t n_z, const int32_t* cols,
                                    int64_t n_cols, double mu_r, double lam_y, double a, double b) {
  double sum = 0.0;
  for (int64_t k = 0; k < n_z; ++k) sum += qrec::expomf_exposure(dot(x, Z + (size_t)k * d, d), mu_r, lam_y);
  for (int64_t k = 0; k < n_cols; ++k)
    sum += qrec::expomf_lift(qrec::expomf_exposure(dot(x, Z + (size_t)cols[k] * d, d), mu_r, lam_y));
  return qrec::expomf_prior(sum, a, b, n_z);
}
