// Host build of qrec_b200/csrc/cofactor_step.cuh (with als_step.cuh): one CoFactor item sweep on the CPU with the
// headers' own right-hand-side, w / c, factorization and substitution functions, item after item in id order as
// cofactor_item_sweep_kernel applies them -- so the CPU suite pins the device source to the reference's golden run.
// (The kernel spreads the sums over threads; only the grouping of the float64 sums differs.)
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>
#define __host__
#define __device__
#define __forceinline__ inline
#include "als_step.cuh"
#include "cofactor_step.cuh"

namespace {

// A (upper triangle, row-major d x d) += sum_k wt_k z_k z_k^T and b += sum_k coef_k z_k over the rows rows[0..n)
void accumulate(std::vector<double>& A, std::vector<double>& b, const double* Z, int d, const int32_t* rows, int64_t n,
                const double* wt, const double* coef) {
  for (int64_t k = 0; k < n; ++k) {
    const double* z = Z + (size_t)rows[k] * d;
    for (int a = 0; a < d; ++a) {
      b[a] += coef[k] * z[a];
      for (int e = a; e < d; ++e) A[(size_t)a * d + e] += (wt[k] * z[a]) * z[e];
    }
  }
}

bool solve(std::vector<double>& A, std::vector<double>& b, int d, double* out) {
  std::vector<double> s(d);
  if (!qrec::als_cholesky(A.data(), d, d, s.data())) return false;
  qrec::als_solve(A.data(), d, d, s.data(), b.data());
  for (int a = 0; a < d; ++a) out[a] = b[a];
  return true;
}

}  // namespace

extern "C" int32_t host_cofactor_item_sweep_f64(double* Y, double* G, double* w, double* c, const double* X, int d,
                                                int64_t n_users, int64_t n_items, const int64_t* irp,
                                                const int32_t* icol, const double* ival, const int64_t* srp,
                                                const int32_t* scol, const double* sval, double lambda, double gamma,
                                                double alpha) {
  std::vector<double> XtX((size_t)d * d, 0.0);
  for (int64_t r = 0; r < n_users; ++r)
    for (int a = 0; a < d; ++a)
      for (int e = 0; e < d; ++e) XtX[(size_t)a * d + e] += X[r * d + a] * X[r * d + e];
  int32_t failed = 0;
  for (int64_t i = 0; i < n_items; ++i) {
    const int64_t nu = irp[i + 1] - irp[i], nc = srp[i + 1] - srp[i];
    const int32_t* users = icol + irp[i];
    const int32_t* ctx = scol + srp[i];
    const double* m = sval + srp[i];
    const double w_i = w[i], c_i = c[i];
    const std::vector<double> y_old(Y + i * d, Y + (i + 1) * d), g_old(G + i * d, G + (i + 1) * d);
    // Y_i: users (weight alpha*r, rhs 1 + alpha*r), then the contexts' G rows (weight 1, rhs ((m - w_i) - c_c))
    std::vector<double> S((size_t)d * d, 0.0), bx(d, 0.0), bg(d, 0.0), wt, coef;
    for (int64_t k = 0; k < nu; ++k) {
      wt.push_back(qrec::als_conf<double>(ival[irp[i] + k], alpha));
      coef.push_back(qrec::als_rhs_weight(wt.back()));
    }
    accumulate(S, bx, X, d, users, nu, wt.data(), coef.data());
    wt.assign(nc, 1.0);
    coef.clear();
    double wsum = 0.0;
    for (int64_t k = 0; k < nc; ++k) {
      coef.push_back(qrec::cof_rhs_y_coef(m[k], w_i, c[ctx[k]]));
      double yg = 0.0;
      for (int a = 0; a < d; ++a) yg += y_old[a] * G[(size_t)ctx[k] * d + a];
      wsum += qrec::cof_w_term(m[k], yg, c[ctx[k]]);
    }
    accumulate(S, bg, G, d, ctx, nc, wt.data(), coef.data());
    std::vector<double> A((size_t)d * d, 0.0), b(d);
    for (int a = 0; a < d; ++a) {
      b[a] = bx[a] + bg[a];
      for (int e = a; e < d; ++e) A[(size_t)a * d + e] = (XtX[(size_t)a * d + e] + S[(size_t)a * d + e]) + (a == e ? lambda : 0.0);
    }
    if (!solve(A, b, d, Y + i * d)) ++failed;            // the row keeps its old value
    if (nc == 0) continue;
    // G_i: the contexts' Y rows (weight 1, rhs ((m - w_c) - c_i)), then w_i and c_i
    std::fill(A.begin(), A.end(), 0.0);
    std::fill(b.begin(), b.end(), 0.0);
    coef.clear();
    double csum = 0.0;
    for (int64_t k = 0; k < nc; ++k) {
      coef.push_back(qrec::cof_rhs_g_coef(m[k], w[ctx[k]], c_i));
      double yg = 0.0;
      for (int a = 0; a < d; ++a) yg += g_old[a] * Y[(size_t)ctx[k] * d + a];
      csum += qrec::cof_c_term(m[k], yg, w[ctx[k]]);
    }
    accumulate(A, b, Y, d, ctx, nc, wt.data(), coef.data());
    for (int a = 0; a < d; ++a) A[(size_t)a * d + a] += gamma;
    if (!solve(A, b, d, G + i * d)) ++failed;
    w[i] = qrec::cof_mean(wsum, (int)nc);
    c[i] = qrec::cof_mean(csum, (int)nc);
  }
  return failed;
}
