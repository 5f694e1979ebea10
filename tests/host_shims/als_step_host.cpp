// Host build of qrec_b200/csrc/als_step.cuh: one WRMF half-epoch on the CPU with the header's own confidence, loss,
// factorization and substitution functions, in the order als_solve_rows_kernel applies them -- so the CPU suite
// pins the device source to the reference's golden run.  (The kernel spreads the sums over threads; only the
// grouping of the float64 sums differs.)
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <vector>
#define __host__
#define __device__
#define __forceinline__ inline
#include "als_step.cuh"

namespace {

template <typename T>
int32_t side(T* X, const T* Z, int d, int64_t n_rows, int64_t n_z, const int64_t* rowptr, const int32_t* cols,
             const T* vals, double lambda, double alpha, double* loss) {
  std::vector<double> G((size_t)d * d, 0.0), A((size_t)d * d), b(d), s(d), x(d);
  for (int64_t r = 0; r < n_z; ++r)
    for (int a = 0; a < d; ++a)
      for (int c = 0; c < d; ++c) G[(size_t)a * d + c] += (double)Z[r * d + a] * (double)Z[r * d + c];
  int32_t failed = 0;
  for (int64_t r = 0; r < n_rows; ++r) {
    std::vector<double> S((size_t)d * d, 0.0);
    std::fill(b.begin(), b.end(), 0.0);
    for (int64_t k = rowptr[r]; k < rowptr[r + 1]; ++k) {
      const T* z = Z + (size_t)cols[k] * d;
      const double w = qrec::als_conf<T>(vals[k], alpha);
      if (loss != nullptr) {
        double xz = 0.0;
        for (int c = 0; c < d; ++c) xz += (double)X[r * d + c] * (double)z[c];
        *loss += qrec::als_loss_term(xz);
      }
      for (int a = 0; a < d; ++a) {
        b[a] += qrec::als_rhs_weight(w) * (double)z[a];
        for (int c = a; c < d; ++c) S[(size_t)a * d + c] += (w * (double)z[a]) * (double)z[c];
      }
    }
    for (int a = 0; a < d; ++a)
      for (int c = a; c < d; ++c)
        A[(size_t)a * d + c] = (G[(size_t)a * d + c] + S[(size_t)a * d + c]) + (a == c ? lambda : 0.0);
    if (!qrec::als_cholesky(A.data(), d, d, s.data())) {
      ++failed;                                    // the row keeps its old value
      continue;
    }
    x = b;
    qrec::als_solve(A.data(), d, d, s.data(), x.data());
    for (int c = 0; c < d; ++c) X[r * d + c] = (T)x[c];
  }
  return failed;
}

}  // namespace

extern "C" {

int32_t host_als_side_f64(double* X, const double* Z, int d, int64_t n_rows, int64_t n_z, const int64_t* rowptr,
                          const int32_t* cols, const double* vals, double lambda, double alpha, double* loss) {
  return side<double>(X, Z, d, n_rows, n_z, rowptr, cols, vals, lambda, alpha, loss);
}

int32_t host_als_side_f32(float* X, const float* Z, int d, int64_t n_rows, int64_t n_z, const int64_t* rowptr,
                          const int32_t* cols, const float* vals, double lambda, double alpha, double* loss) {
  return side<float>(X, Z, d, n_rows, n_z, rowptr, cols, vals, lambda, alpha, loss);
}

// The kernels' tile layout (als_step.cuh), for the CPU suite's shape tables.
int host_als_pad4(int d) { return qrec::pad4(d); }
int host_als_tiles_of(int d) { return qrec::tiles_of(d); }
int host_als_tiles_per_thread(int d) { return qrec::als_tiles_per_thread(d); }
int host_als_groups(int nt, int d) { return qrec::als_groups(nt, d); }
int host_als_threads() { return qrec::kThreads; }
int host_als_stage() { return qrec::kStage; }
int host_als_gram_chunk() { return qrec::kGramChunk; }
int host_als_max_d() { return qrec::kMaxD; }

}  // extern "C"
