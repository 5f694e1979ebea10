// Per-row arithmetic of the WRMF normal-equation solve (als_kernels.cu), kept apart so that the CPU suite can
// compile and run the very same source (tests/host_shims/als_step_host.cpp).
//
//   reference: model/ranking/WRMF.py:19-61
//     A = ZtZ + sum_k alpha*v_k * z_k z_k^T + lambda*I        b = sum_k (1 + alpha*v_k) * z_k
//     x = A^-1 b;   loss += (1 - x_old.z_k)^2 (user side)
//
// A and b are float64 whatever the table type T: with fp32 tables only the stored rows are rounded, so the large
// confidences of play-count data (alpha*v in the millions) do not break the factorization.
//
// A is factored in place as A = U^T U (U upper triangular, row-major, leading dimension ld; only the upper triangle
// is read or written).  The factorization runs column by column (right-looking); step j is split over nt workers,
// so one thread on the host and a whole CTA on the device run the same element updates in the same order.  The
// diagonal of U is kept as s[j] = 1 / U[j][j]; a pivot that is not positive and finite fails the row.
#pragma once
#include <math.h>

namespace qrec {

// Tile layout of the ALS-family row solves (als_kernels.cu), stated once for the kernels and for the CPU suite.
constexpr int kThreads = 256;      // threads per CTA
constexpr int kStage = 32;         // z rows staged in shared memory at a time
constexpr int kGramChunk = 2048;   // rows per partial Gram
constexpr int kMaxD = 128;

// Columns padded to whole 4x4 tiles, and the number of upper-triangle tiles of a d x d system.
__host__ __device__ inline int pad4(int d) { return (d + 3) & ~3; }
__host__ __device__ inline int tiles_of(int d) { const int nb = pad4(d) / 4; return nb * (nb + 1) / 2; }
// Tiles per thread NT of a d-wide system: 1 when the tiles fit one per thread, else 3 (d <= kMaxD).
__host__ __device__ inline int als_tiles_per_thread(int d) { return tiles_of(d) <= kThreads ? 1 : 3; }
// Groups the kStage staged rows are split over at NT tiles per thread: group g takes rows g, g + ngroups, ...
__host__ __device__ inline int als_groups(int nt, int d) {
  const int g = nt * kThreads / tiles_of(d);
  return g > kStage ? kStage : g;
}

// confidence term alpha * v of one entry (WRMF.py:34: 10 * r_ui), and its right-hand-side weight 1 + alpha * v
template <typename T>
__host__ __device__ __forceinline__ double als_conf(T v, double alpha) { return alpha * (double)v; }
__host__ __device__ __forceinline__ double als_rhs_weight(double conf) { return 1.0 + conf; }

// (1 - x.z)^2 with x the row before it is solved (WRMF.py:37-38; P_u[i] = 1 on the rated items)
__host__ __device__ __forceinline__ double als_loss_term(double xz) {
  const double e = 1.0 - xz;
  return e * e;
}

__host__ __device__ __forceinline__ bool als_pivot_ok(double p) { return p > 0.0 && p < INFINITY; }
__host__ __device__ __forceinline__ double als_pivot_scale(double p) { return 1.0 / sqrt(p); }

// Elimination step j (pivot scale s = 1/sqrt(A[j][j])): A[i][k] -= (A[j][i]*s) * (A[j][k]*s) for j < i <= k < d.
// Worker t of nt: rows i = j+1+g, j+1+g+G, ... and columns k = i+l, i+l+w, ... with w = min(nt, 32) lanes and
// G = nt / w row groups (on the device: one warp per row, lanes along it).
__host__ __device__ __forceinline__ void als_chol_step(double* A, int d, int ld, int j, double s, int t, int nt) {
  const int w = nt < 32 ? nt : 32;
  const int G = nt / w, g = t / w, l = t % w;
  if (g >= G) return;
  const double* rj = A + (size_t)j * ld;
  for (int i = j + 1 + g; i < d; i += G) {
    const double ui = rj[i] * s;
    double* ri = A + (size_t)i * ld;
    for (int k = i + l; k < d; k += w) ri[k] -= ui * (rj[k] * s);
  }
}

// After the last step: row j of U off the diagonal, U[j][i] = A[j][i] * s[j] (the values step j eliminated with).
__host__ __device__ __forceinline__ void als_chol_scale_rows(double* A, int d, int ld, const double* s, int t, int nt) {
  for (int e = t; e < d * d; e += nt) {
    const int j = e / d, i = e % d;
    if (i > j) A[(size_t)j * ld + i] *= s[j];
  }
}

// y -= u * x: the update of the substitutions below (column-oriented on both sides)
__host__ __device__ __forceinline__ double als_sub(double y, double u, double x) { return y - u * x; }

// Serial factorization (host): true on success; A then holds U above the diagonal and s the inverse diagonal.
__host__ __device__ inline bool als_cholesky(double* A, int d, int ld, double* s) {
  for (int j = 0; j < d; ++j) {
    const double p = A[(size_t)j * ld + j];
    if (!als_pivot_ok(p)) return false;
    s[j] = als_pivot_scale(p);
    als_chol_step(A, d, ld, j, s[j], 0, 1);
  }
  als_chol_scale_rows(A, d, ld, s, 0, 1);
  return true;
}

// U^T y = b, then U x = y; b is overwritten with x.  Forward: y_j = b_j * s_j, then b_i -= U[j][i] y_j (i > j).
// Back: x_i = y_i * s_i, then y_m -= U[m][i] x_i (m < i).
__host__ __device__ inline void als_solve(const double* U, int d, int ld, const double* s, double* b) {
  for (int j = 0; j < d; ++j) {
    b[j] *= s[j];
    for (int i = j + 1; i < d; ++i) b[i] = als_sub(b[i], U[(size_t)j * ld + i], b[j]);
  }
  for (int i = d - 1; i >= 0; --i) {
    b[i] *= s[i];
    for (int m = 0; m < i; ++m) b[m] = als_sub(b[m], U[(size_t)m * ld + i], b[i]);
  }
}

}  // namespace qrec
