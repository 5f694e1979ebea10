// WRMF (implicit-feedback ALS): the Gram matrix of a table and the per-row normal-equation solve.
//
//   reference: model/ranking/WRMF.py:19-61.  Within one half-epoch every row's solve reads only the other table Z:
//     G = Z^T Z;   for each row r with entries (c_k, v_k):
//       A = G + lambda*I + sum_k alpha*v_k z_k z_k^T,   b = sum_k (1 + alpha*v_k) z_k,   x_r = A^-1 b
//
//   * als_gram_partial_kernel / als_gram_sum_kernel -- G in two stages: every chunk of kGramChunk rows gets its own
//     partial Gram in the caller's workspace, then the partials are summed in chunk order.  Neither the chunking nor
//     any summation order depends on the grid, so G is bitwise the same on every run and every H100.
//   * als_solve_rows_kernel -- one CTA solves one row completely: it stages the row's z vectors into shared memory
//     kStage at a time, accumulates the upper triangle of A in float64 registers (4x4 tiles: each staged element
//     feeds four FMAs), factors A in shared memory (als_step.cuh) and substitutes with one warp.  The grid is
//     persistent and walks the caller's row order (longest rows first keeps one long row from becoming the tail).
//     Nothing depends on scheduling, so the solved tables are bitwise reproducible.
//
//   CoFactor (model/ranking/CoFactor.py): the user half-epoch is WRMF's; the item half-epoch adds the item-item SPPMI
//   co-factorisation (cofactor_step.cuh) and runs in item-id order, updating in place.
//   * cofactor_item_sweep_kernel -- one CTA per item, on the same staging, tiles and Cholesky as the row solve; the
//     in-order dataflow is kept with per-item stamps (see the kernel's comment).
//
//   ExpoMF (model/ranking/ExpoMF.py): every row's system weights EVERY row of the other table by an exposure
//   posterior that depends on the row (expomf_step.cuh), so there is no shared Gram.
//   * exposure_solve_rows_kernel<NT, ExpoPrior> -- one CTA solves one row completely: it streams the whole other
//     table through shared memory, weights each staged row by its posterior, lifts the row's observed entries to 1
//     with a sparse correction pass, and solves on the same tiles and Cholesky.  Fused into the item half, it also
//     sums the posteriors of the new row for the exposure prior.
//
//   SERec (model/ranking/SERec.py): ExpoMF with a prior per (user, item) pair that grows with the user's number of
//   followees (serec_step.cuh).  The reference's dense U x I prior has a closed form in one float64 sum per item and
//   one degree per user, evaluated per pair inside the solve.
//   * exposure_solve_rows_kernel<NT, SocialPrior> -- ExpoMF's row solve with the social prior policy; fused into the
//     item half, it writes each item's summed posterior for the next epoch's prior.
#include <type_traits>

#include "common.h"
#include "device.cuh"
#include "als_step.cuh"
#include "cofactor_step.cuh"
#include "expomf_step.cuh"
#include "serec_step.cuh"

namespace {

using namespace qrec;

constexpr int kThreads = 256;
constexpr int kStage = 32;         // z rows staged in shared memory at a time
constexpr int kGramChunk = 2048;   // rows per partial Gram
constexpr int kMaxD = 128;

__host__ __device__ inline int pad4(int d) { return (d + 3) & ~3; }
__host__ __device__ inline int tiles_of(int d) { const int nb = pad4(d) / 4; return nb * (nb + 1) / 2; }

// Shared-memory carve-up (doubles): A [d][ld] (ld = pad4(d)+1: odd, so column walks are conflict-free),
// Zs [kStage][dp], W [kStage], x_old [dp], b [dp], s [dp].
__host__ __device__ inline int a_words(int d) { return (d * (pad4(d) + 1) + 1) & ~1; }
inline size_t smem_bytes(int d) { return sizeof(double) * ((size_t)a_words(d) + (size_t)(kStage + 3) * pad4(d) + kStage); }

// The upper-triangle 4x4 tiles of A, split into work items (tile, group): group g accumulates the staged entries
// k = g, g + ngroups, ...  Small d has few tiles, so the entries are spread over several groups, reduced in group
// order.  Every tile has a group-0 item (NT * kThreads >= tiles).
template <int NT>
struct Tiles {
  double acc[NT][16];
  int a0[NT], b0[NT], grp[NT];
  int ngroups;

  __device__ void setup(int d) {
    const int nb = pad4(d) / 4, nt = tiles_of(d);
    ngroups = NT * kThreads / nt;
    if (ngroups > kStage) ngroups = kStage;
#pragma unroll
    for (int s = 0; s < NT; ++s) {
      const int id = threadIdx.x + s * kThreads;
      grp[s] = id < nt * ngroups ? id / nt : -1;
      int q = id % nt, I = 0;
      while (q >= nb - I) { q -= nb - I; ++I; }
      a0[s] = 4 * I;
      b0[s] = 4 * (I + q);
    }
  }

  __device__ void zero() {
#pragma unroll
    for (int s = 0; s < NT; ++s)
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[s][e] = 0.0;
  }

  // acc += sum over the staged entries of (W[k] z_k[a]) z_k[b]
  __device__ void accumulate(const double* Zs, const double* W, int dp, int cnt) {
#pragma unroll
    for (int s = 0; s < NT; ++s) {
      if (grp[s] < 0) continue;
      for (int k = grp[s]; k < cnt; k += ngroups) {
        const double w = W[k];
        const double* z = Zs + k * dp;
        const double2 x0 = *reinterpret_cast<const double2*>(z + a0[s]);
        const double2 x1 = *reinterpret_cast<const double2*>(z + a0[s] + 2);
        const double2 y0 = *reinterpret_cast<const double2*>(z + b0[s]);
        const double2 y1 = *reinterpret_cast<const double2*>(z + b0[s] + 2);
        const double za[4] = {w * x0.x, w * x0.y, w * x1.x, w * x1.y};
        const double zb[4] = {y0.x, y0.y, y1.x, y1.y};
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[s][p * 4 + q] = fma(za[p], zb[q], acc[s][p * 4 + q]);
      }
    }
  }

  // S = sum of the groups' tiles, upper triangle of A (ld); ends with a barrier
  __device__ void reduce_into(double* A, int d, int ld) {
    for (int g = 0; g < ngroups; ++g) {
#pragma unroll
      for (int s = 0; s < NT; ++s) {
        if (grp[s] != g) continue;
#pragma unroll
        for (int p = 0; p < 4; ++p)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int a = a0[s] + p, b = b0[s] + q;
            if (a <= b && b < d) A[a * ld + b] = g == 0 ? acc[s][p * 4 + q] : A[a * ld + b] + acc[s][p * 4 + q];
          }
      }
      __syncthreads();
    }
  }
};

// Stages rows row_of(k) of Z (k < cnt) as float64 with zero columns up to dp.  Each warp gathers its kStage/8 rows
// into registers first, so all of a thread's loads are in flight together, then stores them.  kCoherent: Z is written
// by other CTAs of the same launch, so its rows are read from L2 (__ldcg) instead of the read-only path.
template <typename T, bool kCoherent = false, class RowOf>
__device__ __forceinline__ void stage_rows(double* Zs, const T* __restrict__ Z, int d, int dp, int cnt, RowOf row_of) {
  constexpr int kWarps = kThreads / 32, R = kStage / kWarps, C = kMaxD / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double v[R][C];
#pragma unroll
  for (int m = 0; m < R; ++m) {
    const int k = warp + m * kWarps;
    const T* z = Z + (size_t)(k < cnt ? row_of(k) : 0) * d;
#pragma unroll
    for (int e = 0; e < C; ++e) {
      const int c = e * 32 + lane;
      v[m][e] = k < cnt && c < d ? (double)(kCoherent ? __ldcg(z + c) : __ldg(z + c)) : 0.0;
    }
  }
#pragma unroll
  for (int m = 0; m < R; ++m) {
    const int k = warp + m * kWarps;
#pragma unroll
    for (int e = 0; e < C; ++e)
      if (k < cnt && e * 32 + lane < dp) Zs[k * dp + e * 32 + lane] = v[m][e];
  }
}

// Factors the upper triangle of A (d x d, leading dimension ld) in place with the whole CTA (als_step.cuh) and solves
// A x = bv with warp 0, which stores x to out: the tail of the item sweep's and the exposure kernel's solves (WRMF's
// kernel writes the same steps out, see there).  Entered after a barrier that published A and bv.  Returns false on
// every thread when a pivot is not positive and finite; out is then untouched.
template <typename T>
__device__ __forceinline__ bool chol_solve(double* A, int d, int ld, double* sd, const double* bv, T* out) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int j = 0; j < d; ++j) {
    const double p = A[j * ld + j];
    if (!als_pivot_ok(p)) return false;                // uniform: every thread reads the same pivot
    const double s = als_pivot_scale(p);
    if (t == 0) sd[j] = s;
    als_chol_step(A, d, ld, j, s, t, kThreads);
    __syncthreads();
  }
  als_chol_scale_rows(A, d, ld, sd, t, kThreads);
  __syncthreads();
  if (warp == 0) {                                      // U^T y = b, U x = y (als_solve, one warp)
    double y[kMaxD / 32];
#pragma unroll
    for (int e = 0; e < kMaxD / 32; ++e) y[e] = e * 32 + lane < d ? bv[e * 32 + lane] : 0.0;
    for (int j = 0; j < d; ++j) {
      double v = 0.0;
#pragma unroll
      for (int e = 0; e < kMaxD / 32; ++e) if (e == (j >> 5)) v = y[e];
      const double yj = __shfl_sync(0xffffffffu, v, j & 31) * sd[j];
#pragma unroll
      for (int e = 0; e < kMaxD / 32; ++e) {
        const int i = e * 32 + lane;
        if (i == j) y[e] = yj;
        else if (i > j && i < d) y[e] = als_sub(y[e], A[j * ld + i], yj);
      }
    }
    for (int i = d - 1; i >= 0; --i) {
      double v = 0.0;
#pragma unroll
      for (int e = 0; e < kMaxD / 32; ++e) if (e == (i >> 5)) v = y[e];
      const double xi = __shfl_sync(0xffffffffu, v, i & 31) * sd[i];
#pragma unroll
      for (int e = 0; e < kMaxD / 32; ++e) {
        const int m = e * 32 + lane;
        if (m == i) y[e] = xi;
        else if (m < i) y[e] = als_sub(y[e], A[m * ld + i], xi);
      }
    }
#pragma unroll
    for (int e = 0; e < kMaxD / 32; ++e)
      if (e * 32 + lane < d) out[e * 32 + lane] = (T)y[e];
  }
  return true;
}

// The CTA's sum of v as held by lane 0 of each warp: the lanes 0 store it to part (kThreads / 32 doubles) and, after
// a barrier, thread 0 adds them from 0.0 in warp order, so the sum does not depend on scheduling.  Called by every
// thread; returns the sum on thread 0 (0.0 elsewhere).  part must not be written again before the next barrier.
__device__ __forceinline__ double cta_sum(double v, double* part) {
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s += part[w];
  return s;
}

// ------------------------------------------------------------------------------------------
// Gram
// ------------------------------------------------------------------------------------------
template <typename T, int NT>
__global__ void __launch_bounds__(kThreads)
als_gram_partial_kernel(const T* __restrict__ Z, long long n, int d, double* __restrict__ parts) {
  extern __shared__ __align__(16) double smem[];
  const int dp = pad4(d), ld = dp + 1;
  double* A = smem;
  double* Zs = A + a_words(d);
  double* W = Zs + kStage * dp;
  for (int k = threadIdx.x; k < kStage; k += kThreads) W[k] = 1.0;
  Tiles<NT> tl;
  tl.setup(d);
  const long long nchunks = (n + kGramChunk - 1) / kGramChunk;
  for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
    tl.zero();
    const long long r0 = c * kGramChunk;
    const long long r1 = r0 + kGramChunk < n ? r0 + kGramChunk : n;
    for (long long k0 = r0; k0 < r1; k0 += kStage) {
      const int cnt = (int)(r1 - k0 < kStage ? r1 - k0 : kStage);
      __syncthreads();
      stage_rows<T>(Zs, Z, d, dp, cnt, [=](int k) { return k0 + k; });
      __syncthreads();
      tl.accumulate(Zs, W, dp, cnt);
    }
    __syncthreads();
    tl.reduce_into(A, d, ld);
    double* out = parts + (size_t)c * d * d;
    for (int e = threadIdx.x; e < d * d; e += kThreads) {
      const int a = e / d, b = e % d;
      out[e] = a <= b ? A[a * ld + b] : A[b * ld + a];     // mirrored: G is exactly symmetric
    }
  }
}

__global__ void __launch_bounds__(kThreads)
als_gram_sum_kernel(const double* __restrict__ parts, long long nchunks, int dd, double* __restrict__ G) {
  const int e = blockIdx.x * kThreads + threadIdx.x;
  if (e >= dd) return;
  double g = 0.0;
  for (long long c = 0; c < nchunks; ++c) g += parts[(size_t)c * dd + e];
  G[e] = g;
}

// ------------------------------------------------------------------------------------------
// row solve
// ------------------------------------------------------------------------------------------
template <typename T, int NT>
__global__ void __launch_bounds__(kThreads, NT == 1 ? 3 : 1)
als_solve_rows_kernel(T* __restrict__ X, const T* __restrict__ Z, const double* __restrict__ G, int d,
                      long long n_order, const int* __restrict__ order, const long long* __restrict__ rowptr,
                      const int* __restrict__ cols, const T* __restrict__ vals, double lambda, double alpha,
                      double* loss, int* n_failed) {
  extern __shared__ __align__(16) double smem[];
  const int dp = pad4(d), ld = dp + 1;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double* A = smem;
  double* Zs = A + a_words(d);
  double* W = Zs + kStage * dp;
  double* xo = W + kStage;
  double* bv = xo + dp;
  double* sd = bv + dp;
  Tiles<NT> tl;
  tl.setup(d);
  double lsum = 0.0;
  for (long long q = blockIdx.x; q < n_order; q += gridDim.x) {
    const int r = __ldg(order + q);
    const long long beg = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    T* x = X + (size_t)r * d;
    tl.zero();
    double bacc = 0.0;
    __syncthreads();                                   // the previous row's solve is done with the buffers
    if (loss != nullptr)
      for (int c = t; c < dp; c += kThreads) xo[c] = c < d ? (double)x[c] : 0.0;
    for (long long k0 = beg; k0 < end; k0 += kStage) {
      const int cnt = (int)(end - k0 < kStage ? end - k0 : kStage);
      __syncthreads();
      stage_rows<T>(Zs, Z, d, dp, cnt, [=](int k) { return __ldg(cols + k0 + k); });
      for (int k = t; k < cnt; k += kThreads) W[k] = als_conf<T>(__ldg(vals + k0 + k), alpha);
      __syncthreads();
      tl.accumulate(Zs, W, dp, cnt);
      if (t < d)
        for (int k = 0; k < cnt; ++k) bacc = fma(als_rhs_weight(W[k]), Zs[k * dp + t], bacc);
      if (loss != nullptr) {
        for (int k = warp; k < cnt; k += kThreads / 32) {
          double xz = 0.0;
          for (int c = lane; c < d; c += 32) xz = fma(xo[c], Zs[k * dp + c], xz);
          xz = warp_sum(xz);
          if (lane == 0) lsum += als_loss_term(xz);
        }
      }
    }
    __syncthreads();
    tl.reduce_into(A, d, ld);
    // A = (G + S) + lambda*I  (WRMF.py:41: YtY + Y^T C_u Y + regU * eye)
    for (int e = t; e < d * d; e += kThreads) {
      const int a = e / d, b = e % d;
      if (a <= b) A[a * ld + b] = (__ldg(G + e) + A[a * ld + b]) + (a == b ? lambda : 0.0);
    }
    if (t < d) bv[t] = bacc;
    __syncthreads();
    // chol_solve's steps written out: called here, the NT = 1 kernels spill more and solve ~1% slower on an H100
    bool ok = true;
    for (int j = 0; j < d; ++j) {
      const double p = A[j * ld + j];
      if (!als_pivot_ok(p)) { ok = false; break; }      // uniform: every thread reads the same pivot
      const double s = als_pivot_scale(p);
      if (t == 0) sd[j] = s;
      als_chol_step(A, d, ld, j, s, t, kThreads);
      __syncthreads();
    }
    if (!ok) {                                          // the row keeps its old value
      if (t == 0 && n_failed != nullptr) atomicAdd(n_failed, 1);
      continue;
    }
    als_chol_scale_rows(A, d, ld, sd, t, kThreads);
    __syncthreads();
    if (warp == 0) {                                    // U^T y = b, U x = y (als_solve, one warp)
      double y[kMaxD / 32];
#pragma unroll
      for (int e = 0; e < kMaxD / 32; ++e) y[e] = e * 32 + lane < d ? bv[e * 32 + lane] : 0.0;
      for (int j = 0; j < d; ++j) {
        double v = 0.0;
#pragma unroll
        for (int e = 0; e < kMaxD / 32; ++e) if (e == (j >> 5)) v = y[e];
        const double yj = __shfl_sync(0xffffffffu, v, j & 31) * sd[j];
#pragma unroll
        for (int e = 0; e < kMaxD / 32; ++e) {
          const int i = e * 32 + lane;
          if (i == j) y[e] = yj;
          else if (i > j && i < d) y[e] = als_sub(y[e], A[j * ld + i], yj);
        }
      }
      for (int i = d - 1; i >= 0; --i) {
        double v = 0.0;
#pragma unroll
        for (int e = 0; e < kMaxD / 32; ++e) if (e == (i >> 5)) v = y[e];
        const double xi = __shfl_sync(0xffffffffu, v, i & 31) * sd[i];
#pragma unroll
        for (int e = 0; e < kMaxD / 32; ++e) {
          const int m = e * 32 + lane;
          if (m == i) y[e] = xi;
          else if (m < i) y[e] = als_sub(y[e], A[m * ld + i], xi);
        }
      }
#pragma unroll
      for (int e = 0; e < kMaxD / 32; ++e)
        if (e * 32 + lane < d) x[e * 32 + lane] = (T)y[e];
    }
  }
  if (loss != nullptr) {
    __shared__ double part[kThreads / 32];
    const double s = cta_sum(lsum, part);
    if (t == 0 && s != 0.0) atomicAdd(loss, s);
  }
}

// ------------------------------------------------------------------------------------------
// CoFactor item sweep
// ------------------------------------------------------------------------------------------
// Shared-memory carve-up (doubles): A, Zs [kStage][dp], W / M / O [kStage] (tile weight, SPPMI value, the context's
// c or w), y_old, g_old, b, s [dp].
inline size_t cof_smem_bytes(int d) {
  return sizeof(double) * ((size_t)a_words(d) + (size_t)(kStage + 4) * pad4(d) + 3 * kStage);
}

// One in-order item sweep (CoFactor.py, trainModel, item loop; arithmetic in cofactor_step.cuh).  For item i:
//   A_Y = XtX + sum_u alpha*r x x^T + lambda*I + sum_c G_c G_c^T  -> Y_i      (X rows weight alpha*r, G rows weight 1)
//   A_G = sum_c Y_c Y_c^T + gamma*I                               -> G_i, then w_i, c_i   (items with contexts only)
// A and b are float64; a system that is not positive definite leaves its row unchanged and is counted in n_failed.
//
// Order.  The reference updates in place in item-id order, so a context c < i is read after its own update in this
// sweep and c > i before it.  The sweep runs on the in-order protocol of device.cuh with one CTA per item: CTAs take
// items from `ticket` in id order.  Before reading its contexts a CTA waits (acquire) until the stamp of every
// context c < i equals `sweep`; after writing Y_i, G_i, w_i, c_i it publishes its own stamp (release add).  The SPPMI
// is symmetric, so a context c > i has i among its own contexts and waits for i's stamp before it reads anything of
// i or writes its own rows: i reads c's values from before the sweep.
// No deadlock: a CTA takes a ticket only while it runs and holds one at a time, and it waits only on smaller tickets,
// which running CTAs hold; the CTA with the smallest unfinished ticket waits on nobody, so it always finishes.  Every
// CTA of the persistent grid is resident at once (persistent_grid sizes it by occupancy), so no waiting CTA keeps
// another from being scheduled.  Rows other CTAs write (Y, G, w, c) are read through L2.  The schedule only changes
// when a value is computed, never from what, so the result is bitwise the same on every run.
template <typename T, int NT>
__global__ void __launch_bounds__(kThreads, NT == 1 ? 2 : 1)
cofactor_item_sweep_kernel(T* Y, T* G, T* wb, T* cb, const T* __restrict__ X, const double* __restrict__ XtX, int d,
                           int n_items, const long long* __restrict__ irp, const int* __restrict__ icol,
                           const T* __restrict__ ival, const long long* __restrict__ srp, const int* __restrict__ scol,
                           const T* __restrict__ sval, double lambda, double gamma, double alpha, int* stamps,
                           int sweep, unsigned long long* ticket, int* n_failed) {
  extern __shared__ __align__(16) double smem[];
  __shared__ long long s_item;
  __shared__ double part[2][kThreads / 32];
  const int dp = pad4(d), ld = dp + 1;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  double* A = smem;
  double* Zs = A + a_words(d);
  double* W = Zs + kStage * dp;
  double* M = W + kStage;
  double* O = M + kStage;
  double* yo = O + kStage;
  double* go = yo + dp;
  double* bv = go + dp;
  double* sd = bv + dp;
  Tiles<NT> tl;
  tl.setup(d);
  while (true) {
    __syncthreads();                                   // the previous item is done with the buffers and s_item
    if (t == 0) s_item = (long long)atomicAdd(ticket, 1ULL);
    __syncthreads();
    if (s_item >= n_items) break;
    const int i = (int)s_item;
    const long long ub = __ldg(irp + i), ue = __ldg(irp + i + 1), cbeg = __ldg(srp + i), cend = __ldg(srp + i + 1);
    const int nctx = (int)(cend - cbeg);
    T* yi = Y + (size_t)i * d;
    T* gi = G + (size_t)i * d;
    const double w_i = (double)__ldcg(wb + i), c_i = (double)__ldcg(cb + i);
    for (int c = t; c < dp; c += kThreads) {
      yo[c] = c < d ? (double)__ldcg(yi + c) : 0.0;
      go[c] = c < d ? (double)__ldcg(gi + c) : 0.0;
    }
    // users: X rows with weight alpha*r (X is not written in this sweep; nothing to wait for)
    tl.zero();
    double bx = 0.0;
    for (long long k0 = ub; k0 < ue; k0 += kStage) {
      const int cnt = (int)(ue - k0 < kStage ? ue - k0 : kStage);
      __syncthreads();
      stage_rows<T>(Zs, X, d, dp, cnt, [=](int k) { return __ldg(icol + k0 + k); });
      for (int k = t; k < cnt; k += kThreads) W[k] = als_conf<T>(__ldg(ival + k0 + k), alpha);
      __syncthreads();
      tl.accumulate(Zs, W, dp, cnt);
      if (t < d)
        for (int k = 0; k < cnt; ++k) bx = fma(als_rhs_weight(W[k]), Zs[k * dp + t], bx);
    }
    for (long long k = cbeg + t; k < cend; k += kThreads) {
      const int c = __ldg(scol + k);
      if (c < i) spin_until<32, 256>([=] { return ld_acquire_gpu(stamps + c) == sweep; });
    }
    __syncthreads();
    // contexts, first pass: G rows with weight 1 into A_Y and b_Y, and w_i's sum
    double bg = 0.0, wsum = 0.0;
    for (long long k0 = cbeg; k0 < cend; k0 += kStage) {
      const int cnt = (int)(cend - k0 < kStage ? cend - k0 : kStage);
      __syncthreads();
      stage_rows<T, true>(Zs, G, d, dp, cnt, [=](int k) { return __ldg(scol + k0 + k); });
      for (int k = t; k < cnt; k += kThreads) {
        W[k] = 1.0;
        M[k] = (double)__ldg(sval + k0 + k);
        O[k] = (double)__ldcg(cb + __ldg(scol + k0 + k));
      }
      __syncthreads();
      tl.accumulate(Zs, W, dp, cnt);
      if (t < d)
        for (int k = 0; k < cnt; ++k) bg = fma(cof_rhs_y_coef(M[k], w_i, O[k]), Zs[k * dp + t], bg);
      for (int k = warp; k < cnt; k += kThreads / 32) {
        double yg = 0.0;
        for (int c = lane; c < d; c += 32) yg = fma(yo[c], Zs[k * dp + c], yg);
        yg = warp_sum(yg);
        if (lane == 0) wsum += cof_w_term(M[k], yg, O[k]);
      }
    }
    __syncthreads();
    tl.reduce_into(A, d, ld);
    for (int e = t; e < d * d; e += kThreads) {
      const int a = e / d, b = e % d;
      if (a <= b) A[a * ld + b] = (__ldg(XtX + e) + A[a * ld + b]) + (a == b ? lambda : 0.0);
    }
    if (t < d) bv[t] = bx + bg;
    __syncthreads();
    if (!chol_solve<T>(A, d, ld, sd, bv, yi) && t == 0 && n_failed != nullptr) atomicAdd(n_failed, 1);
    if (nctx > 0) {
      // contexts, second pass: Y rows into A_G and b_G, and c_i's sum
      tl.zero();
      double by = 0.0, csum = 0.0;
      for (long long k0 = cbeg; k0 < cend; k0 += kStage) {
        const int cnt = (int)(cend - k0 < kStage ? cend - k0 : kStage);
        __syncthreads();
        stage_rows<T, true>(Zs, Y, d, dp, cnt, [=](int k) { return __ldg(scol + k0 + k); });
        for (int k = t; k < cnt; k += kThreads) {
          W[k] = 1.0;
          M[k] = (double)__ldg(sval + k0 + k);
          O[k] = (double)__ldcg(wb + __ldg(scol + k0 + k));
        }
        __syncthreads();
        tl.accumulate(Zs, W, dp, cnt);
        if (t < d)
          for (int k = 0; k < cnt; ++k) by = fma(cof_rhs_g_coef(M[k], O[k], c_i), Zs[k * dp + t], by);
        for (int k = warp; k < cnt; k += kThreads / 32) {
          double yg = 0.0;
          for (int c = lane; c < d; c += 32) yg = fma(go[c], Zs[k * dp + c], yg);
          yg = warp_sum(yg);
          if (lane == 0) csum += cof_c_term(M[k], yg, O[k]);
        }
      }
      __syncthreads();
      tl.reduce_into(A, d, ld);
      for (int a = t; a < d; a += kThreads) A[a * ld + a] += gamma;
      if (t < d) bv[t] = by;
      const double sw = cta_sum(wsum, part[0]);         // its barrier also publishes A and bv
      const double sc = cta_sum(csum, part[1]);
      if (!chol_solve<T>(A, d, ld, sd, bv, gi) && t == 0 && n_failed != nullptr) atomicAdd(n_failed, 1);
      if (t == 0) {
        wb[i] = (T)cof_mean(sw, nctx);
        cb[i] = (T)cof_mean(sc, nctx);
      }
    }
    __threadfence();
    __syncthreads();
    if (t == 0) red_release_gpu_add(stamps + i, 1);
  }
}

// ------------------------------------------------------------------------------------------
// ExpoMF row solve
// ------------------------------------------------------------------------------------------
// Posteriors of the staged rows Zs[0..cnt) against x (shared, dp columns): one warp per staged row, the dot in float64
// with the lanes along the row.  Each weight is expomf_exposure(s, mu_of(k)), or its lift 1 - A when kLift; it goes to
// W[k] when W is given.  Returns the sum of the weights of the warp's rows on lane 0 (in k order).
template <bool kLift, class MuOf>
__device__ __forceinline__ double expomf_weights(const double* Zs, const double* x, double* W, int d, int dp, int cnt,
                                                 double lam_y, MuOf mu_of) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double sum = 0.0;
  for (int k = warp; k < cnt; k += kThreads / 32) {
    double s = 0.0;
    for (int c = lane; c < d; c += 32) s = fma(x[c], Zs[k * dp + c], s);
    s = warp_sum(s);
    const double A = expomf_exposure(s, mu_of(k), lam_y);
    const double w = kLift ? expomf_lift(A) : A;
    if (lane == 0) {
      if (W != nullptr) W[k] = w;
      sum += w;
    }
  }
  return sum;
}

// Prior policies of exposure_solve_rows_kernel (below).  A policy says what prior each (row r, column k) pair of the solve
// uses, what prior the fused pass after the solve uses, and what that pass writes.  row(r) loads the row's own
// state once; solve(p, k) and out(p, k) take the column as a functor, so that a policy that does not need it does not
// load it.
//
// ExpoMF: one float32 prior per item, indexed by the row (by_row) or by the column.  The fused pass uses mu[r] and
// writes the item's new prior to mu_out.
struct ExpoPrior {
  const float* __restrict__ mu;
  int by_row;
  float* __restrict__ mu_out;
  double a, b;
  long long n_z;
  __device__ __forceinline__ bool has_out() const { return mu_out != nullptr; }
  __device__ __forceinline__ double row(int r) const { return by_row || mu_out != nullptr ? (double)__ldg(mu + r) : 0.0; }
  template <class Col>
  __device__ __forceinline__ double solve(double mu_r, Col col) const { return by_row ? mu_r : (double)__ldg(mu + col()); }
  template <class Col>
  __device__ __forceinline__ double out(double mu_r, Col) const { return mu_r; }
  __device__ __forceinline__ void write(int r, double asum) const { mu_out[r] = (float)expomf_prior(asum, a, b, n_z); }
};

// SERec: the prior of the pair (user u, item i) is serec_prior(A[i], deg[u]) (serec_step.cuh), or the uniform mu0
// when A is null (the first epoch).  row_is_user says which of r and k is the user: the user half has user rows, the
// item half item rows -- except when there are as many users as items, where the reference's item half takes the user
// branch (SERec.py, _solve_batch: mu.shape[1] == X.shape[0]) and so reads mu[i, u].  The fused pass after the solve
// always reads mu[u, i] with the item as the row (SERec.py: _update_expo) and writes the item's summed posterior
// A itself to asum_out; the next epoch evaluates the prior from it.  The social term deg_u * A_i is one float64
// product, where the reference's T.dot adds A_i to itself deg_u times: the two differ by a few ulps once deg_u >= 7
// (about 1e-15 of the prior), far below the float32 rows the prior feeds.
struct SocialPrior {
  const double* __restrict__ A;
  double mu0;
  const int* __restrict__ deg;
  int row_is_user;
  double* __restrict__ asum_out;
  double a, b, s, n_users;
  struct Row {
    double A;                                // A[r]: the row is the item of its pairs
    int deg;                                 // deg[r]: the row is the user of its pairs
  };
  __device__ __forceinline__ bool has_out() const { return asum_out != nullptr; }
  __device__ __forceinline__ Row row(int r) const {
    Row p{0.0, 0};
    if (A != nullptr) {
      if (row_is_user) p.deg = __ldg(deg + r);
      if (!row_is_user || asum_out != nullptr) p.A = __ldg(A + r);
    }
    return p;
  }
  template <class Col>
  __device__ __forceinline__ double solve(const Row& p, Col col) const {
    if (A == nullptr) return mu0;
    const int k = col();
    return row_is_user ? serec_prior(__ldg(A + k), p.deg, a, b, s, n_users)
                       : serec_prior(p.A, __ldg(deg + k), a, b, s, n_users);
  }
  template <class Col>
  __device__ __forceinline__ double out(const Row& p, Col col) const {
    return A == nullptr ? mu0 : serec_prior(p.A, __ldg(deg + col()), a, b, s, n_users);
  }
  __device__ __forceinline__ void write(int r, double asum) const { asum_out[r] = asum; }
};

// One exposure-weighted half-epoch (ExpoMF.py / SERec.py: recompute_factors / _solve, arithmetic in expomf_step.cuh
// and serec_step.cuh).  For row r of X with observed columns Y_r (CSR) against all n_z rows of Z:
//   B = sum_k A_k z_k z_k^T + lambda*I,   A_k = posterior of (x_old.z_k, mu_rk), 1 on Y_r;   x_r = B^-1 sum_{k in Y_r} z_k
// with the prior mu_rk from the policy P.  The dense pass weights every staged row of Z by its posterior; the
// correction pass adds (1 - A) z z^T over Y_r, so the columns need not be sorted.  Every CTA reads only its own old
// row, so X is written in place.  A system that is not positive definite leaves its row unchanged and is counted in
// n_failed.  Fused pass (item half, P::has_out): after the solve the CTA streams Z once more and sums
//   sum_k A_k  with A_k from (x_new.z_k, the policy's out prior), 1 on Y_r   (_update_expo)
// which P::write stores -- never into the prior being read, which other CTAs may still read.  Nothing depends on the
// grid, so X and the fused output are bitwise reproducible.
template <int NT, class P>
__global__ void __launch_bounds__(kThreads, NT == 1 ? 3 : 1)
exposure_solve_rows_kernel(float* X, const float* __restrict__ Z, int d, long long n_z, long long n_order,
                           const int* __restrict__ order, const long long* __restrict__ rowptr,
                           const int* __restrict__ cols, P prior, double lambda, double lam_y, int* n_failed) {
  extern __shared__ __align__(16) double smem[];
  __shared__ double part[kThreads / 32];
  const int dp = pad4(d), ld = dp + 1;
  const int t = threadIdx.x;
  double* A = smem;
  double* Zs = A + a_words(d);
  double* W = Zs + kStage * dp;
  double* xo = W + kStage;
  double* bv = xo + dp;
  double* sd = bv + dp;
  Tiles<NT> tl;
  tl.setup(d);
  for (long long q = blockIdx.x; q < n_order; q += gridDim.x) {
    const int r = __ldg(order + q);
    const long long beg = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    float* x = X + (size_t)r * d;
    const auto pr = prior.row(r);
    tl.zero();
    double bacc = 0.0;
    __syncthreads();                                   // the previous row is done with the buffers
    for (int c = t; c < dp; c += kThreads) xo[c] = c < d ? (double)x[c] : 0.0;
    // every row of Z, weighted by its posterior
    for (long long k0 = 0; k0 < n_z; k0 += kStage) {
      const int cnt = (int)(n_z - k0 < kStage ? n_z - k0 : kStage);
      __syncthreads();
      stage_rows<float>(Zs, Z, d, dp, cnt, [=](int k) { return k0 + k; });
      __syncthreads();
      expomf_weights<false>(Zs, xo, W, d, dp, cnt, lam_y,
                            [=](int k) { return prior.solve(pr, [=] { return k0 + k; }); });
      __syncthreads();
      tl.accumulate(Zs, W, dp, cnt);
    }
    // the observed entries: lifted to A = 1, and the right-hand side
    for (long long k0 = beg; k0 < end; k0 += kStage) {
      const int cnt = (int)(end - k0 < kStage ? end - k0 : kStage);
      __syncthreads();
      stage_rows<float>(Zs, Z, d, dp, cnt, [=](int k) { return __ldg(cols + k0 + k); });
      __syncthreads();
      expomf_weights<true>(Zs, xo, W, d, dp, cnt, lam_y,
                           [=](int k) { return prior.solve(pr, [=] { return __ldg(cols + k0 + k); }); });
      __syncthreads();
      tl.accumulate(Zs, W, dp, cnt);
      if (t < d)
        for (int k = 0; k < cnt; ++k) bacc += Zs[k * dp + t];
    }
    __syncthreads();
    tl.reduce_into(A, d, ld);
    for (int j = t; j < d; j += kThreads) A[j * ld + j] += lambda;     // ExpoMF.py: + lam * np.eye(f)
    if (t < d) bv[t] = bacc;
    __syncthreads();
    if (!chol_solve<float>(A, d, ld, sd, bv, x) && t == 0 && n_failed != nullptr) atomicAdd(n_failed, 1);
    if (!prior.has_out()) continue;
    // the summed posteriors of this row with its new value (the old one if the solve failed)
    __syncthreads();                                   // warp 0's store of x is visible to the CTA
    for (int c = t; c < dp; c += kThreads) xo[c] = c < d ? (double)x[c] : 0.0;
    double asum = 0.0;
    for (long long k0 = 0; k0 < n_z; k0 += kStage) {
      const int cnt = (int)(n_z - k0 < kStage ? n_z - k0 : kStage);
      __syncthreads();
      stage_rows<float>(Zs, Z, d, dp, cnt, [=](int k) { return k0 + k; });
      __syncthreads();
      asum += expomf_weights<false>(Zs, xo, nullptr, d, dp, cnt, lam_y,
                                    [=](int k) { return prior.out(pr, [=] { return k0 + k; }); });
    }
    for (long long k0 = beg; k0 < end; k0 += kStage) {
      const int cnt = (int)(end - k0 < kStage ? end - k0 : kStage);
      __syncthreads();
      stage_rows<float>(Zs, Z, d, dp, cnt, [=](int k) { return __ldg(cols + k0 + k); });
      __syncthreads();
      asum += expomf_weights<true>(Zs, xo, nullptr, d, dp, cnt, lam_y,
                                   [=](int k) { return prior.out(pr, [=] { return __ldg(cols + k0 + k); }); });
    }
    const double s = cta_sum(asum, part);
    if (t == 0) prior.write(r, s);
  }
}

// persistent grid: as many CTAs as fit on the GPU at `bytes` of dynamic shared memory, at most `work`, and at most
// max_ctas when it is > 0.  Never more than fit at once: the CoFactor sweep needs every CTA of its grid resident.
template <class K>
int persistent_grid(K kernel, size_t bytes, long long work, int max_ctas, int* grid) {
  QREC_CUDA(allow_dynamic_smem((const void*)kernel, (int)bytes));
  int per_sm = 0;
  QREC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, bytes));
  *grid = capped_grid(work, per_sm > 0 ? per_sm : 1);
  if (max_ctas > 0 && *grid > max_ctas) *grid = max_ctas;
  return QREC_OK;
}

// Launches kernel_of(std::integral_constant<int, NT>{})(args...) on its persistent grid, with the tile count NT of a
// d-wide system: 1 when the upper triangle's 4x4 tiles fit one per thread, else 3 (d <= kMaxD).
template <class KernelOf, class... Args>
int launch_rows(KernelOf kernel_of, int d, size_t bytes, long long work, int max_ctas, cudaStream_t st,
                Args... args) {
  const auto kernel = tiles_of(d) <= kThreads ? kernel_of(std::integral_constant<int, 1>{})
                                              : kernel_of(std::integral_constant<int, 3>{});
  int grid = 0;
  const int rc = persistent_grid(kernel, bytes, work, max_ctas, &grid);
  if (rc) return rc;
  kernel<<<grid, kThreads, bytes, st>>>(args...);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

long long gram_chunks(long long n) { return (n + kGramChunk - 1) / kGramChunk; }

template <typename T>
int launch_gram(const T* Z, long long n, int d, double* G, void* ws, long long ws_bytes, cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= kMaxD, "als_gram: d=%d unsupported (1..%d)", d, kMaxD);
  QREC_REQUIRE(n >= 0, "als_gram: n < 0");
  QREC_REQUIRE(G != nullptr, "als_gram: null G");
  const long long nchunks = gram_chunks(n);
  QREC_REQUIRE(nchunks == 0 || (Z != nullptr && ws != nullptr), "als_gram: null pointer");
  QREC_REQUIRE(ws_bytes >= nchunks * d * d * (long long)sizeof(double),
               "als_gram: workspace of %lld bytes, %lld needed (qrec_als_gram_workspace_bytes)", ws_bytes,
               nchunks * d * d * (long long)sizeof(double));
  double* parts = (double*)ws;
  if (nchunks > 0) {
    const int rc = launch_rows([](auto nt) { return als_gram_partial_kernel<T, decltype(nt)::value>; }, d,
                               smem_bytes(d), nchunks, 0, st, Z, n, d, parts);
    if (rc) return rc;
  }
  als_gram_sum_kernel<<<(d * d + kThreads - 1) / kThreads, kThreads, 0, st>>>(parts, nchunks, d * d, G);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

template <typename T>
int launch_solve(T* X, const T* Z, const double* G, int d, long long n_order, const int* order,
                 const long long* rowptr, const int* cols, const T* vals, double lambda, double alpha, double* loss,
                 int* n_failed, cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= kMaxD, "als_solve_rows: d=%d unsupported (1..%d)", d, kMaxD);
  QREC_REQUIRE(n_order >= 0, "als_solve_rows: n_rows < 0");
  if (n_order == 0) return QREC_OK;
  QREC_REQUIRE(X && Z && G && order && rowptr, "als_solve_rows: null pointer");
  QREC_REQUIRE((const void*)X != (const void*)Z, "als_solve_rows: X and Z must be different tables");
  return launch_rows([](auto nt) { return als_solve_rows_kernel<T, decltype(nt)::value>; }, d, smem_bytes(d),
                     n_order, 0, st, X, Z, G, d, n_order, order, rowptr, cols, vals, lambda, alpha, loss, n_failed);
}

template <typename T>
int launch_cofactor(T* Y, T* G, T* w, T* c, const T* X, const double* XtX, int d, int n_items, const long long* irp,
                    const int* icol, const T* ival, const long long* srp, const int* scol, const T* sval, double lambda,
                    double gamma, double alpha, int* stamps, int sweep, unsigned long long* ticket, int* n_failed,
                    cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= kMaxD, "cofactor_item_sweep: d=%d unsupported (1..%d)", d, kMaxD);
  QREC_REQUIRE(n_items >= 0, "cofactor_item_sweep: n_items < 0");
  if (n_items == 0) return QREC_OK;
  QREC_REQUIRE(Y && G && w && c && X && XtX && irp && srp && stamps && ticket, "cofactor_item_sweep: null pointer");
  QREC_REQUIRE((const void*)Y != (const void*)G && (const void*)Y != (const void*)X && (const void*)G != (const void*)X,
               "cofactor_item_sweep: Y, G and X must be different tables");
  QREC_REQUIRE(sweep >= 1, "cofactor_item_sweep: sweep=%d (stamps count sweeps from 1)", sweep);
  return launch_rows([](auto nt) { return cofactor_item_sweep_kernel<T, decltype(nt)::value>; }, d,
                     cof_smem_bytes(d), n_items, 0, st, Y, G, w, c, X, XtX, d, n_items, irp, icol, ival, srp, scol,
                     sval, lambda, gamma, alpha, stamps, sweep, ticket, n_failed);
}

int launch_expomf(float* X, const float* Z, int d, long long n_z, long long n_order, const int* order,
                  const long long* rowptr, const int* cols, const float* mu, int mu_by_row, float* mu_out,
                  double lambda, double lam_y, double a, double b, int max_ctas, int* n_failed, cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= kMaxD, "expomf_solve_rows: d=%d unsupported (1..%d)", d, kMaxD);
  QREC_REQUIRE(n_order >= 0 && n_z >= 0, "expomf_solve_rows: n_rows=%lld n_z=%lld", n_order, n_z);
  QREC_REQUIRE(max_ctas >= 0, "expomf_solve_rows: max_ctas=%d < 0", max_ctas);
  if (n_order == 0) return QREC_OK;
  QREC_REQUIRE(X && Z && order && rowptr && mu, "expomf_solve_rows: null pointer");
  QREC_REQUIRE((const void*)X != (const void*)Z, "expomf_solve_rows: X and Z must be different tables");
  QREC_REQUIRE((const void*)mu_out != (const void*)mu, "expomf_solve_rows: mu_out must not be mu");
  const ExpoPrior prior{mu, mu_by_row, mu_out, a, b, n_z};
  return launch_rows([](auto nt) { return exposure_solve_rows_kernel<decltype(nt)::value, ExpoPrior>; }, d,
                     smem_bytes(d), n_order, max_ctas, st, X, Z, d, n_z, n_order, order, rowptr, cols, prior, lambda,
                     lam_y, n_failed);
}

int launch_serec(float* X, const float* Z, int d, long long n_z, long long n_order, const int* order,
                 const long long* rowptr, const int* cols, const double* asum, float mu0, const int* deg,
                 int row_is_user, double* asum_out, double lambda, double lam_y, double a, double b, double s,
                 long long n_users, int max_ctas, int* n_failed, cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= kMaxD, "serec_solve_rows: d=%d unsupported (1..%d)", d, kMaxD);
  QREC_REQUIRE(n_order >= 0 && n_z >= 0, "serec_solve_rows: n_rows=%lld n_z=%lld", n_order, n_z);
  QREC_REQUIRE(max_ctas >= 0, "serec_solve_rows: max_ctas=%d < 0", max_ctas);
  if (n_order == 0) return QREC_OK;
  QREC_REQUIRE(X && Z && order && rowptr && deg, "serec_solve_rows: null pointer");
  QREC_REQUIRE((const void*)X != (const void*)Z, "serec_solve_rows: X and Z must be different tables");
  QREC_REQUIRE(asum_out == nullptr || (const void*)asum_out != (const void*)asum,
               "serec_solve_rows: asum_out must not be asum");
  const SocialPrior prior{asum, (double)mu0, deg, row_is_user, asum_out, a, b, s, (double)n_users};
  return launch_rows([](auto nt) { return exposure_solve_rows_kernel<decltype(nt)::value, SocialPrior>; }, d,
                     smem_bytes(d), n_order, max_ctas, st, X, Z, d, n_z, n_order, order, rowptr, cols, prior, lambda,
                     lam_y, n_failed);
}

}  // namespace

extern "C" {

int64_t qrec_als_gram_workspace_bytes(int64_t n, int32_t d) {
  QREC_REQUIRE(n >= 0 && d >= 1 && d <= kMaxD, "als_gram_workspace_bytes: n=%lld d=%d", (long long)n, d);
  return gram_chunks(n) * d * d * (int64_t)sizeof(double);
}

int qrec_als_gram_f32(const float* Z, int64_t n, int32_t d, double* G, void* workspace, int64_t workspace_bytes,
                      void* stream) {
  return launch_gram<float>(Z, n, d, G, workspace, workspace_bytes, (cudaStream_t)stream);
}

int qrec_als_gram_f64(const double* Z, int64_t n, int32_t d, double* G, void* workspace, int64_t workspace_bytes,
                      void* stream) {
  return launch_gram<double>(Z, n, d, G, workspace, workspace_bytes, (cudaStream_t)stream);
}

int qrec_als_solve_rows_f32(float* X, const float* Z, const double* G, int32_t d, int64_t n_rows,
                            const int32_t* row_order, const int64_t* rowptr, const int32_t* cols, const float* vals,
                            double lambda, double alpha, double* loss, int32_t* n_failed, void* stream) {
  return launch_solve<float>(X, Z, G, d, n_rows, row_order, (const long long*)rowptr, cols, vals, lambda, alpha, loss,
                             n_failed, (cudaStream_t)stream);
}

int qrec_als_solve_rows_f64(double* X, const double* Z, const double* G, int32_t d, int64_t n_rows,
                            const int32_t* row_order, const int64_t* rowptr, const int32_t* cols, const double* vals,
                            double lambda, double alpha, double* loss, int32_t* n_failed, void* stream) {
  return launch_solve<double>(X, Z, G, d, n_rows, row_order, (const long long*)rowptr, cols, vals, lambda, alpha,
                              loss, n_failed, (cudaStream_t)stream);
}

int qrec_cofactor_item_sweep_f32(float* Y, float* G, float* w, float* c, const float* X, const double* XtX, int32_t d,
                                 int32_t n_items, const int64_t* item_rowptr, const int32_t* item_users,
                                 const float* item_vals, const int64_t* sppmi_rowptr, const int32_t* sppmi_cols,
                                 const float* sppmi_vals, double lambda, double gamma, double alpha, int32_t* stamps,
                                 int32_t sweep, unsigned long long* ticket, int32_t* n_failed, void* stream) {
  return launch_cofactor<float>(Y, G, w, c, X, XtX, d, n_items, (const long long*)item_rowptr, item_users, item_vals,
                                (const long long*)sppmi_rowptr, sppmi_cols, sppmi_vals, lambda, gamma, alpha, stamps,
                                sweep, ticket, n_failed, (cudaStream_t)stream);
}

int qrec_cofactor_item_sweep_f64(double* Y, double* G, double* w, double* c, const double* X, const double* XtX,
                                 int32_t d, int32_t n_items, const int64_t* item_rowptr, const int32_t* item_users,
                                 const double* item_vals, const int64_t* sppmi_rowptr, const int32_t* sppmi_cols,
                                 const double* sppmi_vals, double lambda, double gamma, double alpha, int32_t* stamps,
                                 int32_t sweep, unsigned long long* ticket, int32_t* n_failed, void* stream) {
  return launch_cofactor<double>(Y, G, w, c, X, XtX, d, n_items, (const long long*)item_rowptr, item_users, item_vals,
                                 (const long long*)sppmi_rowptr, sppmi_cols, sppmi_vals, lambda, gamma, alpha, stamps,
                                 sweep, ticket, n_failed, (cudaStream_t)stream);
}

int qrec_expomf_solve_rows_f32(float* X, const float* Z, int32_t d, int64_t n_z, int64_t n_rows,
                               const int32_t* row_order, const int64_t* rowptr, const int32_t* cols, const float* mu,
                               int32_t mu_by_row, float* mu_out, double lambda, double lam_y, double a, double b,
                               int32_t max_ctas, int32_t* n_failed, void* stream) {
  return launch_expomf(X, Z, d, n_z, n_rows, row_order, (const long long*)rowptr, cols, mu, mu_by_row, mu_out, lambda,
                       lam_y, a, b, max_ctas, n_failed, (cudaStream_t)stream);
}

int qrec_serec_solve_rows_f32(float* X, const float* Z, int32_t d, int64_t n_z, int64_t n_rows,
                              const int32_t* row_order, const int64_t* rowptr, const int32_t* cols,
                              const double* asum, float mu0, const int32_t* deg, int32_t row_is_user,
                              double* asum_out, double lambda, double lam_y, double a, double b, double s,
                              int64_t n_users, int32_t max_ctas, int32_t* n_failed, void* stream) {
  return launch_serec(X, Z, d, n_z, n_rows, row_order, (const long long*)rowptr, cols, asum, mu0, deg, row_is_user,
                      asum_out, lambda, lam_y, a, b, s, n_users, max_ctas, n_failed, (cudaStream_t)stream);
}

}  // extern "C"
