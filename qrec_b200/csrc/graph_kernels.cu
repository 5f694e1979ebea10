// K2/K3/K4: the kernels behind the graph models' training step
// (reference: model/ranking/LightGCN.py:11-41, util/loss.py:3-6, base/graphRecommender.py:10-39).
//
//   K2  spmm_csr_balanced_kernel Y = A X (+ fused layer accumulation), CSR, nnz-balanced chunks
//       spmm_csr_kernel          the row-partitioned product, for graphs without very long rows:
//                                LPR lanes own one row of Y (d=64: a half warp, float4 per lane);
//                                the lane group streams the row's (col,val) pairs coalesced,
//                                broadcasts them with group-masked shuffles and keeps 4 or 8 gathered
//                                X rows in flight per lane.
//       spmm_csr_d64_kernel      its d = 64 specialisation, 4 CTAs per SM.
//   K3  bpr_grad_scatter_kernel  gather 3 rows of the propagated tables, -ln(sigmoid(y)+eps)
//                                + batch L2, gradient scatter-added (REDG.ADD.F32x4) into the
//                                dense gradient buffers.
//   K4  adam_dense_tf1_kernel    TF1 AdamOptimizer dense update (every row moves every step), in
//                                the ApplyAdam form  m += (g-m)(1-b1); v += (g*g-v)(1-b2);
//                                var -= m*alpha/(sqrt(v)+eps).
#include <cmath>

#include "common.h"
#include "device.cuh"
#include "lane_shape.h"

namespace {

using namespace qrec;

// ------------------------------------------------------------------------------------------ K2
template <int LPR, int VPL>
__global__ void __launch_bounds__(256)
spmm_csr_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                const float* __restrict__ vals, const float* __restrict__ X,
                float* __restrict__ Y, int nvec, float* __restrict__ acc, float acc_scale) {
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (sub * LPR));
  const int d = nvec * 4;
  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * GPW + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * GPW;
  for (long long r = group; r < n_rows; r += ngroups) {
    const long long start = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    float4 a[VPL];
#pragma unroll
    for (int v = 0; v < VPL; ++v) a[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    // software pipeline: the (col,val) pairs of the next LPR non-zeros are fetched while the current
    // ones are gathered; G gathered X rows are in flight per lane at any time.
    constexpr int G = (VPL == 1) ? 8 : 4;
    int c = 0;
    float w = 0.f;
    if (start + l < end) {
      c = __ldg(cols + start + l);
      w = __ldg(vals + start + l);
    }
    for (long long base = start; base < end; base += LPR) {
      const int m = (end - base) < LPR ? (int)(end - base) : LPR;
      int cn = 0;
      float wn = 0.f;
      if (base + LPR + l < end) {
        cn = __ldg(cols + base + LPR + l);
        wn = __ldg(vals + base + LPR + l);
      }
      for (int t = 0; t < m; t += G) {
        int cc[G];
        float ww[G];
        float4 x[G][VPL];
#pragma unroll
        for (int q = 0; q < G; ++q) {
          // lanes beyond m carry c=0,w=0: masked below
          cc[q] = __shfl_sync(gmask, c, sub * LPR + ((t + q) & (LPR - 1)));
          ww[q] = __shfl_sync(gmask, w, sub * LPR + ((t + q) & (LPR - 1)));
          if (t + q >= m) ww[q] = 0.f;
        }
#pragma unroll
        for (int q = 0; q < G; ++q) {
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            if ((t + q) < m && (l + v * LPR) < nvec)
              x[q][v] = __ldg(reinterpret_cast<const float4*>(X + (size_t)cc[q] * d) + l + v * LPR);
            else
              x[q][v] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
#pragma unroll
        for (int q = 0; q < G; ++q)
#pragma unroll
          for (int v = 0; v < VPL; ++v) fma4(a[v], ww[q], x[q][v]);
      }
      c = cn;
      w = wn;
    }
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      if ((l + v * LPR) < nvec) {
        float4* yp = reinterpret_cast<float4*>(Y + (size_t)r * d) + l + v * LPR;
        *yp = a[v];
        if (acc != nullptr) {
          float4* ap = reinterpret_cast<float4*>(acc + (size_t)r * d) + l + v * LPR;
          float4 o = *ap;
          fma4(o, acc_scale, a[v]);
          *ap = o;
        }
      }
    }
  }
}

// Y[r] = a (lane l's float4 of a d = 64 row); acc[r] += acc_scale * a.  A function of its own: written inline, nvcc
// allocates the kernel's registers in a different order.
__device__ __forceinline__ void store_row_d64(float* __restrict__ Y, float* __restrict__ acc, float acc_scale, long long r,
                                              int l, float4 a) {
  float4* yp = reinterpret_cast<float4*>(Y + (size_t)r * 64) + l;
  *yp = a;
  if (acc != nullptr) {
    float4* ap = reinterpret_cast<float4*>(acc + (size_t)r * 64) + l;
    float4 o = *ap;
    fma4(o, acc_scale, a);
    *ap = o;
  }
}

// d = 64: spmm_csr_kernel<16, 1> with the width fixed at compile time and 4 CTAs per SM -- the same lane groups and
// floating-point order, 8 gathered rows in flight per lane, issued and consumed in lock step.
__global__ void __launch_bounds__(256, 4)
spmm_csr_d64_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                    const float* __restrict__ vals, const float* __restrict__ X, float* __restrict__ Y,
                    float* __restrict__ acc, float acc_scale) {
  constexpr int LPR = 16, G = 8;   // a half warp per row, one float4 per lane
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const unsigned gmask = ((1u << LPR) - 1u) << (sub * LPR);
  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 2 + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * 2;
  for (long long r = group; r < n_rows; r += ngroups) {
    const long long start = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    int c = 0;
    float w = 0.f;
    if (start + l < end) {
      c = __ldg(cols + start + l);
      w = __ldg(vals + start + l);
    }
    for (long long base = start; base < end; base += LPR) {
      const int m = (end - base) < LPR ? (int)(end - base) : LPR;
      int cn = 0;
      float wn = 0.f;
      if (base + LPR + l < end) {
        cn = __ldg(cols + base + LPR + l);
        wn = __ldg(vals + base + LPR + l);
      }
      for (int t = 0; t < m; t += G) {
        int cc[G];
        float ww[G];
        float4 x[G];
#pragma unroll
        for (int q = 0; q < G; ++q) {
          cc[q] = __shfl_sync(gmask, c, sub * LPR + ((t + q) & (LPR - 1)));
          ww[q] = __shfl_sync(gmask, w, sub * LPR + ((t + q) & (LPR - 1)));
          if (t + q >= m) ww[q] = 0.f;
        }
#pragma unroll
        for (int q = 0; q < G; ++q)
          x[q] = (t + q) < m ? __ldg(reinterpret_cast<const float4*>(X + (size_t)cc[q] * 64) + l)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int q = 0; q < G; ++q) fma4(a, ww[q], x[q]);
      }
      c = cn;
      w = wn;
    }
    store_row_d64(Y, acc, acc_scale, r, l, a);
  }
}

// nnz-balanced variant: every lane group owns QN consecutive non-zeros instead of whole rows, so a
// 150 K-entry row of a power-law graph is spread over ~300 lane groups.  The group finds the row
// of its first non-zero by binary search in rowptr, walks the row segments inside its chunk, stores
// rows that lie completely inside the chunk and RED-adds the partial sums of rows that straddle a
// chunk boundary (Y is zero-filled beforehand; the fused `acc += s*Y` epilogue is linear, so
// partial rows add s*partial to acc).
template <int LPR, int VPL, int QN>
__global__ void __launch_bounds__(256)
spmm_csr_balanced_kernel(int n_rows, long long nnz, const long long* __restrict__ rowptr,
                         const int* __restrict__ cols, const float* __restrict__ vals,
                         const float* __restrict__ X, float* __restrict__ Y, int nvec,
                         float* __restrict__ acc, float acc_scale) {
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (sub * LPR));
  const int d = nvec * 4;
  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * GPW + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * GPW;
  const long long nchunks = (nnz + QN - 1) / QN;
  for (long long ch = group; ch < nchunks; ch += ngroups) {
    const long long lo = ch * QN;
    const long long hi = (lo + QN) < nnz ? (lo + QN) : nnz;
    // first row whose end lies beyond lo: smallest r with rowptr[r+1] > lo.  LPR-ary search: the
    // lanes of the group probe LPR segment ends at once (ballot), 16x shrink per round at d=64.
    int a = 0, b = n_rows - 1;
    while (a < b) {
      const int len = b - a + 1;
      const int step = (len + LPR - 1) / LPR;
      int p = a + (l + 1) * step - 1;
      if (p > b) p = b;
      const bool pred = __ldg(rowptr + p + 1) > lo;
      const unsigned bal = (__ballot_sync(gmask, pred) & gmask) >> (sub * LPR);
      const int f = __ffs(bal) - 1;            // pred(b) is true, so some lane fires
      int pf = a + (f + 1) * step - 1;
      if (pf > b) pf = b;
      a = a + f * step;
      b = pf;
    }
    int r = a;
    long long rs = __ldg(rowptr + r), re = __ldg(rowptr + r + 1);
    while (true) {
      const long long start = rs > lo ? rs : lo;
      const long long end = re < hi ? re : hi;
      float4 acc4[VPL];
#pragma unroll
      for (int v = 0; v < VPL; ++v) acc4[v] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (long long base = start; base < end; base += LPR) {
        const long long idx = base + l;
        int c = 0;
        float w = 0.f;
        if (idx < end) { c = __ldg(cols + idx); w = __ldg(vals + idx); }
        const int m = (end - base) < LPR ? (int)(end - base) : LPR;
        for (int t = 0; t < m; t += 4) {
          int cc[4];
          float ww[4];
          float4 x[4][VPL];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            cc[q] = __shfl_sync(gmask, c, sub * LPR + ((t + q) & (LPR - 1)));
            ww[q] = __shfl_sync(gmask, w, sub * LPR + ((t + q) & (LPR - 1)));
            if (t + q >= m) ww[q] = 0.f;
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
#pragma unroll
            for (int v = 0; v < VPL; ++v) {
              if ((t + q) < m && (l + v * LPR) < nvec)
                x[q][v] = __ldg(reinterpret_cast<const float4*>(X + (size_t)cc[q] * d) + l + v * LPR);
              else
                x[q][v] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q)
#pragma unroll
            for (int v = 0; v < VPL; ++v) fma4(acc4[v], ww[q], x[q][v]);
        }
      }
      const bool whole = (rs >= lo) && (re <= hi);
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        if ((l + v * LPR) < nvec && end > start) {
          float* yp = Y + (size_t)r * d + (l + v * LPR) * 4;
          if (whole) {
            *reinterpret_cast<float4*>(yp) = acc4[v];
            if (acc != nullptr) {
              float4* ap = reinterpret_cast<float4*>(acc + (size_t)r * d) + l + v * LPR;
              float4 o = *ap;
              fma4(o, acc_scale, acc4[v]);
              *ap = o;
            }
          } else {
            red_add_v4(yp, acc4[v]);
            if (acc != nullptr) {
              float4 sc = make_float4(acc_scale * acc4[v].x, acc_scale * acc4[v].y,
                                      acc_scale * acc4[v].z, acc_scale * acc4[v].w);
              red_add_v4(acc + (size_t)r * d + (l + v * LPR) * 4, sc);
            }
          }
        }
      }
      if (re >= hi) break;
      // next non-empty row
      do {
        ++r;
        rs = re;
        re = __ldg(rowptr + r + 1);
      } while (re == rs && r < n_rows - 1);
      if (rs >= hi) break;
    }
  }
}

// Sparse-input product for the FIRST backward SpMM of a minibatch step: the gradient w.r.t. the
// propagated table is non-zero only in the batch's rows (<= 3B of N), so Y = A X reduces to scattering
// X[r] along the edges of those rows (A is symmetric: column r = row r):  Y[c] += a_rc * X[r].
// One lane group per 64-edge slice of a source row; Y (and acc) receive REDG.ADD.F32x4.
template <int LPR>
__global__ void __launch_bounds__(256)
spmm_scatter_rows_kernel(int n_src, const int* __restrict__ src_rows, const long long* __restrict__ rowptr,
                         const int* __restrict__ cols, const float* __restrict__ vals,
                         const float* __restrict__ X, float* __restrict__ Y, int nvec,
                         float* __restrict__ acc, float acc_scale) {
  constexpr int GPW = 32 / LPR, SLICE = 64;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (sub * LPR));
  const int d = nvec * 4;
  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * GPW + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * GPW;
  // work items: (source row, slice) enumerated row-major with a fixed number of slices per row
  // (rows shorter than slice*SLICE simply skip the slice)
  for (long long w = group;; w += ngroups) {
    const long long si = w / 64;                 // up to 64 slices (4096 edges) per pass over a row
    if (si >= n_src) break;
    const int slice = (int)(w % 64);
    const int r = __ldg(src_rows + si);
    if (r < 0) continue;                           // padding entry of a de-duplicated, fixed-length row list
    const long long start = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    for (long long lo = start + (long long)slice * SLICE; lo < end; lo += 64LL * SLICE) {
      const long long hi = (lo + SLICE) < end ? (lo + SLICE) : end;
      const float4 x = (l < nvec) ? __ldg(reinterpret_cast<const float4*>(X + (size_t)r * d) + l)
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
      for (long long base = lo; base < hi; base += LPR) {
        int c = 0;
        float a = 0.f;
        if (base + l < hi) {
          c = __ldg(cols + base + l);
          a = __ldg(vals + base + l);
        }
        const int m = (hi - base) < LPR ? (int)(hi - base) : LPR;
        for (int t = 0; t < m; ++t) {
          const int cc = __shfl_sync(gmask, c, sub * LPR + t);
          const float aa = __shfl_sync(gmask, a, sub * LPR + t);
          if (l < nvec) {
            const float4 v = make_float4(aa * x.x, aa * x.y, aa * x.z, aa * x.w);
            red_add_v4(Y + (size_t)cc * d + l * 4, v);
            if (acc != nullptr)
              red_add_v4(acc + (size_t)cc * d + l * 4,
                         make_float4(acc_scale * v.x, acc_scale * v.y, acc_scale * v.z, acc_scale * v.w));
          }
        }
      }
    }
  }
}

// Pull-side product on a LIST of output rows: out[k] = sum_e a_e X[col_e] over the CSR row rows[k].  One warp per
// listed row; the warp's 32/LPR lane groups take the row's entries round-robin, four gathers in flight each, and
// their partial sums meet in a butterfly at the end (a fixed order: the result is deterministic).  Used for the
// LAST forward layer of a minibatch step, of which the loss reads only the batch's rows.
template <int LPR>
__global__ void __launch_bounds__(256)
spmm_list_rows_kernel(int n_list, const int* __restrict__ rows, const long long* __restrict__ rowptr,
                      const int* __restrict__ cols, const float* __restrict__ vals, const float* __restrict__ X,
                      float* __restrict__ Y, int compact, int nvec, float* __restrict__ acc, float acc_scale) {
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const int d = nvec * 4;
  const bool live = l < nvec;
  const int warp = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int nwarps = (int)(((long long)gridDim.x * blockDim.x) >> 5);
  for (int w = warp; w < n_list; w += nwarps) {
    const int r = __ldg(rows + w);
    if (r < 0) {                                           // padding entry of a fixed-length row list
      if (compact && Y != nullptr && sub == 0 && live)
        *reinterpret_cast<float4*>(Y + (size_t)w * d + l * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const long long start = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long base = start + sub; base < end; base += 4 * GPW) {
      int c[4];
      float a[4];
      float4 x[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const long long e = base + (long long)t * GPW;
        const bool ok = e < end;
        c[t] = ok ? __ldg(cols + e) : -1;
        a[t] = ok ? __ldg(vals + e) : 0.f;
      }
#pragma unroll
      for (int t = 0; t < 4; ++t)
        x[t] = (live && c[t] >= 0) ? __ldg(reinterpret_cast<const float4*>(X + (size_t)c[t] * d) + l)
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        s.x = fmaf(a[t], x[t].x, s.x);
        s.y = fmaf(a[t], x[t].y, s.y);
        s.z = fmaf(a[t], x[t].z, s.z);
        s.w = fmaf(a[t], x[t].w, s.w);
      }
    }
#pragma unroll
    for (int off = LPR; off < 32; off <<= 1) {
      s.x += __shfl_xor_sync(0xffffffffu, s.x, off);
      s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
      s.z += __shfl_xor_sync(0xffffffffu, s.z, off);
      s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
    }
    if (sub == 0 && live) {
      if (Y != nullptr) *reinterpret_cast<float4*>(Y + (size_t)(compact ? w : r) * d + l * 4) = s;
      if (acc != nullptr) {                                // listed rows are distinct: a plain read-modify-write
        float4* ap = reinterpret_cast<float4*>(acc + (size_t)r * d + l * 4);
        float4 o = *ap;
        o.x = fmaf(acc_scale, s.x, o.x);
        o.y = fmaf(acc_scale, s.y, o.y);
        o.z = fmaf(acc_scale, s.z, o.z);
        o.w = fmaf(acc_scale, s.w, o.w);
        *ap = o;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ K3
// MODE 0: the fused kernel.  MODE 1 / 2: the same step for a COLUMN block of the tables (feature-parallel ranks, each
// holding d/world columns of every row): 1 = partial scores y_k = sum over the local columns (+ the local part of the
// batch L2 term into `loss`), no gradients; 2 = gradients of the local columns from the FULL scores (the ranks' partial
// scores summed), the -ln term weighted by log_weight (1 on one rank, 0 elsewhere: it is a function of the full score).
template <int LPR, int VPL, int UNROLL, int MODE = 0>
__global__ void __launch_bounds__(256)
bpr_grad_scatter_kernel(const float* __restrict__ U, const float* __restrict__ V, int nvec,
                        long long n, const int* __restrict__ u, const int* __restrict__ i,
                        const int* __restrict__ j, float eps, float reg, float* __restrict__ gU,
                        float* __restrict__ gV, double* loss, float* __restrict__ y_buf = nullptr,
                        float log_weight = 1.f, const float* __restrict__ y_scale = nullptr) {
  constexpr int TPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int d = nvec * 4;
  float lsum = 0.f;
  for (long long base = warp * 32; base < n; base += nwarps * 32) {
    const long long k = base + lane;
    int mu = 0, mi = 0, mj = 0;
    if (k < n) { mu = __ldg(u + k); mi = __ldg(i + k); mj = __ldg(j + k); }
    const int cnt = (n - base) < 32 ? (int)(n - base) : 32;
    for (int s0 = 0; s0 < cnt; s0 += TPW * UNROLL) {
      float4 p[UNROLL][VPL], qi[UNROLL][VPL], qj[UNROLL][VPL];
      size_t ou[UNROLL], oi[UNROLL], oj[UNROLL];
      bool ok[UNROLL];
#pragma unroll
      for (int r = 0; r < UNROLL; ++r) {
        const int t = s0 + r * TPW + sub;
        const int uu = __shfl_sync(0xffffffffu, mu, t & 31);
        const int ii = __shfl_sync(0xffffffffu, mi, t & 31);
        const int jj = __shfl_sync(0xffffffffu, mj, t & 31);
        ok[r] = t < cnt && uu >= 0;                     // u < 0: not this rank's triple (sharded callers pad instead of compacting)
        ou[r] = (size_t)uu * d + l * 4;
        oi[r] = (size_t)ii * d + l * 4;
        oj[r] = (size_t)jj * d + l * 4;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          if (ok[r] && (l + v * LPR) < nvec) {
            p[r][v] = __ldg(reinterpret_cast<const float4*>(U + ou[r] + v * LPR * 4));
            qi[r][v] = __ldg(reinterpret_cast<const float4*>(V + oi[r] + v * LPR * 4));
            qj[r][v] = __ldg(reinterpret_cast<const float4*>(V + oj[r] + v * LPR * 4));
          } else {
            p[r][v] = qi[r][v] = qj[r][v] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < UNROLL; ++r) {
        float y = 0.f, sq = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          y += dot4(p[r][v], qi[r][v]) - dot4(p[r][v], qj[r][v]);
          sq += dot4(p[r][v], p[r][v]) + dot4(qi[r][v], qi[r][v]) + dot4(qj[r][v], qj[r][v]);
        }
        y = group_sum<LPR>(y);
        sq = group_sum<LPR>(sq);
        if (MODE == 1) {                                  // partial score out, local part of the L2 term, nothing else
          const int t = s0 + r * TPW + sub;
          if (t < cnt && l == 0) {
            y_buf[base + t] = ok[r] ? y : 0.f;
            if (ok[r]) lsum += reg * 0.5f * sq;
          }
          continue;
        }
        if (MODE == 2) {
          const int t = s0 + r * TPW + sub;
          y = (t < cnt) ? __ldg(y_buf + base + t) : 0.f;  // the full score (sum of the ranks' partial scores)
        }
        // optional per-sample score scale c_k: the term is -ln(sigmoid(c_k y) + eps) (SBPR.py:112-113, c = 1/(weight+1))
        float c = 1.f;
        if (MODE == 0 && y_scale != nullptr) {
          const int t = s0 + r * TPW + sub;
          c = (t < cnt) ? __ldg(y_scale + base + t) : 1.f;
          y *= c;
        }
        const float s = 1.0f / (1.0f + expf(-y));
        // d/dy of -ln(s+eps) = -s(1-s)/(s+eps)      (SURVEY A5); chain rule through the score scale
        const float gy = -s * (1.0f - s) / (s + eps) * c;
        if (ok[r]) {
          if (l == 0) lsum += (MODE == 2) ? log_weight * -logf(s + eps) : (-logf(s + eps) + reg * 0.5f * sq);
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            if ((l + v * LPR) < nvec) {
              const float4 P4 = p[r][v], I4 = qi[r][v], J4 = qj[r][v];
              float4 gu, gi, gj;
              gu.x = gy * (I4.x - J4.x) + reg * P4.x; gu.y = gy * (I4.y - J4.y) + reg * P4.y;
              gu.z = gy * (I4.z - J4.z) + reg * P4.z; gu.w = gy * (I4.w - J4.w) + reg * P4.w;
              gi.x = gy * P4.x + reg * I4.x; gi.y = gy * P4.y + reg * I4.y;
              gi.z = gy * P4.z + reg * I4.z; gi.w = gy * P4.w + reg * I4.w;
              gj.x = -gy * P4.x + reg * J4.x; gj.y = -gy * P4.y + reg * J4.y;
              gj.z = -gy * P4.z + reg * J4.z; gj.w = -gy * P4.w + reg * J4.w;
              red_add_v4(gU + ou[r] + v * LPR * 4, gu);
              red_add_v4(gV + oi[r] + v * LPR * 4, gi);
              red_add_v4(gV + oj[r] + v * LPR * 4, gj);
            }
          }
        }
      }
    }
  }
  block_add_loss(lsum, loss);
}

// ------------------------------------------------------------------------------------------ K4
__global__ void __launch_bounds__(256)
adam_dense_tf1_kernel(float* __restrict__ var, float* __restrict__ m, float* __restrict__ v,
                      const float* __restrict__ g, long long n, float lr_t, float b1, float b2,
                      float eps, const float* __restrict__ lr_t_dev) {
  if (lr_t_dev != nullptr) lr_t = __ldg(lr_t_dev);      // step-dependent factor read at run time (CUDA-graph replays)
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = n >> 2;
  const float ob1 = 1.0f - b1, ob2 = 1.0f - b2;
  for (long long k = tid; k < n4; k += stride) {
    float4 G = __ldg(reinterpret_cast<const float4*>(g) + k);
    float4 M = reinterpret_cast<float4*>(m)[k];
    float4 Vv = reinterpret_cast<float4*>(v)[k];
    float4 W = reinterpret_cast<float4*>(var)[k];
#define QREC_ADAM(c)                              \
  M.c = M.c + (G.c - M.c) * ob1;                  \
  Vv.c = Vv.c + (G.c * G.c - Vv.c) * ob2;         \
  W.c = W.c - (M.c * lr_t) / (sqrtf(Vv.c) + eps);
    QREC_ADAM(x) QREC_ADAM(y) QREC_ADAM(z) QREC_ADAM(w)
    reinterpret_cast<float4*>(m)[k] = M;
    reinterpret_cast<float4*>(v)[k] = Vv;
    reinterpret_cast<float4*>(var)[k] = W;
  }
  for (long long k = (n4 << 2) + tid; k < n; k += stride) {
    float G = g[k], M = m[k], Vv = v[k], W = var[k];
    M = M + (G - M) * ob1;
    Vv = Vv + (G * G - Vv) * ob2;
    W = W - (M * lr_t) / (sqrtf(Vv) + eps);
    m[k] = M; v[k] = Vv; var[k] = W;
  }
#undef QREC_ADAM
}

__global__ void __launch_bounds__(256)
axpby_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ b,
             float alpha, float beta, long long n) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long n4 = n >> 2;
  for (long long k = tid; k < n4; k += stride) {
    const float4 A = reinterpret_cast<const float4*>(a)[k];
    const float4 B = reinterpret_cast<const float4*>(b)[k];
    float4 o;
    o.x = alpha * A.x + beta * B.x; o.y = alpha * A.y + beta * B.y;
    o.z = alpha * A.z + beta * B.z; o.w = alpha * A.w + beta * B.w;
    reinterpret_cast<float4*>(dst)[k] = o;
  }
  for (long long k = (n4 << 2) + tid; k < n; k += stride) dst[k] = alpha * a[k] + beta * b[k];
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// K3's launch, shared by its four entry points (MODE as in bpr_grad_scatter_kernel); they check the arguments.
template <int MODE>
int launch_k3(const float* U, const float* V, int d, long long n, const int* u, const int* i, const int* j, float eps,
              float reg, float* gU, float* gV, double* loss, float* y_buf, float log_weight, const float* y_scale,
              cudaStream_t st) {
  const int nvec = d / 4;
  const int grid = capped_grid(((n + 31) / 32 + 7) / 8, 8);
  with_row_shape<256>(nvec, [&](auto s) {
    using S = decltype(s);
    bpr_grad_scatter_kernel<S::LPR, S::VPL, S::UNROLL, MODE><<<grid, 256, 0, st>>>(
        U, V, nvec, n, u, i, j, eps, reg, gU, gV, loss, y_buf, log_weight, y_scale);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // namespace

extern "C" {

int qrec_spmm_csr_f32(int32_t n_rows, int64_t nnz, const int64_t* rowptr, const int32_t* cols,
                      const float* vals, const float* X, float* Y, int32_t d, float* acc,
                      float acc_scale, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && nnz >= 0, "qrec_spmm_csr_f32: n_rows or nnz < 0");
  QREC_REQUIRE(d >= 4 && d <= 256 && d % 4 == 0, "qrec_spmm_csr_f32: d=%d unsupported (multiple of 4, 4..256)", d);
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && X && Y, "qrec_spmm_csr_f32: null pointer");
  QREC_REQUIRE(aligned16(X) && aligned16(Y) && aligned16(acc), "qrec_spmm_csr_f32: tables must be 16-byte aligned");
  QREC_REQUIRE(X != Y, "qrec_spmm_csr_f32: X and Y must not alias");
  cudaStream_t st = (cudaStream_t)stream;
  QREC_CUDA(cudaMemsetAsync(Y, 0, sizeof(float) * (size_t)n_rows * d, st));
  if (nnz == 0) return QREC_OK;
  QREC_REQUIRE(cols && vals, "qrec_spmm_csr_f32: null cols/vals");
  const int nvec = d / 4;
  constexpr int QN = 1024;
  with_row_shape<256>(nvec, [&](auto s) {
    using S = decltype(s);
    const long long groups_per_block = 8 * (32 / S::LPR);
    const int grid = capped_grid(((nnz + QN - 1) / QN + groups_per_block - 1) / groups_per_block, 8);
    spmm_csr_balanced_kernel<S::LPR, S::VPL, QN><<<grid, 256, 0, st>>>(
        n_rows, nnz, reinterpret_cast<const long long*>(rowptr), cols, vals, X, Y, nvec, acc, acc_scale);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_spmm_csr_rowsplit_f32(int32_t n_rows, int64_t nnz, const int64_t* rowptr, const int32_t* cols,
                      const float* vals, const float* X, float* Y, int32_t d, float* acc,
                      float acc_scale, void* stream) {
  QREC_REQUIRE(n_rows >= 0, "qrec_spmm_csr_rowsplit_f32: n_rows < 0");
  QREC_REQUIRE(d >= 4 && d <= 256 && d % 4 == 0, "qrec_spmm_csr_rowsplit_f32: d=%d unsupported (multiple of 4, 4..256)", d);
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && X && Y, "qrec_spmm_csr_rowsplit_f32: null pointer");
  QREC_REQUIRE(aligned16(X) && aligned16(Y) && aligned16(acc), "qrec_spmm_csr_rowsplit_f32: tables must be 16-byte aligned");
  QREC_REQUIRE(X != Y, "qrec_spmm_csr_rowsplit_f32: X and Y must not alias");
  cudaStream_t st = (cudaStream_t)stream;
  if (d == 64) {
    const int grid = capped_grid(((long long)n_rows + 15) / 16, 8);   // 16 lane groups (rows) per 256-thread block
    spmm_csr_d64_kernel<<<grid, 256, 0, st>>>(n_rows, reinterpret_cast<const long long*>(rowptr), cols, vals, X, Y, acc,
                                              acc_scale);
    QREC_LAUNCH_CHECK();
    return QREC_OK;
  }
  const int nvec = d / 4;
  with_row_shape<256>(nvec, [&](auto s) {
    using S = decltype(s);
    const long long groups_per_block = 8 * (32 / S::LPR);
    const int grid = capped_grid((n_rows + groups_per_block - 1) / groups_per_block, 8);
    spmm_csr_kernel<S::LPR, S::VPL><<<grid, 256, 0, st>>>(
        n_rows, reinterpret_cast<const long long*>(rowptr), cols, vals, X, Y, nvec, acc, acc_scale);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_spmm_csr_scatter_rows_f32(int32_t n_rows, int32_t n_src, const int32_t* src_rows,
                                   const int64_t* rowptr, const int32_t* cols, const float* vals,
                                   const float* X, float* Y, int32_t d, float* acc, float acc_scale,
                                   void* stream) {
  QREC_REQUIRE(n_rows >= 0 && n_src >= 0, "qrec_spmm_csr_scatter_rows_f32: negative size");
  QREC_REQUIRE(d >= 4 && d <= 128 && d % 4 == 0, "qrec_spmm_csr_scatter_rows_f32: d=%d unsupported (multiple of 4, 4..128)", d);
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && X && Y, "qrec_spmm_csr_scatter_rows_f32: null pointer");
  QREC_REQUIRE(X != Y, "qrec_spmm_csr_scatter_rows_f32: X and Y must not alias");
  cudaStream_t st = (cudaStream_t)stream;
  QREC_CUDA(cudaMemsetAsync(Y, 0, sizeof(float) * (size_t)n_rows * d, st));
  if (n_src == 0) return QREC_OK;
  QREC_REQUIRE(src_rows && cols && vals, "qrec_spmm_csr_scatter_rows_f32: null index pointer");
  const int nvec = d / 4;
  with_row_shape<128>(nvec, [&](auto s) {
    constexpr int LPR = decltype(s)::LPR;
    const long long per_block = 8 * (32 / LPR);
    const int grid = capped_grid(((long long)n_src * 64 + per_block - 1) / per_block, 8);
    spmm_scatter_rows_kernel<LPR><<<grid, 256, 0, st>>>(
        n_src, src_rows, reinterpret_cast<const long long*>(rowptr), cols, vals, X, Y, nvec, acc, acc_scale);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_spmm_csr_rows_f32(int32_t n_list, const int32_t* rows, const int64_t* rowptr, const int32_t* cols,
                           const float* vals, const float* X, float* Y, int32_t compact, int32_t d, float* acc,
                           float acc_scale, void* stream) {
  QREC_REQUIRE(d >= 4 && d <= 128 && d % 4 == 0, "qrec_spmm_csr_rows_f32: d=%d unsupported (multiple of 4, <= 128)", d);
  QREC_REQUIRE(n_list >= 0, "qrec_spmm_csr_rows_f32: n_list < 0");
  if (n_list == 0) return QREC_OK;
  QREC_REQUIRE(rows && rowptr && cols && vals && X && (Y || acc), "qrec_spmm_csr_rows_f32: null pointer");
  QREC_REQUIRE(aligned16(X) && (!Y || aligned16(Y)) && (!acc || aligned16(acc)),
               "qrec_spmm_csr_rows_f32: matrices must be 16-byte aligned");
  const int nvec = d / 4;
  const int grid = capped_grid(((long long)n_list + 7) / 8, 8);   // one warp per listed row, 8 warps per block
  cudaStream_t st = (cudaStream_t)stream;
  with_row_shape<128>(nvec, [&](auto s) {
    spmm_list_rows_kernel<decltype(s)::LPR><<<grid, 256, 0, st>>>(
        n_list, rows, reinterpret_cast<const long long*>(rowptr), cols, vals, X, Y, compact, nvec, acc, acc_scale);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_bpr_grad_scatter_f32(const float* U, const float* V, int32_t d, int64_t n,
                              const int32_t* u, const int32_t* i, const int32_t* j, float eps,
                              float reg, float* gU, float* gV, double* loss, void* stream) {
  QREC_REQUIRE(d >= 4 && d <= 256 && d % 4 == 0, "qrec_bpr_grad_scatter_f32: d=%d unsupported", d);
  QREC_REQUIRE(n >= 0, "qrec_bpr_grad_scatter_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(U && V && u && i && j && gU && gV && loss, "qrec_bpr_grad_scatter_f32: null pointer");
  QREC_REQUIRE(aligned16(U) && aligned16(V) && aligned16(gU) && aligned16(gV),
               "qrec_bpr_grad_scatter_f32: tables must be 16-byte aligned");
  return launch_k3<0>(U, V, d, n, u, i, j, eps, reg, gU, gV, loss, nullptr, 1.f, nullptr, (cudaStream_t)stream);
}

int qrec_bpr_grad_scatter_scaled_f32(const float* U, const float* V, int32_t d, int64_t n,
                                     const int32_t* u, const int32_t* i, const int32_t* j, const float* y_scale,
                                     float eps, float reg, float* gU, float* gV, double* loss, void* stream) {
  QREC_REQUIRE(d >= 4 && d <= 256 && d % 4 == 0, "qrec_bpr_grad_scatter_scaled_f32: d=%d unsupported", d);
  QREC_REQUIRE(n >= 0, "qrec_bpr_grad_scatter_scaled_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(U && V && u && i && j && y_scale && gU && gV && loss, "qrec_bpr_grad_scatter_scaled_f32: null pointer");
  QREC_REQUIRE(aligned16(U) && aligned16(V) && aligned16(gU) && aligned16(gV),
               "qrec_bpr_grad_scatter_scaled_f32: tables must be 16-byte aligned");
  return launch_k3<0>(U, V, d, n, u, i, j, eps, reg, gU, gV, loss, nullptr, 1.f, y_scale, (cudaStream_t)stream);
}

int qrec_bpr_partial_scores_f32(const float* U, const float* V, int32_t d, int64_t n, const int32_t* u, const int32_t* i,
                                const int32_t* j, float reg, float* y_part, double* loss, void* stream) {
  QREC_REQUIRE(d >= 4 && d <= 256 && d % 4 == 0, "qrec_bpr_partial_scores_f32: d=%d unsupported", d);
  QREC_REQUIRE(n >= 0, "qrec_bpr_partial_scores_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(U && V && u && i && j && y_part && loss, "qrec_bpr_partial_scores_f32: null pointer");
  QREC_REQUIRE(aligned16(U) && aligned16(V), "qrec_bpr_partial_scores_f32: tables must be 16-byte aligned");
  return launch_k3<1>(U, V, d, n, u, i, j, 0.f, reg, nullptr, nullptr, loss, y_part, 0.f, nullptr, (cudaStream_t)stream);
}

int qrec_bpr_grad_from_scores_f32(const float* U, const float* V, int32_t d, int64_t n, const int32_t* u, const int32_t* i,
                                  const int32_t* j, const float* y_full, float eps, float reg, float log_weight, float* gU,
                                  float* gV, double* loss, void* stream) {
  QREC_REQUIRE(d >= 4 && d <= 256 && d % 4 == 0, "qrec_bpr_grad_from_scores_f32: d=%d unsupported", d);
  QREC_REQUIRE(n >= 0, "qrec_bpr_grad_from_scores_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(U && V && u && i && j && y_full && gU && gV && loss, "qrec_bpr_grad_from_scores_f32: null pointer");
  QREC_REQUIRE(aligned16(U) && aligned16(V) && aligned16(gU) && aligned16(gV),
               "qrec_bpr_grad_from_scores_f32: tables must be 16-byte aligned");
  return launch_k3<2>(U, V, d, n, u, i, j, eps, reg, gU, gV, loss, const_cast<float*>(y_full), log_weight, nullptr,
                      (cudaStream_t)stream);
}

int qrec_adam_dense_tf1_f32(float* var, float* m, float* v, const float* g, int64_t n, float lr,
                            float beta1, float beta2, float eps, int64_t t, void* stream) {
  QREC_REQUIRE(n >= 0 && t >= 1, "qrec_adam_dense_tf1_f32: bad n or t");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(var && m && v && g, "qrec_adam_dense_tf1_f32: null pointer");
  QREC_REQUIRE(aligned16(var) && aligned16(m) && aligned16(v) && aligned16(g),
               "qrec_adam_dense_tf1_f32: buffers must be 16-byte aligned");
  // TF1 evaluates alpha in the variable dtype (fp32); beta^t is rounded to fp32 once here (TF keeps
  // a running fp32 product, which differs in the last bits only)
  const float b1p = (float)pow((double)beta1, (double)t), b2p = (float)pow((double)beta2, (double)t);
  const float lr_t = lr * sqrtf(1.0f - b2p) / (1.0f - b1p);
  adam_dense_tf1_kernel<<<capped_grid((n / 4 + 255) / 256 + 1, 8), 256, 0, (cudaStream_t)stream>>>(
      var, m, v, g, n, lr_t, beta1, beta2, eps, nullptr);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_adam_dense_tf1_devstep_f32(float* var, float* m, float* v, const float* g, int64_t n, const float* dev_lr_t,
                                    float beta1, float beta2, float eps, void* stream) {
  QREC_REQUIRE(n >= 0, "qrec_adam_dense_tf1_devstep_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(var && m && v && g && dev_lr_t, "qrec_adam_dense_tf1_devstep_f32: null pointer");
  QREC_REQUIRE(aligned16(var) && aligned16(m) && aligned16(v) && aligned16(g),
               "qrec_adam_dense_tf1_devstep_f32: buffers must be 16-byte aligned");
  adam_dense_tf1_kernel<<<capped_grid((n / 4 + 255) / 256 + 1, 8), 256, 0, (cudaStream_t)stream>>>(
      var, m, v, g, n, 0.f, beta1, beta2, eps, dev_lr_t);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_axpby_f32(float* dst, const float* a, const float* b, float alpha, float beta, int64_t n,
                   void* stream) {
  QREC_REQUIRE(n >= 0, "qrec_axpby_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(dst && a && b, "qrec_axpby_f32: null pointer");
  QREC_REQUIRE(aligned16(dst) && aligned16(a) && aligned16(b), "qrec_axpby_f32: buffers must be 16-byte aligned");
  axpby_kernel<<<capped_grid((n / 4 + 255) / 256 + 1, 8), 256, 0, (cudaStream_t)stream>>>(dst, a, b, alpha, beta, n);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
