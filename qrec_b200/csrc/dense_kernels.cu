// K6 and the small dense helpers of the graph models:
//   * simgcl_perturb_kernel      E += sign(E) * l2_normalize(U[0,1)^d) * eps   (SimGCL.py:33-35),
//                                Philox noise generated in registers, optional fused layer mean
//   * gather_normalize_kernel    Z = l2_normalize(T[idx])                      (SimGCL.py:61-69)
//   * infonce_rows_kernel        row log-sum-exp of S/tau, loss, dS in place   (SimGCL.py:70-78)
//   * normalize_bwd_scatter      gradient through l2_normalize, added to the dense grad rows
//   * sgemm_f32                  C = alpha*op(A)*op(B) + beta*C, fp32 SIMT tiles -- the B' x B' x d
//                                similarity products and NGCF's [N,d]x[d,d] layer transforms are
//                                bandwidth-sized, not tensor-core-sized (SURVEY.md 2.5: tensor
//                                cores only for NeuMF's MLP)
//   * leaky_relu / dropout / row l2-normalise forward+backward for NGCF (NGCF.py:29-40)
#include <cmath>

#include "common.h"
#include "device.cuh"
#include "philox.cuh"

namespace {

using qrec::philox4x32_10;
using qrec::red_add_v4;
using qrec::capped_grid;
using qrec::sm_count;

__device__ __forceinline__ float u01(uint32_t w) { return (float)(w >> 8) * (1.0f / 16777216.0f); }
__device__ __forceinline__ float sgn(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

// one warp per row, lanes stride over float4 slices (d multiple of 4, any size)
__global__ void __launch_bounds__(256)
simgcl_perturb_kernel(float* __restrict__ E, long long n_rows, int nvec, int d_valid, float eps, uint32_t k0,
                      uint32_t k1, uint32_t tag, uint32_t step, float* __restrict__ acc,
                      float acc_scale, long long row_off,     // row_off: global id of row 0 (row-sharded tables)
                      const int* __restrict__ row_list) {     // non-null: E is compact, row k belongs to table row row_list[k]
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += nwarps) {
    float4* row = reinterpret_cast<float4*>(E) + r * nvec;
    long long tr = r;                                         // row of the table (and of acc) this row of E stands for
    if (row_list != nullptr) {
      tr = __ldg(row_list + r);
      if (tr < 0) continue;                                   // padding entry of a fixed-length row list
    }
    const unsigned long long gr = (unsigned long long)(tr + row_off);   // the noise is a function of the GLOBAL row
    float ss = 0.f;
    // first pass: squared norm of the row's noise (regenerated below; Philox is cheaper than HBM)
    for (int v = lane; v < nvec; v += 32) {
      uint32_t w[4];
      philox4x32_10((uint32_t)gr, (uint32_t)(gr >> 32) ^ (uint32_t)v, tag, step, k0, k1, w);
      // columns >= d_valid are zero padding of the table: they carry no noise
      const float a = (v * 4 + 0 < d_valid) ? u01(w[0]) : 0.f, b = (v * 4 + 1 < d_valid) ? u01(w[1]) : 0.f;
      const float c = (v * 4 + 2 < d_valid) ? u01(w[2]) : 0.f, d4 = (v * 4 + 3 < d_valid) ? u01(w[3]) : 0.f;
      ss += a * a + b * b + c * c + d4 * d4;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float inv = eps * rsqrtf(fmaxf(ss, 1e-12f));       // tf.nn.l2_normalize epsilon
    for (int v = lane; v < nvec; v += 32) {
      uint32_t w[4];
      philox4x32_10((uint32_t)gr, (uint32_t)(gr >> 32) ^ (uint32_t)v, tag, step, k0, k1, w);
      float4 e = row[v];
      e.x += sgn(e.x) * u01(w[0]) * inv;
      e.y += sgn(e.y) * u01(w[1]) * inv;
      e.z += sgn(e.z) * u01(w[2]) * inv;
      e.w += sgn(e.w) * u01(w[3]) * inv;
      row[v] = e;
      if (acc != nullptr) {
        float4* ap = reinterpret_cast<float4*>(acc) + tr * nvec + v;
        float4 o = *ap;
        o.x += acc_scale * e.x; o.y += acc_scale * e.y; o.z += acc_scale * e.z; o.w += acc_scale * e.w;
        *ap = o;
      }
    }
  }
}

// Z[r,:] = T[idx[r],:] / max(|T[idx[r]]|, 1e-6); norms[r] = that denominator.  warp per row.
__global__ void __launch_bounds__(256)
gather_normalize_kernel(const float* __restrict__ T, const int* __restrict__ idx, int n, int d,
                        float* __restrict__ Z, float* __restrict__ norms) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r = warp; r < n; r += nwarps) {
    const float* src = T + (size_t)idx[r] * d;
    float ss = 0.f;
    for (int c = lane; c < d; c += 32) { const float x = src[c]; ss += x * x; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float nrm = sqrtf(fmaxf(ss, 1e-12f));
    for (int c = lane; c < d; c += 32) Z[(size_t)r * d + c] = src[c] / nrm;
    if (lane == 0) norms[r] = nrm;
  }
}

// S holds raw dots z1_i . z2_j (n x n, row-major).  Per row i: lse_i = log sum_j exp(S_ij/tau);
// loss += lse_i - S_ii/tau;  S_ij <- (exp(S_ij/tau - lse_i) - [i==j]) / tau   (= dLoss/dS_ij raw).
__global__ void __launch_bounds__(256)
infonce_rows_kernel(float* __restrict__ S, int n, float inv_tau, double* loss) {
  __shared__ float red[8];
  __shared__ float bcast;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    float* row = S + (size_t)i * n;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, row[j] * inv_tau);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = red[0];
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) t = fmaxf(t, red[w]);
      bcast = t;
    }
    __syncthreads();
    const float mx = bcast;
    float s = 0.f;
    for (int j = threadIdx.x; j < n; j += blockDim.x) s += expf(row[j] * inv_tau - mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
      const float lse = mx + logf(t);
      atomicAdd(loss, (double)(lse - row[i] * inv_tau));
      bcast = lse;
    }
    __syncthreads();
    const float lse = bcast;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
      const float p = expf(row[j] * inv_tau - lse);
      row[j] = (p - (j == i ? 1.f : 0.f)) * inv_tau;
    }
    __syncthreads();
  }
}

// G[idx[r],:] += scale * (dZ_r - Z_r * (Z_r . dZ_r)) / norm_r        (idx unique within a call)
__global__ void __launch_bounds__(256)
normalize_bwd_scatter_kernel(const float* __restrict__ dZ, const float* __restrict__ Z,
                             const float* __restrict__ norms, const int* __restrict__ idx, int n,
                             int d, float scale, float* __restrict__ G) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int r = warp; r < n; r += nwarps) {
    const float* z = Z + (size_t)r * d;
    const float* g = dZ + (size_t)r * d;
    float dot = 0.f;
    for (int c = lane; c < d; c += 32) dot += z[c] * g[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    const float k = scale / norms[r];
    float* dst = G + (size_t)idx[r] * d;
    for (int c = lane; c < d; c += 32) atomicAdd(dst + c, k * (g[c] - z[c] * dot));
  }
}

// C[M,N] = alpha * op(A) * op(B) + beta * C, row-major, 64x64 tile, 16x16 threads, 4x4 micro-tile.
// ksplit > 1: the K range is cut into `ksplit` slabs (work item = tile x slab) and partial products
// are atomically added into C, which the host has pre-scaled by beta (the [d,N]x[N,d] weight
// gradients of NGCF have one output tile and K = #nodes).
template <bool TA, bool TB>
__global__ void __launch_bounds__(256)
sgemm_kernel(int M, int N, int K, float alpha, const float* __restrict__ A, int lda,
             const float* __restrict__ B, int ldb, float beta, float* __restrict__ C, int ldc,
             int ksplit) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const long long ntiles = (long long)((M + BM - 1) / BM) * ((N + BN - 1) / BN);
  const int kslab = ((K + ksplit - 1) / ksplit + BK - 1) / BK * BK;
  for (long long work = blockIdx.x; work < ntiles * ksplit; work += gridDim.x) {
    const long long tile = work / ksplit;
    const int slab = (int)(work % ksplit);
    const int kbeg = slab * kslab, kend = (kbeg + kslab) < K ? (kbeg + kslab) : K;
    const int tn = (N + BN - 1) / BN;
    const int m0 = (int)(tile / tn) * BM, n0 = (int)(tile % tn) * BN;
    float acc[4][4] = {};
    for (int k0 = kbeg; k0 < kend; k0 += BK) {
      for (int e = threadIdx.x; e < BM * BK; e += 256) {
        int m, k;
        if (TA) { m = e % BM; k = e / BM; } else { k = e % BK; m = e / BK; }
        const int gm = m0 + m, gk = k0 + k;
        float v = 0.f;
        if (gm < M && gk < kend) v = TA ? A[(size_t)gk * lda + gm] : A[(size_t)gm * lda + gk];
        As[k][m] = v;
      }
      for (int e = threadIdx.x; e < BN * BK; e += 256) {
        int n, k;
        if (TB) { k = e % BK; n = e / BK; } else { n = e % BN; k = e / BN; }
        const int gn = n0 + n, gk = k0 + k;
        float v = 0.f;
        if (gn < N && gk < kend) v = TB ? B[(size_t)gn * ldb + gk] : B[(size_t)gk * ldb + gn];
        Bs[k][n] = v;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        // rows of As / Bs are 68 floats apart (272 B): 16-byte aligned, so one LDS.128 each instead of four LDS.32
        const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
        const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
        const float a[4] = {av.x, av.y, av.z, av.w}, b[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int p = 0; p < 4; ++p) acc[q][p] = fmaf(a[q], b[p], acc[q][p]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int gm = m0 + ty * 4 + q;
      if (gm >= M) continue;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int gn = n0 + tx * 4 + p;
        if (gn < N) {
          float* c = C + (size_t)gm * ldc + gn;
          if (ksplit > 1) atomicAdd(c, alpha * acc[q][p]);
          else *c = alpha * acc[q][p] + (beta != 0.f ? beta * *c : 0.f);
        }
      }
    }
  }
}


// Tall-skinny product for the NGCF layer transforms: C[M,N] = alpha * A[M,K] * op(B) + beta * C with
// N, K <= 64 (a d x d weight) and M = #nodes.  One thread owns one output row: op(B) sits in shared
// memory (read as broadcast LDS.128), the row's N accumulators in registers; the row of A is streamed
// with 16-byte loads.  FFMA : LDS = 4 : 1, no cross-thread reduction, no __syncthreads in the loop.
template <bool TB>
__global__ void __launch_bounds__(128)
sgemm_skinny_kernel(int M, int N, int K, float alpha, const float* __restrict__ A, int lda,
                    const float* __restrict__ B, int ldb, float beta, float* __restrict__ C, int ldc) {
  __shared__ __align__(16) float W[64 * 64];            // W[k][n], row pitch 64
  for (int e = threadIdx.x; e < 64 * 64; e += blockDim.x) {
    const int k = e >> 6, n = e & 63;
    float v = 0.f;
    if (k < K && n < N) v = TB ? B[(size_t)n * ldb + k] : B[(size_t)k * ldb + n];
    W[e] = v;
  }
  __syncthreads();
  const int n4 = (N + 3) >> 2;
  for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < M;
       row += (long long)gridDim.x * blockDim.x) {
    float acc[64];
#pragma unroll
    for (int n = 0; n < 64; ++n) acc[n] = 0.f;
    const float* a = A + (size_t)row * lda;
    for (int k0 = 0; k0 < K; k0 += 4) {
      const float4 av = *reinterpret_cast<const float4*>(a + k0);
      const float ak[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const float4* wrow = reinterpret_cast<const float4*>(W + (k0 + kk) * 64);
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          if (q < n4) {
            const float4 w = wrow[q];
            acc[4 * q + 0] = fmaf(ak[kk], w.x, acc[4 * q + 0]);
            acc[4 * q + 1] = fmaf(ak[kk], w.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(ak[kk], w.z, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(ak[kk], w.w, acc[4 * q + 3]);
          }
        }
      }
    }
    float* c = C + (size_t)row * ldc;
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      if (q < n4) {
        float4 o = make_float4(alpha * acc[4 * q], alpha * acc[4 * q + 1], alpha * acc[4 * q + 2], alpha * acc[4 * q + 3]);
        if (beta != 0.f) {
          const float4 old = *reinterpret_cast<const float4*>(c + 4 * q);
          o.x += beta * old.x; o.y += beta * old.y; o.z += beta * old.z; o.w += beta * old.w;
        }
        *reinterpret_cast<float4*>(c + 4 * q) = o;
      }
    }
  }
}

// ---- NGCF elementwise pieces (NGCF.py:29-40) ------------------------------------------------------
// forward: H = leaky_relu(Z, 0.2); H *= mask/keep (mask from Philox, keep prob); Nrm = |H| row norm;
// out = H / max(|H|, 1e-6).  Stores H (post-dropout) for the backward pass.  warp per row.
__global__ void __launch_bounds__(256)
ngcf_act_fwd_kernel(const float* __restrict__ Zin, long long n_rows, int d, float keep, int training,
                    uint32_t k0, uint32_t k1, uint32_t tag, uint32_t step, float* __restrict__ H,
                    float* __restrict__ out, int ld_out, float* __restrict__ norms) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += nwarps) {
    float ss = 0.f;
    for (int c = lane; c < d; c += 32) {
      float z = Zin[r * d + c];
      float h = z > 0.f ? z : 0.2f * z;
      if (training) {
        uint32_t w[4];
        philox4x32_10((uint32_t)r, (uint32_t)((unsigned long long)r >> 32) ^ (uint32_t)(c >> 2), tag, step, k0, k1, w);
        h = (u01(w[c & 3]) < keep) ? h / keep : 0.f;
      }
      H[r * d + c] = h;
      ss += h * h;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float nrm = sqrtf(fmaxf(ss, 1e-12f));
    for (int c = lane; c < d; c += 32) out[r * ld_out + c] = H[r * d + c] / nrm;
    if (lane == 0) norms[r] = nrm;
  }
}

// backward: given dOut (grad wrt normalised output) and dH_extra (grad wrt H from the next layer's
// use of the un-normalised ego embedding), produce dZ (grad wrt the pre-activation).
__global__ void __launch_bounds__(256)
ngcf_act_bwd_kernel(const float* __restrict__ dOut, int ld_dout, const float* __restrict__ dH_extra,
                    const float* __restrict__ H, const float* __restrict__ Zin,
                    const float* __restrict__ norms, long long n_rows, int d, float keep,
                    int training, uint32_t k0, uint32_t k1, uint32_t tag, uint32_t step,
                    float* __restrict__ dZ) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += nwarps) {
    const float nrm = norms[r];
    float dot = 0.f;
    for (int c = lane; c < d; c += 32) dot += (H[r * d + c] / nrm) * dOut[r * ld_dout + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
    for (int c = lane; c < d; c += 32) {
      const float o = H[r * d + c] / nrm;
      float g = (dOut[r * ld_dout + c] - o * dot) / nrm;
      if (dH_extra != nullptr) g += dH_extra[r * d + c];
      if (training) {
        uint32_t w[4];
        philox4x32_10((uint32_t)r, (uint32_t)((unsigned long long)r >> 32) ^ (uint32_t)(c >> 2), tag, step, k0, k1, w);
        g = (u01(w[c & 3]) < keep) ? g / keep : 0.f;
      }
      const float z = Zin[r * d + c];
      dZ[r * d + c] = z > 0.f ? g : 0.2f * g;
    }
  }
}

__global__ void __launch_bounds__(256)
scale_matrix_kernel(float* __restrict__ C, int M, int N, int ldc, float beta) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < (long long)M * N; k += stride) {
    float* c = C + (k / N) * ldc + (k % N);
    *c = beta != 0.f ? beta * *c : 0.f;
  }
}

__global__ void __launch_bounds__(256)
mul_kernel(float* __restrict__ dst, const float* __restrict__ a, const float* __restrict__ b, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride) dst[k] = a[k] * b[k];
}


// ---- NeuMF pieces (model/ranking/NeuMF.py:27-75) ------------------------------------------------
// out[b, 0:d] = T[idx[b], :]   (row stride ld_out: writes one half of the concatenated MLP input)
__global__ void __launch_bounds__(256)
gather_rows_kernel(const float* __restrict__ T, const int* __restrict__ idx, long long n, int nvec,
                   float* __restrict__ out, int ld_out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n * nvec; k += stride) {
    const long long b = k / nvec;
    const int v = (int)(k % nvec);
    const int row = __ldg(idx + b);                      // row < 0: an empty slot of a fixed-capacity exchange -> zeros
    const float4 x = row >= 0 ? __ldg(reinterpret_cast<const float4*>(T + (size_t)row * nvec * 4) + v) : make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(out + (size_t)b * ld_out + v * 4) = x;
  }
}

// G[idx[b], :] += scale * src[b, 0:d]   (duplicates in idx accumulate: REDG.ADD.F32x4)
__global__ void __launch_bounds__(256)
scatter_add_rows_kernel(float* __restrict__ G, const int* __restrict__ idx, long long n, int nvec,
                        const float* __restrict__ src, int ld_src, float scale) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n * nvec; k += stride) {
    const long long b = k / nvec;
    const int v = (int)(k % nvec);
    const int row = __ldg(idx + b);
    if (row < 0) continue;                                // empty slot
    float4 x = *reinterpret_cast<const float4*>(src + (size_t)b * ld_src + v * 4);
    x.x *= scale; x.y *= scale; x.z *= scale; x.w *= scale;
    red_add_v4(G + (size_t)row * nvec * 4 + v * 4, x);
  }
}

// K7 (row-sharded item table): request k asks for item ids[k]; its owner is ids[k] / rows_per_rank.  Every
// (requester, owner) pair has a FIXED number of slots (cap), so the three exchanges are equal-split all-to-alls
// whose sizes the host knows without looking at the data: slot = atomicAdd(count[owner]); send[owner*cap + slot] =
// LOCAL row at the owner; pos[k] = owner*cap + slot (where the row will arrive and the delta must be left).
// A bucket that overflows raises *overflow (the step is then invalid; the caller re-runs with a larger cap).
__global__ void __launch_bounds__(256)
bucket_requests_kernel(const int* __restrict__ ids, long long n, int rows_per_rank, int world, int cap,
                       int* __restrict__ count, int* __restrict__ send, int* __restrict__ pos, int* __restrict__ overflow) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  const long long first = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  // uniform trip count per warp so that the warp-aggregated reservation below sees all 32 lanes
  for (long long k0 = first - lane; k0 < n; k0 += stride) {
    const long long k = k0 + lane;
    const bool valid = k < n;
    int id = 0, owner = 0;
    if (valid) {
      id = __ldg(ids + k);
      owner = id / rows_per_rank;
      if (owner >= world) owner = world - 1;
    }
    // one atomicAdd per (warp, owner) instead of one per request: with few owners every request of a minibatch
    // would otherwise hit the same handful of counters
    const unsigned act = __ballot_sync(0xffffffffu, valid);
    if (!valid) continue;
    const unsigned peers = __match_any_sync(act, owner);
    const int leader = __ffs(peers) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(count + owner, __popc(peers));
    base = __shfl_sync(peers, base, leader);
    const int slot = base + __popc(peers & ((1u << lane) - 1u));
    if (slot < cap) {
      send[(long long)owner * cap + slot] = id - owner * rows_per_rank;
      pos[k] = owner * cap + slot;
    } else {
      pos[k] = owner * cap;                                // stays in bounds; the step is flagged invalid
      atomicExch(overflow, 1);
    }
  }
}

// out[c] += alpha * sum_b A[b, c] * v[b]   (v == nullptr: column sums).  The bias / head-vector gradients of NeuMF
// (NeuMF.py:39-57: d b_k = column sums of dH_k, d h = X^T dz) are matrix^T-vector products over the B samples of a
// minibatch; through the tiled sgemm they cost a 64x64 tile per useful column.  Here a block owns a slab of rows,
// threads own columns (coalesced row reads), partial sums meet in shared memory and leave with one atomic per
// column and block.
__global__ void __launch_bounds__(256)
gemv_t_kernel(const float* __restrict__ A, int lda, long long rows, int cols, const float* __restrict__ v, float alpha,
              float* __restrict__ out, int rows_per_block) {
  __shared__ float part[256];
  const int cw = cols < 256 ? (cols <= 32 ? 32 : (cols <= 64 ? 64 : (cols <= 128 ? 128 : 256))) : 256;   // threads per row
  const int ry = threadIdx.x / cw, cx = threadIdx.x % cw, rstep = 256 / cw;
  const long long r0 = (long long)blockIdx.x * rows_per_block;
  const long long r1 = (r0 + rows_per_block) < rows ? (r0 + rows_per_block) : rows;
  for (int c0 = 0; c0 < cols; c0 += cw) {
    const int c = c0 + cx;
    float acc = 0.f;
    if (c < cols)
      for (long long r = r0 + ry; r < r1; r += rstep) acc = fmaf(__ldg(A + (size_t)r * lda + c), v ? __ldg(v + r) : 1.0f, acc);
    part[threadIdx.x] = acc;
    __syncthreads();
    if (ry == 0 && c < cols) {
      float t = 0.f;
      for (int q = 0; q < rstep; ++q) t += part[q * cw + cx];
      atomicAdd(out + c, alpha * t);
    }
    __syncthreads();
  }
}

// Prediction heads and their gradients.  mode 0 = GMF (NeuMF.py:52-58), 1 = MLP (:60-65),
// 2 = fused NeuMF (:67-73).  One warp per sample.
//   z = wg * (UG*IG).h_mf + wm * H3.h_mlp,  (wg, wm) = (1,0) | (0,1) | (.5,.5);  y = sigmoid(z)
//   loss += -(r ln(y+1e-9) + (1-r) ln(1-y+1e-9)) [+ reg*0.5(|UG|^2+|IG|^2) unless mode 1]
//   dz = dLoss/dz;  GMF = UG*IG;  dUG = wg*dz*h_mf*IG + reg*UG;  dIG likewise;
//   dH3 = wm*dz*h_mlp masked by H3 > 0 (ReLU);  training = 0: only y is written.
__global__ void __launch_bounds__(256)
neumf_head_kernel(int mode, int training, const float* __restrict__ UG, const float* __restrict__ IG,
                  const float* __restrict__ H3, const float* __restrict__ h_mf,
                  const float* __restrict__ h_mlp, const float* __restrict__ r, long long n, int d,
                  float reg, double* loss, float* __restrict__ y_out, float* __restrict__ dz_out,
                  float* __restrict__ GMF, float* __restrict__ dUG, float* __restrict__ dIG,
                  float* __restrict__ dH3) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float wg = mode == 0 ? 1.f : (mode == 1 ? 0.f : 0.5f);
  const float wm = mode == 1 ? 1.f : (mode == 0 ? 0.f : 0.5f);
  double lsum = 0.0;
  for (long long b = warp; b < n; b += nwarps) {
    float z = 0.f, sq = 0.f;
    for (int c = lane; c < d; c += 32) {
      if (mode != 1) {
        const float ug = UG[b * d + c], ig = IG[b * d + c];
        z += wg * ug * ig * h_mf[c];
        sq += ug * ug + ig * ig;
      }
      if (mode != 0) z += wm * H3[b * d + c] * h_mlp[c];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      z += __shfl_xor_sync(0xffffffffu, z, o);
      sq += __shfl_xor_sync(0xffffffffu, sq, o);
    }
    const float y = 1.0f / (1.0f + expf(-z));
    if (lane == 0 && y_out != nullptr) y_out[b] = y;
    if (!training) continue;
    const float rb = r[b];
    const float e = 10e-10f;                                   // the literal in NeuMF.py:55
    const float dy = -rb / (y + e) + (1.f - rb) / (1.f - y + e);
    const float dz = dy * y * (1.f - y);
    if (lane == 0) {
      lsum += -(double)(rb * logf(y + e) + (1.f - rb) * logf(1.f - y + e)) + (mode != 1 ? 0.5 * reg * sq : 0.0);
      dz_out[b] = dz;
    }
    for (int c = lane; c < d; c += 32) {
      if (mode != 1) {
        const float ug = UG[b * d + c], ig = IG[b * d + c];
        GMF[b * d + c] = ug * ig;
        dUG[b * d + c] = wg * dz * h_mf[c] * ig + reg * ug;
        dIG[b * d + c] = wg * dz * h_mf[c] * ug + reg * ig;
      }
      if (mode != 0) dH3[b * d + c] = H3[b * d + c] > 0.f ? wm * dz * h_mlp[c] : 0.f;
    }
  }
  if (training && lane == 0 && lsum != 0.0) atomicAdd(loss, lsum);
}


// K8 helper (base/recommender.py:147-149): scores[b, item] = value for every item user_ids[b] rated
// in the training set -- the reference overwrites rated positions with 0, it does not remove them.
__global__ void __launch_bounds__(256)
mask_rated_kernel(float* __restrict__ scores, int n_rows, long long ld, const int* __restrict__ users,
                  const long long* __restrict__ rowptr, const int* __restrict__ cols, float value) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int b = warp; b < n_rows; b += nwarps) {
    const int u = users[b];
    const long long lo = rowptr[u], hi = rowptr[u + 1];
    for (long long e = lo + lane; e < hi; e += 32) scores[(size_t)b * ld + cols[e]] = value;
  }
}

inline int grid_for(long long work_items, int per_block) { return capped_grid((work_items + per_block - 1) / per_block, 8); }

}  // namespace

extern "C" {

int qrec_simgcl_perturb_rows_f32(float* E, int64_t n_rows, int64_t row_offset, int32_t d, int32_t d_valid, float eps,
                                 uint64_t seed, uint32_t tag, uint32_t step, float* acc, float acc_scale, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && row_offset >= 0 && d >= 4 && d % 4 == 0, "qrec_simgcl_perturb_f32: bad shape (d multiple of 4)");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(E != nullptr, "qrec_simgcl_perturb_f32: null table");
  simgcl_perturb_kernel<<<grid_for(n_rows, 8), 256, 0, (cudaStream_t)stream>>>(
      E, n_rows, d / 4, (d_valid > 0 && d_valid < d) ? d_valid : d, eps, (uint32_t)seed, (uint32_t)(seed >> 32), tag, step, acc,
      acc_scale, row_offset, nullptr);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_simgcl_perturb_listed_f32(float* Ec, const int32_t* rows, int64_t n_list, int64_t row_offset, int32_t d,
                                   int32_t d_valid, float eps, uint64_t seed, uint32_t tag, uint32_t step, float* acc,
                                   float acc_scale, void* stream) {
  QREC_REQUIRE(n_list >= 0 && row_offset >= 0 && d >= 4 && d % 4 == 0, "qrec_simgcl_perturb_listed_f32: bad shape (d multiple of 4)");
  if (n_list == 0) return QREC_OK;
  QREC_REQUIRE(Ec != nullptr && rows != nullptr, "qrec_simgcl_perturb_listed_f32: null pointer");
  simgcl_perturb_kernel<<<grid_for(n_list, 8), 256, 0, (cudaStream_t)stream>>>(
      Ec, n_list, d / 4, (d_valid > 0 && d_valid < d) ? d_valid : d, eps, (uint32_t)seed, (uint32_t)(seed >> 32), tag, step, acc,
      acc_scale, row_offset, rows);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_simgcl_perturb_f32(float* E, int64_t n_rows, int32_t d, int32_t d_valid, float eps, uint64_t seed,
                            uint32_t tag, uint32_t step, float* acc, float acc_scale, void* stream) {
  return qrec_simgcl_perturb_rows_f32(E, n_rows, 0, d, d_valid, eps, seed, tag, step, acc, acc_scale, stream);
}

int qrec_gather_normalize_f32(const float* T, const int32_t* idx, int32_t n, int32_t d, float* Z,
                              float* norms, void* stream) {
  QREC_REQUIRE(n >= 0 && d >= 1, "qrec_gather_normalize_f32: bad shape");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(T && idx && Z && norms, "qrec_gather_normalize_f32: null pointer");
  gather_normalize_kernel<<<grid_for(n, 8), 256, 0, (cudaStream_t)stream>>>(T, idx, n, d, Z, norms);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_infonce_rows_f32(float* S, int32_t n, float tau, double* loss, void* stream) {
  QREC_REQUIRE(n >= 0 && tau > 0.f, "qrec_infonce_rows_f32: bad argument");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(S && loss, "qrec_infonce_rows_f32: null pointer");
  infonce_rows_kernel<<<grid_for(n, 1), 256, 0, (cudaStream_t)stream>>>(S, n, 1.0f / tau, loss);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_normalize_bwd_scatter_f32(const float* dZ, const float* Z, const float* norms,
                                   const int32_t* idx, int32_t n, int32_t d, float scale, float* G,
                                   void* stream) {
  QREC_REQUIRE(n >= 0 && d >= 1, "qrec_normalize_bwd_scatter_f32: bad shape");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(dZ && Z && norms && idx && G, "qrec_normalize_bwd_scatter_f32: null pointer");
  normalize_bwd_scatter_kernel<<<grid_for(n, 8), 256, 0, (cudaStream_t)stream>>>(dZ, Z, norms, idx, n, d, scale, G);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_sgemm_f32(int32_t trans_a, int32_t trans_b, int32_t M, int32_t N, int32_t K, float alpha,
                   const float* A, int32_t lda, const float* B, int32_t ldb, float beta, float* C,
                   int32_t ldc, void* stream) {
  QREC_REQUIRE(M >= 0 && N >= 0 && K >= 0, "qrec_sgemm_f32: negative dimension");
  if (M == 0 || N == 0) return QREC_OK;
  QREC_REQUIRE(A && B && C, "qrec_sgemm_f32: null pointer");
  const long long tiles = (long long)((M + 63) / 64) * ((N + 63) / 64);
  cudaStream_t st = (cudaStream_t)stream;
  // tall-skinny fast path: [M, <=64] x [<=64, <=64] with 16-byte aligned rows (the NGCF layer transforms)
  if (!trans_a && M >= 4096 && N <= 64 && K <= 64 && (N % 4) == 0 && (K % 4) == 0 && (lda % 4) == 0 && (ldc % 4) == 0 &&
      (reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(C) & 15) == 0) {
    const int grid = grid_for(M, 128);
    if (trans_b) sgemm_skinny_kernel<true><<<grid, 128, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    else sgemm_skinny_kernel<false><<<grid, 128, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc);
    QREC_LAUNCH_CHECK();
    return QREC_OK;
  }
  int ksplit = 1;
  const long long target = (long long)sm_count() * 4;
  if (tiles < target / 2 && K >= 4096) {
    ksplit = (int)((target + tiles - 1) / tiles);
    if (ksplit > (K + 1023) / 1024) ksplit = (K + 1023) / 1024;
    if (ksplit < 1) ksplit = 1;
  }
  if (ksplit > 1) {
    scale_matrix_kernel<<<grid_for((long long)M * N, 1024), 256, 0, st>>>(C, M, N, ldc, beta);
    QREC_LAUNCH_CHECK();
  }
  const int grid = grid_for(tiles * ksplit, 1);
  if (!trans_a && !trans_b) sgemm_kernel<false, false><<<grid, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, ksplit);
  else if (trans_a && !trans_b) sgemm_kernel<true, false><<<grid, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, ksplit);
  else if (!trans_a && trans_b) sgemm_kernel<false, true><<<grid, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, ksplit);
  else sgemm_kernel<true, true><<<grid, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, beta, C, ldc, ksplit);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_ngcf_act_fwd_f32(const float* Zin, int64_t n_rows, int32_t d, float keep, int32_t training,
                          uint64_t seed, uint32_t tag, uint32_t step, float* H, float* out,
                          int32_t ld_out, float* norms, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && d >= 1 && keep > 0.f && keep <= 1.f, "qrec_ngcf_act_fwd_f32: bad argument");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(Zin && H && out && norms, "qrec_ngcf_act_fwd_f32: null pointer");
  ngcf_act_fwd_kernel<<<grid_for(n_rows, 8), 256, 0, (cudaStream_t)stream>>>(
      Zin, n_rows, d, keep, training, (uint32_t)seed, (uint32_t)(seed >> 32), tag, step, H, out, ld_out, norms);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_ngcf_act_bwd_f32(const float* dOut, int32_t ld_dout, const float* dH_extra, const float* H, const float* Zin,
                          const float* norms, int64_t n_rows, int32_t d, float keep, int32_t training,
                          uint64_t seed, uint32_t tag, uint32_t step, float* dZ, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && d >= 1 && keep > 0.f && keep <= 1.f, "qrec_ngcf_act_bwd_f32: bad argument");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(dOut && H && Zin && norms && dZ, "qrec_ngcf_act_bwd_f32: null pointer");
  ngcf_act_bwd_kernel<<<grid_for(n_rows, 8), 256, 0, (cudaStream_t)stream>>>(
      dOut, ld_dout, dH_extra, H, Zin, norms, n_rows, d, keep, training, (uint32_t)seed, (uint32_t)(seed >> 32), tag, step, dZ);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_mul_f32(float* dst, const float* a, const float* b, int64_t n, void* stream) {
  QREC_REQUIRE(n >= 0, "qrec_mul_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(dst && a && b, "qrec_mul_f32: null pointer");
  mul_kernel<<<grid_for(n, 1024), 256, 0, (cudaStream_t)stream>>>(dst, a, b, n);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_gather_rows_f32(const float* T, const int32_t* idx, int64_t n, int32_t d, float* out,
                         int32_t ld_out, void* stream) {
  QREC_REQUIRE(n >= 0 && d >= 4 && d % 4 == 0 && ld_out % 4 == 0, "qrec_gather_rows_f32: bad shape (d, ld multiples of 4)");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(T && idx && out, "qrec_gather_rows_f32: null pointer");
  gather_rows_kernel<<<grid_for(n * (d / 4), 256), 256, 0, (cudaStream_t)stream>>>(T, idx, n, d / 4, out, ld_out);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_scatter_add_rows_f32(float* G, const int32_t* idx, int64_t n, int32_t d, const float* src,
                              int32_t ld_src, float scale, void* stream) {
  QREC_REQUIRE(n >= 0 && d >= 4 && d % 4 == 0 && ld_src % 4 == 0, "qrec_scatter_add_rows_f32: bad shape");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(G && idx && src, "qrec_scatter_add_rows_f32: null pointer");
  scatter_add_rows_kernel<<<grid_for(n * (d / 4), 256), 256, 0, (cudaStream_t)stream>>>(G, idx, n, d / 4, src, ld_src, scale);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_bucket_requests(const int32_t* ids, int64_t n, int32_t rows_per_rank, int32_t world, int32_t cap, int32_t* count,
                         int32_t* send, int32_t* pos, int32_t* overflow, void* stream) {
  QREC_REQUIRE(n >= 0 && rows_per_rank >= 1 && world >= 1 && cap >= 1, "qrec_bucket_requests: bad argument");
  QREC_REQUIRE(count && send && overflow && (n == 0 || (ids && pos)), "qrec_bucket_requests: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  QREC_CUDA(cudaMemsetAsync(count, 0, sizeof(int32_t) * world, st));
  QREC_CUDA(cudaMemsetAsync(send, 0xff, sizeof(int32_t) * (size_t)world * cap, st));      // -1 = empty slot
  if (n == 0) return QREC_OK;
  bucket_requests_kernel<<<grid_for(n, 256), 256, 0, st>>>(ids, n, rows_per_rank, world, cap, count, send, pos, overflow);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_gemv_t_f32(const float* A, int32_t lda, int64_t rows, int32_t cols, const float* v, float alpha, float beta, float* out,
                    void* stream) {
  QREC_REQUIRE(rows >= 0 && cols >= 1 && lda >= cols, "qrec_gemv_t_f32: bad shape");
  QREC_REQUIRE(out && (A || rows == 0), "qrec_gemv_t_f32: null pointer");
  QREC_REQUIRE(beta == 0.f || beta == 1.f, "qrec_gemv_t_f32: beta must be 0 (overwrite) or 1 (accumulate)");
  cudaStream_t st = (cudaStream_t)stream;
  if (beta == 0.f) QREC_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)cols, st));
  if (rows == 0) return QREC_OK;
  const int rows_per_block = 128;
  const long long blocks = (rows + rows_per_block - 1) / rows_per_block;
  gemv_t_kernel<<<(int)blocks, 256, 0, st>>>(A, lda, rows, cols, v, alpha, out, rows_per_block);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_neumf_head_f32(int32_t mode, int32_t training, const float* UG, const float* IG,
                        const float* H3, const float* h_mf, const float* h_mlp, const float* r,
                        int64_t n, int32_t d, float reg, double* loss, float* y_out, float* dz_out,
                        float* GMF, float* dUG, float* dIG, float* dH3, void* stream) {
  QREC_REQUIRE(mode >= 0 && mode <= 2 && n >= 0 && d >= 1, "qrec_neumf_head_f32: bad argument");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(mode == 1 || (UG && IG && h_mf), "qrec_neumf_head_f32: GMF inputs missing");
  QREC_REQUIRE(mode == 0 || (H3 && h_mlp), "qrec_neumf_head_f32: MLP inputs missing");
  QREC_REQUIRE(!training || (r && loss && dz_out), "qrec_neumf_head_f32: training outputs missing");
  QREC_REQUIRE(!training || mode == 1 || (GMF && dUG && dIG), "qrec_neumf_head_f32: GMF gradient buffers missing");
  QREC_REQUIRE(!training || mode == 0 || dH3, "qrec_neumf_head_f32: dH3 missing");
  neumf_head_kernel<<<grid_for(n, 8), 256, 0, (cudaStream_t)stream>>>(mode, training, UG, IG, H3, h_mf, h_mlp, r, n, d, reg,
                                                                      loss, y_out, dz_out, GMF, dUG, dIG, dH3);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_mask_rated_f32(float* scores, int32_t n_rows, int64_t ld, const int32_t* users,
                        const int64_t* rowptr, const int32_t* cols, float value, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && ld >= 0, "qrec_mask_rated_f32: bad shape");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(scores && users && rowptr, "qrec_mask_rated_f32: null pointer");
  mask_rated_kernel<<<grid_for(n_rows, 8), 256, 0, (cudaStream_t)stream>>>(scores, n_rows, ld, users,
                                                                         reinterpret_cast<const long long*>(rowptr), cols, value);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
