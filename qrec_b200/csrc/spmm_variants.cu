// K2 experiments (d = 64, row-split): the production kernel is spmm_csr_kernel<16,1> in
// graph_kernels.cu -- 8 gathered rows in flight per lane group, issued and consumed in lock step.  The variants here change only HOW MANY loads are outstanding and how
// many warps are resident, never the order of the floating-point operations, so every variant must
// reproduce the production kernel bit for bit:
//   0  G=8,  4 CTAs/SM   the production configuration (A/B control)
//   1  G=8,  5 CTAs/SM   <= 48 registers
//   2  G=8,  6 CTAs/SM   <= 40 registers
//   3  G=16, 3 CTAs/SM   16 gathers per batch
//   4  G=4 x 2 buffers, 3 CTAs/SM   software pipeline: the next group's gathers are issued before the
//                                   current group is consumed (8 in flight continuously)
//   5  G=8 x 2 buffers, 2 CTAs/SM   the same with 16 in flight
//   6  variant 0 + L2 residency hints: (col, val) streamed (L2::evict_first, no L1 allocation), X rows evict_last
// Reached only through qrec_spmm_csr_rowsplit_var_f32 (tests/test_gpu_spmm_variants.py, tools/bench_graph.py).
#include "common.h"
#include "device.cuh"

namespace {

using qrec::fma4;

constexpr int LPR = 16;   // lanes per row: d = 64, one float4 per lane

__device__ __forceinline__ void store_row(float* __restrict__ Y, float* __restrict__ acc, float acc_scale, long long r,
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

// L2 residency hints (variant 6): the (col, val) arrays are read once and only pollute the L2, the gathered X rows are
// what should stay -- stream the former (evict_first, no L1 allocation), pin the latter (evict_last).
__device__ __forceinline__ unsigned long long l2_policy_evict_first() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
template <bool HINT>
__device__ __forceinline__ int ld_index(const int* p, unsigned long long pol) {
  if (!HINT) return __ldg(p);
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
template <bool HINT>
__device__ __forceinline__ float ld_value(const float* p, unsigned long long pol) {
  if (!HINT) return __ldg(p);
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
  return v;
}
template <bool HINT>
__device__ __forceinline__ float4 ld_row(const float4* p, unsigned long long pol) {
  if (!HINT) return __ldg(p);
  float4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}

// lock-step batches of G gathers (the production structure with G and the occupancy as parameters)
template <int G, int MINB, bool HINT = false>
__global__ void __launch_bounds__(256, MINB)
spmm_rowsplit_batch_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                           const float* __restrict__ vals, const float* __restrict__ X, float* __restrict__ Y,
                           float* __restrict__ acc, float acc_scale) {
  const unsigned long long pol_stream = HINT ? l2_policy_evict_first() : 0ULL, pol_keep = HINT ? l2_policy_evict_last() : 0ULL;
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
      c = ld_index<HINT>(cols + start + l, pol_stream);
      w = ld_value<HINT>(vals + start + l, pol_stream);
    }
    for (long long base = start; base < end; base += LPR) {
      const int m = (end - base) < LPR ? (int)(end - base) : LPR;
      int cn = 0;
      float wn = 0.f;
      if (base + LPR + l < end) {
        cn = ld_index<HINT>(cols + base + LPR + l, pol_stream);
        wn = ld_value<HINT>(vals + base + LPR + l, pol_stream);
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
          x[q] = (t + q) < m ? ld_row<HINT>(reinterpret_cast<const float4*>(X + (size_t)cc[q] * 64) + l, pol_keep)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int q = 0; q < G; ++q) fma4(a, ww[q], x[q]);
      }
      c = cn;
      w = wn;
    }
    store_row(Y, acc, acc_scale, r, l, a);
  }
}

// software pipeline: two register buffers of G gathered rows; group g+1 is issued before group g is
// consumed.  Groups never straddle a 16-entry index chunk (G divides 16); the chunk's (col, val)
// registers advance inside issue().  FMAs run in non-zero order, exactly as in the batch kernel.
template <int G, int MINB>
__global__ void __launch_bounds__(256, MINB)
spmm_rowsplit_pipe_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                          const float* __restrict__ vals, const float* __restrict__ X, float* __restrict__ Y,
                          float* __restrict__ acc, float acc_scale) {
  static_assert(LPR % G == 0, "a group must not straddle an index chunk");
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const unsigned gmask = ((1u << LPR) - 1u) << (sub * LPR);
  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 2 + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * 2;
  for (long long r = group; r < n_rows; r += ngroups) {
    const long long start = __ldg(rowptr + r), end = __ldg(rowptr + r + 1);
    const int len = (int)(end - start);
    const int ng = (len + G - 1) / G;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    // index registers of the chunk being issued from, and of the one after it
    int c = 0, cn = 0, cur_chunk = 0;
    float w = 0.f, wn = 0.f;
    if (l < len) {
      c = __ldg(cols + start + l);
      w = __ldg(vals + start + l);
    }
    if (LPR + l < len) {
      cn = __ldg(cols + start + LPR + l);
      wn = __ldg(vals + start + LPR + l);
    }
    float4 xa[G], xb[G];
    float wa[G], wb[G];
    auto issue = [&](float4* x, float* ww, int g) {
      const int t0 = g * G;                              // first non-zero of the group, relative to start
      if (t0 / LPR > cur_chunk) {                        // groups are issued in order: at most one step
        c = cn;
        w = wn;
        ++cur_chunk;
        const int nxt = (cur_chunk + 1) * LPR + l;
        cn = 0;
        wn = 0.f;
        if (nxt < len) {
          cn = __ldg(cols + start + nxt);
          wn = __ldg(vals + start + nxt);
        }
      }
#pragma unroll
      for (int q = 0; q < G; ++q) {
        const int cc = __shfl_sync(gmask, c, sub * LPR + ((t0 + q) & (LPR - 1)));
        ww[q] = __shfl_sync(gmask, w, sub * LPR + ((t0 + q) & (LPR - 1)));
        if (t0 + q < len) {
          x[q] = __ldg(reinterpret_cast<const float4*>(X + (size_t)cc * 64) + l);
        } else {
          x[q] = make_float4(0.f, 0.f, 0.f, 0.f);
          ww[q] = 0.f;
        }
      }
    };
    if (ng > 0) issue(xa, wa, 0);
    for (int g = 0; g < ng; g += 2) {
      if (g + 1 < ng) issue(xb, wb, g + 1);
#pragma unroll
      for (int q = 0; q < G; ++q) fma4(a, wa[q], xa[q]);
      if (g + 2 < ng) issue(xa, wa, g + 2);
      if (g + 1 < ng) {
#pragma unroll
        for (int q = 0; q < G; ++q) fma4(a, wb[q], xb[q]);
      }
    }
    store_row(Y, acc, acc_scale, r, l, a);
  }
}

}  // namespace

extern "C" int qrec_spmm_csr_rowsplit_var_f32(int32_t variant, int32_t n_rows, const int64_t* rowptr,
                                              const int32_t* cols, const float* vals, const float* X, float* Y,
                                              int32_t d, float* acc, float acc_scale, void* stream) {
  QREC_REQUIRE(variant >= 0 && variant <= 6, "qrec_spmm_csr_rowsplit_var_f32: variant %d (0..6)", variant);
  QREC_REQUIRE(d == 64, "qrec_spmm_csr_rowsplit_var_f32: experiments are d = 64 only (got %d)", d);
  QREC_REQUIRE(n_rows >= 0, "qrec_spmm_csr_rowsplit_var_f32: n_rows < 0");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && X && Y, "qrec_spmm_csr_rowsplit_var_f32: null pointer");   // cols / vals may be null when nnz = 0
  QREC_REQUIRE(X != Y, "qrec_spmm_csr_rowsplit_var_f32: X and Y must not alias");
  QREC_REQUIRE(((reinterpret_cast<uintptr_t>(X) | reinterpret_cast<uintptr_t>(Y) | reinterpret_cast<uintptr_t>(acc)) & 15) == 0,
               "qrec_spmm_csr_rowsplit_var_f32: tables must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = qrec::capped_grid(((long long)n_rows + 15) / 16, 8);   // 16 lane groups (rows) per 256-thread block
  const long long* rp = reinterpret_cast<const long long*>(rowptr);
#define QREC_VAR(KERNEL) KERNEL<<<grid, 256, 0, st>>>(n_rows, rp, cols, vals, X, Y, acc, acc_scale)
  switch (variant) {
    case 0: QREC_VAR((spmm_rowsplit_batch_kernel<8, 4>)); break;
    case 1: QREC_VAR((spmm_rowsplit_batch_kernel<8, 5>)); break;
    case 2: QREC_VAR((spmm_rowsplit_batch_kernel<8, 6>)); break;
    case 3: QREC_VAR((spmm_rowsplit_batch_kernel<16, 3>)); break;
    case 4: QREC_VAR((spmm_rowsplit_pipe_kernel<4, 3>)); break;
    case 6: QREC_VAR((spmm_rowsplit_batch_kernel<8, 4, true>)); break;
    default: QREC_VAR((spmm_rowsplit_pipe_kernel<8, 2>)); break;
  }
#undef QREC_VAR
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
