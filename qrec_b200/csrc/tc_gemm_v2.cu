// K5 v2: the same product as tc_gemm.cu,
//     C[M,N] = epilogue( A[M,K] * B )          fp32 in HBM, TF32 wgmma, fp32 accumulate in registers
// rebuilt as a persistent, warp-specialised pipeline (model/ranking/NeuMF.py:39-50 is still the caller):
//   * one CTA per SM keeps ONE 64-column block of B resident in shared memory for its whole life
//     (all K/32 k-blocks, transposed / rounded to TF32 once) and walks the 128-row tiles of A that
//     belong to that column block;
//   * warp 4 (one lane): TMA producer -- cp.async.bulk.tensor.2d loads 128 x 32 fp32 boxes of A through
//     a SWIZZLE_128B tensor map straight into the K-major layout the wgmma descriptors expect, NSTAGE-deep
//     ring, mbarrier complete_tx; out-of-range rows / columns are zero-filled by the copy engine;
//   * warps 0-3 (one warpgroup) consume the ring in order: per stage two wgmma.mma_async m64n64k8 TF32 per
//     8-wide k-step (csrc/wgmma.cuh), accumulator in registers; the stage goes back to the producer once the
//     group has retired, so the copy engine runs ahead into the next tile while the epilogue applies
//     bias / ReLU / ReLU-mask and writes whole 256-byte rows through a shared-memory tile.
//     (The ring is consumed strictly in order: an mbarrier parity wait cannot tell a phase two ahead from
//     the one before, so a second consumer taking every other tile could not wait on the same ring.)
// A reaches the tensor cores as raw fp32 bits (the TF32 MMA drops the low 13 mantissa bits: truncation,
// error <= 2^-10 per operand instead of 2^-11 with the cvt.rna staging of v1); B is rounded (rna) while
// it is staged.  K <= 320 (B block + 4-stage ring + epilogue tile = 178 KB of the 227 KB).
#include <cuda.h>

#include "common.h"
#include "device.cuh"
#include "wgmma.cuh"

namespace {

using namespace qrec;
using wg::sw_off;
using wg::to_tf32;

constexpr int BM = 128, BN = 64, BK = 32;           // BK fp32 = 128 B = one swizzle span
constexpr int NSTAGE = 4;
constexpr int STAGE_A = BM * 128;                   // 16 KB per A stage
constexpr int KB_B = BN * 128;                      // 8 KB per resident B k-block
constexpr int MAX_K = 320;
constexpr int EPI_PITCH = BN + 4;                   // floats; 272-byte rows
constexpr int EPI_BYTES = BM * EPI_PITCH * 4;
constexpr int NTHREADS = 160;                       // the consumer warpgroup + the producer warp

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void group_sync() {     // the 128 threads of the consumer warpgroup
  asm volatile("bar.sync 1, 128;" ::: "memory");
}

enum Epilogue { EPI_NONE = 0, EPI_BIAS_RELU = 1, EPI_RELU_MASK = 2, EPI_BIAS = 3 };

// grid = n_blocks * ctas_per_n; CTA c owns column block c % n_blocks and the row tiles
// c / n_blocks, c / n_blocks + ctas_per_n, ...
template <bool B_IS_NK>
__global__ void __launch_bounds__(NTHREADS, 1)
tc_gemm_tf32_v2_kernel(const __grid_constant__ CUtensorMap mapA, int M, int N, int K,
                       const float* __restrict__ B, int ldb, float* __restrict__ C, int ldc, int epi,
                       const float* __restrict__ bias, const float* __restrict__ mask, int ldmask,
                       int n_blocks, int ctas_per_n) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[NSTAGE], empty_bar[NSTAGE];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int nkb = (K + BK - 1) / BK;
  uint8_t* sA = smem;                                // NSTAGE x 16 KB
  uint8_t* sB = smem + NSTAGE * STAGE_A;             // nkb x 8 KB, resident
  uint8_t* sE = sB + nkb * KB_B;                     // EPI_BYTES
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nb = blockIdx.x % n_blocks, first_tile = blockIdx.x / n_blocks;
  const int n0 = nb * BN;
  const int m_tiles = (M + BM - 1) / BM;

  if (tid == 0) {
    for (int s = 0; s < NSTAGE; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 4);                   // one arrival per warp of the consuming warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
  }
  // resident B block: every thread stages a share of the nkb k-blocks, rounded to TF32, K-major
  for (int kb = 0; kb < nkb; ++kb) {
    uint8_t* dst = sB + kb * KB_B;
    const int k0 = kb * BK;
    if (B_IS_NK) {                                   // B [N,K] row-major: already K-major
      for (int e = tid; e < BN * 8; e += NTHREADS) {
        const int row = e >> 3, c = e & 7;
        const int gn = n0 + row, gk = k0 + c * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gn < N && gk < K) v = __ldg(reinterpret_cast<const float4*>(B + (size_t)gn * ldb + gk));
        *reinterpret_cast<float4*>(dst + sw_off(row, c * 4)) = to_tf32(v);
      }
    } else {                                         // B [K,N] row-major: transposed on the way in
      for (int e = tid; e < BN * BK; e += NTHREADS) {
        const int n = e & 63, k = e >> 6;
        const int gn = n0 + n, gk = k0 + k;
        const float v = (gn < N && gk < K) ? __ldg(B + (size_t)gk * ldb + gn) : 0.f;      // coalesced along n
        *reinterpret_cast<float*>(dst + sw_off(n, k)) = to_tf32(v);
      }
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy writes -> async proxy (wgmma)
  __syncthreads();

  if (warp == 4) {
    // ===== TMA producer =====
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int mt = first_tile; mt < m_tiles; mt += ctas_per_n) {
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);                    // slot free (passes on first use)
          mbar_expect_tx(&full_bar[stage], STAGE_A);
          tma_load_2d(sA + stage * STAGE_A, &mapA, kb * BK, mt * BM, &full_bar[stage]);
          if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===== consumer warpgroup =====
    float* tile = reinterpret_cast<float*>(sE);
    const int c4 = (tid & 15) * 4;                   // 16 threads cover one 64-float row on the way out
    const int col = n0 + c4;
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((epi == EPI_BIAS_RELU || epi == EPI_BIAS) && col < N) {
      bv.x = bias[col];
      if (col + 1 < N) bv.y = bias[col + 1];
      if (col + 2 < N) bv.z = bias[col + 2];
      if (col + 3 < N) bv.w = bias[col + 3];
    }
    const bool vec_ok = (col + 3 < N) && ((ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int mt = first_tile; mt < m_tiles; mt += ctas_per_n) {
      float acc[2][32];
      for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);                           // the copy engine has landed this stage
        __syncwarp();                                                  // wgmma is warp-aligned: reconverge after the spin
        wg::fence();
        const uint64_t da = wg::desc_sw128(smem_u32(sA + stage * STAGE_A));
        const uint64_t db = wg::desc_sw128(smem_u32(sB + kb * KB_B));
#pragma unroll
        for (int k4 = 0; k4 < BK / 8; ++k4) {                          // +2 = 32 bytes (8 tf32) along K
          const uint32_t accumulate = (kb > 0 || k4 > 0) ? 1u : 0u;
          wg::mma_m64n64k8_tf32(acc[0], da + (uint64_t)(k4 * 2), db + (uint64_t)(k4 * 2), accumulate);
          wg::mma_m64n64k8_tf32(acc[1], da + (uint64_t)(STAGE_A / 2 >> 4) + (uint64_t)(k4 * 2), db + (uint64_t)(k4 * 2), accumulate);
        }
        wg::commit();
        wg::wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[stage]);                 // this warp's share of the stage is read
        if (++stage == NSTAGE) { stage = 0; phase ^= 1; }
      }
      group_sync();                                  // the previous tile's rows are out of the staging tile
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 32; e += 2)
          *reinterpret_cast<float2*>(tile + (64 * h + wg::frag_row(warp, lane, e)) * EPI_PITCH + wg::frag_col(lane, e)) =
              make_float2(acc[h][e], acc[h][e + 1]);
      group_sync();
      for (int rr = tid >> 4; rr < BM; rr += 8) {    // eight rows per pass, 256 B each
        const int row = mt * BM + rr;
        if (row >= M || col >= N) continue;
        float4 v = *reinterpret_cast<const float4*>(tile + rr * EPI_PITCH + c4);
        if (epi == EPI_BIAS_RELU) {
          v.x = fmaxf(v.x + bv.x, 0.f); v.y = fmaxf(v.y + bv.y, 0.f); v.z = fmaxf(v.z + bv.z, 0.f); v.w = fmaxf(v.w + bv.w, 0.f);
        } else if (epi == EPI_BIAS) {
          v.x += bv.x; v.y += bv.y; v.z += bv.z; v.w += bv.w;
        } else if (epi == EPI_RELU_MASK) {
          const float* mk = mask + (size_t)row * ldmask + col;
          v.x = mk[0] > 0.f ? v.x : 0.f;
          if (col + 1 < N) v.y = mk[1] > 0.f ? v.y : 0.f;
          if (col + 2 < N) v.z = mk[2] > 0.f ? v.z : 0.f;
          if (col + 3 < N) v.w = mk[3] > 0.f ? v.w : 0.f;
        }
        float* dst = C + (size_t)row * ldc + col;
        if (vec_ok) {
          *reinterpret_cast<float4*>(dst) = v;
        } else {
          dst[0] = v.x;
          if (col + 1 < N) dst[1] = v.y;
          if (col + 2 < N) dst[2] = v.z;
          if (col + 3 < N) dst[3] = v.w;
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled through the runtime (libqrec.so links cudart statically and never libcuda)
EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

}  // namespace

extern "C" int qrec_tc_gemm_tf32_v2(int32_t b_is_nk, int32_t M, int32_t N, int32_t K, const float* A,
                                    int32_t lda, const float* B, int32_t ldb, float* C, int32_t ldc,
                                    int32_t epilogue, const float* bias, const float* mask,
                                    int32_t ldmask, void* stream) {
  QREC_REQUIRE(M >= 0 && N >= 0 && K >= 1, "qrec_tc_gemm_tf32_v2: bad dimensions");
  if (M == 0 || N == 0) return QREC_OK;
  QREC_REQUIRE(A && B && C, "qrec_tc_gemm_tf32_v2: null pointer");
  QREC_REQUIRE(K <= MAX_K, "qrec_tc_gemm_tf32_v2: K=%d exceeds %d (the resident B block); use qrec_tc_gemm_tf32", K, MAX_K);
  QREC_REQUIRE(K % 4 == 0 && lda % 4 == 0 && lda >= K && (reinterpret_cast<uintptr_t>(A) & 15) == 0,
               "qrec_tc_gemm_tf32_v2: A must be 16-byte aligned with K and lda multiples of 4");
  QREC_REQUIRE(!b_is_nk || (ldb % 4 == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0),
               "qrec_tc_gemm_tf32_v2: [N,K] B must be 16-byte aligned with ldb a multiple of 4");
  QREC_REQUIRE(epilogue >= 0 && epilogue <= 3, "qrec_tc_gemm_tf32_v2: unknown epilogue %d", epilogue);
  QREC_REQUIRE((epilogue != EPI_BIAS_RELU && epilogue != EPI_BIAS) || bias, "qrec_tc_gemm_tf32_v2: bias epilogue without bias");
  QREC_REQUIRE(epilogue != EPI_RELU_MASK || mask, "qrec_tc_gemm_tf32_v2: mask epilogue without mask");
  const int sms = sm_count();
  const int n_blocks = (N + BN - 1) / BN;
  QREC_REQUIRE(n_blocks <= sms, "qrec_tc_gemm_tf32_v2: N=%d needs more column blocks than SMs; use qrec_tc_gemm_tf32", N);
  EncodeTiledFn enc = encode_tiled();
  QREC_REQUIRE(enc != nullptr, "qrec_tc_gemm_tf32_v2: cuTensorMapEncodeTiled not available from this driver");
  alignas(64) CUtensorMap mapA;
  const cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)M};             // innermost first
  const cuuint64_t gstride[1] = {(cuuint64_t)lda * sizeof(float)};       // bytes between rows
  const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};            // 32 fp32 (128 B) x 128 rows
  const cuuint32_t estride[2] = {1, 1};
  const CUresult rc = enc(&mapA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(A), gdim, gstride, box, estride,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  QREC_REQUIRE(rc == CUDA_SUCCESS, "qrec_tc_gemm_tf32_v2: cuTensorMapEncodeTiled failed (%d)", (int)rc);
  const int m_tiles = (M + BM - 1) / BM;
  int ctas_per_n = sms / n_blocks;
  if (ctas_per_n > m_tiles) ctas_per_n = m_tiles;
  if (ctas_per_n < 1) ctas_per_n = 1;
  const int nkb = (K + BK - 1) / BK;
  const int smem = NSTAGE * STAGE_A + nkb * KB_B + EPI_BYTES + 1024;
  QREC_CUDA(allow_dynamic_smem(b_is_nk ? (const void*)tc_gemm_tf32_v2_kernel<true> : (const void*)tc_gemm_tf32_v2_kernel<false>, smem));
  const int grid = n_blocks * ctas_per_n;
  cudaStream_t st = (cudaStream_t)stream;
  if (b_is_nk)
    tc_gemm_tf32_v2_kernel<true><<<grid, NTHREADS, smem, st>>>(mapA, M, N, K, B, ldb, C, ldc, epilogue, bias, mask, ldmask, n_blocks, ctas_per_n);
  else
    tc_gemm_tf32_v2_kernel<false><<<grid, NTHREADS, smem, st>>>(mapA, M, N, K, B, ldb, C, ldc, epilogue, bias, mask, ldmask, n_blocks, ctas_per_n);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
