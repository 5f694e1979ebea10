// K5 building block: the tensor-core GEMM of NeuMF's MLP (model/ranking/NeuMF.py:39-50),
//     C[M,N] = epilogue( A[M,K] * B )          fp32 in HBM, TF32 wgmma, fp32 accumulate in registers
// written directly against the sm_90a tensor-core path:
//   * operands are staged in shared memory in the canonical K-major SWIZZLE_128B layout
//     (rows of 32 fp32 = 128 B, 8-row 1024 B atoms, 16-byte chunk index XOR row%8) -- the MLP's
//     weight matrices are [K,N] row-major, so they are transposed on the way into shared memory;
//   * the CTA is one warpgroup: per 8-wide k-step it issues two wgmma.mma_async m64n64k8 TF32
//     (rows 0-63 and 64-127 of the tile) from shared-memory descriptors (csrc/wgmma.cuh); the
//     128 x 64 fp32 accumulator lives in registers (64 per thread);
//   * 2-stage ring: the MMAs of k-block kb run while the stores of k-block kb+1 wait only for the
//     group of kb-1 (wgmma.wait_group 1 + a CTA barrier before a stage is rewritten);
//   * global loads are register-staged one k-block ahead (their latency overlaps the MMAs), the
//     epilogue is parked in shared memory and written as whole 256-byte rows with bias / ReLU /
//     ReLU-mask applied.
// Tile: 128 x 64 per CTA, 128 threads.
#include "common.h"
#include "device.cuh"
#include "wgmma.cuh"

namespace {

using qrec::smem_u32;
using wg::sw_off;
using wg::to_tf32;

constexpr int BM = 128, BN = 64, BK = 32;           // BK fp32 = 128 B = one swizzle span
constexpr int STAGE_A = BM * 128, STAGE_B = BN * 128;
constexpr int SMEM_BYTES = 2 * (STAGE_A + STAGE_B) + 1024;   // + alignment slack

enum Epilogue { EPI_NONE = 0, EPI_BIAS_RELU = 1, EPI_RELU_MASK = 2, EPI_BIAS = 3 };

template <bool B_IS_NK>
__global__ void __launch_bounds__(128)
tc_gemm_tf32_kernel(int M, int N, int K, const float* __restrict__ A, int lda,
                    const float* __restrict__ B, int ldb, float* __restrict__ C, int ldc,
                    int epi, const float* __restrict__ bias, const float* __restrict__ mask,
                    int ldmask) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  // stage s: A tile at smem + s*(STAGE_A+STAGE_B), B tile right behind it (computed, not looked up:
  // a pointer array indexed by the stage lands in local memory)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  float acc[2][32];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 32; ++e) acc[h][e] = 0.f;

  const int nkb = (K + BK - 1) / BK;
  // Register-staged global loads, one k-block ahead: the loads of block kb+1 are issued before the
  // shared-memory stores / MMAs of block kb, so their latency overlaps the tensor-core work.
  float4 ra[8];
  float4 rb4[4];
  float rb1[16];
  auto load_block = [&](int kb) {
    const int k0 = kb * BK;
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int row = (tid >> 3) + 16 * p, c = tid & 7;
      const int gm = m0 + row, gk = k0 + c * 4;
      ra[p] = (gm < M && gk < K) ? __ldg(reinterpret_cast<const float4*>(A + (size_t)gm * lda + gk))
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (B_IS_NK) {
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int row = (tid >> 3) + 16 * p, c = tid & 7;
        const int gn = n0 + row, gk = k0 + c * 4;
        rb4[p] = (gn < N && gk < K) ? __ldg(reinterpret_cast<const float4*>(B + (size_t)gn * ldb + gk))
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else {
#pragma unroll
      for (int p = 0; p < 16; ++p) {
        const int n = tid & 63, k = (tid >> 6) + 2 * p;
        const int gn = n0 + n, gk = k0 + k;
        rb1[p] = (gn < N && gk < K) ? __ldg(B + (size_t)gk * ldb + gn) : 0.f;     // coalesced along n
      }
    }
  };
  load_block(0);
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb & 1;
    uint8_t* const sA_s = smem + s * (STAGE_A + STAGE_B);
    uint8_t* const sB_s = sA_s + STAGE_A;
    if (kb >= 2) __syncthreads();          // every warp has retired the MMAs of kb-2 (wait_group 1 below): stage s is free
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int row = (tid >> 3) + 16 * p, c = tid & 7;
      *reinterpret_cast<float4*>(sA_s + sw_off(row, c * 4)) = to_tf32(ra[p]);
    }
    if (B_IS_NK) {
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int row = (tid >> 3) + 16 * p, c = tid & 7;
        *reinterpret_cast<float4*>(sB_s + sw_off(row, c * 4)) = to_tf32(rb4[p]);
      }
    } else {
#pragma unroll
      for (int p = 0; p < 16; ++p) {
        const int n = tid & 63, k = (tid >> 6) + 2 * p;
        *reinterpret_cast<float*>(sB_s + sw_off(n, k)) = to_tf32(rb1[p]);        // transposed into K-major
      }
    }
    if (kb + 1 < nkb) load_block(kb + 1);                                        // in flight during the MMAs
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes -> async proxy (wgmma)
    __syncthreads();
    wg::fence();
    const uint64_t da = wg::desc_sw128(smem_u32(sA_s)), db = wg::desc_sw128(smem_u32(sB_s));
#pragma unroll
    for (int k4 = 0; k4 < BK / 8; ++k4) {                              // +2 = 32 bytes (8 tf32) along K
      wg::mma_m64n64k8_tf32(acc[0], da + (uint64_t)(k4 * 2), db + (uint64_t)(k4 * 2), 1u);
      wg::mma_m64n64k8_tf32(acc[1], da + (uint64_t)(STAGE_A / 2 >> 4) + (uint64_t)(k4 * 2), db + (uint64_t)(k4 * 2), 1u);
    }
    wg::commit();
    wg::wait<1>();
  }
  wg::wait<0>();
  __syncthreads();                                  // every warp's MMAs are done: the operand stages are free
  // ---- epilogue: registers -> shared memory -> coalesced global rows.  The accumulator is parked in a
  // [128][64+4] fp32 tile (row pitch 272 B); then every warp writes whole 256-byte rows.
  float* tile = reinterpret_cast<float*>(smem);
  constexpr int PITCH = BN + 4;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 32; e += 2)
      *reinterpret_cast<float2*>(tile + (64 * h + wg::frag_row(warp, lane, e)) * PITCH + wg::frag_col(lane, e)) =
          make_float2(acc[h][e], acc[h][e + 1]);
  __syncthreads();
  {
    const int c4 = (tid & 15) * 4;                 // 16 threads cover one 64-float row
    const int col = n0 + c4;
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool vec_ok = (col + 3 < N) && ((ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
    if ((epi == EPI_BIAS_RELU || epi == EPI_BIAS) && col < N) {
      bv.x = bias[col];
      if (col + 1 < N) bv.y = bias[col + 1];
      if (col + 2 < N) bv.z = bias[col + 2];
      if (col + 3 < N) bv.w = bias[col + 3];
    }
    for (int rr = tid >> 4; rr < BM; rr += 8) {
      const int row = m0 + rr;
      if (row >= M || col >= N) continue;
      float4 v = *reinterpret_cast<const float4*>(tile + rr * PITCH + c4);
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

}  // namespace

extern "C" int qrec_tc_gemm_tf32(int32_t b_is_nk, int32_t M, int32_t N, int32_t K, const float* A,
                                 int32_t lda, const float* B, int32_t ldb, float* C, int32_t ldc,
                                 int32_t epilogue, const float* bias, const float* mask,
                                 int32_t ldmask, void* stream) {
  QREC_REQUIRE(M >= 0 && N >= 0 && K >= 1, "qrec_tc_gemm_tf32: bad dimensions");
  if (M == 0 || N == 0) return QREC_OK;
  QREC_REQUIRE(A && B && C, "qrec_tc_gemm_tf32: null pointer");
  QREC_REQUIRE(K % 4 == 0 && lda % 4 == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0,
               "qrec_tc_gemm_tf32: A must be 16-byte aligned with K and lda multiples of 4");
  QREC_REQUIRE(!b_is_nk || (ldb % 4 == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0),
               "qrec_tc_gemm_tf32: [N,K] B must be 16-byte aligned with ldb a multiple of 4");
  QREC_REQUIRE((M + BM - 1) / BM <= 65535, "qrec_tc_gemm_tf32: M=%d exceeds the 65535 x 128 rows of one launch; split the batch", M);
  QREC_REQUIRE(epilogue >= 0 && epilogue <= 3, "qrec_tc_gemm_tf32: unknown epilogue %d", epilogue);
  QREC_REQUIRE((epilogue != EPI_BIAS_RELU && epilogue != EPI_BIAS) || bias, "qrec_tc_gemm_tf32: bias epilogue without bias");
  QREC_REQUIRE(epilogue != EPI_RELU_MASK || mask, "qrec_tc_gemm_tf32: mask epilogue without mask");
  QREC_CUDA(qrec::allow_dynamic_smem(b_is_nk ? (const void*)tc_gemm_tf32_kernel<true> : (const void*)tc_gemm_tf32_kernel<false>,
                                      SMEM_BYTES));
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
  cudaStream_t st = (cudaStream_t)stream;
  if (b_is_nk) tc_gemm_tf32_kernel<true><<<grid, 128, SMEM_BYTES, st>>>(M, N, K, A, lda, B, ldb, C, ldc, epilogue, bias, mask, ldmask);
  else tc_gemm_tf32_kernel<false><<<grid, 128, SMEM_BYTES, st>>>(M, N, K, A, lda, B, ldb, C, ldc, epilogue, bias, mask, ldmask);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
