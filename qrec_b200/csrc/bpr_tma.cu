// K1, user-major, with the item rows staged through shared memory by the bulk-copy (TMA) engine -- the variant the
// north star names ("128-bit vectorised coalesced HBM row reads, TMA staging to shared memory").  Same step, same
// order, same sampler and the same scatter-add as bpr_sgd_usermajor_kernel (bpr_kernels.cu; reference:
// model/ranking/BPR.py:29-53): what changes is HOW the two item rows of a triple reach the lane group.  There every
// lane issues an LDG.E.128 per row (32 LSU lane-operations per triple); here ONE lane per row issues a 256-byte
// cp.async.bulk.shared::cluster.global into the group's staging slot, completion is signalled on an mbarrier, and the
// lanes read their 16-byte slices with LDS.128 -- the gathers leave the LSU/L1TEX path, which then carries only the
// scatter-adds (REDG.E.ADD.F32x4).  d = 64 only (16 lanes x float4 = one 256-byte row per bulk copy).
//
// Pipeline per lane group (16 lanes): the rows of the next 4 triples (8 rows, 2 KB) are requested while the current
// 4 are being computed: two staging slots, two mbarriers, phase bits tracked in registers.
#include "common.h"
#include "device.cuh"
#include "philox.cuh"
#include "bpr_step.cuh"

namespace {

using namespace qrec;
using namespace qrec::bpr;

constexpr int LPR = 16, G = 4, CH = 32, ROWS = 2 * G, GROUPS = 16;   // 256 threads = 16 lane groups
constexpr int STAGE_FLOATS = ROWS * 64;

// one 256-byte row: global -> this CTA's shared memory, completion counted on `bar`
__device__ __forceinline__ void bulk_row_load(float* smem_dst, const float* gsrc, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 256, [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(smem_u32(bar)) : "memory");
}

template <bool SAMPLE>
__global__ void __launch_bounds__(256, 3)
bpr_sgd_usermajor_tma_kernel(float* __restrict__ P, float* __restrict__ Q, int n_users, long long n,
                             const long long* __restrict__ rowptr, const int* __restrict__ i, const int* __restrict__ j,
                             float lr, float reg_u, float reg_i, double* loss, FusedSampler fs) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* stage_all = reinterpret_cast<float*>(smem_raw);                               // [GROUPS][2][ROWS][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage_all + GROUPS * 2 * STAGE_FLOATS);    // [GROUPS][2]
  constexpr int d = 64;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const int g_in_cta = (threadIdx.x >> 5) * 2 + sub;
  const unsigned gmask = ((1u << LPR) - 1u) << (sub * LPR);
  float* stage = stage_all + (size_t)g_in_cta * 2 * STAGE_FLOATS;
  uint64_t* bar = bars + g_in_cta * 2;
  if (l == 0) { mbar_init(bar, 1); mbar_init(bar + 1, 1); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  uint32_t phase0 = 0, phase1 = 0;

  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 2 + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * 2;
  const float a_u = lr * reg_u, a_i = lr * reg_i;
  const float one_m_au = 1.0f - a_u, one_m_ai = 1.0f - a_i;
  const long long nchunks = (n + CH - 1) / CH;
  float lsum = 0.f;
  for (long long ch = group; ch < nchunks; ch += ngroups) {
    const long long lo = ch * CH;
    const long long hi = (lo + CH) < n ? (lo + CH) : n;
    int a = 0, b = n_users - 1;                                   // user of triple lo: LPR-ary search of rowptr
    while (a < b) {
      const int len = b - a + 1;
      const int step = (len + LPR - 1) / LPR;
      int pp = a + (l + 1) * step - 1;
      if (pp > b) pp = b;
      const bool pred = __ldg(rowptr + pp + 1) > lo;
      const unsigned bal = (__ballot_sync(gmask, pred) & gmask) >> (sub * LPR);
      const int f = __ffs(bal) - 1;
      int pf = a + (f + 1) * step - 1;
      if (pf > b) pf = b;
      a = a + f * step;
      b = pf;
    }
    int uu = a;
    long long uend = __ldg(rowptr + uu + 1);
    float* prow = P + (size_t)uu * d + l * 4;
    float4 p = *reinterpret_cast<const float4*>(prow);
    float4 p0 = p;
    for (long long base = lo; base < hi; base += LPR) {
      const int m = (hi - base) < LPR ? (int)(hi - base) : LPR;
      int mi = 0, mj = 0;
      if (l < m) {
        mi = __ldg(i + base + l);
        if (SAMPLE) {
          int us = uu;
          long long ue = uend;
          while (ue <= base + l) { ++us; ue = __ldg(rowptr + us + 1); }
          mj = qrec::sample_negative(base + l, fs.epoch, fs.seed_lo, fs.seed_hi, fs.num_items, fs.rated_cols,
                                     __ldg(fs.rated_rowptr + us), __ldg(fs.rated_rowptr + us + 1));
          if (fs.j_out != nullptr) fs.j_out[base + l] = mj;
        } else {
          mj = __ldg(j + base + l);
        }
      }
      const int nsb = (m + G - 1) / G;
      // request the rows of sub-batch sb into staging slot sb & 1: lane 2f -> Q[i_f], lane 2f+1 -> Q[j_f]
      auto issue = [&](int sb) {
        const int t0 = sb * G;
        const int src = sub * LPR + ((t0 + (l >> 1)) & (LPR - 1));
        const int idi = __shfl_sync(gmask, mi, src), idj = __shfl_sync(gmask, mj, src);
        const int rows_now = 2 * ((m - t0) < G ? (m - t0) : G);
        uint64_t* bb = bar + (sb & 1);
        if (l == 0) mbar_expect_tx(bb, 256u * rows_now);
        __syncwarp(gmask);
        if (l < rows_now) bulk_row_load(stage + (sb & 1) * STAGE_FLOATS + l * 64, Q + (size_t)((l & 1) ? idj : idi) * d, bb);
      };
      issue(0);
      for (int sb = 0; sb < nsb; ++sb) {
        const int t0 = sb * G;
        if (sb + 1 < nsb) issue(sb + 1);
        uint64_t* bb = bar + (sb & 1);
        const uint32_t par = (sb & 1) ? phase1 : phase0;
        while (!mbar_try_wait(bb, par)) {}
        if (sb & 1) phase1 ^= 1u; else phase0 ^= 1u;
        float4 qi[G], qj[G];
        int ri[G], rj[G];
        const float* st = stage + (sb & 1) * STAGE_FLOATS;
#pragma unroll
        for (int f = 0; f < G; ++f) {
          ri[f] = __shfl_sync(gmask, mi, sub * LPR + ((t0 + f) & (LPR - 1)));
          rj[f] = __shfl_sync(gmask, mj, sub * LPR + ((t0 + f) & (LPR - 1)));
          if (t0 + f < m) {
            qi[f] = *reinterpret_cast<const float4*>(st + (2 * f) * 64 + l * 4);
            qj[f] = *reinterpret_cast<const float4*>(st + (2 * f + 1) * 64 + l * 4);
          } else {
            qi[f] = qj[f] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
        __syncwarp(gmask);                                        // the slot may be requested again two sub-batches on
#pragma unroll
        for (int f = 0; f < G; ++f) {
          const long long t = base + t0 + f;
          if (t0 + f < m) {
            if (t >= uend) {                                      // next user: flush the P delta, load the new row
              red_add_v4(prow, make_float4(p.x - p0.x, p.y - p0.y, p.z - p0.z, p.w - p0.w));
              do { ++uu; uend = __ldg(rowptr + uu + 1); } while (uend <= t);
              prow = P + (size_t)uu * d + l * 4;
              p = *reinterpret_cast<const float4*>(prow);
              p0 = p;
            }
            float x = dot4(p, qi[f]) - dot4(p, qj[f]);
            x = group_sum<LPR>(x, gmask);
            const float s = fast_sigmoid(x);
            const float g = lr * (1.0f - s);
            if (l == 0) lsum += fast_neg_log(s);
            float4 dqi, dqj;
            bpr_step4_inplace(p, qi[f], qj[f], g, one_m_au, g * one_m_ai, a_i, dqi, dqj);
            red_add_v4(Q + (size_t)ri[f] * d + l * 4, dqi);
            red_add_v4(Q + (size_t)rj[f] * d + l * 4, dqj);
          }
        }
      }
    }
    red_add_v4(prow, make_float4(p.x - p0.x, p.y - p0.y, p.z - p0.z, p.w - p0.w));
  }
  block_add_loss(lsum, loss);
}

}  // namespace

extern "C" int qrec_bpr_epoch_usermajor_tma_f32(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, const int64_t* rowptr,
                                                const int32_t* i, const int64_t* rated_rowptr, const int32_t* rated_cols,
                                                int32_t num_items, uint64_t seed, uint32_t epoch, int32_t* j_out, float lr,
                                                float reg_u, float reg_i, double* loss, void* stream) {
  QREC_REQUIRE(P && Q && loss, "qrec_bpr_epoch_usermajor_tma_f32: null pointer");
  QREC_REQUIRE(d == 64, "qrec_bpr_epoch_usermajor_tma_f32: d=%d unsupported (64 only: one 256-byte bulk copy per row); use "
                        "qrec_bpr_epoch_usermajor_f32", d);
  QREC_REQUIRE(n_users >= 0 && n >= 0 && num_items >= 1, "qrec_bpr_epoch_usermajor_tma_f32: bad size");
  if (n_users == 0 || n == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && i && rated_rowptr && rated_cols, "qrec_bpr_epoch_usermajor_tma_f32: null index pointer");
  QREC_REQUIRE((reinterpret_cast<uintptr_t>(Q) & 15) == 0, "qrec_bpr_epoch_usermajor_tma_f32: Q must be 16-byte aligned");
  constexpr size_t smem = (size_t)GROUPS * 2 * STAGE_FLOATS * 4 + GROUPS * 2 * 8;
  QREC_CUDA(allow_dynamic_smem((const void*)bpr_sgd_usermajor_tma_kernel<true>, (int)smem));
  int occ = 3;                                       // one sweep over the stream: grid = resident CTAs (see launch_usermajor)
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, bpr_sgd_usermajor_tma_kernel<true>, 256, smem) != cudaSuccess || occ < 1) occ = 3;
  const int grid = capped_grid(((n + CH - 1) / CH + GROUPS - 1) / GROUPS, occ);
  FusedSampler fs = {reinterpret_cast<const long long*>(rated_rowptr), rated_cols, num_items, (uint32_t)seed,
                     (uint32_t)(seed >> 32), epoch, j_out};
  bpr_sgd_usermajor_tma_kernel<true><<<grid, 256, smem, (cudaStream_t)stream>>>(
      P, Q, n_users, n, reinterpret_cast<const long long*>(rowptr), i, nullptr, lr, reg_u, reg_i, loss, fs);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
