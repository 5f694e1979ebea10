// K1: BPR.optimization(u,i,j) on the GPU (reference: model/ranking/BPR.py:45-53).
//
//   x = P[u].Q[i] - P[u].Q[j];  s = 1/(1+exp(-x));  g = lr*(1-s)
//   P[u] += g*(Q[i]-Q[j]);  Q[i] += g*P[u](new);  Q[j] -= g*P[u](new)
//   P[u] -= lr*regU*P[u];   Q[i] -= lr*regI*Q[i];  Q[j] -= lr*regI*Q[j];   loss += -ln(s)
//
// Two kernels:
//   * bpr_sgd_ordered_kernel  -- parity mode.  The reference loop is Gauss-Seidel: triple k
//     must see every earlier update of its three rows.  Instead of level-by-level launches
//     the kernel runs the epoch as a dataflow: warps claim triples in array order from a
//     ticket counter and spin until each of their three rows has reached the version
//     (= number of earlier touches) computed by qrec_bpr_order_prepare.  Because tickets are
//     handed out in order to running warps, the oldest unfinished triple always has its
//     dependencies satisfied, so the scheme cannot deadlock whatever the grid size.
//   * bpr_sgd_batch_kernel    -- throughput mode.  LPR lanes own one triple (d=64: a half
//     warp, one float4 per lane = one 128-bit LDG per row), the dot products are reduced with
//     xor-shuffles inside the lane group and the three row deltas go back with
//     REDG.E.ADD.F32x4 (red.global.add.v4.f32).  UNROLL triples per lane group are in flight
//     before the first use so each warp keeps 2*UNROLL*3 row loads outstanding.
#include <cmath>

#include "common.h"
#include "device.cuh"
#include "philox.cuh"
#include "bpr_step.cuh"
#include "um_waves.cuh"

namespace {

using namespace qrec;
using namespace qrec::bpr;

// ------------------------------------------------------------------------------------------
// parity mode
// ------------------------------------------------------------------------------------------
template <typename T, int E>  // E = ceil(d/32) elements per lane, element index e*32+lane
__global__ void __launch_bounds__(256)
bpr_sgd_ordered_kernel(T* __restrict__ P, T* __restrict__ Q, int d, long long n,
                       const int* __restrict__ u, const int* __restrict__ i,
                       const int* __restrict__ j, const int* __restrict__ wu,
                       const int* __restrict__ wi, const int* __restrict__ wj, int* ver_p,
                       int* ver_q, unsigned long long* ticket, T lr, T reg_u, T reg_i,
                       double* loss) {
  const int lane = threadIdx.x & 31;
  double local_loss = 0.0;
  const T a_u = mul_rn(lr, reg_u), a_i = mul_rn(lr, reg_i);
  while (true) {
    unsigned long long k = 0;
    if (lane == 0) k = atomicAdd(ticket, 1ULL);
    k = __shfl_sync(0xffffffffu, k, 0);
    if (k >= (unsigned long long)n) break;
    const int uu = u[k], ii = i[k], jj = j[k];
    // lanes 0..2 each watch one row version
    const int* vp = lane == 0 ? ver_p + uu : (lane == 1 ? ver_q + ii : ver_q + jj);
    const int need = lane == 0 ? wu[k] : (lane == 1 ? wi[k] : wj[k]);
    unsigned backoff = 8, polls = 0;
    while (true) {
      const int have = lane < 3 ? ld_acquire_gpu(vp) : need;
      if (__all_sync(0xffffffffu, have == need)) break;
      __nanosleep(backoff);
      if (backoff < 64) backoff <<= 1;
      // a ticket waits for at most (#resident warps) predecessors, i.e. milliseconds; ~10 s of polling
      // means the wait_* arrays do not describe this triple stream -- abort the launch instead of
      // hanging the GPU (the host sees a launch failure)
      if (++polls > (1u << 27)) __trap();
    }
    T* pr = P + (size_t)uu * d;
    T* qir = Q + (size_t)ii * d;
    T* qjr = Q + (size_t)jj * d;
    T p[E], qi[E], qj[E];
    T di = 0, dj = 0;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      if (c < d) {
        p[e] = __ldcg(pr + c);  // L2-coherent: the row was last written by another SM
        qi[e] = __ldcg(qir + c);
        qj[e] = __ldcg(qjr + c);
        di += p[e] * qi[e];
        dj += p[e] * qj[e];
      } else {
        p[e] = qi[e] = qj[e] = 0;
      }
    }
    di = warp_sum(di);
    dj = warp_sum(dj);
    const T s = sigmoid_full(sub_rn(di, dj));
    const T g = mul_rn(lr, sub_rn((T)1, s));
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      if (c < d) {
        T pn, qin, qjn;
        bpr_update_parity(p[e], qi[e], qj[e], g, a_u, a_i, pn, qin, qjn);
        __stcg(pr + c, pn);
        __stcg(qir + c, qin);
        __stcg(qjr + c, qjn);
      }
    }
    __threadfence();
    __syncwarp();
    if (lane < 3) red_release_gpu_add(const_cast<int*>(vp), 1);
    if (lane == 0) local_loss += neg_log(s);
  }
  if (lane == 0 && local_loss != 0.0) atomicAdd(loss, local_loss);
}

// ------------------------------------------------------------------------------------------
// throughput mode
// ------------------------------------------------------------------------------------------
// sigmoid and -ln(s) on the SFU (fast_sigmoid / fast_neg_log, device.cuh); parity mode keeps expf/logf.
template <int LPR, int VPL, int UNROLL>
__global__ void __launch_bounds__(256)
bpr_sgd_batch_kernel(float* __restrict__ P, float* __restrict__ Q, int nvec, long long n,
                     const int* __restrict__ u, const int* __restrict__ i,
                     const int* __restrict__ j, float lr, float reg_u, float reg_i,
                     double* loss) {
  constexpr int TPW = 32 / LPR;  // triples processed side by side in one warp
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int d = nvec * 4;
  const float a_u = lr * reg_u, a_i = lr * reg_i;
  float lsum = 0.f;

  for (long long base = warp * 32; base < n; base += nwarps * 32) {
    const long long k = base + lane;
    int mu = 0, mi = 0, mj = 0;
    if (k < n) {
      mu = __ldg(u + k);
      mi = __ldg(i + k);
      mj = __ldg(j + k);
    }
    const int cnt = (n - base) < 32 ? (int)(n - base) : 32;
    for (int s0 = 0; s0 < cnt; s0 += TPW * UNROLL) {
      float4 p[UNROLL][VPL], qi[UNROLL][VPL], qj[UNROLL][VPL];
      float* pr[UNROLL];
      float* qir[UNROLL];
      float* qjr[UNROLL];
      bool ok[UNROLL];
#pragma unroll
      for (int r = 0; r < UNROLL; ++r) {
        const int t = s0 + r * TPW + sub;
        const int uu = __shfl_sync(0xffffffffu, mu, t & 31);
        const int ii = __shfl_sync(0xffffffffu, mi, t & 31);
        const int jj = __shfl_sync(0xffffffffu, mj, t & 31);
        ok[r] = t < cnt;
        pr[r] = P + (size_t)uu * d + l * 4;
        qir[r] = Q + (size_t)ii * d + l * 4;
        qjr[r] = Q + (size_t)jj * d + l * 4;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          if (ok[r] && (l + v * LPR) < nvec) {
            p[r][v] = *reinterpret_cast<const float4*>(pr[r] + v * LPR * 4);
            qi[r][v] = *reinterpret_cast<const float4*>(qir[r] + v * LPR * 4);
            qj[r][v] = *reinterpret_cast<const float4*>(qjr[r] + v * LPR * 4);
          } else {
            p[r][v] = qi[r][v] = qj[r][v] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
#pragma unroll
      for (int r = 0; r < UNROLL; ++r) {
        float x = 0.f;
#pragma unroll
        for (int v = 0; v < VPL; ++v) x += dot4(p[r][v], qi[r][v]) - dot4(p[r][v], qj[r][v]);
        x = group_sum<LPR>(x);
        const float s = fast_sigmoid(x);
        const float g = lr * (1.0f - s);
        if (ok[r]) {
          if (l == 0) lsum += fast_neg_log(s);
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            if ((l + v * LPR) < nvec) {
              float4 dp, dqi, dqj;
              bpr_step4(p[r][v], qi[r][v], qj[r][v], g, a_u, a_i, dp, dqi, dqj);
              red_add_v4(pr[r] + v * LPR * 4, dp);
              red_add_v4(qir[r] + v * LPR * 4, dqi);
              red_add_v4(qjr[r] + v * LPR * 4, dqj);
            }
          }
        }
      }
    }
  }
  // block reduction of the loss: one double atomic per block
  block_add_loss(lsum, loss);
}


// ------------------------------------------------------------------------------------------
// K1 on staged item rows (row-sharded Q, SURVEY 8e): the rows of i and j were fetched from their
// owner ranks into R[pos]; the step is the same, P is updated in place (REDG.ADD.F32x4) and the item
// deltas are written next to the fetched rows (D[pos]) to be sent back and scatter-added by the
// owner.  LPR = d/4 lanes per triple like the batch kernel; one triple per lane group per step.
// ------------------------------------------------------------------------------------------
template <int LPR>
__global__ void __launch_bounds__(256)
bpr_sgd_staged_kernel(float* __restrict__ P, int nvec, long long n, const int* __restrict__ u,
                      const int* __restrict__ pos_i, const int* __restrict__ pos_j,
                      const float* __restrict__ R, float* __restrict__ D, float lr, float reg_u,
                      float reg_i, double* loss) {
  constexpr int TPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const long long group = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5) * TPW + sub;
  const long long ngroups = (((long long)gridDim.x * blockDim.x) >> 5) * TPW;
  const int d = nvec * 4;
  const float a_u = lr * reg_u, a_i = lr * reg_i;
  float lsum = 0.f;
  const long long rounds = (n + ngroups - 1) / ngroups;
  for (long long it = 0; it < rounds; ++it) {
    const long long k = it * ngroups + group;
    const bool ok = k < n && l < nvec;
    float4 p = make_float4(0.f, 0.f, 0.f, 0.f), qi = p, qj = p;
    float* pr = nullptr;
    size_t oi = 0, oj = 0;
    if (ok) {
      pr = P + (size_t)__ldg(u + k) * d + l * 4;
      oi = (size_t)__ldg(pos_i + k) * d + l * 4;
      oj = (size_t)__ldg(pos_j + k) * d + l * 4;
      p = *reinterpret_cast<const float4*>(pr);
      qi = __ldg(reinterpret_cast<const float4*>(R + oi));
      qj = __ldg(reinterpret_cast<const float4*>(R + oj));
    }
    float x = dot4(p, qi) - dot4(p, qj);
    x = group_sum<LPR>(x);
    const float s = fast_sigmoid(x);
    const float g = lr * (1.0f - s);
    if (ok) {
      if (l == 0) lsum += fast_neg_log(s);
      float4 dp, dqi, dqj;
      bpr_step4(p, qi, qj, g, a_u, a_i, dp, dqi, dqj);
      red_add_v4(pr, dp);
      *reinterpret_cast<float4*>(D + oi) = dqi;
      *reinterpret_cast<float4*>(D + oj) = dqj;
    }
  }
  block_add_loss(lsum, loss);
}


// ------------------------------------------------------------------------------------------
// throughput mode, TMA scatter variant (d = 64): identical gather/compute, but the three row deltas
// of a triple are parked in shared memory and added to the tables by the bulk-copy engine
//   cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [row], [smem], 256
// (one instruction per 256-byte row, issued by one lane, executed by the TMA unit against L2)
// instead of 16 lanes x REDG.E.ADD.F32x4 through the LSU/L1TEX path that bounds the plain kernel.
// Shared memory: per warp 2 buffers x (UNROLL*TPW triples x 3 rows x 256 B); a buffer is rewritten
// only after cp.async.bulk.wait_group.read shows that the engine has read it.
// ------------------------------------------------------------------------------------------
// TMA_MASK selects which rows go through the bulk engine (bit 0: P[u], bit 1: Q[i], bit 2: Q[j]);
// the others keep the REDG path, so the two scatter paths can run side by side.
template <int UNROLL, int TMA_MASK>
__global__ void __launch_bounds__(256)
bpr_sgd_batch_tma_kernel(float* __restrict__ P, float* __restrict__ Q, long long n,
                         const int* __restrict__ u, const int* __restrict__ i,
                         const int* __restrict__ j, float lr, float reg_u, float reg_i,
                         double* loss) {
  constexpr int LPR = 16, TPW = 2, D = 64;
  constexpr int ROWS = ((TMA_MASK >> 0) & 1) + ((TMA_MASK >> 1) & 1) + ((TMA_MASK >> 2) & 1);
  constexpr int SLOT_P = 0, SLOT_I = (TMA_MASK & 1), SLOT_J = (TMA_MASK & 1) + ((TMA_MASK >> 1) & 1);
  constexpr int SLOT_FLOATS = UNROLL * TPW * ROWS * D;         // per warp, per buffer
  extern __shared__ __align__(128) float stage[];              // [8 warps][2 buffers][SLOT_FLOATS]
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int sub = lane / LPR, l = lane % LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float a_u = lr * reg_u, a_i = lr * reg_i;
  float* my_stage = stage + (size_t)wib * 2 * SLOT_FLOATS;
  float lsum = 0.f;
  int buf = 0;

  for (long long base = warp * 32; base < n; base += nwarps * 32) {
    const long long k = base + lane;
    int mu = 0, mi = 0, mj = 0;
    if (k < n) {
      mu = __ldg(u + k);
      mi = __ldg(i + k);
      mj = __ldg(j + k);
    }
    const int cnt = (n - base) < 32 ? (int)(n - base) : 32;
    for (int s0 = 0; s0 < cnt; s0 += TPW * UNROLL) {
      float4 p[UNROLL], qi[UNROLL], qj[UNROLL];
      int uu[UNROLL], ii[UNROLL], jj[UNROLL];
      bool ok[UNROLL];
#pragma unroll
      for (int r = 0; r < UNROLL; ++r) {
        const int t = s0 + r * TPW + sub;
        uu[r] = __shfl_sync(0xffffffffu, mu, t & 31);
        ii[r] = __shfl_sync(0xffffffffu, mi, t & 31);
        jj[r] = __shfl_sync(0xffffffffu, mj, t & 31);
        ok[r] = t < cnt;
        if (ok[r]) {
          p[r] = *reinterpret_cast<const float4*>(P + (size_t)uu[r] * D + l * 4);
          qi[r] = *reinterpret_cast<const float4*>(Q + (size_t)ii[r] * D + l * 4);
          qj[r] = *reinterpret_cast<const float4*>(Q + (size_t)jj[r] * D + l * 4);
        } else {
          p[r] = qi[r] = qj[r] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      // the engine must have finished READING the buffer we are about to overwrite (issued two
      // iterations ago by lanes 0..2 of each lane group; bulk groups are tracked per thread)
      if (l < 3) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      __syncwarp();
      float* slot = my_stage + (size_t)buf * SLOT_FLOATS;
#pragma unroll
      for (int r = 0; r < UNROLL; ++r) {
        float x = dot4(p[r], qi[r]) - dot4(p[r], qj[r]);
        x = group_sum<LPR>(x);
        const float s = fast_sigmoid(x);
        const float g = lr * (1.0f - s);
        if (ok[r]) {
          if (l == 0) lsum += fast_neg_log(s);
          float4 dp, dqi, dqj;
          bpr_step4(p[r], qi[r], qj[r], g, a_u, a_i, dp, dqi, dqj);
          float* trip = slot + (size_t)(r * TPW + sub) * ROWS * D;
          if (TMA_MASK & 1) *reinterpret_cast<float4*>(trip + SLOT_P * D + l * 4) = dp;
          else red_add_v4(P + (size_t)uu[r] * D + l * 4, dp);
          if (TMA_MASK & 2) *reinterpret_cast<float4*>(trip + SLOT_I * D + l * 4) = dqi;
          else red_add_v4(Q + (size_t)ii[r] * D + l * 4, dqi);
          if (TMA_MASK & 4) *reinterpret_cast<float4*>(trip + SLOT_J * D + l * 4) = dqj;
          else red_add_v4(Q + (size_t)jj[r] * D + l * 4, dqj);
        }
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // st.shared -> visible to the bulk engine
      __syncwarp();
      if (l < 3 && ((TMA_MASK >> l) & 1)) {
        const int srow = (l == 0) ? SLOT_P : (l == 1 ? SLOT_I : SLOT_J);
#pragma unroll
        for (int r = 0; r < UNROLL; ++r) {
          if (ok[r]) {
            float* dst = (l == 0) ? (P + (size_t)uu[r] * D) : (Q + (size_t)(l == 1 ? ii[r] : jj[r]) * D);
            const float* src = slot + (size_t)(r * TPW + sub) * ROWS * D + srow * D;
            asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst),
                         "r"((uint32_t)__cvta_generic_to_shared(src)), "n"(D * 4)
                         : "memory");
          }
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      buf ^= 1;
    }
  }
  if (l < 3) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all reductions performed
  block_add_loss(lsum, loss);
}


// ------------------------------------------------------------------------------------------
// throughput mode, user-major (P-stationary): the reference's own iteration order
// (model/ranking/BPR.py:31-33: for user: for item).  A lane group takes one user, keeps P[u] in
// registers across that user's triples -- so P[u] is updated SEQUENTIALLY inside a user exactly as
// in the reference, and costs one row load + one row RED per user instead of per triple -- while
// the two item rows of every triple are gathered (PF triples ahead) and scatter-added with
// REDG.E.ADD.F32x4 as in the batch kernel.  Per triple: 2 row loads + 2 row REDs instead of 3 + 3.
// Input: CSR over users (rowptr), i[] / j[] in that order.
// ------------------------------------------------------------------------------------------
// The launch runs in waves (um_waves.cuh); inside a wave the item rows are READ from Qr, the table as it was when
// the wave started, and scatter-added into Q.  Lane group g of a wave's launch takes the wave's users ua + g,
// ua + g + ngroups, ... and runs each one whole (P[u] register-resident, updated sequentially, one row RED at the
// end).  Nothing a triple reads depends on timing: the result is the same every run up to the summation order of
// the float REDs, and an item row is read at most about one wave late.
// SAMPLE: the negatives are drawn inside the kernel (lane l draws the negative of triple base+l with
// the same Philox counter as the stand-alone sampler, so both give identical j) instead of being
// read from j[] (FusedSampler, philox.cuh); they are optionally written to j_out.
// SIG: the sampler pre-tests every draw against the user's 512-bit rated signature (philox.cuh).
// TMA (d = 64 only): the item rows reach the lane group through shared memory instead of one LDG.128 per lane
// and row.  One lane per row issues a 256-byte cp.async.bulk from Qr into the group's staging slot, completion is
// signalled on the slot's mbarrier and the lanes read their slices with LDS.128, so the gathers leave the
// LSU/L1TEX path, which then carries only the scatter-adds.  Two slots per lane group: the rows of the next G
// triples are requested while the current G are computed.
constexpr int UM_STAGE_FLOATS = 2 * 4 * 64;                  // one slot: the 2 x G rows of G = 4 triples, d = 64
constexpr int UM_STAGE_GROUPS = 16;                          // lane groups of 16 lanes in a 256-thread CTA
constexpr int UM_STAGE_SMEM = UM_STAGE_GROUPS * 2 * (UM_STAGE_FLOATS * 4 + 8);   // two slots + two mbarriers per group

// one 256-byte row: global -> this CTA's shared memory, completion counted on `bar`
__device__ __forceinline__ void bulk_row_load(float* smem_dst, const float* gsrc, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], 256, [%2];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(smem_u32(bar)) : "memory");
}

template <int LPR, int G, bool FULL, bool SAMPLE, bool SIG, bool TMA>   // FULL: d == 4*LPR (every lane owns a slice)
__device__ __forceinline__ void
usermajor_epoch(float* __restrict__ P, float* __restrict__ Q, const float* __restrict__ Qr, int nvec, long long n,
                const int* __restrict__ wave_user, const long long* __restrict__ rowptr, const int* __restrict__ i,
                const int* __restrict__ j, float lr, float reg_u, float reg_i, double* loss, FusedSampler fs,
                long long trip_off, const uint32_t* __restrict__ rated_sig) {
  // rowptr holds GLOBAL triple offsets; i/j are indexed relative to trip_off (a chunk of users of a
  // larger epoch: the host pipeline stages one chunk at a time).  Philox counters use global indices.
  // wave_user[0 .. 1]: the wave's users [ua, ub).
  static_assert(!TMA || (LPR == 16 && G == 4 && FULL), "the TMA fetch is laid out for d = 64, G = 4");
  constexpr int GPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (sub * LPR));
  const int group = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * GPW + sub;
  const int ngroups = (int)((gridDim.x * blockDim.x) >> 5) * GPW;
  const int d = FULL ? LPR * 4 : nvec * 4;
  const bool act = FULL ? true : (l < nvec);
  const float a_u = lr * reg_u, a_i = lr * reg_i;
  const float one_m_au = 1.0f - a_u, one_m_ai = 1.0f - a_i;
  float lsum = 0.f;
  // launch_usermajor chains the waves with programmatic dependent launch: the next wave's snapshot copy may be
  // launched now, and this wave reads neither Q nor Qr, nor writes anything, before pdl_wait() (`waited`)
  qrec::pdl_launch_dependents();
  bool waited = false;
  float* stage = nullptr;                                    // TMA: this group's two slots and their mbarriers
  uint64_t* bar = nullptr;
  uint32_t phase0 = 0, phase1 = 0;
  if constexpr (TMA) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* stage_all = reinterpret_cast<float*>(smem_raw);                                         // [GROUPS][2][8][64]
    uint64_t* bars = reinterpret_cast<uint64_t*>(stage_all + UM_STAGE_GROUPS * 2 * UM_STAGE_FLOATS);  // [GROUPS][2]
    const int g_in_cta = (threadIdx.x >> 5) * GPW + sub;
    stage = stage_all + (size_t)g_in_cta * 2 * UM_STAGE_FLOATS;
    bar = bars + g_in_cta * 2;
    if (l == 0) { mbar_init(bar, 1); mbar_init(bar + 1, 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }
  const int ub = __ldg(wave_user + 1);
  for (int uu = __ldg(wave_user) + group; uu < ub; uu += ngroups) {
    // the launch's first and last users are cut where the caller cut the launch
    long long lo = __ldg(rowptr + uu) - trip_off, hi = __ldg(rowptr + uu + 1) - trip_off;
    lo = lo > 0 ? lo : 0;
    hi = hi < n ? hi : n;
    if (lo >= hi) continue;
    float* prow = P + (size_t)uu * d + l * 4;
    float4 p = act ? *reinterpret_cast<const float4*>(prow) : make_float4(0.f, 0.f, 0.f, 0.f);
    long long rated_lo = 0, rated_hi = 0;
    if (SAMPLE) {
      rated_lo = __ldg(fs.rated_rowptr + uu);
      rated_hi = __ldg(fs.rated_rowptr + uu + 1);
    }
    for (long long base = lo; base < hi; base += LPR) {
      const int m = (hi - base) < LPR ? (int)(hi - base) : LPR;
      int mi = 0, mj = 0;
      if (l < m) {
        mi = __ldg(i + base + l);
        if (SAMPLE) {
          if (SIG)
            mj = qrec::sample_negative_sig(base + l + trip_off, fs.epoch, fs.seed_lo, fs.seed_hi, fs.num_items,
                                           fs.rated_cols, rated_lo, rated_hi,
                                           rated_sig + (size_t)uu * qrec::RATED_SIG_WORDS);
          else
            mj = qrec::sample_negative(base + l + trip_off, fs.epoch, fs.seed_lo, fs.seed_hi, fs.num_items, fs.rated_cols,
                                       rated_lo, rated_hi);
        } else {
          mj = __ldg(j + base + l);
        }
      }
      if (!waited) {                                     // the first table access of this thread
        qrec::pdl_wait();
        waited = true;
      }
      if (SAMPLE && l < m && fs.j_out != nullptr) fs.j_out[base + l] = mj;
      // TMA: request the rows of triples t0 .. t0+G-1 into slot (t0 / G) & 1: lane 2f -> Qr[i_f], lane 2f+1 -> Qr[j_f]
      auto issue = [&](int t0) {
        const int src = sub * LPR + ((t0 + (l >> 1)) & (LPR - 1));
        const int idi = __shfl_sync(gmask, mi, src), idj = __shfl_sync(gmask, mj, src);
        const int rows_now = 2 * ((m - t0) < G ? (m - t0) : G);
        uint64_t* bb = bar + ((t0 / G) & 1);
        if (l == 0) mbar_expect_tx(bb, 256u * rows_now);
        __syncwarp(gmask);
        if (l < rows_now) bulk_row_load(stage + ((t0 / G) & 1) * UM_STAGE_FLOATS + l * 64, Qr + (size_t)((l & 1) ? idj : idi) * d, bb);
      };
      if constexpr (TMA) issue(0);
      for (int t0 = 0; t0 < m; t0 += G) {
        const float* slot = nullptr;
        if constexpr (TMA) {
          if (t0 + G < m) issue(t0 + G);
          const int s = (t0 / G) & 1;
          mbar_wait(bar + s, s ? phase1 : phase0);
          if (s) phase1 ^= 1u; else phase0 ^= 1u;
          slot = stage + s * UM_STAGE_FLOATS;
        }
        float4 qi[G], qj[G];
        int ri[G], rj[G];
#pragma unroll
        for (int f = 0; f < G; ++f) {                    // G triples' item rows in flight
          ri[f] = __shfl_sync(gmask, mi, sub * LPR + ((t0 + f) & (LPR - 1)));
          rj[f] = __shfl_sync(gmask, mj, sub * LPR + ((t0 + f) & (LPR - 1)));
          if (t0 + f < m && act) {
            if constexpr (TMA) {
              qi[f] = *reinterpret_cast<const float4*>(slot + (2 * f) * 64 + l * 4);
              qj[f] = *reinterpret_cast<const float4*>(slot + (2 * f + 1) * 64 + l * 4);
            } else {
              // not through L1: the previous wave's rows of Qr may still sit there (launch_usermajor)
              qi[f] = qrec::ldg_no_l1_v4(reinterpret_cast<const float4*>(Qr + (size_t)ri[f] * d + l * 4));
              qj[f] = qrec::ldg_no_l1_v4(reinterpret_cast<const float4*>(Qr + (size_t)rj[f] * d + l * 4));
            }
          } else {
            qi[f] = qj[f] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
        if constexpr (TMA) __syncwarp(gmask);         // the slot may be requested again G triples on
#pragma unroll
        for (int f = 0; f < G; ++f) {
          if (t0 + f < m) {                              // uniform inside the lane group
            float x = dot4(p, qi[f]) - dot4(p, qj[f]);
            x = group_sum<LPR>(x, gmask);
            const float s = fast_sigmoid(x);
            const float g = lr * (1.0f - s);
            if (l == 0) lsum += fast_neg_log(s);
            if (act) {
              float4 dqi, dqj;
              bpr_step4_inplace(p, qi[f], qj[f], g, one_m_au, g * one_m_ai, a_i, dqi, dqj);   // P[u] stays in registers
              red_add_v4(Q + (size_t)ri[f] * d + l * 4, dqi);
              red_add_v4(Q + (size_t)rj[f] * d + l * 4, dqj);
            }
          }
        }
      }
    }
    if (act) {
      // only this lane group touches P[u] in the launch: the row still holds what p was loaded from
      const float4 p0 = __ldcg(reinterpret_cast<const float4*>(prow));
      red_add_v4(prow, make_float4(p.x - p0.x, p.y - p0.y, p.z - p0.z, p.w - p0.w));
    }
  }
  if (!waited) qrec::pdl_wait();
  block_add_loss(lsum, loss);
}

template <int LPR, int G, bool FULL, bool SAMPLE, int MINB = 3, bool SIG = false>
__global__ void __launch_bounds__(256, MINB)
bpr_sgd_usermajor_kernel(float* __restrict__ P, float* __restrict__ Q, const float* __restrict__ Qr, int nvec, long long n,
                         const int* __restrict__ wave_user, const long long* __restrict__ rowptr,
                         const int* __restrict__ i, const int* __restrict__ j, float lr, float reg_u, float reg_i,
                         double* loss, FusedSampler fs, long long trip_off, const uint32_t* __restrict__ rated_sig) {
  usermajor_epoch<LPR, G, FULL, SAMPLE, SIG, false>(P, Q, Qr, nvec, n, wave_user, rowptr, i, j, lr, reg_u, reg_i, loss, fs,
                                                    trip_off, rated_sig);
}

// d = 64 with fused sampling, item rows staged in shared memory (UM_STAGE_SMEM bytes of dynamic shared memory)
__global__ void __launch_bounds__(256, 3)
bpr_sgd_usermajor_tma_kernel(float* __restrict__ P, float* __restrict__ Q, const float* __restrict__ Qr, int nvec,
                             long long n, const int* __restrict__ wave_user, const long long* __restrict__ rowptr,
                             const int* __restrict__ i, const int* __restrict__ j, float lr, float reg_u, float reg_i,
                             double* loss, FusedSampler fs, long long trip_off, const uint32_t* __restrict__ rated_sig) {
  usermajor_epoch<16, 4, true, true, false, true>(P, Q, Qr, nvec, n, wave_user, rowptr, i, j, lr, reg_u, reg_i, loss, fs,
                                                  trip_off, rated_sig);
}

using UserMajorKernel = decltype(&bpr_sgd_usermajor_tma_kernel);

// The instantiation for lane groups of LPR lanes: FULL when d = 4 LPR; the signature pre-test only then.  With FULL
// fused sampling, G = 2 triples in flight fit 64 registers, so four 256-thread CTAs are resident per SM instead of
// three: 8,448 lane groups on an H100, one round for the 8,000 users of a benchmark wave (400K triples / 50).
template <int LPR>
UserMajorKernel usermajor_kernel(int nvec, bool sample, bool sig) {
  if (nvec != LPR)
    return sample ? bpr_sgd_usermajor_kernel<LPR, 4, false, true> : bpr_sgd_usermajor_kernel<LPR, 4, false, false>;
  if (sig) return bpr_sgd_usermajor_kernel<LPR, 2, true, true, 4, true>;
  return sample ? bpr_sgd_usermajor_kernel<LPR, 2, true, true, 4> : bpr_sgd_usermajor_kernel<LPR, 4, true, false>;
}

// The snapshot a wave reads: Qr = Q (n4 float4s), both tables kept in L2 (evict_last), so that the wave's gathers and
// scatter-adds find them there.  Neither table is read through L1 (launch_usermajor).  It runs on the whole GPU, four
// 512-thread CTAs per SM at <= 32 registers: the next wave's K1 can do little but wait for it, so the copy is made as
// short as possible rather than leaving room for K1 CTAs beside it (measured on an H100 80GB HBM3 at 400 W: 16.8 ms per
// benchmark epoch against 17.2 ms with one copy CTA per SM).
constexpr int UM_SNAPSHOT_THREADS = 512, UM_SNAPSHOT_CTAS_PER_SM = 4;
__global__ void __launch_bounds__(UM_SNAPSHOT_THREADS, UM_SNAPSHOT_CTAS_PER_SM)
um_snapshot_kernel(const float4* __restrict__ Q, float4* __restrict__ Qr, long long n4) {
  const unsigned long long keep = qrec::l2_policy_evict_last();
  qrec::pdl_wait();                  // the previous wave's scatter-adds into Q are complete and visible
  qrec::pdl_launch_dependents();     // the next wave's K1 may run its prologue (see launch_usermajor)
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (; k + 3 * stride < n4; k += 4 * stride) {
    float4 v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r] = qrec::ld_stream_v4(Q + k + r * stride, keep);
#pragma unroll
    for (int r = 0; r < 4; ++r) qrec::st_hint_v4(Qr + k + r * stride, v[r], keep);
  }
  for (; k < n4; k += stride) qrec::st_hint_v4(Qr + k, qrec::ld_stream_v4(Q + k, keep), keep);
}

// wave_user[w] = first user of wave w, w = 0 .. nwaves (um_waves.cuh)
__global__ void __launch_bounds__(256)
um_wave_table_kernel(const long long* __restrict__ rowptr, int n_users, long long n, long long trip_off,
                     long long wave_chunks, long long nwaves, int* __restrict__ wave_user) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w <= nwaves) wave_user[w] = um_wave_first_user(rowptr, n_users, n, trip_off, wave_chunks, w);
}

// one warp per user: bit (c & 511) of the user's 16-word signature for every rated column c
__global__ void __launch_bounds__(256)
rated_signature_kernel(int n_users, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                       uint32_t* __restrict__ sig) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long uu = warp; uu < n_users; uu += nwarps) {
    const long long lo = __ldg(rowptr + uu), hi = __ldg(rowptr + uu + 1);
    for (long long e = lo + lane; e < hi; e += 32) {
      const int c = __ldg(cols + e);
      atomicOr(sig + (size_t)uu * qrec::RATED_SIG_WORDS + ((c >> 5) & (qrec::RATED_SIG_WORDS - 1)), 1u << (c & 31));
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
sumsq_kernel(const T* __restrict__ x, long long n, double* out) {
  double acc = 0.0;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  if constexpr (sizeof(T) == 4) {
    const long long n4 = n >> 2;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    for (long long k = tid; k < n4; k += stride) {
      const float4 v = __ldg(x4 + k);
      acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
    }
    for (long long k = (n4 << 2) + tid; k < n; k += stride) acc += (double)x[k] * x[k];
  } else {
    for (long long k = tid; k < n; k += stride) acc += (double)x[k] * (double)x[k];
  }
  acc = warp_sum(acc);
  __shared__ double wsum[8];
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += wsum[w];
    atomicAdd(out, t);
  }
}

template <typename T>
int launch_ordered(T* P, T* Q, int d, long long n, const int* u, const int* i, const int* j,
                   const int* wu, const int* wi, const int* wj, int* ver_p, int* ver_q,
                   unsigned long long* ticket, T lr, T reg_u, T reg_i, double* loss,
                   int n_warps, cudaStream_t st) {
  QREC_REQUIRE(P && Q && loss && ticket && ver_p && ver_q, "bpr_sgd_ordered: null pointer");
  QREC_REQUIRE(d >= 1 && d <= 256, "bpr_sgd_ordered: d=%d unsupported (1..256)", d);
  QREC_REQUIRE(n >= 0, "bpr_sgd_ordered: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && j && wu && wi && wj, "bpr_sgd_ordered: null index pointer");
  const int e = (d + 31) / 32;
  // 2 CTAs of 8 warps per SM: enough warps to cover the dependency DAG's width at the
  // synthetic scale (~25 independent triples per level in user-major order) without
  // drowning the LSU in pollers.
  // n_warps > 0: the caller knows the width of the dependency DAG (qrec_bpr_order_depth) and asks
  // for about that many pollers -- thousands of idle warps hammering the version counters slow the
  // few that can make progress (1.4 independent triples per level on FilmTrust, ~25 at SYN scale)
  const int grid = n_warps > 0 ? capped_grid((n_warps + 7) / 8, 2) : sm_count() * 2;
#define QREC_ORD(E)                                                                              \
  bpr_sgd_ordered_kernel<T, E><<<grid, 256, 0, st>>>(P, Q, d, n, u, i, j, wu, wi, wj, ver_p,     \
                                                     ver_q, ticket, lr, reg_u, reg_i, loss)
  if (e <= 1) QREC_ORD(1);
  else if (e <= 2) QREC_ORD(2);
  else if (e <= 4) QREC_ORD(4);
  else QREC_ORD(8);
#undef QREC_ORD
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // namespace

namespace qrec {
// shared with runtime.cu (pipelined host path)
int launch_bpr_batch(float* P, float* Q, int d, long long n, const int* u, const int* i,
                     const int* j, float lr, float reg_u, float reg_i, double* loss,
                     cudaStream_t st) {
  QREC_REQUIRE(P && Q && loss, "bpr_sgd_batch: null pointer");
  QREC_REQUIRE(d >= 4 && d <= 256 && (d % 4) == 0, "bpr_sgd_batch: d=%d unsupported (multiple of 4, 4..256)", d);
  QREC_REQUIRE(n >= 0, "bpr_sgd_batch: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && j, "bpr_sgd_batch: null index pointer");
  const int nvec = d / 4;
  const long long warps_needed = (n + 31) / 32;
  const int grid = capped_grid((warps_needed + 7) / 8, 8);  // 8 CTAs x 8 warps per SM, grid-stride beyond
#define QREC_BATCH(LPR, VPL, UN)                                                                \
  bpr_sgd_batch_kernel<LPR, VPL, UN><<<grid, 256, 0, st>>>(P, Q, nvec, n, u, i, j, lr, reg_u,   \
                                                           reg_i, loss)
  if (nvec <= 4) QREC_BATCH(4, 1, 2);
  else if (nvec <= 8) QREC_BATCH(8, 1, 4);
  else if (nvec <= 16) QREC_BATCH(16, 1, 4);
  else if (nvec <= 32) QREC_BATCH(32, 1, 4);
  else QREC_BATCH(32, 2, 2);
#undef QREC_BATCH
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
}  // namespace qrec

extern "C" {

int qrec_bpr_sgd_ordered_f32(float* P, float* Q, int32_t d, int64_t n, const int32_t* u,
                             const int32_t* i, const int32_t* j, const int32_t* wu,
                             const int32_t* wi, const int32_t* wj, int32_t* ver_p,
                             int32_t* ver_q, unsigned long long* ticket, float lr, float reg_u,
                             float reg_i, double* loss, int32_t n_warps, void* stream) {
  return launch_ordered<float>(P, Q, d, n, u, i, j, wu, wi, wj, ver_p, ver_q, ticket, lr, reg_u,
                               reg_i, loss, n_warps, (cudaStream_t)stream);
}

int qrec_bpr_sgd_ordered_f64(double* P, double* Q, int32_t d, int64_t n, const int32_t* u,
                             const int32_t* i, const int32_t* j, const int32_t* wu,
                             const int32_t* wi, const int32_t* wj, int32_t* ver_p,
                             int32_t* ver_q, unsigned long long* ticket, double lr,
                             double reg_u, double reg_i, double* loss, int32_t n_warps, void* stream) {
  return launch_ordered<double>(P, Q, d, n, u, i, j, wu, wi, wj, ver_p, ver_q, ticket, lr, reg_u,
                                reg_i, loss, n_warps, (cudaStream_t)stream);
}

int qrec_bpr_sgd_batch_f32(float* P, float* Q, int32_t d, int64_t n, const int32_t* u,
                           const int32_t* i, const int32_t* j, float lr, float reg_u,
                           float reg_i, double* loss, void* stream) {
  return qrec::launch_bpr_batch(P, Q, d, n, u, i, j, lr, reg_u, reg_i, loss, (cudaStream_t)stream);
}

int qrec_bpr_sgd_batch_tma_f32(float* P, float* Q, int32_t d, int64_t n, const int32_t* u,
                               const int32_t* i, const int32_t* j, float lr, float reg_u,
                               float reg_i, double* loss, void* stream) {
  QREC_REQUIRE(P && Q && loss, "qrec_bpr_sgd_batch_tma_f32: null pointer");
  QREC_REQUIRE(d == 64, "qrec_bpr_sgd_batch_tma_f32: only d=64 (got %d); use qrec_bpr_sgd_batch_f32", d);
  QREC_REQUIRE(n >= 0, "qrec_bpr_sgd_batch_tma_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && j, "qrec_bpr_sgd_batch_tma_f32: null index pointer");
  // only P's row goes through the bulk engine (TMA_MASK 1: the fewest bytes through the copy engine); the item rows
  // keep REDG
  constexpr int UN = 4, MASK = 1;
  constexpr int smem = 8 * 2 * UN * 2 * 64 * 4;   // 8 warps x 2 buffers x UN*2 triples x one 256-byte row
  QREC_CUDA(allow_dynamic_smem((const void*)bpr_sgd_batch_tma_kernel<UN, MASK>, smem));
  const int grid = capped_grid(((n + 31) / 32 + 7) / 8, 2);
  bpr_sgd_batch_tma_kernel<UN, MASK><<<grid, 256, smem, (cudaStream_t)stream>>>(P, Q, n, u, i, j, lr, reg_u, reg_i, loss);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C" (reopened below)

namespace qrec {
int launch_usermajor(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, const int64_t* rowptr,
                     const int32_t* i, const int32_t* j, float lr, float reg_u, float reg_i, double* loss,
                     bool sample, const int64_t* rated_rowptr, const int32_t* rated_cols, int32_t num_items,
                     uint64_t seed, uint32_t epoch, int32_t* j_out, long long trip_off, cudaStream_t st,
                     const uint32_t* rated_sig, bool tma) {
  if (n <= 0) return QREC_OK;
  QREC_REQUIRE(num_items >= 1, "qrec user-major epoch: num_items=%d (the item table's rows) must be given", num_items);
  QREC_REQUIRE(!tma || (d == 64 && sample), "qrec user-major epoch: the TMA fetch needs d = 64 and fused sampling");
  FusedSampler fs = {reinterpret_cast<const long long*>(rated_rowptr), rated_cols, num_items, (uint32_t)seed,
                     (uint32_t)(seed >> 32), epoch, j_out};
  const int nvec = d / 4;
  const int lpr = nvec <= 4 ? 4 : nvec <= 8 ? 8 : nvec <= 16 ? 16 : 32;
  const bool sig = sample && rated_sig != nullptr;
  const UserMajorKernel kernel = tma        ? bpr_sgd_usermajor_tma_kernel
                                 : lpr == 4  ? usermajor_kernel<4>(nvec, sample, sig)
                                 : lpr == 8  ? usermajor_kernel<8>(nvec, sample, sig)
                                 : lpr == 16 ? usermajor_kernel<16>(nvec, sample, sig)
                                             : usermajor_kernel<32>(nvec, sample, sig);
  const int smem = tma ? UM_STAGE_SMEM : 0;
  if (tma) QREC_CUDA(allow_dynamic_smem((const void*)kernel, smem));
  // Grid = exactly the CTAs that are resident at once (occupancy API per instantiation); the stream is swept in
  // waves (um_waves.cuh), each reading the item table as the previous waves left it (a snapshot copied on the stream).
  int occ = 3;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, 256, smem) != cudaSuccess || occ < 1) occ = 3;
  const long long per_block = 8 * (32 / lpr);                                 // lane groups per CTA
  const long long max_users = n < n_users ? n : n_users;                      // users with triples in the launch
  const int grid = capped_grid((max_users + per_block - 1) / per_block, occ);
  const size_t q_bytes = (size_t)num_items * d * sizeof(float);
  const long long wave = um_wave_chunks(n, num_items, d);
  const long long nwaves = um_num_waves(n, wave);
  float* Qr = nullptr;                                // the item table as the current wave started (stream-ordered scratch)
  int* wave_user = nullptr;                           // first user of every wave, and one past the last (nwaves + 1)
  QREC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&Qr), q_bytes, st));
  const int rc = [&]() -> int {
    QREC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&wave_user), sizeof(int) * (size_t)(nwaves + 1), st));
    um_wave_table_kernel<<<(unsigned)((nwaves + 256) / 256), 256, 0, st>>>(reinterpret_cast<const long long*>(rowptr), n_users,
                                                                          n, trip_off, wave, nwaves, wave_user);
    QREC_CUDA(cudaGetLastError());
    count_launch();
    // Every snapshot copy and K1 after the call's first copy is launched with programmatic stream serialization: a
    // kernel may start while its predecessor on the stream still runs, and waits (pdl_wait) for the predecessor's
    // completion before its first access to Q / Qr, the loss or j_out.  The first copy is a normal launch, so all
    // earlier work on the stream is complete before the call's first kernel starts.  A copy kernel lets its successor
    // launch only after its own wait, so when a K1 starts, every kernel before its copy has completed.  What a K1 does
    // before its wait -- the wave's user bounds, the users' rowptr and rated bounds, i, the sampled negatives and the
    // P rows -- is therefore safe: those inputs are read-only, and no earlier wave of the call touches the P rows of
    // this wave's users (users are processed whole, each in one wave).  Q and Qr are never read through L1 (the copy's
    // loads and K1's gathers do not allocate there), so no line of an earlier wave's snapshot can be served after a wait.
    cudaLaunchAttribute pdl;
    pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    pdl.val.programmaticStreamSerializationAllowed = 1;
    const auto launch = [&](auto* fn, dim3 g, dim3 b, size_t shm, bool chained, auto... args) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = g;
      cfg.blockDim = b;
      cfg.dynamicSmemBytes = shm;
      cfg.stream = st;
      cfg.attrs = chained ? &pdl : nullptr;
      cfg.numAttrs = chained ? 1 : 0;
      return cudaLaunchKernelEx(&cfg, fn, args...);
    };
    const long long n4 = (long long)(q_bytes / sizeof(float4));
    const int copy_grid = sm_count() * UM_SNAPSHOT_CTAS_PER_SM;
    for (long long w = 0; w < nwaves; ++w) {
      QREC_CUDA(launch(um_snapshot_kernel, dim3(copy_grid), dim3(UM_SNAPSHOT_THREADS), 0, w > 0,
                       reinterpret_cast<const float4*>(Q), reinterpret_cast<float4*>(Qr), n4));
      count_launch();
      QREC_CUDA(launch(kernel, dim3(grid), dim3(256), (size_t)smem, true, P, Q, static_cast<const float*>(Qr), nvec,
                       (long long)n, static_cast<const int*>(wave_user + w), reinterpret_cast<const long long*>(rowptr), i, j,
                       lr, reg_u, reg_i, loss, fs, trip_off, rated_sig));
      if (w + 1 < nwaves) count_launch();
    }
    return QREC_OK;
  }();
  if (wave_user != nullptr) QREC_CUDA(cudaFreeAsync(wave_user, st));
  QREC_CUDA(cudaFreeAsync(Qr, st));
  if (rc != QREC_OK) return rc;
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
}  // namespace qrec

extern "C" {

int qrec_bpr_sgd_usermajor_f32(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, int32_t num_items,
                               const int64_t* rowptr, const int32_t* i, const int32_t* j, float lr, float reg_u, float reg_i,
                               double* loss, void* stream) {
  QREC_REQUIRE(P && Q && loss, "qrec_bpr_sgd_usermajor_f32: null pointer");
  QREC_REQUIRE(d >= 4 && d <= 128 && (d % 4) == 0, "qrec_bpr_sgd_usermajor_f32: d=%d unsupported (multiple of 4, 4..128)", d);
  QREC_REQUIRE(n_users >= 0 && n >= 0, "qrec_bpr_sgd_usermajor_f32: negative size");
  if (n_users == 0 || n == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && i && j, "qrec_bpr_sgd_usermajor_f32: null index pointer");
  return qrec::launch_usermajor(P, Q, d, n_users, n, rowptr, i, j, lr, reg_u, reg_i, loss, false, nullptr, nullptr, num_items,
                                0, 0, nullptr, 0, (cudaStream_t)stream, nullptr, false);
}

int qrec_bpr_epoch_usermajor_f32(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, const int64_t* rowptr,
                                 const int32_t* i, const int64_t* rated_rowptr, const int32_t* rated_cols,
                                 int32_t num_items, uint64_t seed, uint32_t epoch, int32_t* j_out, float lr,
                                 float reg_u, float reg_i, double* loss, void* stream) {
  QREC_REQUIRE(P && Q && loss, "qrec_bpr_epoch_usermajor_f32: null pointer");
  QREC_REQUIRE(d >= 4 && d <= 128 && (d % 4) == 0, "qrec_bpr_epoch_usermajor_f32: d=%d unsupported (multiple of 4, 4..128)", d);
  QREC_REQUIRE(n_users >= 0 && n >= 0 && num_items >= 1, "qrec_bpr_epoch_usermajor_f32: bad size");
  if (n_users == 0 || n == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && i && rated_rowptr && rated_cols, "qrec_bpr_epoch_usermajor_f32: null index pointer");
  return qrec::launch_usermajor(P, Q, d, n_users, n, rowptr, i, nullptr, lr, reg_u, reg_i, loss, true, rated_rowptr,
                                rated_cols, num_items, seed, epoch, j_out, 0, (cudaStream_t)stream, nullptr, false);
}

int qrec_rated_signature_build(int32_t n_users, const int64_t* rated_rowptr, const int32_t* rated_cols,
                               uint32_t* sig, void* stream) {
  QREC_REQUIRE(n_users >= 0, "qrec_rated_signature_build: n_users < 0");
  if (n_users == 0) return QREC_OK;
  QREC_REQUIRE(rated_rowptr && rated_cols && sig, "qrec_rated_signature_build: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  QREC_CUDA(cudaMemsetAsync(sig, 0, (size_t)n_users * qrec::RATED_SIG_WORDS * sizeof(uint32_t), st));
  rated_signature_kernel<<<capped_grid(((long long)n_users + 7) / 8, 8), 256, 0, st>>>(n_users, reinterpret_cast<const long long*>(rated_rowptr),
                                                     rated_cols, sig);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_bpr_epoch_usermajor_sig_f32(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, const int64_t* rowptr,
                                     const int32_t* i, const int64_t* rated_rowptr, const int32_t* rated_cols,
                                     const uint32_t* rated_sig, int32_t num_items, uint64_t seed, uint32_t epoch,
                                     int32_t* j_out, float lr, float reg_u, float reg_i, double* loss, void* stream) {
  QREC_REQUIRE(P && Q && loss, "qrec_bpr_epoch_usermajor_sig_f32: null pointer");
  QREC_REQUIRE(d == 16 || d == 32 || d == 64 || d == 128,
               "qrec_bpr_epoch_usermajor_sig_f32: d=%d unsupported (16, 32, 64 or 128); use qrec_bpr_epoch_usermajor_f32", d);
  QREC_REQUIRE(n_users >= 0 && n >= 0 && num_items >= 1, "qrec_bpr_epoch_usermajor_sig_f32: bad size");
  if (n_users == 0 || n == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && i && rated_rowptr && rated_cols && rated_sig, "qrec_bpr_epoch_usermajor_sig_f32: null index pointer");
  return qrec::launch_usermajor(P, Q, d, n_users, n, rowptr, i, nullptr, lr, reg_u, reg_i, loss, true, rated_rowptr,
                                rated_cols, num_items, seed, epoch, j_out, 0, (cudaStream_t)stream, rated_sig, false);
}

int qrec_bpr_epoch_usermajor_tma_f32(float* P, float* Q, int32_t d, int32_t n_users, int64_t n, const int64_t* rowptr,
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
  return qrec::launch_usermajor(P, Q, d, n_users, n, rowptr, i, nullptr, lr, reg_u, reg_i, loss, true, rated_rowptr,
                                rated_cols, num_items, seed, epoch, j_out, 0, (cudaStream_t)stream, nullptr, true);
}

int qrec_bpr_sgd_staged_f32(float* P, int32_t d, int64_t n, const int32_t* u, const int32_t* pos_i,
                            const int32_t* pos_j, const float* R, float* D, float lr, float reg_u,
                            float reg_i, double* loss, void* stream) {
  QREC_REQUIRE(d >= 4 && d <= 128 && (d % 4) == 0, "qrec_bpr_sgd_staged_f32: d=%d unsupported (multiple of 4, 4..128)", d);
  QREC_REQUIRE(n >= 0, "qrec_bpr_sgd_staged_f32: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(P && u && pos_i && pos_j && R && D && loss, "qrec_bpr_sgd_staged_f32: null pointer");
  const int nvec = d / 4;
  cudaStream_t st = (cudaStream_t)stream;
#define QREC_STAGED(LPR)                                                                        \
  {                                                                                             \
    const long long per_block = 8 * (32 / LPR);                                                 \
    const int grid = capped_grid((n + per_block - 1) / per_block, 8);                           \
    bpr_sgd_staged_kernel<LPR><<<grid, 256, 0, st>>>(P, nvec, n, u, pos_i, pos_j, R, D,         \
                                                     lr, reg_u, reg_i, loss);                   \
  }
  if (nvec <= 4) QREC_STAGED(4)
  else if (nvec <= 8) QREC_STAGED(8)
  else if (nvec <= 16) QREC_STAGED(16)
  else QREC_STAGED(32)
#undef QREC_STAGED
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_sumsq_f32(const float* x, int64_t n, double* out, void* stream) {
  QREC_REQUIRE(out && (x || n == 0) && n >= 0, "qrec_sumsq_f32: bad argument");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "qrec_sumsq_f32: x not 16-byte aligned");
  sumsq_kernel<float><<<capped_grid((n / 4 + 255) / 256 + 1, 8), 256, 0, (cudaStream_t)stream>>>(x, n, out);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_table_snapshot_f32(const float* src, float* dst, int64_t n, void* stream) {
  QREC_REQUIRE(n >= 0 && (n % 4) == 0, "qrec_table_snapshot_f32: n=%lld must be a multiple of 4", (long long)n);
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(src && dst, "qrec_table_snapshot_f32: null pointer");
  QREC_REQUIRE(((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0,
               "qrec_table_snapshot_f32: src and dst must be 16-byte aligned");
  um_snapshot_kernel<<<sm_count() * UM_SNAPSHOT_CTAS_PER_SM, UM_SNAPSHOT_THREADS, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(src),
                                                                                 reinterpret_cast<float4*>(dst), n / 4);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_sumsq_f64(const double* x, int64_t n, double* out, void* stream) {
  QREC_REQUIRE(out && (x || n == 0) && n >= 0, "qrec_sumsq_f64: bad argument");
  if (n == 0) return QREC_OK;
  sumsq_kernel<double><<<capped_grid((n + 255) / 256, 8), 256, 0, (cudaStream_t)stream>>>(x, n, out);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
