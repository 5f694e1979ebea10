// K9: the pointwise MF step of the rating-prediction family on the GPU (SURVEY.md §8 f-4).
//
//   reference: model/rating/BasicMF.py:13-23 (kind 0), model/rating/PMF.py:13-22 (kind 1),
//              model/rating/SVD.py:17-32 + predictForRating SVD.py:84-90 (kind 2),
//              model/rating/SoRec.py:42-60 (kind 3: the trust-edge pass, on the tables (P, Z)),
//              model/rating/SocialMF.py:15-24 (kind 4: kind 1 on copies of the rows),
//              model/rating/EE.py:15-36 + predictForRating EE.py:81-87 (kind 5: Euclidean embedding)
//
//   e = r - P[u].Q[i]                (SVD: - globalMean - Bi[i] - Bu[u], added in that order)
//   kind 0:  P[u] += (lr*e)*Q[i];                  Q[i] += (lr*e)*P[u](new)
//   kind 1:  P[u] += lr*(e*Q[i] - regU*P[u]);      Q[i] += lr*(e*P[u](new) - regI*Q[i](old))
//   kind 2:  kind 1 + Bu[u] += lr*(e - regB*Bu[u]);  Bi[i] += lr*(e - regB*Bi[i])
//   kind 3:  P[u] += lr*((regS*e)*Z[v]);  Z[v] += lr*((regS*e)*P[u](new) - regZ*Z[v](old))
//            (regS / regZ in the reg_u / reg_i slots, no bias vectors; the parity kernel only)
//   kind 4:  P[u] += lr*(e*Q[i] - regU*P[u]);      Q[i] += lr*(e*P[u](old) - regI*Q[i](old))
//            (no bias vectors; the parity kernel only)
//   kind 5:  dist = |P[u]-Q[i]|^2,  e = r - (((globalMean + Bi[i]) + Bu[u]) - dist)
//            P[u] -= (lr*(e+regU))*(P[u]-Q[i]);     Q[i] += (lr*(e+regI))*(P[u](new)-Q[i])
//            Bu / Bi as kind 2 (from the biases before the update; the parity kernel only)
//   loss += e^2  (kind 3: regS*e^2; kind 5: e^2 + regU*dist)
//
// `p = self.P[u]` is a numpy view in the reference, so the item row is updated from the already
// updated user row -- both kernels keep that.  SocialMF copies both rows first (kind 4).
//
//   * mf_sgd_ordered_kernel -- parity mode, on the in-order protocol of device.cuh: warps take
//     entries in array order and wait until their two rows have reached the version (= number
//     of earlier touches) computed by qrec_mf_order_prepare; mul/add are kept apart (no FMA) in
//     numpy's evaluation order.  Bu[u] / Bi[i] ride on the version counters of P[u] / Q[i].
//   * mf_sgd_batch_kernel   -- throughput mode: LPR lanes own one entry (one float4 per lane and
//     row), xor-shuffle dot, both row deltas go back with red.global.add.v4.f32; rows shared by
//     in-flight entries receive the sum of their deltas.
//   * mf_predict_pairs_kernel -- predictForRating for a list of (u,i) pairs (the per-epoch
//     rating_performance of iterativeRecommender.py:104-113 without moving the tables).
#include "common.h"
#include "device.cuh"
#include "lane_shape.h"
#include "mf_step.cuh"

namespace {

using namespace qrec;

// ------------------------------------------------------------------------------------------
// parity mode
// ------------------------------------------------------------------------------------------
template <typename T, int E, int KIND>  // E = ceil(d/32) elements per lane, element index e*32+lane
__global__ void __launch_bounds__(256)
mf_sgd_ordered_kernel(T* __restrict__ P, T* __restrict__ Q, int d, long long n,
                      const int* __restrict__ u, const int* __restrict__ i, const T* __restrict__ r,
                      const int* __restrict__ wu, const int* __restrict__ wi, int* ver_p, int* ver_q,
                      unsigned long long* ticket, T lr, T reg_u, T reg_i, T* Bu, T* Bi, T reg_b,
                      T global_mean, double* loss) {
  const int lane = threadIdx.x & 31;
  double local_loss = 0.0;
  while (true) {
    const unsigned long long k = warp_next_ticket(ticket);
    if (k >= (unsigned long long)n) break;
    const int uu = u[k], ii = i[k];
    const T rating = r[k];
    const int* vp = lane == 0 ? ver_p + uu : ver_q + ii;   // lanes 0 and 1 each watch one row version
    const int need = lane == 0 ? wu[k] : wi[k];
    spin_until<8, 64>([=] { return __all_sync(0xffffffffu, (lane < 2 ? ld_acquire_gpu(vp) : need) == need); });
    T* pr = P + (size_t)uu * d;
    T* qr = Q + (size_t)ii * d;
    T p[E], q[E];
    T dot = 0;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      if (c < d) {
        p[e] = __ldcg(pr + c);  // L2-coherent: the row was last written by another SM
        q[e] = __ldcg(qr + c);
        if (KIND == 5) {
          const T df = p[e] - q[e];
          dot += df * df;
        } else {
          dot += p[e] * q[e];
        }
      } else {
        p[e] = q[e] = 0;
      }
    }
    dot = warp_sum(dot);
    T bu = 0, bi = 0;
    if (KIND == 2 || KIND == 5) {
      bu = __ldcg(Bu + uu);
      bi = __ldcg(Bi + ii);
    }
    const T err = qrec::mf_sub(rating, qrec::mf_prediction<T, KIND>(dot, global_mean, bi, bu));   // SVD.py:88
    const T g = qrec::mf_step_scale<T, KIND>(err, lr, reg_u);    // BasicMF.py:22: lRate*error; SoRec.py:58: regS*euv
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      if (c < d) {
        T pn, qn;
        qrec::mf_update_parity<T, KIND>(p[e], q[e], err, g, lr, reg_u, reg_i, pn, qn);
        __stcg(pr + c, pn);
        __stcg(qr + c, qn);
      }
    }
    if (KIND == 2 || KIND == 5) {
      if (lane == 0) __stcg(Bu + uu, qrec::mf_bias_parity<T>(bu, err, lr, reg_b));
      if (lane == 1) __stcg(Bi + ii, qrec::mf_bias_parity<T>(bi, err, lr, reg_b));
    }
    warp_fence();
    if (lane < 2) red_release_gpu_add(const_cast<int*>(vp), 1);
    if (lane == 0) local_loss += qrec::mf_loss_term<T, KIND>(err, reg_u, dot);
  }
  if (lane == 0 && local_loss != 0.0) atomicAdd(loss, local_loss);
}

// ------------------------------------------------------------------------------------------
// throughput mode
// ------------------------------------------------------------------------------------------
template <int LPR, int KIND, int UNROLL>
__global__ void __launch_bounds__(256)
mf_sgd_batch_kernel(float* __restrict__ P, float* __restrict__ Q, int nvec, long long n,
                    const int* __restrict__ u, const int* __restrict__ i, const float* __restrict__ r,
                    float lr, float reg_u, float reg_i, float* Bu, float* Bi, float reg_b,
                    float global_mean, double* loss) {
  constexpr int EPW = 32 / LPR;  // entries processed side by side in one warp
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, l = lane % LPR;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int d = nvec * 4;
  const bool act = l < nvec;
  float lsum = 0.f;
  for (long long base = warp * 32; base < n; base += nwarps * 32) {
    const long long k = base + lane;
    int mu = 0, mi = 0;
    float mr = 0.f;
    if (k < n) {
      mu = __ldg(u + k);
      mi = __ldg(i + k);
      mr = __ldg(r + k);
    }
    const int cnt = (n - base) < 32 ? (int)(n - base) : 32;
    for (int s0 = 0; s0 < cnt; s0 += EPW * UNROLL) {
      float4 p[UNROLL], q[UNROLL];
      float* pr[UNROLL];
      float* qr[UNROLL];
      float rt[UNROLL], bu[UNROLL], bi[UNROLL];
      int ru[UNROLL], ri[UNROLL];
      bool ok[UNROLL];
#pragma unroll
      for (int f = 0; f < UNROLL; ++f) {                 // UNROLL entries' rows in flight
        const int t = s0 + f * EPW + sub;
        ru[f] = __shfl_sync(0xffffffffu, mu, t & 31);
        ri[f] = __shfl_sync(0xffffffffu, mi, t & 31);
        rt[f] = __shfl_sync(0xffffffffu, mr, t & 31);
        ok[f] = t < cnt;
        pr[f] = P + (size_t)ru[f] * d + l * 4;
        qr[f] = Q + (size_t)ri[f] * d + l * 4;
        if (ok[f] && act) {
          p[f] = *reinterpret_cast<const float4*>(pr[f]);
          q[f] = *reinterpret_cast<const float4*>(qr[f]);
        } else {
          p[f] = q[f] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        bu[f] = bi[f] = 0.f;
        if (KIND == 2 && ok[f]) {
          bu[f] = Bu[ru[f]];
          bi[f] = Bi[ri[f]];
        }
      }
#pragma unroll
      for (int f = 0; f < UNROLL; ++f) {
        const float dot = group_sum<LPR>(dot4(p[f], q[f]));
        float pred = dot;
        if (KIND == 2) pred = ((dot + global_mean) + bi[f]) + bu[f];
        const float e = rt[f] - pred;
        if (ok[f]) {
          if (act) {
            float4 dp, dq;
            qrec::mf_delta_fast<KIND>(p[f].x, q[f].x, e, lr, reg_u, reg_i, dp.x, dq.x);
            qrec::mf_delta_fast<KIND>(p[f].y, q[f].y, e, lr, reg_u, reg_i, dp.y, dq.y);
            qrec::mf_delta_fast<KIND>(p[f].z, q[f].z, e, lr, reg_u, reg_i, dp.z, dq.z);
            qrec::mf_delta_fast<KIND>(p[f].w, q[f].w, e, lr, reg_u, reg_i, dp.w, dq.w);
            red_add_v4(pr[f], dp);
            red_add_v4(qr[f], dq);
          }
          if (l == 0) {
            lsum += e * e;
            if (KIND == 2) {
              atomicAdd(Bu + ru[f], lr * (e - reg_b * bu[f]));
              atomicAdd(Bi + ri[f], lr * (e - reg_b * bi[f]));
            }
          }
        }
      }
    }
  }
  block_add_loss(lsum, loss);
}

// one warp per pair; out[k] = P[u].Q[i] (+ globalMean + Bi[i] + Bu[u] when Bu != null)
template <typename T>
__global__ void __launch_bounds__(256)
mf_predict_pairs_kernel(const T* __restrict__ P, const T* __restrict__ Q, int d, long long n,
                        const int* __restrict__ u, const int* __restrict__ i, const T* __restrict__ Bu,
                        const T* __restrict__ Bi, T global_mean, T* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long k = warp; k < n; k += nwarps) {
    const int uu = __ldg(u + k), ii = __ldg(i + k);
    const T* pr = P + (size_t)uu * d;
    const T* qr = Q + (size_t)ii * d;
    T dot = 0;
    for (int c = lane; c < d; c += 32) dot += pr[c] * qr[c];
    dot = warp_sum(dot);
    if (lane == 0) out[k] = Bu != nullptr ? ((dot + global_mean) + Bi[ii]) + Bu[uu] : dot;
  }
}

template <typename T>
int launch_ordered(int kind, T* P, T* Q, int d, long long n, const int* u, const int* i, const T* r,
                   const int* wu, const int* wi, int* ver_p, int* ver_q, unsigned long long* ticket, T lr,
                   T reg_u, T reg_i, T* Bu, T* Bi, T reg_b, T global_mean, double* loss, int n_warps,
                   cudaStream_t st) {
  QREC_REQUIRE(kind >= 0 && kind <= 5,
               "mf_sgd_ordered: kind=%d (0 BasicMF, 1 PMF, 2 SVD, 3 SoRec edges, 4 SocialMF, 5 EE)", kind);
  QREC_REQUIRE(P && Q && loss && ticket && ver_p && ver_q, "mf_sgd_ordered: null pointer");
  QREC_REQUIRE(kind != 2 || (Bu && Bi), "mf_sgd_ordered: kind 2 needs the bias vectors");
  QREC_REQUIRE(kind != 5 || (Bu && Bi), "mf_sgd_ordered: kind 5 needs the bias vectors");
  QREC_REQUIRE((kind != 3 && kind != 4) || (!Bu && !Bi), "mf_sgd_ordered: kind %d takes no bias vectors", kind);
  QREC_REQUIRE(d >= 1 && d <= 256, "mf_sgd_ordered: d=%d unsupported (1..256)", d);
  QREC_REQUIRE(n >= 0, "mf_sgd_ordered: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && r && wu && wi, "mf_sgd_ordered: null entry pointer");
  const int grid = ordered_grid(n_warps);
  with_lane_elems(d, [&](auto e) {
    constexpr int E = decltype(e)::E;
    const auto kernel = kind == 0   ? mf_sgd_ordered_kernel<T, E, 0>
                        : kind == 1 ? mf_sgd_ordered_kernel<T, E, 1>
                        : kind == 2 ? mf_sgd_ordered_kernel<T, E, 2>
                        : kind == 3 ? mf_sgd_ordered_kernel<T, E, 3>
                        : kind == 4 ? mf_sgd_ordered_kernel<T, E, 4>
                                    : mf_sgd_ordered_kernel<T, E, 5>;
    kernel<<<grid, 256, 0, st>>>(P, Q, d, n, u, i, r, wu, wi, ver_p, ver_q, ticket, lr, reg_u, reg_i, Bu, Bi, reg_b,
                                 global_mean, loss);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

template <typename T>
int launch_predict(const T* P, const T* Q, int d, long long n, const int* u, const int* i, const T* Bu,
                   const T* Bi, T global_mean, T* out, cudaStream_t st) {
  QREC_REQUIRE(n >= 0 && d >= 1, "mf_predict_pairs: bad sizes");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(P && Q && u && i && out, "mf_predict_pairs: null pointer");
  QREC_REQUIRE((Bu == nullptr) == (Bi == nullptr), "mf_predict_pairs: give both bias vectors or neither");
  mf_predict_pairs_kernel<T><<<capped_grid((n + 7) / 8, 8), 256, 0, st>>>(P, Q, d, n, u, i, Bu, Bi, global_mean, out);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // namespace

extern "C" {

int qrec_mf_sgd_ordered_f64(int32_t kind, double* P, double* Q, int32_t d, int64_t n, const int32_t* u,
                            const int32_t* i, const double* r, const int32_t* wait_u, const int32_t* wait_i,
                            int32_t* ver_p, int32_t* ver_q, unsigned long long* ticket, double lr, double reg_u,
                            double reg_i, double* Bu, double* Bi, double reg_b, double global_mean, double* loss,
                            int32_t n_warps, void* stream) {
  return launch_ordered<double>(kind, P, Q, d, n, u, i, r, wait_u, wait_i, ver_p, ver_q, ticket, lr, reg_u,
                                reg_i, Bu, Bi, reg_b, global_mean, loss, n_warps, (cudaStream_t)stream);
}

int qrec_mf_sgd_ordered_f32(int32_t kind, float* P, float* Q, int32_t d, int64_t n, const int32_t* u,
                            const int32_t* i, const float* r, const int32_t* wait_u, const int32_t* wait_i,
                            int32_t* ver_p, int32_t* ver_q, unsigned long long* ticket, float lr, float reg_u,
                            float reg_i, float* Bu, float* Bi, float reg_b, float global_mean, double* loss,
                            int32_t n_warps, void* stream) {
  return launch_ordered<float>(kind, P, Q, d, n, u, i, r, wait_u, wait_i, ver_p, ver_q, ticket, lr, reg_u,
                               reg_i, Bu, Bi, reg_b, global_mean, loss, n_warps, (cudaStream_t)stream);
}

int qrec_mf_sgd_batch_f32(int32_t kind, float* P, float* Q, int32_t d, int64_t n, const int32_t* u,
                          const int32_t* i, const float* r, float lr, float reg_u, float reg_i, float* Bu,
                          float* Bi, float reg_b, float global_mean, double* loss, int64_t max_inflight,
                          void* stream) {
  QREC_REQUIRE(kind >= 0 && kind <= 2, "mf_sgd_batch: kind=%d (0 BasicMF, 1 PMF, 2 SVD)", kind);
  QREC_REQUIRE(max_inflight >= 0, "mf_sgd_batch: max_inflight < 0");
  QREC_REQUIRE(P && Q && loss, "mf_sgd_batch: null pointer");
  QREC_REQUIRE(kind != 2 || (Bu && Bi), "mf_sgd_batch: kind 2 needs the bias vectors");
  QREC_REQUIRE(d >= 4 && d <= 128 && d % 4 == 0, "mf_sgd_batch: d=%d unsupported (multiple of 4, 4..128)", d);
  QREC_REQUIRE(n >= 0, "mf_sgd_batch: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && r, "mf_sgd_batch: null entry pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int nvec = d / 4;
  long long blocks = capped_grid((n + 255) / 256, 8);    // 32 entries per warp and pass
  if (max_inflight > 0) {
    // a lane group has UNROLL = 4 entries between their row reads and their reductions: bound the
    // number of such entries across the grid (the staleness window of the Hogwild update)
    const long long per_block = 8LL * (32 / row_lpr(nvec)) * 4;
    long long want = (max_inflight + per_block - 1) / per_block;
    if (want < 1) want = 1;
    if (blocks > want) blocks = want;
  }
  with_row_shape<128>(nvec, [&](auto s) {
    constexpr int LPR = decltype(s)::LPR;
    const auto kernel = kind == 0   ? mf_sgd_batch_kernel<LPR, 0, 4>
                        : kind == 1 ? mf_sgd_batch_kernel<LPR, 1, 4>
                                    : mf_sgd_batch_kernel<LPR, 2, 4>;
    kernel<<<(int)blocks, 256, 0, st>>>(P, Q, nvec, n, u, i, r, lr, reg_u, reg_i, Bu, Bi, reg_b, global_mean, loss);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_mf_predict_pairs_f32(const float* P, const float* Q, int32_t d, int64_t n, const int32_t* u,
                              const int32_t* i, const float* Bu, const float* Bi, float global_mean, float* out,
                              void* stream) {
  return launch_predict<float>(P, Q, d, n, u, i, Bu, Bi, global_mean, out, (cudaStream_t)stream);
}

int qrec_mf_predict_pairs_f64(const double* P, const double* Q, int32_t d, int64_t n, const int32_t* u,
                              const int32_t* i, const double* Bu, const double* Bi, double global_mean,
                              double* out, void* stream) {
  return launch_predict<double>(P, Q, d, n, u, i, Bu, Bi, global_mean, out, (cudaStream_t)stream);
}

}  // extern "C"
