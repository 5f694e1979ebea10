// K16: RSTE's rating pass (model/rating/RSTE.py:20-64) on the GPU.
//
//   rste_sgd_ordered_kernel -- the epoch in list order, sequential-equivalent, on the in-order protocol of
//     device.cuh (one warp per entry, lanes across d).  An entry (u, i) reads its own rows P[u], Q[i] and the rows
//     P[f] of all u's followees, and writes P[u] and Q[i] only (rste_step.cuh has the formulas).  Before it reads,
//     entry k waits until
//       ver_p[u]   == wait_u[k]        writes to P[u] by earlier entries        (read/write after write)
//       reads_p[u] == wait_reads_u[k]  earlier entries' reads of P[u] as a followee row   (write after read)
//       ver_q[i]   == wait_i[k]        writes to Q[i] by earlier entries
//       ver_p[f]   == earlier writes to P[f], for each followee f != u   (read after write)
//     The last count is the number of u == f entries before position k: a bisection of k in user f's sorted
//     entry positions (pos[pos_rowptr[f] .. pos_rowptr[f+1]), qrec_rste_order_prepare), so no table of
//     n x out-degree wait numbers is kept.  After reading its followee rows and before writing its own, the warp
//     adds one to reads_p[f] of each f != u; after writing, one to ver_p[u] and ver_q[i].  A self-follow reads
//     the pre-update P[u] the warp already holds and counts as no foreign read.  Every wait is on earlier
//     entries only, so the result is that of the serial loop whatever the grid.
//   rste_predict_pairs_kernel -- predictForRating for a list of known (u, i) pairs, one warp per pair.
#include "common.h"
#include "device.cuh"
#include "lane_shape.h"
#include "rste_step.cuh"

namespace {

using namespace qrec;

// number of entries of `a[0..n)` (ascending) below k
__device__ __forceinline__ int count_below(const int* __restrict__ a, int n, long long k) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if ((long long)__ldg(a + mid) < k) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// warp-wide P[row].q over the lane's E elements (element e*32+lane)
template <typename T, int E>
__device__ __forceinline__ T row_dot(const T* __restrict__ row, const T (&q)[E], int d, int lane) {
  T dot = 0;
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int c = e * 32 + lane;
    if (c < d) dot += __ldcg(row + c) * q[e];
  }
  return warp_sum(dot);
}

template <typename T, int E>
__global__ void __launch_bounds__(256)
rste_sgd_ordered_kernel(T* __restrict__ P, T* __restrict__ Q, int d, long long n, const int* __restrict__ u,
                        const int* __restrict__ i, const T* __restrict__ r, const int* __restrict__ wu,
                        const int* __restrict__ wi, const int* __restrict__ wr, const long long* __restrict__ pos_rowptr,
                        const int* __restrict__ pos, const long long* __restrict__ f_rowptr,
                        const int* __restrict__ f_cols, const T* __restrict__ f_w, const T* __restrict__ denom,
                        int* ver_p, int* ver_q, int* reads_p, unsigned long long* ticket, T lr, T reg_u, T reg_i,
                        T alpha, double* loss) {
  const int lane = threadIdx.x & 31;
  double local_loss = 0.0;
  while (true) {
    const unsigned long long k = warp_next_ticket(ticket);
    if (k >= (unsigned long long)n) break;
    const int uu = u[k], ii = i[k];
    const T rating = r[k];
    const long long fb = f_rowptr[uu], fe = f_rowptr[uu + 1];

    // own rows: lane 0 watches ver_p[u], lane 1 ver_q[i], lane 2 reads_p[u]
    {
      const int* vp = lane == 0 ? ver_p + uu : lane == 1 ? ver_q + ii : reads_p + uu;
      const int need = lane == 0 ? wu[k] : lane == 1 ? wi[k] : lane == 2 ? wr[k] : 0;
      spin_until<8, 64>([=] { return __all_sync(0xffffffffu, (lane < 3 ? ld_acquire_gpu(vp) : 0) == need); });
    }
    // followee rows, 32 at a time: each lane finds its followee's write count before position k
    for (long long base = fb; base < fe; base += 32) {
      const long long j = base + lane;
      int f = uu, need = 0;
      if (j < fe) f = f_cols[j];
      if (f != uu) {
        const long long pb = pos_rowptr[f];
        need = count_below(pos + pb, (int)(pos_rowptr[f + 1] - pb), (long long)k);
      }
      spin_until<8, 64>([=] { return __all_sync(0xffffffffu, (f != uu ? ld_acquire_gpu(ver_p + f) : 0) == need); });
    }

    T* pr = P + (size_t)uu * d;
    T* qr = Q + (size_t)ii * d;
    T p[E], q[E];
    T dot = 0;
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      if (c < d) {
        p[e] = __ldcg(pr + c);  // L2-coherent: the rows were last written by other SMs
        q[e] = __ldcg(qr + c);
        dot += p[e] * q[e];
      } else {
        p[e] = q[e] = 0;
      }
    }
    dot = warp_sum(dot);
    T social = 0;
    for (long long j = fb; j < fe; ++j) {
      const int f = __ldg(f_cols + j);
      // a self-follow reads the pre-update row this warp holds: its dot is `dot`
      const T fdot = f == uu ? dot : row_dot<T, E>(P + (size_t)f * d, q, d, lane);
      social = qrec::rste_social_add(social, __ldg(f_w + j), fdot);
    }
    // the followee rows are read: let their owners' later entries write them
    warp_fence();
    for (long long j = fb + lane; j < fe; j += 32) {
      const int f = __ldg(f_cols + j);
      if (f != uu) red_release_gpu_add(reads_p + f, 1);
    }

    const T pred = qrec::rste_prediction(dot, social, alpha, __ldg(denom + uu));
    const T err = qrec::mf_sub(rating, pred);
    const T aerr = qrec::mf_mul(alpha, err);  // RSTE.py:33: self.alpha*error
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      if (c < d) {
        T pn, qn;
        qrec::mf_update_parity<T, 1>(p[e], q[e], aerr, aerr, lr, reg_u, reg_i, pn, qn);
        __stcg(pr + c, pn);
        __stcg(qr + c, qn);
      }
    }
    warp_fence();
    if (lane == 0) red_release_gpu_add(ver_p + uu, 1);
    if (lane == 1) red_release_gpu_add(ver_q + ii, 1);
    if (lane == 0) local_loss += (double)err * (double)err;
  }
  if (lane == 0 && local_loss != 0.0) atomicAdd(loss, local_loss);
}

template <typename T, int E>
__global__ void __launch_bounds__(256)
rste_predict_pairs_kernel(const T* __restrict__ P, const T* __restrict__ Q, int d, long long n,
                          const int* __restrict__ u, const int* __restrict__ i, const long long* __restrict__ f_rowptr,
                          const int* __restrict__ f_cols, const T* __restrict__ f_w, const T* __restrict__ denom,
                          T alpha, T* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long k = warp; k < n; k += nwarps) {
    const int uu = __ldg(u + k), ii = __ldg(i + k);
    const T* qr = Q + (size_t)ii * d;
    T q[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      q[e] = c < d ? __ldg(qr + c) : T(0);
    }
    const T dot = row_dot<T, E>(P + (size_t)uu * d, q, d, lane);
    T social = 0;
    const long long fe = __ldg(f_rowptr + uu + 1);
    for (long long j = __ldg(f_rowptr + uu); j < fe; ++j) {
      const int f = __ldg(f_cols + j);
      social = qrec::rste_social_add(social, __ldg(f_w + j), row_dot<T, E>(P + (size_t)f * d, q, d, lane));
    }
    if (lane == 0) out[k] = qrec::rste_prediction(dot, social, alpha, __ldg(denom + uu));
  }
}

template <typename T>
int launch_ordered(T* P, T* Q, int d, long long n, const int* u, const int* i, const T* r, const int* wu,
                   const int* wi, const int* wr, const long long* pos_rowptr, const int* pos,
                   const long long* f_rowptr, const int* f_cols, const T* f_w, const T* denom, int* ver_p, int* ver_q,
                   int* reads_p, unsigned long long* ticket, T lr, T reg_u, T reg_i, T alpha, double* loss,
                   int n_warps, cudaStream_t st) {
  QREC_REQUIRE(P && Q && loss && ticket && ver_p && ver_q && reads_p, "rste_sgd_ordered: null pointer");
  QREC_REQUIRE(d >= 1 && d <= 256, "rste_sgd_ordered: d=%d unsupported (1..256)", d);
  QREC_REQUIRE(n >= 0 && n < (1LL << 31), "rste_sgd_ordered: n=%lld outside [0, 2^31)", (long long)n);
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && r && wu && wi && wr && pos_rowptr && pos && f_rowptr && denom,
               "rste_sgd_ordered: null entry pointer");
  const int grid = ordered_grid(n_warps);
  with_lane_elems(d, [&](auto e) {
    constexpr int E = decltype(e)::E;
    rste_sgd_ordered_kernel<T, E><<<grid, 256, 0, st>>>(P, Q, d, n, u, i, r, wu, wi, wr, pos_rowptr, pos, f_rowptr,
                                                       f_cols, f_w, denom, ver_p, ver_q, reads_p, ticket, lr, reg_u,
                                                       reg_i, alpha, loss);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

template <typename T>
int launch_predict(const T* P, const T* Q, int d, long long n, const int* u, const int* i, const long long* f_rowptr,
                   const int* f_cols, const T* f_w, const T* denom, T alpha, T* out, cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= 256, "rste_predict_pairs: d=%d unsupported (1..256)", d);
  QREC_REQUIRE(n >= 0, "rste_predict_pairs: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(P && Q && u && i && f_rowptr && denom && out, "rste_predict_pairs: null pointer");
  with_lane_elems(d, [&](auto e) {
    constexpr int E = decltype(e)::E;
    rste_predict_pairs_kernel<T, E><<<capped_grid((n + 7) / 8, 8), 256, 0, st>>>(P, Q, d, n, u, i, f_rowptr, f_cols,
                                                                                 f_w, denom, alpha, out);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // namespace

extern "C" {

int qrec_rste_sgd_ordered_f64(double* P, double* Q, int32_t d, int64_t n, const int32_t* u, const int32_t* i,
                              const double* r, const int32_t* wait_u, const int32_t* wait_i,
                              const int32_t* wait_reads_u, const int64_t* pos_rowptr, const int32_t* pos,
                              const int64_t* f_rowptr, const int32_t* f_cols, const double* f_w, const double* denom,
                              int32_t* ver_p, int32_t* ver_q, int32_t* reads_p, unsigned long long* ticket, double lr,
                              double reg_u, double reg_i, double alpha, double* loss, int32_t n_warps, void* stream) {
  return launch_ordered<double>(P, Q, d, n, u, i, r, wait_u, wait_i, wait_reads_u, (const long long*)pos_rowptr, pos,
                                (const long long*)f_rowptr, f_cols, f_w, denom, ver_p, ver_q, reads_p, ticket, lr,
                                reg_u, reg_i, alpha, loss, n_warps, (cudaStream_t)stream);
}

int qrec_rste_sgd_ordered_f32(float* P, float* Q, int32_t d, int64_t n, const int32_t* u, const int32_t* i,
                              const float* r, const int32_t* wait_u, const int32_t* wait_i,
                              const int32_t* wait_reads_u, const int64_t* pos_rowptr, const int32_t* pos,
                              const int64_t* f_rowptr, const int32_t* f_cols, const float* f_w, const float* denom,
                              int32_t* ver_p, int32_t* ver_q, int32_t* reads_p, unsigned long long* ticket, float lr,
                              float reg_u, float reg_i, float alpha, double* loss, int32_t n_warps, void* stream) {
  return launch_ordered<float>(P, Q, d, n, u, i, r, wait_u, wait_i, wait_reads_u, (const long long*)pos_rowptr, pos,
                               (const long long*)f_rowptr, f_cols, f_w, denom, ver_p, ver_q, reads_p, ticket, lr,
                               reg_u, reg_i, alpha, loss, n_warps, (cudaStream_t)stream);
}

int qrec_rste_predict_pairs_f64(const double* P, const double* Q, int32_t d, int64_t n, const int32_t* u,
                                const int32_t* i, const int64_t* f_rowptr, const int32_t* f_cols, const double* f_w,
                                const double* denom, double alpha, double* out, void* stream) {
  return launch_predict<double>(P, Q, d, n, u, i, (const long long*)f_rowptr, f_cols, f_w, denom, alpha, out,
                                (cudaStream_t)stream);
}

int qrec_rste_predict_pairs_f32(const float* P, const float* Q, int32_t d, int64_t n, const int32_t* u,
                                const int32_t* i, const int64_t* f_rowptr, const int32_t* f_cols, const float* f_w,
                                const float* denom, float alpha, float* out, void* stream) {
  return launch_predict<float>(P, Q, d, n, u, i, (const long long*)f_rowptr, f_cols, f_w, denom, alpha, out,
                               (cudaStream_t)stream);
}

}  // extern "C"
