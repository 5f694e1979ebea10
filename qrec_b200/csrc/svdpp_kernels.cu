// K11: SVD++ (model/rating/SVDPlusPlus.py) on the GPU.  The arithmetic lives in svdpp_step.cuh.
//
// Every entry (u, i, r) reads the implicit rows Y[j] of all the user's items N(u) and updates all but Y[i], so one
// entry depends on nearly every entry before it (on FilmTrust the dependency chain covers 32 884 of 33 750 entries).
//
//   * svdpp_sgd_ordered_kernel -- parity mode: ONE CTA walks the entries in array order and is parallel only inside
//     an entry.  The w rows of N(u) are staged in shared memory a chunk at a time; thread c forms the two sequential
//     column sums of column c (all w rows for the prediction, the w-1 rows j != i for the Q step), block reductions
//     give the two dot products, then the w-1 row updates run elementwise over the block.  No spinning across CTAs,
//     no tickets: nothing can wait on anything but the CTA's own barriers.
//   * svdpp_usermajor_kernel -- throughput mode: one lane group per user (LPR lanes, one float4 per lane), users
//     taken from a row order.  A user's entries run in CSR order through the closed form of svdpp_step.cuh, which
//     keeps the user's Y rows implicit (S = their sum, B = the shared part of their updates), so a step moves the
//     rows Q[i_t], Y[i_t] once instead of all W rows of the user.  P[u] and Bu[u] stay in registers and are stored
//     once; Q / Y deltas go back with red.global.add.v4.f32, Bi with atomicAdd.  A user's items are distinct, so the
//     reads of Q[i_t], Bi[i_t], Y[i_t] run kPrefetch steps ahead of the writes of the steps before.
#include "common.h"
#include "device.cuh"
#include "lane_shape.h"
#include "svdpp_step.cuh"

namespace {

using namespace qrec;

constexpr int kThreads = 256;
constexpr int kStageBytes = 16384;   // parity kernel: staged Y rows per chunk (2048 doubles / 4096 floats)
constexpr int kPrefetch = 4;         // throughput kernel: steps whose row reads are in flight ahead of the update

// ------------------------------------------------------------------------------------------
// parity mode
// ------------------------------------------------------------------------------------------
// Sum over the block of one value per thread: xor-butterfly inside each warp, then the warp sums in warp order
// (tests/host_shims/svdpp_step_host.cpp replays the same grouping).  Ends with the result in every thread.
template <typename T>
__device__ __forceinline__ void block_sum2(T& a, T& b, T* red) {
  a = warp_sum(a);
  b = warp_sum(b);
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[warp] = a;
    red[8 + warp] = b;
  }
  __syncthreads();
  a = red[0];
  b = red[8];
#pragma unroll
  for (int w = 1; w < kThreads / 32; ++w) {
    a = sp_add(a, red[w]);
    b = sp_add(b, red[8 + w]);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
svdpp_sgd_ordered_kernel(T* P, T* Q, T* Y, T* Bu, T* Bi, int d, long long n, const int* __restrict__ u,
                         const int* __restrict__ i, const T* __restrict__ r, const long long* __restrict__ rowptr,
                         const int* __restrict__ cols, T lr, T reg_u, T reg_i, T reg_b, T reg_y, T global_mean,
                         double* loss) {
  constexpr int kStage = kStageBytes / sizeof(T);
  __shared__ T stage[kStage];
  __shared__ int stage_ids[kStage];
  __shared__ T q_old[kThreads];
  __shared__ T red[16];
  __shared__ T err_s;
  const int tid = threadIdx.x;
  const int rows_per_chunk = kStage / d;
  double local_loss = 0.0;
  for (long long k = 0; k < n; ++k) {
    const int uu = u[k], ii = i[k];
    const long long beg = rowptr[uu], end = rowptr[uu + 1];
    const int w = (int)(end - beg);
    // 1. the two sequential column sums of N(u) (SVDPlusPlus.py:76-79 over all w rows; :52 over j != i)
    T s_all = 0, s_ex = 0;
    for (long long c0 = beg; c0 < end; c0 += rows_per_chunk) {
      const int nr = (int)(end - c0 < rows_per_chunk ? end - c0 : rows_per_chunk);
      for (int t = tid; t < nr; t += kThreads) stage_ids[t] = cols[c0 + t];
      __syncthreads();
      for (int x = tid; x < nr * d; x += kThreads) {
        const int row = x / d, col = x - row * d;
        stage[x] = Y[(size_t)stage_ids[row] * d + col];
      }
      __syncthreads();
      if (tid < d) {
        for (int row = 0; row < nr; ++row) {
          const T y = stage[row * d + tid];
          s_all = sp_add(s_all, y);
          if (stage_ids[row] != ii) s_ex = sp_add(s_ex, y);
        }
      }
      __syncthreads();
    }
    // 2. the two dot products, the error and the biases (SVDPlusPlus.py:33-45)
    T p = 0, q = 0, ty = 0, tp = 0;
    if (tid < d) {
      p = P[(size_t)uu * d + tid];
      q = Q[(size_t)ii * d + tid];
      q_old[tid] = q;
      svdpp_dot_terms_parity<T>(s_all, (T)w, p, q, ty, tp);
    }
    block_sum2<T>(ty, tp, red);
    if (tid == 0) {
      const T bu = Bu[uu], bi = Bi[ii];
      const T err = svdpp_error_parity<T>(r[k], ty, tp, global_mean, bi, bu);
      Bu[uu] = svdpp_bias_parity<T>(bu, err, lr, reg_b);
      Bi[ii] = svdpp_bias_parity<T>(bi, err, lr, reg_b);
      err_s = err;
      local_loss += (double)err * (double)err;
    }
    __syncthreads();
    const T err = err_s;
    const T wm1 = (T)(w - 1);
    // 3. the implicit rows j != i against the old Q[i] (SVDPlusPlus.py:54), then P[u] and Q[i] (:55-58)
    if (w > 1) {
      for (long long x = tid; x < (long long)w * d; x += kThreads) {
        const int row = (int)(x / d), col = (int)(x - (long long)row * d);
        const int j = cols[beg + row];
        if (j != ii) {
          T* yp = Y + (size_t)j * d + col;
          *yp = svdpp_y_parity<T>(*yp, err, q_old[col], wm1, lr, reg_y);
        }
      }
    }
    if (tid < d) {
      T pn, qn;
      svdpp_pq_parity<T>(p, q, s_ex, w > 1, err, wm1, lr, reg_u, reg_i, pn, qn);
      P[(size_t)uu * d + tid] = pn;
      Q[(size_t)ii * d + tid] = qn;
    }
    __syncthreads();
  }
  if (tid == 0 && local_loss != 0.0) atomicAdd(loss, local_loss);
}

template <typename T>
int launch_ordered(T* P, T* Q, T* Y, T* Bu, T* Bi, int d, long long n, const int* u, const int* i, const T* r,
                   const int64_t* rowptr, const int* cols, T lr, T reg_u, T reg_i, T reg_b, T reg_y, T global_mean,
                   double* loss, cudaStream_t st) {
  QREC_REQUIRE(P && Q && Y && Bu && Bi && loss, "svdpp_sgd_ordered: null pointer");
  QREC_REQUIRE(d >= 1 && d <= 256, "svdpp_sgd_ordered: d=%d unsupported (1..256)", d);
  QREC_REQUIRE(n >= 0, "svdpp_sgd_ordered: n < 0");
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(u && i && r && rowptr && cols, "svdpp_sgd_ordered: null entry pointer");
  svdpp_sgd_ordered_kernel<T><<<1, kThreads, 0, st>>>(P, Q, Y, Bu, Bi, d, n, u, i, r, (const long long*)rowptr, cols,
                                                       lr, reg_u, reg_i, reg_b, reg_y, global_mean, loss);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

// ------------------------------------------------------------------------------------------
// throughput mode
// ------------------------------------------------------------------------------------------
struct Step {
  float4 q, y;
  float bi, rating;
  int j;
};

template <int LPR>
__device__ __forceinline__ Step load_step(const float* Q, const float* Y, const float* Bi, const int* cols,
                                          const float* vals, long long at, int d, int l, bool act) {
  Step s;
  s.j = __ldg(cols + at);
  s.rating = __ldg(vals + at);
  // L2-coherent loads: other lane groups add into these rows during the launch
  s.q = act ? __ldcg(reinterpret_cast<const float4*>(Q + (size_t)s.j * d) + l) : make_float4(0.f, 0.f, 0.f, 0.f);
  s.y = act ? __ldcg(reinterpret_cast<const float4*>(Y + (size_t)s.j * d) + l) : make_float4(0.f, 0.f, 0.f, 0.f);
  s.bi = l == 0 ? __ldcg(Bi + s.j) : 0.f;
  return s;
}

template <int LPR>
__global__ void __launch_bounds__(kThreads, 2)
svdpp_usermajor_kernel(float* P, float* Q, float* Y, float* Bu, float* Bi, int nvec, int n_rows,
                       const int* __restrict__ row_order, const long long* __restrict__ rowptr,
                       const int* __restrict__ cols, const float* __restrict__ vals, float lr, float reg_u,
                       float reg_i, float reg_b, float reg_y, float global_mean, long long n_groups, double* loss) {
  const int lane = threadIdx.x & 31;
  const int l = lane % LPR;
  const unsigned gmask = LPR == 32 ? 0xffffffffu : (((1u << LPR) - 1u) << (lane - l));
  const long long group = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / LPR;
  const int d = nvec * 4;
  const bool act = l < nvec;
  const float omc = lr * reg_y, c = 1.f - omc;
  const float lc = log1pf(-omc);   // ln c
  float lsum = 0.f;
  for (long long pos = group; group < n_groups && pos < n_rows; pos += n_groups) {
    const int uu = __ldg(row_order + pos);
    const long long beg = __ldg(rowptr + uu);
    const int W = (int)(__ldg(rowptr + uu + 1) - beg);
    if (W == 0) continue;
    float4* prow = reinterpret_cast<float4*>(P + (size_t)uu * d) + l;
    float4 p = act ? *prow : make_float4(0.f, 0.f, 0.f, 0.f);
    float bu = __shfl_sync(gmask, l == 0 ? Bu[uu] : 0.f, 0, LPR);
    const bool implicit = W > 1;
    // S_0: the sum of the user's Y rows (W = 1: the prediction still reads Y[i_0])
    float4 S = make_float4(0.f, 0.f, 0.f, 0.f);
    if (act) {
#pragma unroll 4
      for (int t = 0; t < W; ++t) {
        const float4 y = __ldcg(reinterpret_cast<const float4*>(Y + (size_t)__ldg(cols + beg + t) * d) + l);
        S.x += y.x; S.y += y.y; S.z += y.z; S.w += y.w;
      }
    }
    float4 B = make_float4(0.f, 0.f, 0.f, 0.f);
    SvdppCfScalars k;
    k.lr = lr; k.reg_u = reg_u; k.reg_i = reg_i; k.c = c; k.omc = omc;
    k.wm1 = (float)(W - 1);
    k.cw1m1 = expm1f((float)(W - 1) * lc);
    k.ct = 1.f;
    const float inv_w = 1.f / (float)W;
    Step ring[kPrefetch];
#pragma unroll
    for (int f = 0; f < kPrefetch; ++f)
      if (f < W) ring[f] = load_step<LPR>(Q, Y, Bi, cols, vals, beg + f, d, l, act);
    for (int t0 = 0; t0 < W; t0 += kPrefetch) {
#pragma unroll
      for (int f = 0; f < kPrefetch; ++f) {
        const int t = t0 + f;
        if (t >= W) break;
        const Step s = ring[f];
        if (t + kPrefetch < W) ring[f] = load_step<LPR>(Q, Y, Bi, cols, vals, beg + t + kPrefetch, d, l, act);
        float4 z;                                   // S/W + p: both dot products in one reduction
        z.x = S.x * inv_w + p.x; z.y = S.y * inv_w + p.y; z.z = S.z * inv_w + p.z; z.w = S.w * inv_w + p.w;
        const float dot = group_sum<LPR>(dot4(z, s.q), gmask);
        const float bi = __shfl_sync(gmask, s.bi, 0, LPR);
        const float e = s.rating - (((dot + global_mean) + bi) + bu);
        bu += lr * (e - reg_b * bu);
        k.e = e;
        k.le = implicit ? lr * e / k.wm1 : 0.f;
        k.crest = implicit ? expf((float)(W - 1 - t) * lc) : 0.f;
        float4 dq, dy;
        svdpp_cf_component(k, implicit, p.x, s.q.x, s.y.x, S.x, B.x, dq.x, dy.x);
        svdpp_cf_component(k, implicit, p.y, s.q.y, s.y.y, S.y, B.y, dq.y, dy.y);
        svdpp_cf_component(k, implicit, p.z, s.q.z, s.y.z, S.z, B.z, dq.z, dy.z);
        svdpp_cf_component(k, implicit, p.w, s.q.w, s.y.w, S.w, B.w, dq.w, dy.w);
        k.ct *= c;
        if (act) {
          red_add_v4(Q + (size_t)s.j * d + 4 * l, dq);
          if (implicit) red_add_v4(Y + (size_t)s.j * d + 4 * l, dy);
        }
        if (l == 0) {
          atomicAdd(Bi + s.j, lr * (e - reg_b * bi));
          lsum += e * e;
        }
      }
    }
    // B_W belongs to every Y row of the user
    if (implicit && act) {
      for (int t = 0; t < W; ++t) red_add_v4(Y + (size_t)__ldg(cols + beg + t) * d + 4 * l, B);
    }
    if (act) *prow = p;
    if (l == 0) Bu[uu] = bu;
  }
  block_add_loss(lsum, loss);
}

}  // namespace

extern "C" {

int qrec_svdpp_sgd_ordered_f64(double* P, double* Q, double* Y, double* Bu, double* Bi, int32_t d, int64_t n,
                               const int32_t* u, const int32_t* i, const double* r, const int64_t* rowptr,
                               const int32_t* cols, double lr, double reg_u, double reg_i, double reg_b, double reg_y,
                               double global_mean, double* loss, void* stream) {
  return launch_ordered<double>(P, Q, Y, Bu, Bi, d, n, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y,
                                global_mean, loss, (cudaStream_t)stream);
}

int qrec_svdpp_sgd_ordered_f32(float* P, float* Q, float* Y, float* Bu, float* Bi, int32_t d, int64_t n,
                               const int32_t* u, const int32_t* i, const float* r, const int64_t* rowptr,
                               const int32_t* cols, float lr, float reg_u, float reg_i, float reg_b, float reg_y,
                               float global_mean, double* loss, void* stream) {
  return launch_ordered<float>(P, Q, Y, Bu, Bi, d, n, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y,
                               global_mean, loss, (cudaStream_t)stream);
}

int qrec_svdpp_epoch_usermajor_f32(float* P, float* Q, float* Y, float* Bu, float* Bi, int32_t d, int32_t n_rows,
                                   const int32_t* row_order, const int64_t* rowptr, const int32_t* cols,
                                   const float* vals, float lr, float reg_u, float reg_i, float reg_b, float reg_y,
                                   float global_mean, double* loss, int64_t max_users_in_flight, void* stream) {
  QREC_REQUIRE(max_users_in_flight >= 0, "svdpp_epoch_usermajor: max_users_in_flight < 0");
  QREC_REQUIRE(P && Q && Y && Bu && Bi && loss, "svdpp_epoch_usermajor: null pointer");
  QREC_REQUIRE(d >= 4 && d <= 128 && d % 4 == 0, "svdpp_epoch_usermajor: d=%d unsupported (multiple of 4, 4..128)", d);
  QREC_REQUIRE(n_rows >= 0, "svdpp_epoch_usermajor: n_rows < 0");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(row_order && rowptr && cols && vals, "svdpp_epoch_usermajor: null CSR pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int nvec = d / 4;
  const long long per_block = kThreads / row_lpr(nvec);
  long long groups = max_users_in_flight > 0 && max_users_in_flight < n_rows ? max_users_in_flight : n_rows;
  const int blocks = capped_grid((groups + per_block - 1) / per_block, 8);
  if (groups > (long long)blocks * per_block) groups = (long long)blocks * per_block;
  with_row_shape<128>(nvec, [&](auto s) {
    svdpp_usermajor_kernel<decltype(s)::LPR><<<blocks, kThreads, 0, st>>>(
        P, Q, Y, Bu, Bi, nvec, n_rows, row_order, (const long long*)rowptr, cols, vals, lr, reg_u, reg_i, reg_b, reg_y,
        global_mean, groups, loss);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
