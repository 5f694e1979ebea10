// K17: the trust-neighbourhood user pass of SocialMF (model/rating/SocialMF.py:26-43), SoReg
// (model/rating/SoReg.py:54-72) and SREE (model/rating/SREE.py:48-61) on the GPU.
//
//   social_user_pass_kernel -- the pass over the visiting order (the reference's `self.social.user` restricted to
//     training users), sequential-equivalent, on the in-order protocol of device.cuh (one warp per visit position,
//     lanes across d).  User u reads its own row and the rows of its followees (SoReg: and of its followers), and
//     writes its own row only; social_pass_step.cuh has the formulas.  Each user is visited at most once, so one
//     done flag per user records every dependency: before it reads, the warp at position k waits until done[v] is
//     set for every followee and follower v != u with 0 <= pos[v] < k.  Followees cover the reads of rows written
//     earlier; followers cover the other direction, an earlier follower having to read P[u] before u writes it
//     (SocialMF and SREE read no follower row, but still wait for them).  After writing P[u] the warp release-sets done[u].
//     A self-follow reads the pre-update row the warp holds; SREE moves the row after each followee in turn, so there
//     it reads the row as the followees before it left it.  Every wait is on earlier positions only, so the result
//     is that of the serial loop whatever the grid.
#include "common.h"
#include "device.cuh"
#include "lane_shape.h"
#include "social_pass_step.cuh"

namespace {

using namespace qrec;

constexpr int kSocialMF = 0;
constexpr int kSoReg = 1;
constexpr int kSREE = 2;    // reached through qrec_sree_user_pass_* only

// waits until done[v] is set for every neighbour v = cols[j] (j in [b, e)) visited before position k
__device__ __forceinline__ void wait_neighbours(const int* __restrict__ cols, long long b, long long e, int uu,
                                                const int* __restrict__ pos, long long k, const int* done, int lane) {
  for (long long base = b; base < e; base += 32) {
    const long long j = base + lane;
    const int* flag = nullptr;
    if (j < e) {
      const int v = __ldg(cols + j);
      const int pv = v != uu ? __ldg(pos + v) : -1;
      if (pv >= 0 && pv < k) flag = done + v;
    }
    spin_until<8, 64>([=] { return __all_sync(0xffffffffu, flag == nullptr || ld_acquire_gpu(flag) != 0); });
  }
}

template <typename T, int E, int KIND>
__global__ void __launch_bounds__(256)
social_user_pass_kernel(T* __restrict__ P, int d, long long n, const int* __restrict__ visit,
                        const int* __restrict__ pos, const long long* __restrict__ f_rowptr,
                        const int* __restrict__ f_cols, const T* __restrict__ f_val,
                        const long long* __restrict__ g_rowptr, const int* __restrict__ g_cols,
                        const T* __restrict__ g_val, int* done, unsigned long long* ticket, T lr, T coef,
                        double* loss) {
  const int lane = threadIdx.x & 31;
  double local_loss = 0.0;
  while (true) {
    const unsigned long long k = warp_next_ticket(ticket);
    if (k >= (unsigned long long)n) break;
    const int uu = __ldg(visit + k);
    const long long fb = __ldg(f_rowptr + uu), fe = __ldg(f_rowptr + uu + 1);
    const long long gb = __ldg(g_rowptr + uu), ge = __ldg(g_rowptr + uu + 1);
    wait_neighbours(f_cols, fb, fe, uu, pos, (long long)k, done, lane);
    wait_neighbours(g_cols, gb, ge, uu, pos, (long long)k, done, lane);

    T* pr = P + (size_t)uu * d;
    T p[E], a1[E], a2[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int c = e * 32 + lane;
      p[e] = c < d ? __ldcg(pr + c) : T(0);  // L2-coherent: the rows were last written by other SMs
      a1[e] = a2[e] = T(0);
    }
    if (KIND == kSocialMF) {
      T denom = 0;
      for (long long j = fb; j < fe; ++j) {
        const int f = __ldg(f_cols + j);
        const T w = __ldg(f_val + j);
        const T* row = P + (size_t)f * d;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int c = e * 32 + lane;
          if (c < d) a1[e] = socialmf_add(a1[e], w, f == uu ? p[e] : __ldcg(row + c));
        }
        denom = mf_add(denom, w);
      }
      if (denom != T(0)) {
        const T lr_regs = mf_mul(lr, coef);
        double sq = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int c = e * 32 + lane;
          if (c < d) {
            const T rl = socialmf_residual(p[e], a1[e], denom);
            sq += (double)rl * (double)rl;
            __stcg(pr + c, socialmf_step(p[e], lr_regs, rl));
          }
        }
        sq = warp_sum(sq);
        local_loss += (double)coef * sq;
      }
    } else if (KIND == kSREE) {
      const T lr_alpha = mf_mul(lr, coef);
      for (long long j = fb; j < fe; ++j) {
        const int f = __ldg(f_cols + j);
        const T w = __ldg(f_val + j);
        const T* row = P + (size_t)f * d;
        double sq = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int c = e * 32 + lane;
          if (c < d) {
            const T pf = f == uu ? p[e] : __ldcg(row + c);
            p[e] = sree_step(p[e], lr_alpha, w, pf);
            const T df = mf_sub(p[e], pf);
            sq += (double)df * (double)df;
          }
        }
        sq = warp_sum(sq);
        local_loss += (double)mf_mul(coef, w) * sq;    // SREE.py:60: alpha*weight*|p - z|^2 after the step
      }
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int c = e * 32 + lane;
        if (c < d) __stcg(pr + c, p[e]);
      }
    } else {
      double sim_sum = 0.0;
      for (long long j = fb; j < fe; ++j) {
        const int f = __ldg(f_cols + j);
        const T s = __ldg(f_val + j);
        const T* row = P + (size_t)f * d;
        double sq = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int c = e * 32 + lane;
          if (c < d) {
            const T pf = f == uu ? p[e] : __ldcg(row + c);
            a1[e] = soreg_add(a1[e], s, p[e], pf);
            const double df = (double)p[e] - (double)pf;
            sq += df * df;
          }
        }
        sq = warp_sum(sq);
        sim_sum += (double)s * sq;
        local_loss += sim_sum;  // SoReg.py:65: the running simSum, after every followee
      }
      for (long long j = gb; j < ge; ++j) {
        const int g = __ldg(g_cols + j);
        const T s = __ldg(g_val + j);
        const T* row = P + (size_t)g * d;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int c = e * 32 + lane;
          if (c < d) a2[e] = soreg_add(a2[e], s, p[e], g == uu ? p[e] : __ldcg(row + c));
        }
      }
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int c = e * 32 + lane;
        if (c < d) __stcg(pr + c, soreg_step(p[e], lr, coef, a1[e], a2[e]));
      }
    }
    warp_fence();
    if (lane == 0) red_release_gpu_add(done + uu, 1);
  }
  if (lane == 0 && local_loss != 0.0) atomicAdd(loss, local_loss);
}

// name: the entry point's name, as its messages show it; kind: checked by the caller
template <typename T>
int launch_pass(const char* name, int kind, T* P, int d, long long n, const int* visit, const int* pos,
                const long long* f_rowptr, const int* f_cols, const T* f_val, const long long* g_rowptr,
                const int* g_cols, const T* g_val, int* done, unsigned long long* ticket, T lr, T coef, double* loss,
                int n_warps, cudaStream_t st) {
  QREC_REQUIRE(d >= 1 && d <= 256, "%s: d=%d unsupported (1..256)", name, d);
  QREC_REQUIRE(n >= 0 && n < (1LL << 31), "%s: n=%lld outside [0, 2^31)", name, (long long)n);
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(P && visit && pos && f_rowptr && g_rowptr && done && ticket && loss, "%s: null pointer", name);
  QREC_REQUIRE(kind != kSoReg || g_val, "%s: SoReg needs the followers' similarities", name);
  const int grid = ordered_grid(n_warps);
  with_lane_elems(d, [&](auto e) {
    constexpr int E = decltype(e)::E;
    const auto kernel = kind == kSocialMF ? social_user_pass_kernel<T, E, kSocialMF>
                        : kind == kSoReg  ? social_user_pass_kernel<T, E, kSoReg>
                                          : social_user_pass_kernel<T, E, kSREE>;
    kernel<<<grid, 256, 0, st>>>(P, d, n, visit, pos, f_rowptr, f_cols, f_val, g_rowptr, g_cols, g_val, done, ticket,
                                 lr, coef, loss);
  });
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

template <typename T>
int launch_social(int kind, T* P, int d, long long n, const int* visit, const int* pos, const int64_t* f_rowptr,
                  const int* f_cols, const T* f_val, const int64_t* g_rowptr, const int* g_cols, const T* g_val,
                  int* done, unsigned long long* ticket, T lr, T coef, double* loss, int n_warps, void* stream) {
  QREC_REQUIRE(kind == kSocialMF || kind == kSoReg, "social_user_pass: kind=%d (0 SocialMF, 1 SoReg)", kind);
  return launch_pass<T>("social_user_pass", kind, P, d, n, visit, pos, (const long long*)f_rowptr, f_cols, f_val,
                        (const long long*)g_rowptr, g_cols, g_val, done, ticket, lr, coef, loss, n_warps,
                        (cudaStream_t)stream);
}

template <typename T>
int launch_sree(T* P, int d, long long n, const int* visit, const int* pos, const int64_t* f_rowptr, const int* f_cols,
                const T* f_w, const int64_t* g_rowptr, const int* g_cols, int* done, unsigned long long* ticket, T lr,
                T alpha, double* loss, int n_warps, void* stream) {
  return launch_pass<T>("sree_user_pass", kSREE, P, d, n, visit, pos, (const long long*)f_rowptr, f_cols, f_w,
                        (const long long*)g_rowptr, g_cols, (const T*)nullptr, done, ticket, lr, alpha, loss, n_warps,
                        (cudaStream_t)stream);
}

}  // namespace

extern "C" {

int qrec_social_user_pass_f64(int32_t kind, double* P, int32_t d, int64_t n, const int32_t* visit,
                              const int32_t* pos, const int64_t* f_rowptr, const int32_t* f_cols,
                              const double* f_val, const int64_t* g_rowptr, const int32_t* g_cols,
                              const double* g_val, int32_t* done, unsigned long long* ticket, double lr, double coef,
                              double* loss, int32_t n_warps, void* stream) {
  return launch_social<double>(kind, P, d, n, visit, pos, f_rowptr, f_cols, f_val, g_rowptr, g_cols, g_val, done,
                               ticket, lr, coef, loss, n_warps, stream);
}

int qrec_social_user_pass_f32(int32_t kind, float* P, int32_t d, int64_t n, const int32_t* visit, const int32_t* pos,
                              const int64_t* f_rowptr, const int32_t* f_cols, const float* f_val,
                              const int64_t* g_rowptr, const int32_t* g_cols, const float* g_val, int32_t* done,
                              unsigned long long* ticket, float lr, float coef, double* loss, int32_t n_warps,
                              void* stream) {
  return launch_social<float>(kind, P, d, n, visit, pos, f_rowptr, f_cols, f_val, g_rowptr, g_cols, g_val, done,
                              ticket, lr, coef, loss, n_warps, stream);
}

int qrec_sree_user_pass_f64(double* P, int32_t d, int64_t n, const int32_t* visit, const int32_t* pos,
                            const int64_t* f_rowptr, const int32_t* f_cols, const double* f_w, const int64_t* g_rowptr,
                            const int32_t* g_cols, int32_t* done, unsigned long long* ticket, double lr, double alpha,
                            double* loss, int32_t n_warps, void* stream) {
  return launch_sree<double>(P, d, n, visit, pos, f_rowptr, f_cols, f_w, g_rowptr, g_cols, done, ticket, lr, alpha,
                             loss, n_warps, stream);
}

int qrec_sree_user_pass_f32(float* P, int32_t d, int64_t n, const int32_t* visit, const int32_t* pos,
                            const int64_t* f_rowptr, const int32_t* f_cols, const float* f_w, const int64_t* g_rowptr,
                            const int32_t* g_cols, int32_t* done, unsigned long long* ticket, float lr, float alpha,
                            double* loss, int32_t n_warps, void* stream) {
  return launch_sree<float>(P, d, n, visit, pos, f_rowptr, f_cols, f_w, g_rowptr, g_cols, done, ticket, lr, alpha,
                            loss, n_warps, stream);
}

}  // extern "C"
