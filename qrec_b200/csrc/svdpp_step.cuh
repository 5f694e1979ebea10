// Arithmetic of the K11 (SVD++) kernels (svdpp_kernels.cu), kept apart so that the CPU suite can compile and run
// the very same source (tests/host_shims/svdpp_step_host.cpp).
//
//   reference: model/rating/SVDPlusPlus.py:30-61 (step), 70-88 (predictForRating).  Per entry (u, i, r), with N(u)
//   the user's distinct items and w = |N(u)|:
//     pred = (sum_{N(u)} Y / w).Q[i] + (((P[u].Q[i] + mean) + Bi[i]) + Bu[u]);   e = r - pred
//     Bu[u], Bi[i] += lr*(e - regB*b)
//     w > 1:  Y[j] += lr*((e*q)/(w-1) - regY*Y[j])  (j in N(u), j != i; q = old Q[i]);  Q[i] += ((lr*e)*sum)/(w-1)
//     P[u] += lr*(e*Q[i] - regU*P[u]);  Q[i] += lr*(e*P[u] - regI*Q[i])
//
// Parity flavour (svdpp_*_parity): numpy's evaluation order, every product, quotient and sum rounded separately
// (the __*_rn intrinsics never contract into an FMA; the host build uses -ffp-contract=off).
//
// Closed-form flavour (svdpp_cf_component, fp32, contraction allowed): one user's W distinct items i_0..i_{W-1} in
// order.  With c = 1 - lr*regY and v_t = lr*e_t*q_t/(W-1), the Y rows of the user after step t are
//     Y_j(t) = c^t Y_j(0) + B_t  for items not yet visited,  B_0 = 0,  B_{t+1} = c B_t + v_t,
// and S_t = sum_j Y_j(t) follows S_{t+1} = c (S_t - y_t) + (W-1) v_t + y_t with y_t = c^t Y_{i_t}(0) + B_t.  The
// final row of j = i_s is c^{W-1} Y_j(0) + B_W + c^{W-1-s} ((1-c) B_s - v_s): the kernel adds the part that does not
// involve B_W at step s and B_W to every row of the user at the end.
#pragma once

#ifndef __CUDACC__
#define __host__
#define __device__
#define __forceinline__ inline
#endif

namespace qrec {

__host__ __device__ __forceinline__ float sp_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float sp_add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float sp_sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float sp_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__host__ __device__ __forceinline__ double sp_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double sp_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double sp_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ double sp_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// ---- parity flavour
// one column's terms of the two dot products: (s_all/w)*q and p*q
template <typename T>
__host__ __device__ __forceinline__ void svdpp_dot_terms_parity(T s_all, T w, T p, T q, T& ty, T& tp) {
  ty = sp_mul(sp_div(s_all, w), q);
  tp = sp_mul(p, q);
}

// SVDPlusPlus.py:80-81: pred = dot_y; pred += P.Q + mean + Bi + Bu (left to right)
template <typename T>
__host__ __device__ __forceinline__ T svdpp_error_parity(T rating, T dot_y, T dot_p, T global_mean, T bi, T bu) {
  return sp_sub(rating, sp_add(dot_y, sp_add(sp_add(sp_add(dot_p, global_mean), bi), bu)));
}

template <typename T>
__host__ __device__ __forceinline__ T svdpp_bias_parity(T b, T err, T lr, T reg_b) {
  return sp_add(b, sp_mul(lr, sp_sub(err, sp_mul(reg_b, b))));
}

// SVDPlusPlus.py:54: one element of an implicit row j != i; q = the old Q[i]
template <typename T>
__host__ __device__ __forceinline__ T svdpp_y_parity(T y, T err, T q, T wm1, T lr, T reg_y) {
  return sp_add(y, sp_mul(lr, sp_sub(sp_div(sp_mul(err, q), wm1), sp_mul(reg_y, y))));
}

// SVDPlusPlus.py:55,57-58: one column of Q[i] and P[u]; wm1 = w - 1, s_ex = the old Y rows of N(u)\{i} summed in order
template <typename T>
__host__ __device__ __forceinline__ void svdpp_pq_parity(T p, T q, T s_ex, bool implicit, T err, T wm1, T lr, T reg_u,
                                                         T reg_i, T& pn, T& qn) {
  const T q1 = implicit ? sp_add(q, sp_div(sp_mul(sp_mul(lr, err), s_ex), wm1)) : q;
  pn = sp_add(p, sp_mul(lr, sp_sub(sp_mul(err, q1), sp_mul(reg_u, p))));
  qn = sp_add(q1, sp_mul(lr, sp_sub(sp_mul(err, pn), sp_mul(reg_i, q1))));
}

// ---- closed-form flavour: one column of step t of a user with W > 1 items (W = 1: implicit = false, no Y terms).
// In: p, q (row values now), y0 = Y_{i_t}(0), S = S_t, B = B_t; ct = c^t, c, omc = 1 - c, cw1m1 = c^{W-1} - 1,
// crest = c^{W-1-t}, le = lr*e/(W-1), wm1 = W - 1.  Out: the new p, the deltas of Q[i_t] and (partially) Y[i_t], S and B
// advanced to step t+1.
struct SvdppCfScalars {
  float e, lr, reg_u, reg_i, c, omc, cw1m1, ct, crest, le, wm1;
};

__host__ __device__ __forceinline__ void svdpp_cf_component(const SvdppCfScalars& k, bool implicit, float& p, float q,
                                                            float y0, float& S, float& B, float& dq, float& dy) {
  float qn = q;
  if (implicit) {
    const float yt = k.ct * y0 + B;
    const float v = k.le * q;
    qn = q + k.le * (S - yt);
    dy = k.cw1m1 * y0 + k.crest * (k.omc * B - v);
    S = k.c * (S - yt) + k.wm1 * v + yt;
    B = k.c * B + v;
  } else {
    dy = 0.f;
  }
  p = p + k.lr * (k.e * qn - k.reg_u * p);
  dq = (qn - q) + k.lr * (k.e * p - k.reg_i * qn);
}

}  // namespace qrec
