// Scalar pieces of the K9 step (mf_kernels.cu), kept apart so that the CPU suite can compile and run
// the very same source (tests/host_shims/mf_step_host.cpp).  Parity flavour: numpy's evaluation order,
// every product and sum rounded separately (__fmul_rn / __fadd_rn never contract into an FMA).
//   kind 0  BasicMF.py:22-23   P[u] += (lr*e)*q ;           Q[i] += (lr*e)*P[u]
//   kind 1  PMF.py:21-22       P[u] += lr*(e*q - regU*p) ;  Q[i] += lr*(e*P[u] - regI*q)
//   kind 2  SVD.py:27-30,88    kind 1 + biases; prediction = ((dot + mean) + Bi[i]) + Bu[u]
//   kind 3  SoRec.py:42-60     one trust edge (u, v) on the tables (P, Z); the "rating" is weight*tuv, regS and
//                              regZ travel in the reg_u / reg_i slots and g = regS*e:
//                              P[u] += lr*(g*z) ;  Z[v] += lr*(g*P[u] - regZ*z) ;  loss += regS*e^2
//   kind 4  SocialMF.py:15-24  kind 1 on copies of both rows: the item step reads the user row as it was before
//                              P[u] += lr*(e*q - regU*p) ;  Q[i] += lr*(e*p - regI*q)
//   kind 5  EE.py:15-36        Euclidean embedding with biases; `dot` is dist = |p-q|^2 and the
//                              prediction ((globalMean + Bi[i]) + Bu[u]) - dist:
//                              P[u] -= (lr*(e+regU))*(p-q) ;  Q[i] += (lr*(e+regI))*(P[u]-q) ;
//                              loss += e^2 + regU*dist
#pragma once

namespace qrec {

__device__ __forceinline__ float mf_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float mf_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float mf_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double mf_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double mf_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double mf_sub(double a, double b) { return __dsub_rn(a, b); }

template <typename T, int KIND>
__device__ __forceinline__ T mf_prediction(T dot, T global_mean, T bi, T bu) {
  if (KIND == 5) return mf_sub(mf_add(mf_add(global_mean, bi), bu), dot);
  return KIND == 2 ? mf_add(mf_add(mf_add(dot, global_mean), bi), bu) : dot;
}

// the scalar the kernels hand to mf_update_parity as g: lr*err for kind 0, regS*err for kind 3 (unused otherwise)
template <typename T, int KIND>
__device__ __forceinline__ T mf_step_scale(T err, T lr, T reg_u) {
  return KIND == 3 ? mf_mul(reg_u, err) : mf_mul(lr, err);
}

// one component of both rows; g = mf_step_scale(err, lr, reg_u) (kinds 0 and 3)
template <typename T, int KIND>
__device__ __forceinline__ void mf_update_parity(T p, T q, T err, T g, T lr, T reg_u, T reg_i, T& pn, T& qn) {
  if (KIND == 0) {
    pn = mf_add(p, mf_mul(g, q));
    qn = mf_add(q, mf_mul(g, pn));
  } else if (KIND == 3) {
    pn = mf_add(p, mf_mul(lr, mf_mul(g, q)));
    qn = mf_add(q, mf_mul(lr, mf_sub(mf_mul(g, pn), mf_mul(reg_i, q))));
  } else if (KIND == 4) {
    pn = mf_add(p, mf_mul(lr, mf_sub(mf_mul(err, q), mf_mul(reg_u, p))));
    qn = mf_add(q, mf_mul(lr, mf_sub(mf_mul(err, p), mf_mul(reg_i, q))));
  } else if (KIND == 5) {
    pn = mf_sub(p, mf_mul(mf_mul(lr, mf_add(err, reg_u)), mf_sub(p, q)));
    qn = mf_add(q, mf_mul(mf_mul(lr, mf_add(err, reg_i)), mf_sub(pn, q)));
  } else {
    pn = mf_add(p, mf_mul(lr, mf_sub(mf_mul(err, q), mf_mul(reg_u, p))));
    qn = mf_add(q, mf_mul(lr, mf_sub(mf_mul(err, pn), mf_mul(reg_i, q))));
  }
}

// the entry's term of the epoch loss: e^2, regS*e^2 for a trust edge (kind 3), e^2 + regU*dist for EE (kind 5)
template <typename T, int KIND>
__device__ __forceinline__ double mf_loss_term(T err, T reg_u, T dist = T(0)) {
  const double sq = (double)err * (double)err;
  if (KIND == 5) return sq + (double)reg_u * (double)dist;
  return KIND == 3 ? (double)reg_u * sq : sq;
}

template <typename T>
__device__ __forceinline__ T mf_bias_parity(T b, T err, T lr, T reg_b) {
  return mf_add(b, mf_mul(lr, mf_sub(err, mf_mul(reg_b, b))));
}

// throughput flavour: the row DELTAS of one component (fp32, contraction allowed)
template <int KIND>
__device__ __forceinline__ void mf_delta_fast(float p, float q, float e, float lr, float reg_u, float reg_i,
                                              float& dp, float& dq) {
  if (KIND == 0) {
    dp = (lr * e) * q;
    dq = (lr * e) * (p + dp);
  } else {
    dp = lr * (e * q - reg_u * p);
    dq = lr * (e * (p + dp) - reg_i * q);
  }
}

}  // namespace qrec
