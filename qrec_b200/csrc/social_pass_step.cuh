// Scalar pieces of the trust-neighbourhood user pass (social_pass_kernels.cu, K17), kept apart so that the CPU suite
// can compile and run the very same source (tests/host_shims/social_pass_step_host.cpp).  numpy's evaluation order,
// every product, sum and quotient rounded separately (the mf_* helpers never contract into an FMA).
//
//   SocialMF.py:26-43, one training user u, its cleaned followees f with weights w_f in dict order:
//     fPred = sum_f w_f*P[f],  denom = sum_f w_f                     both from 0, in the followee order
//     rl    = P[u] - fPred/denom   (0 when denom == 0)
//     P[u] -= (lr*regS)*rl ;  loss += regS*(rl.rl)
//   SoReg.py:54-72, one training user u, followees f and followers g with the similarities Sim[u][.]:
//     f1 = sum_f Sim[u][f]*(P[u]-P[f]),  f2 = sum_g Sim[u][g]*(P[u]-P[g])     both from 0, in dict order
//     P[u] += lr*((-alpha)*(f1+f2))
//     loss += simSum after every followee, simSum += Sim[u][f]*|P[u]-P[f]|^2 (the running sum, as the reference)
//   P[u] on the right-hand sides is u's row before the update, also where u follows itself.
//   SREE.py:48-61, one training user u, its cleaned followees f with weights w_f in dict order, one after another:
//     P[u] -= ((lr*alpha)*w_f)*(P[u]-P[f]) ;  loss += (alpha*w_f)*|P[u]-P[f]|^2 with the updated P[u]
//   Here P[u] is the row as moved by the followees before f; a self-follow reads that row and moves nothing.
#pragma once

#include "rste_step.cuh"

namespace qrec {

// SocialMF: one followee's term of fPred (one component) and of denom
template <typename T>
__device__ __forceinline__ T socialmf_add(T fpred, T w, T pf) {
  return mf_add(fpred, mf_mul(w, pf));
}

// SocialMF: rl = P[u] - fPred/denom (one component; the caller skips the update when denom == 0)
template <typename T>
__device__ __forceinline__ T socialmf_residual(T p, T fpred, T denom) {
  return mf_sub(p, mf_div(fpred, denom));
}

// SocialMF: P[u] -= lr_regs*rl, lr_regs = lr*regS formed first
template <typename T>
__device__ __forceinline__ T socialmf_step(T p, T lr_regs, T rl) {
  return mf_sub(p, mf_mul(lr_regs, rl));
}

// SoReg: one neighbour's term of f1 or f2 (one component): f + s*(p - pv)
template <typename T>
__device__ __forceinline__ T soreg_add(T f, T s, T p, T pv) {
  return mf_add(f, mf_mul(s, mf_sub(p, pv)));
}

// SoReg: P[u] += lr*((-alpha)*(f1+f2))
template <typename T>
__device__ __forceinline__ T soreg_step(T p, T lr, T alpha, T f1, T f2) {
  return mf_add(p, mf_mul(lr, mf_mul(-alpha, mf_add(f1, f2))));
}

// SREE: one followee's step on one component, P[u] -= (lr_alpha*w)*(p - pf), lr_alpha = lr*alpha formed first
template <typename T>
__device__ __forceinline__ T sree_step(T p, T lr_alpha, T w, T pf) {
  return mf_sub(p, mf_mul(mf_mul(lr_alpha, w), mf_sub(p, pf)));
}

}  // namespace qrec
