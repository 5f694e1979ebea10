// Per-item arithmetic of the CoFactor item sweep (als_kernels.cu) that als_step.cuh does not already hold: the SPPMI
// terms of the two right-hand sides and the w / c updates.  Kept apart so that the CPU suite can compile and run the
// very same source (tests/host_shims/cofactor_step_host.cpp).
//
//   reference: model/ranking/CoFactor.py, trainModel, item loop.  For item i with contexts c (SPPMI values m):
//     A_Y = XtX + sum_u alpha*r x x^T + regU*I + sum_c G_c G_c^T     b_Y = sum_u (1 + alpha*r) x + sum_c ((m - w_i) - c_c) G_c
//     A_G = sum_c Y_c Y_c^T + gamma*I                                 b_G = sum_c ((m - w_c) - c_i) Y_c
//     w_i = mean_c ((m - Y_i.G_c) - c_c)                              c_i = mean_c ((m - Y_c.G_i) - w_c)
//   with Y_i, G_i, w_i, c_i the item's values from before its own update.  The operand order of every difference is
//   the reference's.
#pragma once

namespace qrec {

// coefficient of G_c in b_Y
__host__ __device__ __forceinline__ double cof_rhs_y_coef(double m, double w_i, double c_c) { return (m - w_i) - c_c; }
// coefficient of Y_c in b_G
__host__ __device__ __forceinline__ double cof_rhs_g_coef(double m, double w_c, double c_i) { return (m - w_c) - c_i; }
// one context's term of w_i's sum (yg = Y_i.G_c) and of c_i's sum (yg = Y_c.G_i)
__host__ __device__ __forceinline__ double cof_w_term(double m, double yg, double c_c) { return (m - yg) - c_c; }
__host__ __device__ __forceinline__ double cof_c_term(double m, double yg, double w_c) { return (m - yg) - w_c; }
// update_w / len(SPPMI[item]) (called only for items that have contexts)
__host__ __device__ __forceinline__ double cof_mean(double sum, int n) { return sum / (double)n; }

}  // namespace qrec
