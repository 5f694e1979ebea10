// Host build of the scalar steps of SoRec's trust-edge pass (K9 kind 3, qrec_b200/csrc/mf_step.cuh) and of RSTE's
// prediction (qrec_b200/csrc/rste_step.cuh), so that the CPU suite can check the device source's arithmetic
// against Python floats.  Built with -ffp-contract=off: every product, sum and quotient is rounded on its own.
#include <cstdint>
#define __device__
#define __forceinline__ inline
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
#include "rste_step.cuh"

extern "C" {

// one trust edge on rows p, z of length d, given e = target - p.z: both rows in place; returns the loss term
double host_sorec_edge_f64(double* p, double* z, int d, double err, double lr, double reg_s, double reg_z) {
  const double g = qrec::mf_step_scale<double, 3>(err, lr, reg_s);
  for (int c = 0; c < d; ++c) {
    double pn, zn;
    qrec::mf_update_parity<double, 3>(p[c], z[c], err, g, lr, reg_s, reg_z, pn, zn);
    p[c] = pn;
    z[c] = zn;
  }
  return qrec::mf_loss_term<double, 3>(err, reg_s);
}

// the social sum over n followee dots in order, then the blend
double host_rste_prediction_f64(double dot, const double* w, const double* fdot, int n, double alpha, double denom) {
  double s = 0;
  for (int k = 0; k < n; ++k) s = qrec::rste_social_add(s, w[k], fdot[k]);
  return qrec::rste_prediction(dot, s, alpha, denom);
}

}  // extern "C"
