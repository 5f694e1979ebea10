// Host build of EE's rating step (K9 kind 5, qrec_b200/csrc/mf_step.cuh) and SREE's followee step (K17,
// qrec_b200/csrc/social_pass_step.cuh), so that the CPU suite can check the device source's arithmetic against Python
// floats.  Built with -ffp-contract=off: every product, sum and difference is rounded on its own.
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
#include "social_pass_step.cuh"

extern "C" {

// one EE entry on rows p, q of length d and the biases *bu, *bi, given dist = |p-q|^2 (summed by the caller): rows
// and biases in place; returns the entry's loss term
double host_ee_rating_f64(double* p, double* q, int d, double dist, double r, double gm, double* bu, double* bi,
                          double lr, double reg_u, double reg_i, double reg_b) {
  const double err = qrec::mf_sub(r, qrec::mf_prediction<double, 5>(dist, gm, *bi, *bu));
  const double g = qrec::mf_step_scale<double, 5>(err, lr, reg_u);
  for (int c = 0; c < d; ++c) {
    double pn, qn;
    qrec::mf_update_parity<double, 5>(p[c], q[c], err, g, lr, reg_u, reg_i, pn, qn);
    p[c] = pn;
    q[c] = qn;
  }
  const double b_u = *bu, b_i = *bi;
  *bu = qrec::mf_bias_parity<double>(b_u, err, lr, reg_b);
  *bi = qrec::mf_bias_parity<double>(b_i, err, lr, reg_b);
  return qrec::mf_loss_term<double, 5>(err, reg_u, dist);
}

// SREE's user step on p (length d) from its n followee rows (n x d, row-major) and weights, in turn; is_self[k] marks
// a self-follow, which reads p itself.  In place; returns the loss terms, each followee's squared distance summed in
// column order
double host_sree_user_f64(double* p, int d, const double* rows, const double* w, const int* is_self, int n, double lr,
                          double alpha) {
  const double lr_alpha = qrec::mf_mul(lr, alpha);
  double loss = 0.0;
  for (int k = 0; k < n; ++k) {
    double sq = 0.0;
    for (int c = 0; c < d; ++c) {
      const double pf = is_self[k] ? p[c] : rows[k * d + c];
      p[c] = qrec::sree_step(p[c], lr_alpha, w[k], pf);
      const double df = qrec::mf_sub(p[c], pf);
      sq += df * df;
    }
    loss += qrec::mf_mul(alpha, w[k]) * sq;
  }
  return loss;
}

}  // extern "C"
