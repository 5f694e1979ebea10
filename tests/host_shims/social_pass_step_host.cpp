// Host build of the user-pass formulas of SocialMF and SoReg (K17, qrec_b200/csrc/social_pass_step.cuh) and of
// SocialMF's rating step (K9 kind 4, qrec_b200/csrc/mf_step.cuh), so that the CPU suite can check the device
// source's arithmetic against Python floats.  Built with -ffp-contract=off: every product, sum and quotient is
// rounded on its own.
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

// one rating entry of SocialMF on rows p, q of length d, given e = r - p.q: both rows in place (kind 4)
void host_socialmf_rating_f64(double* p, double* q, int d, double err, double lr, double reg_u, double reg_i) {
  for (int c = 0; c < d; ++c) {
    double pn, qn;
    qrec::mf_update_parity<double, 4>(p[c], q[c], err, qrec::mf_step_scale<double, 4>(err, lr, reg_u), lr, reg_u,
                                      reg_i, pn, qn);
    p[c] = pn;
    q[c] = qn;
  }
}

// SocialMF's user step on p (length d) from its n followee rows (n x d, row-major) and weights; in place
void host_socialmf_user_f64(double* p, int d, const double* rows, const double* w, int n, double lr, double reg_s) {
  double denom = 0;
  for (int k = 0; k < n; ++k) denom = qrec::mf_add(denom, w[k]);
  if (denom == 0) return;
  for (int c = 0; c < d; ++c) {
    double f = 0;
    for (int k = 0; k < n; ++k) f = qrec::socialmf_add(f, w[k], rows[k * d + c]);
    p[c] = qrec::socialmf_step(p[c], qrec::mf_mul(lr, reg_s), qrec::socialmf_residual(p[c], f, denom));
  }
}

// SoReg's user step on p (length d) from its nf followee rows / similarities and ng follower rows / similarities
void host_soreg_user_f64(double* p, int d, const double* frows, const double* fs, int nf, const double* grows,
                         const double* gs, int ng, double lr, double alpha) {
  for (int c = 0; c < d; ++c) {
    double f1 = 0, f2 = 0;
    for (int k = 0; k < nf; ++k) f1 = qrec::soreg_add(f1, fs[k], p[c], frows[k * d + c]);
    for (int k = 0; k < ng; ++k) f2 = qrec::soreg_add(f2, gs[k], p[c], grows[k * d + c]);
    p[c] = qrec::soreg_step(p[c], lr, alpha, f1, f2);
  }
}

}  // extern "C"
