// Host build of qrec_b200/csrc/svdpp_step.cuh: replays svdpp_sgd_ordered_kernel's arithmetic entry by entry on the
// CPU -- sequential column sums, per-column dot terms, the warp xor-butterfly and the warp-order sum of the block
// reduction, then the header's own step functions -- and svdpp_usermajor_kernel's closed form with one user in
// flight, so the CPU suite pins the device source to the reference's golden run and to the numpy oracle.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <vector>

#include "svdpp_step.cuh"

namespace {

// the 256 per-thread values of one block reduction (thread c holds column c's term, the rest 0)
template <typename T>
T block_sum(const T* terms, int d) {
  T warp_total[8];
  for (int w = 0; w < 8; ++w) {
    T v[32];
    for (int lane = 0; lane < 32; ++lane) {
      const int c = w * 32 + lane;
      v[lane] = c < d ? terms[c] : (T)0;
    }
    for (int o = 16; o > 0; o >>= 1) {          // v += __shfl_xor_sync(v, o) on all lanes at once
      T x[32];
      for (int lane = 0; lane < 32; ++lane) x[lane] = v[lane] + v[lane ^ o];
      for (int lane = 0; lane < 32; ++lane) v[lane] = x[lane];
    }
    warp_total[w] = v[0];
  }
  T s = warp_total[0];
  for (int w = 1; w < 8; ++w) s = qrec::sp_add(s, warp_total[w]);
  return s;
}

template <typename T>
double ordered_epoch(T* P, T* Q, T* Y, T* Bu, T* Bi, int d, int64_t n, const int32_t* u, const int32_t* i, const T* r,
                     const int64_t* rowptr, const int32_t* cols, T lr, T reg_u, T reg_i, T reg_b, T reg_y, T gm) {
  double loss = 0.0;
  std::vector<T> s_all(d), s_ex(d), ty(d), tp(d), q_old(d);
  for (int64_t k = 0; k < n; ++k) {
    const int uu = u[k], ii = i[k];
    const int64_t beg = rowptr[uu], end = rowptr[uu + 1];
    const int w = (int)(end - beg);
    for (int c = 0; c < d; ++c) {
      T a = 0, b = 0;
      for (int64_t x = beg; x < end; ++x) {
        const T y = Y[(size_t)cols[x] * d + c];
        a = qrec::sp_add(a, y);
        if (cols[x] != ii) b = qrec::sp_add(b, y);
      }
      s_all[c] = a;
      s_ex[c] = b;
    }
    T* p = P + (size_t)uu * d;
    T* q = Q + (size_t)ii * d;
    for (int c = 0; c < d; ++c) {
      q_old[c] = q[c];
      qrec::svdpp_dot_terms_parity<T>(s_all[c], (T)w, p[c], q[c], ty[c], tp[c]);
    }
    const T dot_y = block_sum<T>(ty.data(), d), dot_p = block_sum<T>(tp.data(), d);
    const T bu = Bu[uu], bi = Bi[ii];
    const T err = qrec::svdpp_error_parity<T>(r[k], dot_y, dot_p, gm, bi, bu);
    Bu[uu] = qrec::svdpp_bias_parity<T>(bu, err, lr, reg_b);
    Bi[ii] = qrec::svdpp_bias_parity<T>(bi, err, lr, reg_b);
    loss += (double)err * (double)err;
    const T wm1 = (T)(w - 1);
    if (w > 1) {
      for (int64_t x = beg; x < end; ++x) {
        if (cols[x] == ii) continue;
        T* yr = Y + (size_t)cols[x] * d;
        for (int c = 0; c < d; ++c) yr[c] = qrec::svdpp_y_parity<T>(yr[c], err, q_old[c], wm1, lr, reg_y);
      }
    }
    for (int c = 0; c < d; ++c) {
      T pn, qn;
      qrec::svdpp_pq_parity<T>(p[c], q_old[c], s_ex[c], w > 1, err, wm1, lr, reg_u, reg_i, pn, qn);
      p[c] = pn;
      q[c] = qn;
    }
  }
  return loss;
}

}  // namespace

extern "C" {

double host_svdpp_ordered_f64(double* P, double* Q, double* Y, double* Bu, double* Bi, int d, int64_t n,
                              const int32_t* u, const int32_t* i, const double* r, const int64_t* rowptr,
                              const int32_t* cols, double lr, double reg_u, double reg_i, double reg_b, double reg_y,
                              double gm) {
  return ordered_epoch<double>(P, Q, Y, Bu, Bi, d, n, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y, gm);
}

double host_svdpp_ordered_f32(float* P, float* Q, float* Y, float* Bu, float* Bi, int d, int64_t n, const int32_t* u,
                              const int32_t* i, const float* r, const int64_t* rowptr, const int32_t* cols, float lr,
                              float reg_u, float reg_i, float reg_b, float reg_y, float gm) {
  return ordered_epoch<float>(P, Q, Y, Bu, Bi, d, n, u, i, r, rowptr, cols, lr, reg_u, reg_i, reg_b, reg_y, gm);
}

// svdpp_usermajor_kernel with one user in flight: the users row_order[0..n_rows) one after another (fp32)
double host_svdpp_usermajor_f32(float* P, float* Q, float* Y, float* Bu, float* Bi, int d, int n_rows,
                                const int32_t* row_order, const int64_t* rowptr, const int32_t* cols,
                                const float* vals, float lr, float reg_u, float reg_i, float reg_b, float reg_y,
                                float gm) {
  double loss = 0.0;
  const float omc = lr * reg_y, c = 1.f - omc, lc = std::log1p(-omc);
  std::vector<float> S(d), B(d), dq(d), dy(d), y0(d), q(d);
  for (int pos = 0; pos < n_rows; ++pos) {
    const int uu = row_order[pos];
    const int64_t beg = rowptr[uu];
    const int W = (int)(rowptr[uu + 1] - beg);
    if (W == 0) continue;
    float* p = P + (size_t)uu * d;
    float bu = Bu[uu];
    const bool implicit = W > 1;
    for (int x = 0; x < d; ++x) S[x] = B[x] = 0.f;
    for (int t = 0; t < W; ++t)
      for (int x = 0; x < d; ++x) S[x] += Y[(size_t)cols[beg + t] * d + x];
    qrec::SvdppCfScalars k;
    k.lr = lr; k.reg_u = reg_u; k.reg_i = reg_i; k.c = c; k.omc = omc;
    k.wm1 = (float)(W - 1);
    k.cw1m1 = std::expm1((float)(W - 1) * lc);
    k.ct = 1.f;
    for (int t = 0; t < W; ++t) {
      const int j = cols[beg + t];
      float dot = 0.f;
      for (int x = 0; x < d; ++x) {
        q[x] = Q[(size_t)j * d + x];
        y0[x] = Y[(size_t)j * d + x];
        dot += (S[x] / (float)W + p[x]) * q[x];
      }
      const float bi = Bi[j];
      const float e = vals[beg + t] - (((dot + gm) + bi) + bu);
      bu += lr * (e - reg_b * bu);
      k.e = e;
      k.le = implicit ? lr * e / k.wm1 : 0.f;
      k.crest = implicit ? std::exp((float)(W - 1 - t) * lc) : 0.f;
      for (int x = 0; x < d; ++x) qrec::svdpp_cf_component(k, implicit, p[x], q[x], y0[x], S[x], B[x], dq[x], dy[x]);
      k.ct *= c;
      for (int x = 0; x < d; ++x) {
        Q[(size_t)j * d + x] += dq[x];
        if (implicit) Y[(size_t)j * d + x] += dy[x];
      }
      Bi[j] += lr * (e - reg_b * bi);
      loss += (double)e * (double)e;
    }
    if (implicit)
      for (int t = 0; t < W; ++t)
        for (int x = 0; x < d; ++x) Y[(size_t)cols[beg + t] * d + x] += B[x];
    Bu[uu] = bu;
  }
  return loss;
}

}  // extern "C"
