// Per-pair arithmetic of the memory-based rating models (knn_kernels.cu): the co-rated sums of the three similarities
// and of SlopeOne's deviation, and how each sum becomes a similarity.  Kept apart so that the CPU suite can compile
// and run the very same source (tests/host_shims/knn_step_host.cpp).
//
//   reference: util/qmath.py (pearson_sp, cosine_sp, euclidean_sp) and model/rating/SlopeOne.py (computeAverage).
//   Every sum runs over x1's entries in insertion order, restricted to the keys x2 shares, from 0:
//     pcc        t += (a-m1)*(b-m2),  d1 += (a-m1)**2,  d2 += (b-m2)**2     -> t / (sqrt(d1)*sqrt(d2))
//     cos        t += a*b,            d1 += a**2,       d2 += b**2           -> t / (sqrt(d1)*sqrt(d2))
//     euclidean  t += a**2 - b**2                                            -> 1 / t
//     SlopeOne   t += a - b,          n += 1                                 -> t / n
//   `** 2` is CPython's float pow (glibc pow(x, 2.0)), which is not always the correctly rounded x*x, so the squares
//   are not formed here: each entry carries its own square `sa` / `sb`, computed on the host.  Every other product,
//   sum, quotient and root is a separately rounded IEEE operation, as in the reference.
//   A zero denominator raises ZeroDivisionError in the reference and returns: pcc 1 when a key was shared, else 0;
//   cos 0; euclidean 0.
#pragma once

namespace qrec {

enum KnnMetric { kPearson = 0, kCosine = 1, kEuclidean = 2 };

struct KnnAcc {
  double t, d1, d2;
  int n;                 // shared keys seen so far
};

#ifdef __CUDA_ARCH__
#define QREC_KNN_ADD(x, y) __dadd_rn(x, y)
#define QREC_KNN_SUB(x, y) __dsub_rn(x, y)
#define QREC_KNN_MUL(x, y) __dmul_rn(x, y)
#define QREC_KNN_DIV(x, y) __ddiv_rn(x, y)
#define QREC_KNN_SQRT(x) __dsqrt_rn(x)
#else
#define QREC_KNN_ADD(x, y) ((x) + (y))
#define QREC_KNN_SUB(x, y) ((x) - (y))
#define QREC_KNN_MUL(x, y) ((x) * (y))
#define QREC_KNN_DIV(x, y) ((x) / (y))
#define QREC_KNN_SQRT(x) sqrt(x)
#endif

// one shared key: x1's entry (a, its square sa, x1's mean m1) against x2's (b, sb, m2).  The means are read by pcc
// only; the squares already hold (a-m1)**2 for pcc and a**2 for cos / euclidean.
template <int M>
__host__ __device__ __forceinline__ void knn_add(KnnAcc& acc, double a, double sa, double m1, double b, double sb,
                                                 double m2) {
  if (M == kPearson) {
    acc.t = QREC_KNN_ADD(acc.t, QREC_KNN_MUL(QREC_KNN_SUB(a, m1), QREC_KNN_SUB(b, m2)));
    acc.d1 = QREC_KNN_ADD(acc.d1, sa);
    acc.d2 = QREC_KNN_ADD(acc.d2, sb);
  } else if (M == kCosine) {
    acc.t = QREC_KNN_ADD(acc.t, QREC_KNN_MUL(a, b));
    acc.d1 = QREC_KNN_ADD(acc.d1, sa);
    acc.d2 = QREC_KNN_ADD(acc.d2, sb);
  } else {
    acc.t = QREC_KNN_ADD(acc.t, QREC_KNN_SUB(sa, sb));
  }
  acc.n += 1;
}

template <int M>
__host__ __device__ __forceinline__ double knn_similarity(const KnnAcc& acc) {
  if (acc.n == 0) return 0.0;
  if (M == kEuclidean) return acc.t == 0.0 ? 0.0 : QREC_KNN_DIV(1.0, acc.t);
  const double den = QREC_KNN_MUL(QREC_KNN_SQRT(acc.d1), QREC_KNN_SQRT(acc.d2));
  if (den == 0.0) return M == kPearson ? 1.0 : 0.0;
  return QREC_KNN_DIV(acc.t, den);
}

// SlopeOne: one user who rated both items, x_i[u] = a and x_j[u] = b
__host__ __device__ __forceinline__ void slopeone_add(KnnAcc& acc, double a, double b) {
  acc.t = QREC_KNN_ADD(acc.t, QREC_KNN_SUB(a, b));
  acc.n += 1;
}

// the stored average deviation: diff / count, or 0 when no user rated both
__host__ __device__ __forceinline__ double slopeone_average(const KnnAcc& acc) {
  return acc.n == 0 ? 0.0 : QREC_KNN_DIV(acc.t, (double)acc.n);
}

// one of the user's rated items j (rating r) in SlopeOne's prediction: sum += (r + diffAvg[i][j]) * count[i][j]
__host__ __device__ __forceinline__ double slopeone_vote(double sum, double r, const KnnAcc& acc) {
  return QREC_KNN_ADD(sum, QREC_KNN_MUL(QREC_KNN_ADD(r, slopeone_average(acc)), (double)acc.n));
}

// one neighbour n (similarity s, rating r, mean m) in a KNN prediction: sum += s*(r - m), denom += s
__host__ __device__ __forceinline__ void knn_vote(double& sum, double& denom, double s, double r, double m) {
  sum = QREC_KNN_ADD(sum, QREC_KNN_MUL(s, QREC_KNN_SUB(r, m)));
  denom = QREC_KNN_ADD(denom, s);
}

}  // namespace qrec
