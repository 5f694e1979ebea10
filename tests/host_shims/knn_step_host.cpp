// Host build of qrec_b200/csrc/knn_step.cuh: the similarity of listed row pairs (x1, x2) of a CSR, with the header's
// own knn_add / knn_similarity walking x1's entries in order -- so the CPU suite pins the device source to the float64
// oracle.  Compiled with -ffp-contract=off, as the device code keeps every product and sum separately rounded.
#include <cmath>
#include <cstdint>
#include <vector>
#define __host__
#define __device__
#define __forceinline__ inline
#include "knn_step.cuh"

template <int M>
static double pair_similarity(const int64_t* rowptr, const int32_t* cols, const double* vals, const double* sq,
                              const double* means, int32_t n_cols, int32_t a, int32_t b) {
  std::vector<int64_t> at(n_cols, -1);
  for (int64_t f = rowptr[b]; f < rowptr[b + 1]; ++f) at[cols[f]] = f;
  qrec::KnnAcc acc{0.0, 0.0, 0.0, 0};
  for (int64_t e = rowptr[a]; e < rowptr[a + 1]; ++e) {
    const int64_t f = at[cols[e]];
    if (f >= 0) qrec::knn_add<M>(acc, vals[e], sq[e], means[a], vals[f], sq[f], means[b]);
  }
  return qrec::knn_similarity<M>(acc);
}

// out[k] = similarity(row x1[k], row x2[k]) under metric (0 pcc, 1 cos, 2 euclidean)
extern "C" void host_knn_similarity(int32_t metric, const int64_t* rowptr, const int32_t* cols, const double* vals,
                                    const double* sq, const double* means, int32_t n_cols, const int32_t* x1,
                                    const int32_t* x2, int64_t n_pairs, double* out) {
  for (int64_t k = 0; k < n_pairs; ++k)
    out[k] = metric == 0   ? pair_similarity<qrec::kPearson>(rowptr, cols, vals, sq, means, n_cols, x1[k], x2[k])
             : metric == 1 ? pair_similarity<qrec::kCosine>(rowptr, cols, vals, sq, means, n_cols, x1[k], x2[k])
                           : pair_similarity<qrec::kEuclidean>(rowptr, cols, vals, sq, means, n_cols, x1[k], x2[k]);
}
