// Host build of qrec_b200/csrc/serec_step.cuh: the social exposure prior of every (user, item) pair listed, with the
// header's own serec_prior -- so the CPU suite pins the device source to the float64 oracle.  Compiled with
// -ffp-contract=off, as the device code keeps every product and sum separately rounded.
#include <cstdint>
#define __host__
#define __device__
#define __forceinline__ inline
#include "serec_step.cuh"

// out[u][i] = serec_prior(A[i], deg[u]) for u < n_rows, i < n_items (row-major)
extern "C" void host_serec_prior(const double* A, int64_t n_items, const int32_t* deg, int64_t n_rows, double a,
                                 double b, double s, double n_users, double* out) {
  for (int64_t u = 0; u < n_rows; ++u)
    for (int64_t i = 0; i < n_items; ++i) out[u * n_items + i] = qrec::serec_prior(A[i], deg[u], a, b, s, n_users);
}
