// Host build of qrec_b200/csrc/lane_shape.h: the lane-group shape the row-parallel launchers pick for each row width,
// so that the CPU suite can pin the table.
#include "lane_shape.h"

namespace {

template <int MAX_D>
void row_shape(int nvec, int* out) {
  qrec::with_row_shape<MAX_D>(nvec, [&](auto s) {
    using S = decltype(s);
    out[0] = S::LPR;
    out[1] = S::VPL;
    out[2] = S::UNROLL;
  });
}

}  // namespace

extern "C" {

// out[0..2] = LPR, VPL, UNROLL of the shape with_row_shape<max_d> (max_d 128 or 256) picks for nvec; -1 for other max_d
int row_shape_host(int nvec, int max_d, int* out) {
  if (max_d == 128) row_shape<128>(nvec, out);
  else if (max_d == 256) row_shape<256>(nvec, out);
  else return -1;
  return 0;
}

int row_lpr_host(int nvec) { return qrec::row_lpr(nvec); }

int lane_elems_host(int d) {
  return qrec::with_lane_elems(d, [](auto e) { return decltype(e)::E; });
}

}  // extern "C"
