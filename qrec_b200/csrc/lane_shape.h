// How the row-parallel launchers shape their lane groups.  Host code only (no CUDA headers), so that the CPU suite can
// compile it with g++ and pin the table (tests/host_shims/lane_shape_host.cpp).
//
// A row-parallel kernel runs one lane group per row: LPR lanes (4, 8, 16 or 32) that each own VPL 16-byte slices
// (float4s) of the row.  The group is the smallest power of two >= 4 that gives every lane one slice of a row of
// nvec = d / 4 float4s, so that each lane issues one 128-bit load per row and the group's dot products reduce in
// log2(LPR) shuffles; rows wider than a warp (d > 128) give each of the 32 lanes two slices.  Launchers whose d is
// capped at 128 instantiate no two-slice kernel.
//
// The parity kernels run one warp per triple instead, E = ceil(d / 32) elements per lane, rounded up to 1, 2, 4 or 8.
#pragma once

namespace qrec {

// Lanes per row for a row of nvec float4s.  Launchers that size their grid before choosing the kernel use it.
constexpr int row_lpr(int nvec) { return nvec <= 4 ? 4 : nvec <= 8 ? 8 : nvec <= 16 ? 16 : 32; }

template <int LPR_, int VPL_>
struct RowShape {
  static constexpr int LPR = LPR_;
  static constexpr int VPL = VPL_;
  // Triples in flight per lane group in the throughput triple kernels (the BPR batch step and the BPR gradient
  // kernels): 4, but 2 where the group is small (LPR = 4: more groups per warp already) or each lane holds two slices
  // (register pressure).
  static constexpr int UNROLL = (LPR == 4 || VPL == 2) ? 2 : 4;
};

// Calls f(RowShape<LPR, VPL>{}) for a row of nvec float4s and returns its result.  MAX_D is the largest d the launcher
// accepts: the two-slice shape (32, 2) exists only above 128.
template <int MAX_D, class F>
auto with_row_shape(int nvec, F&& f) {
  static_assert(MAX_D == 128 || MAX_D == 256, "rows hold at most 256 floats");
  switch (row_lpr(nvec)) {
    case 4: return f(RowShape<4, 1>{});
    case 8: return f(RowShape<8, 1>{});
    case 16: return f(RowShape<16, 1>{});
    default: break;
  }
  if constexpr (MAX_D > 128) {
    if (nvec > 32) return f(RowShape<32, 2>{});
  }
  return f(RowShape<32, 1>{});
}

template <int E_>
struct LaneElems {
  static constexpr int E = E_;
};

// Calls f(LaneElems<E>{}) for the warp-per-triple parity kernels and returns its result: E = ceil(d / 32) rounded up
// to 1, 2, 4 or 8 (d <= 256).
template <class F>
auto with_lane_elems(int d, F&& f) {
  const int e = (d + 31) / 32;
  if (e <= 1) return f(LaneElems<1>{});
  if (e <= 2) return f(LaneElems<2>{});
  if (e <= 4) return f(LaneElems<4>{});
  return f(LaneElems<8>{});
}

}  // namespace qrec
