// CoFactor's item co-occurrence counts (model/ranking/CoFactor.py, initModel): for every pair of eligible items
// (each with at least `filter` distinct users), i != j, the number of users they share, kept when it is > filter.
//
// Row by row like Gustavson's product C = B^T B, without forming B^T B or any per-user list of pairs (the sum of the
// squared user degrees is in the billions at benchmark scale).  One CTA builds one row i (persistent grid, rows in the
// caller's order, longest first): for every user u of item i (item-major CSR) it walks u's items (user-major CSR,
// ascending ids) that fall into the current column tile and counts them into a shared-memory strip of kTile
// counters; each user's first item in the tile is found by binary search.  The tile is then read in ascending column
// order, 256 columns at a time, with a block-wide ordered compaction.  Two passes over the same counts: the first
// writes each row's number of kept entries, the second (given the scanned row pointer) the kept columns with their
// counts.  Integer counts: the output is exact and the same on every run.
#include "common.h"

namespace {

constexpr int kThreads = 256;
constexpr int kTile = 8192;          // counters per column tile (32 KB of shared memory)

__global__ void __launch_bounds__(kThreads)
cooc_count_kernel(int n_items, const long long* __restrict__ irp, const int* __restrict__ iusers,
                  const long long* __restrict__ urp, const int* __restrict__ uitems, int n_rows,
                  const int* __restrict__ order, int filter, const long long* __restrict__ out_rowptr,
                  long long* __restrict__ row_nnz, int* __restrict__ out_cols, int* __restrict__ out_counts) {
  __shared__ int cnt[kTile];
  __shared__ int wtot[kThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int q = blockIdx.x; q < n_rows; q += gridDim.x) {
    const int i = __ldg(order + q);
    const long long ub = __ldg(irp + i), ue = __ldg(irp + i + 1);
    long long pos = out_rowptr != nullptr ? __ldg(out_rowptr + i) : 0;   // next output slot (uniform)
    long long kept = 0;
    for (int j0 = 0; j0 < n_items; j0 += kTile) {
      const int j1 = n_items - j0 < kTile ? n_items : j0 + kTile;
      __syncthreads();                                 // the previous tile's counts have been read
      for (int k = t; k < kTile; k += kThreads) cnt[k] = 0;
      __syncthreads();
      int touched = 0;
      for (long long e = ub + warp; e < ue; e += kThreads / 32) {      // one warp per user of item i
        const int u = __ldg(iusers + e);
        long long lo = __ldg(urp + u), hi = __ldg(urp + u + 1);
        const long long end = hi;
        while (lo < hi) {                              // first of u's items >= j0
          const long long mid = (lo + hi) >> 1;
          if (__ldg(uitems + mid) < j0) lo = mid + 1; else hi = mid;
        }
        for (long long p = lo + lane; p < end; p += 32) {
          const int j = __ldg(uitems + p);
          if (j >= j1) break;
          atomicAdd(&cnt[j - j0], 1);
          touched = 1;
        }
      }
      if (!__syncthreads_or(touched)) continue;
      for (int b = 0; b < j1 - j0; b += kThreads) {    // ascending columns, kThreads at a time
        const int k = b + t, j = j0 + k;
        bool keep = false;
        int n = 0;
        if (j < j1 && j != i) {
          n = cnt[k];
          keep = n > filter && __ldg(irp + j + 1) - __ldg(irp + j) >= filter;
        }
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wtot[warp] = __popc(m);
        __syncthreads();
        int before = __popc(m & ((1u << lane) - 1u)), total = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
          const int c = wtot[w];
          if (w < warp) before += c;
          total += c;
        }
        if (keep && out_cols != nullptr) {
          out_cols[pos + before] = j;
          out_counts[pos + before] = n;
        }
        pos += total;
        kept += total;
        __syncthreads();                               // wtot is rewritten by the next chunk
      }
    }
    if (t == 0 && out_rowptr == nullptr) row_nnz[i] = kept;
  }
}

}  // namespace

extern "C" {

int qrec_cooc_count(int32_t n_items, const int64_t* item_rowptr, const int32_t* item_users, const int64_t* user_rowptr,
                    const int32_t* user_items, int32_t n_rows, const int32_t* row_order, int32_t filter,
                    const int64_t* out_rowptr, int64_t* row_nnz, int32_t* out_cols, int32_t* out_counts,
                    void* stream) {
  QREC_REQUIRE(n_items >= 0 && n_rows >= 0 && n_rows <= n_items, "cooc_count: n_items=%d n_rows=%d", n_items, n_rows);
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(item_rowptr && item_users && user_rowptr && user_items && row_order, "cooc_count: null pointer");
  QREC_REQUIRE(out_rowptr != nullptr ? (out_cols && out_counts) : row_nnz != nullptr,
               "cooc_count: the count pass needs row_nnz, the fill pass out_cols and out_counts");
  const int grid = qrec::capped_grid(n_rows, 6);
  cooc_count_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(
      n_items, (const long long*)item_rowptr, item_users, (const long long*)user_rowptr, user_items, n_rows, row_order,
      filter, (const long long*)out_rowptr, (long long*)row_nnz, out_cols, out_counts);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
