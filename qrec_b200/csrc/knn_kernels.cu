// Memory-based rating models: UserKNN, ItemKNN (neighbour lists and predictions) and SlopeOne.
//
//   reference: model/rating/UserKNN.py, ItemKNN.py, SlopeOne.py and util/qmath.py.  One side's training rows ("rows":
//   users for UserKNN, items for ItemKNN and SlopeOne) are compared over the keys they share; the arithmetic of one
//   shared key is in knn_step.cuh.  All of it is float64 with every operation separately rounded and no
//   floating-point atomics, so the results are bitwise reproducible and do not depend on the grid.
//
//   * corated_scatter -- the primitive all three models use: one CTA walks its query row's entries in insertion
//     order and adds each entry's term to every row sharing that column (the other side's CSR lists them), with a
//     barrier between entries.  Every candidate meets a column at most once, so each accumulator receives its terms
//     in the query's order -- the reference's order when the query is x1.
//   * knn_neighbours_kernel<M> -- one persistent CTA per query.  The reference's candidate list for the query at
//     position p (computeSimilarities with its SymmetricMatrix) is: every earlier query (cold ones included) at list
//     position p' < p, with the similarity the EARLIER query computed (x1 = the earlier row), then every other
//     training row v at position Q + v with x1 = the query.  A cold query lists every training row at Q + v with
//     similarity 0.  Only rows that share a key with the query can be non-zero: they are scattered, and the earlier
//     queries among them are redone in their own entry order against the query staged densely by column.  The
//     stably sorted list is (similarity descending, position ascending); its first K entries are selected exactly:
//     positives by a radix select on the 96-bit key (order-preserving similarity, inverted position), then the
//     zeros in position order, then negatives by the same select.
//   * knn_predict_kernel -- one thread per test line walks its query's neighbours in order and looks the probe up by
//     bisection in the neighbour's sorted row.
//   * slopeone_predict_kernel -- one persistent CTA per test item: the item's diff / count row against every item is
//     scattered into per-CTA scratch, then every test line of the item is served from it.
//   * knn_pair_similarity_kernel -- one thread per listed pair (a, b): pcc(a, b) with a's row walked in insertion
//     order and each key looked up by bisection in b's sorted row, then (pcc + w) / 2.0 (SoReg's similarity).
//   Scratch is per CTA and O(rows + columns): no queries x rows table is ever formed.
#include "common.h"
#include "knn_step.cuh"

namespace {

using namespace qrec;

constexpr int kThreads = 256;
constexpr int kCold = -2;          // ids <= kCold: the cold earlier query at position kCold - id
constexpr int kPad = -1;


// Adds a term for every entry of row q, in insertion order, to the accumulator of every row that shares the entry's
// column: the other side's CSR lists those rows (orows[orowptr[c] ..]).  Row `skip` is left out.  term(acc, e, v, k)
// adds query entry e against row v, whose entry is the other side's k.  The first term a row receives appends it to
// list[*n_list].  Every row meets a column at most once, so no two threads share an accumulator between the barriers.
// Called by the whole CTA; ends on a barrier.
template <class Term>
__device__ void corated_scatter(const long long* __restrict__ rowptr, const int* __restrict__ cols, int q, int skip,
                                const long long* __restrict__ orowptr, const int* __restrict__ orows,
                                KnnAcc* __restrict__ acc, int* __restrict__ list, int* n_list, Term term) {
  for (long long e = rowptr[q]; e < rowptr[q + 1]; ++e) {
    const int c = cols[e];
    for (long long k = orowptr[c] + threadIdx.x; k < orowptr[c + 1]; k += kThreads) {
      const int v = orows[k];
      if (v == skip) continue;
      KnnAcc& a = acc[v];
      if (a.n == 0) list[atomicAdd(n_list, 1)] = v;
      term(a, e, v, k);
    }
    __syncthreads();
  }
  __syncthreads();
}

__device__ __forceinline__ unsigned long long ord_of(double s) {   // monotone double -> uint64, -0.0 as +0.0
  const unsigned long long u = (unsigned long long)__double_as_longlong(s + 0.0);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// The sort key of a candidate: descending keys are (similarity descending, list position ascending), and no two
// candidates share a key.
struct Key {
  unsigned long long hi;
  unsigned lo;
  __device__ bool operator>(const Key& o) const { return hi != o.hi ? hi > o.hi : lo > o.lo; }
  __device__ unsigned byte(int b) const {             // byte b, most significant first (12 bytes)
    return b < 8 ? (unsigned)(hi >> (56 - 8 * b)) & 255u : (lo >> (24 - 8 * (b - 8))) & 255u;
  }
  __device__ bool prefix_is(const Key& p, int b) const {   // the first b bytes equal p's
    if (b == 0) return true;
    if (b <= 8) return (hi >> (64 - 8 * b)) == (p.hi >> (64 - 8 * b));
    return hi == p.hi && (b == 12 || (lo >> (96 - 8 * b)) == (p.lo >> (96 - 8 * b)));
  }
};

struct Shared {
  Key thr;
  int n_list, count, npos, nneg;
  int hist[256];
  int warp_cnt[kThreads / 32];
};

__device__ __forceinline__ bool in_class(double s, int sign) { return sign > 0 ? s > 0.0 : s < 0.0; }

// The k-th largest key among the listed rows of class `sign` (1: similarity > 0, -1: < 0), 1 <= k <= their number:
// a radix select over the 12 key bytes with a shared-memory histogram (integer atomics only).
template <class KeyOf>
__device__ Key radix_select(const int* list, int n_list, const double* simd, int sign, int k, KeyOf key_of,
                            Shared& sh) {
  Key p{0ull, 0u};
  for (int b = 0; b < 12; ++b) {
    for (int d = threadIdx.x; d < 256; d += kThreads) sh.hist[d] = 0;
    __syncthreads();
    for (int j = threadIdx.x; j < n_list; j += kThreads) {
      const int v = list[j];
      if (!in_class(simd[v], sign)) continue;
      const Key kv = key_of(v);
      if (kv.prefix_is(p, b)) atomicAdd(&sh.hist[kv.byte(b)], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int d = 255;
      for (; d > 0 && k > sh.hist[d]; --d) k -= sh.hist[d];
      if (b < 8) p.hi |= (unsigned long long)d << (56 - 8 * b);
      else p.lo |= (unsigned)d << (24 - 8 * (b - 8));
      sh.thr = p;
    }
    __syncthreads();
    p = sh.thr;                                       // (k is thread 0's)
    __syncthreads();
  }
  return p;
}

// Writes the `take` largest keys of class `sign` to ids / sims [base, base + take), in descending key order.  The
// selected keys are ranked by counting, O(take^2 / kThreads) key reads per thread: cheap at the K of the models'
// configs (num.neighbors is tens), quadratic when K reaches the whole candidate list of a large set.
template <class KeyOf, class IdOf>
__device__ void emit_class(const int* list, int n_list, const double* simd, int sign, int take, int* sel,
                           KeyOf key_of, IdOf id_of, int* ids, double* sims, int base, Shared& sh) {
  if (take <= 0) return;
  const Key thr = radix_select(list, n_list, simd, sign, take, key_of, sh);
  if (threadIdx.x == 0) sh.count = 0;
  __syncthreads();
  for (int j = threadIdx.x; j < n_list; j += kThreads) {
    const int v = list[j];
    if (in_class(simd[v], sign) && !(thr > key_of(v))) sel[atomicAdd(&sh.count, 1)] = v;
  }
  __syncthreads();
  const int n = sh.count;          // == take: the keys are distinct
  for (int j = threadIdx.x; j < n; j += kThreads) {
    const int v = sel[j];
    const Key kv = key_of(v);
    int rank = 0;
    for (int m = 0; m < n; ++m) rank += key_of(sel[m]) > kv;
    ids[base + rank] = id_of(v);
    sims[base + rank] = simd[v];
  }
  __syncthreads();
}

// per-CTA scratch of knn_neighbours_kernel
__host__ __device__ inline size_t knn_scratch_stride(int n_rows, int n_cols) {
  const size_t b = sizeof(KnnAcc) * (size_t)n_rows + sizeof(double) * (size_t)n_rows +
                   sizeof(int) * (2 * (size_t)n_rows + (size_t)n_cols);
  return (b + 255) & ~(size_t)255;
}

template <int M>
__global__ void __launch_bounds__(kThreads)
knn_neighbours_kernel(const long long* __restrict__ rowptr, const int* __restrict__ cols,
                      const double* __restrict__ vals, const double* __restrict__ sq, const double* __restrict__ means,
                      const long long* __restrict__ crowptr, const int* __restrict__ crows,
                      const long long* __restrict__ cent, int n_rows, int n_cols, const int* __restrict__ queries,
                      const int* __restrict__ pos_of_row, int n_queries, int K, int* __restrict__ out_ids,
                      double* __restrict__ out_sims, int* __restrict__ out_cnt, unsigned char* __restrict__ scratch) {
  __shared__ Shared sh;
  unsigned char* mine = scratch + knn_scratch_stride(n_rows, n_cols) * blockIdx.x;
  KnnAcc* acc = (KnnAcc*)mine;                                   // [n_rows], zero between queries
  double* simd = (double*)(acc + n_rows);                        // [n_rows], 0.0 between queries
  int* list = (int*)(simd + n_rows);                             // [n_rows]
  int* sel = list + n_rows;                                      // [n_rows]
  int* stage = sel + n_rows;                                     // [n_cols], 0 between queries
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  for (int p = blockIdx.x; p < n_queries; p += gridDim.x) {
    const int q = queries[p];
    int* ids = out_ids + (size_t)p * K;
    double* sims = out_sims + (size_t)p * K;
    if (threadIdx.x == 0) { sh.n_list = 0; sh.npos = 0; sh.nneg = 0; }
    __syncthreads();
    if (q >= 0) {
      const long long q0 = rowptr[q];
      for (long long e = q0 + threadIdx.x; e < rowptr[q + 1]; e += kThreads) stage[cols[e]] = (int)(e - q0) + 1;
      const double mq = means[q];
      corated_scatter(rowptr, cols, q, q, crowptr, crows, acc, list, &sh.n_list,
                      [&](KnnAcc& a, long long e, int v, long long k) {
                        const long long f = cent[k];
                        knn_add<M>(a, vals[e], sq[e], mq, vals[f], sq[f], means[v]);
                      });
    }
    __syncthreads();
    const int n_list = sh.n_list;
    // the similarity of every row that shares a key; an earlier query's in its own entry order (x1 = that row)
    int npos = 0, nneg = 0;
    for (int j = threadIdx.x; j < n_list; j += kThreads) {
      const int v = list[j];
      const int pv = pos_of_row[v];
      double s;
      if (pv >= 0 && pv < p) {
        KnnAcc a2{0.0, 0.0, 0.0, 0};
        const long long q0 = rowptr[q] - 1;
        for (long long f = rowptr[v]; f < rowptr[v + 1]; ++f) {
          const int at = stage[cols[f]];
          if (at) knn_add<M>(a2, vals[f], sq[f], means[v], vals[q0 + at], sq[q0 + at], means[q]);
        }
        s = knn_similarity<M>(a2);
      } else {
        s = knn_similarity<M>(acc[v]);
      }
      simd[v] = s;
      acc[v] = KnnAcc{0.0, 0.0, 0.0, 0};
      npos += s > 0.0;
      nneg += s < 0.0;
    }
    atomicAdd(&sh.npos, npos);
    atomicAdd(&sh.nneg, nneg);
    __syncthreads();
    int filled = 0;
    if (K > 0) {
      const int n_pos = sh.npos, n_neg = sh.nneg;
      const auto key_of = [&](int v) {
        const int pv = pos_of_row[v];
        const unsigned pos = pv >= 0 && pv < p ? (unsigned)pv : (unsigned)n_queries + (unsigned)v;
        return Key{ord_of(simd[v]), 0xffffffffu - pos};
      };
      const auto id_of = [](int v) { return v; };
      const int take_pos = n_pos < K ? n_pos : K;
      emit_class(list, n_list, simd, 1, take_pos, sel, key_of, id_of, ids, sims, 0, sh);
      filled = take_pos;
      // the zeros in list position order: the earlier queries (for a training query), then the training rows
      const int off = q >= 0 ? p : 0;
      const long long n_virtual = (long long)off + n_rows;
      for (long long c0 = 0; c0 < n_virtual && filled < K; c0 += kThreads) {
        const long long idx = c0 + threadIdx.x;
        bool zero = false;
        int id = kPad;
        if (idx < off) {
          const int v = queries[idx];
          zero = v < 0 || simd[v] == 0.0;
          id = v >= 0 ? v : kCold - (int)idx;
        } else if (idx < n_virtual) {
          const int v = (int)(idx - off);
          const int pv = pos_of_row[v];
          zero = v != q && !(q >= 0 && pv >= 0 && pv < p) && simd[v] == 0.0;
          id = v;
        }
        const unsigned ballot = __ballot_sync(0xffffffffu, zero);
        if (lane == 0) sh.warp_cnt[warp] = __popc(ballot);
        __syncthreads();
        int before = filled, total = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
          if (w < warp) before += sh.warp_cnt[w];
          total += sh.warp_cnt[w];
        }
        const int at = before + __popc(ballot & ((1u << lane) - 1u));
        if (zero && at < K) {
          ids[at] = id;
          sims[at] = 0.0;
        }
        filled = filled + total < K ? filled + total : K;
        __syncthreads();
      }
      const int take_neg = K - filled < n_neg ? K - filled : n_neg;
      emit_class(list, n_list, simd, -1, take_neg, sel, key_of, id_of, ids, sims, filled, sh);
      filled += take_neg;
      for (int j = filled + threadIdx.x; j < K; j += kThreads) {
        ids[j] = kPad;
        sims[j] = 0.0;
      }
    }
    if (threadIdx.x == 0) out_cnt[p] = filled;
    // leave the scratch as it was found
    for (int j = threadIdx.x; j < n_list; j += kThreads) simd[list[j]] = 0.0;
    if (q >= 0)
      for (long long e = rowptr[q] + threadIdx.x; e < rowptr[q + 1]; e += kThreads) stage[cols[e]] = 0;
    __syncthreads();
  }
}

// One thread per test line: the line's query is at list position qpos[l] (row queries[qpos[l]], -1 when cold) and
// its probe is the other side's id (-1 when cold), looked up by bisection in each neighbour's row of the sorted view
// (scols / svals: every row's columns ascending, with their values).  minus_one_unrated: a stored -1 counts as
// unrated (UserKNN's `rating(n, i) != -1`; ItemKNN asks `contains`).  status: 0 prediction, 1 mean fallback
// (sum == 0), 2 the reference's ZeroDivisionError (denominator 0 with sum != 0; pred is then 0).
__global__ void __launch_bounds__(kThreads)
knn_predict_kernel(const long long* __restrict__ rowptr, const int* __restrict__ scols, const double* __restrict__ svals,
                   const double* __restrict__ means, double global_mean, const int* __restrict__ queries, int K,
                   const int* __restrict__ nbr, const double* __restrict__ nsim, const int* __restrict__ ncnt,
                   long long n_lines, const int* __restrict__ qpos, const int* __restrict__ probe, int minus_one_unrated,
                   double* __restrict__ pred, int* __restrict__ status) {
  for (long long l = blockIdx.x * (long long)kThreads + threadIdx.x; l < n_lines; l += (long long)gridDim.x * kThreads) {
    const int p = qpos[l], x = probe[l], q = queries[p];
    double sum = 0.0, denom = 0.0;
    const int n = x < 0 ? 0 : ncnt[p];
    for (int k = 0; k < n; ++k) {
      const int v = nbr[(size_t)p * K + k];
      if (v < 0) continue;                        // a cold earlier query has no ratings
      long long lo = rowptr[v], hi = rowptr[v + 1];
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (scols[mid] < x) lo = mid + 1; else hi = mid;
      }
      if (lo == rowptr[v + 1] || scols[lo] != x) continue;
      const double r = svals[lo];
      if (minus_one_unrated && r == -1.0) continue;
      knn_vote(sum, denom, nsim[(size_t)p * K + k], r, means[v]);
    }
    const double base = q >= 0 ? means[q] : global_mean;
    if (sum == 0.0) {
      pred[l] = base;
      status[l] = 1;
    } else if (denom == 0.0) {
      pred[l] = 0.0;
      status[l] = 2;
    } else {
      pred[l] = __dadd_rn(base, __ddiv_rn(sum, denom));
      status[l] = 0;
    }
  }
}

// One thread per pair p: out[p] = (pcc(a[p], b[p]) + w[p]) / 2.0 (SoReg.py:35-36, util/qmath.py: pearson_sp).  Row a
// is walked in insertion order (cols / vals / sq); each of its keys is looked up by bisection in row b of the sorted
// view (scols / svals / ssq: the same rows with their columns ascending, values and squares in the same permutation).
__global__ void __launch_bounds__(kThreads)
knn_pair_similarity_kernel(const long long* __restrict__ rowptr, const int* __restrict__ cols,
                           const double* __restrict__ vals, const double* __restrict__ sq,
                           const double* __restrict__ means, const int* __restrict__ scols,
                           const double* __restrict__ svals, const double* __restrict__ ssq, long long n_pairs,
                           const int* __restrict__ pa, const int* __restrict__ pb, const double* __restrict__ w,
                           double* __restrict__ out) {
  for (long long p = blockIdx.x * (long long)kThreads + threadIdx.x; p < n_pairs;
       p += (long long)gridDim.x * kThreads) {
    const int a = pa[p], b = pb[p];
    const double ma = means[a], mb = means[b];
    const long long bb = rowptr[b], be = rowptr[b + 1];
    KnnAcc acc{0.0, 0.0, 0.0, 0};
    for (long long e = rowptr[a]; e < rowptr[a + 1]; ++e) {
      const int x = cols[e];
      long long lo = bb, hi = be;
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (scols[mid] < x) lo = mid + 1; else hi = mid;
      }
      if (lo == be || scols[lo] != x) continue;
      knn_add<kPearson>(acc, vals[e], sq[e], ma, svals[lo], ssq[lo], mb);
    }
    out[p] = __ddiv_rn(__dadd_rn(knn_similarity<kPearson>(acc), w[p]), 2.0);
  }
}

__host__ __device__ inline size_t slopeone_scratch_stride(int n_items) {
  return (sizeof(KnnAcc) * (size_t)n_items + sizeof(int) * (size_t)n_items + 255) & ~(size_t)255;
}

// One persistent CTA per test item p (row items[p] of the item CSR, -1 when cold).  Its diff / count row against every
// item (the item itself included) is scattered from its users in insertion order through the user CSR, then its test
// lines line_rowptr[p] .. [p+1] (user line_user[k], -1 when cold) are served from it into pred[line_out[k]].  A warm
// user walks their rated items in insertion order; status 1 marks the mean fallbacks (no shared user, or a cold user).
__global__ void __launch_bounds__(kThreads)
slopeone_predict_kernel(const long long* __restrict__ irowptr, const int* __restrict__ icols,
                        const double* __restrict__ ivals, const double* __restrict__ item_means,
                        const long long* __restrict__ urowptr, const int* __restrict__ ucols,
                        const double* __restrict__ uvals, const double* __restrict__ user_means, double global_mean,
                        int n_items, const int* __restrict__ items, int n_queries,
                        const long long* __restrict__ line_rowptr, const int* __restrict__ line_user,
                        const long long* __restrict__ line_out, double* __restrict__ pred, int* __restrict__ status,
                        unsigned char* __restrict__ scratch) {
  __shared__ int n_list;
  unsigned char* mine = scratch + slopeone_scratch_stride(n_items) * blockIdx.x;
  KnnAcc* acc = (KnnAcc*)mine;                                   // [n_items], zero between test items
  int* list = (int*)(acc + n_items);                             // [n_items]
  for (int p = blockIdx.x; p < n_queries; p += gridDim.x) {
    const int i = items[p];
    if (threadIdx.x == 0) n_list = 0;
    __syncthreads();
    if (i >= 0)
      corated_scatter(irowptr, icols, i, -1, urowptr, ucols, acc, list, &n_list,
                      [&](KnnAcc& a, long long e, int, long long k) { slopeone_add(a, ivals[e], uvals[k]); });
    for (long long l = line_rowptr[p] + threadIdx.x; l < line_rowptr[p + 1]; l += kThreads) {
      const int u = line_user[l];
      double out;
      int st = 0;
      if (u >= 0) {
        double sum = 0.0;
        long long freq = 0;
        for (long long k = urowptr[u]; k < urowptr[u + 1]; ++k) {
          const KnnAcc& a = acc[ucols[k]];
          sum = slopeone_vote(sum, uvals[k], a);
          freq += a.n;
        }
        if (freq == 0) {
          out = user_means[u];
          st = 1;
        } else {
          out = __ddiv_rn(sum, (double)freq);
        }
      } else {
        out = i >= 0 ? item_means[i] : global_mean;
        st = 1;
      }
      pred[line_out[l]] = out;
      status[line_out[l]] = st;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < n_list; j += kThreads) acc[list[j]] = KnnAcc{0.0, 0.0, 0.0, 0};
    __syncthreads();
  }
}

int grid_of(long long work, int max_ctas) {
  int grid = capped_grid(work, 2);
  if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
  return grid;
}

int launch_neighbours(int metric, const long long* rowptr, const int* cols, const double* vals, const double* sq,
                      const double* means, int n_rows, int n_cols, const long long* crowptr, const int* crows,
                      const long long* cent, const int* queries, const int* pos_of_row, int n_queries, int K,
                      int* out_ids, double* out_sims, int* out_cnt, int max_ctas, cudaStream_t st) {
  QREC_REQUIRE(metric >= kPearson && metric <= kEuclidean, "knn_neighbours: metric=%d (0 pcc, 1 cos, 2 euclidean)",
               metric);
  QREC_REQUIRE(n_rows >= 0 && n_cols >= 0 && n_queries >= 0 && K >= 0,
               "knn_neighbours: n_rows=%d n_cols=%d n_queries=%d K=%d", n_rows, n_cols, n_queries, K);
  QREC_REQUIRE((long long)n_queries + n_rows < 0x7fffffffLL, "knn_neighbours: too many queries and rows");
  QREC_REQUIRE(max_ctas >= 0, "knn_neighbours: max_ctas=%d < 0", max_ctas);
  if (n_queries == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && crowptr && queries && pos_of_row && out_cnt && (K == 0 || (out_ids && out_sims)),
               "knn_neighbours: null pointer");
  const int grid = grid_of(n_queries, max_ctas);
  const size_t stride = knn_scratch_stride(n_rows, n_cols);
  unsigned char* scratch = nullptr;
  QREC_CUDA(cudaMallocAsync((void**)&scratch, stride * grid, st));
  QREC_CUDA(cudaMemsetAsync(scratch, 0, stride * grid, st));
  const auto kernel = metric == kPearson ? knn_neighbours_kernel<kPearson>
                      : metric == kCosine ? knn_neighbours_kernel<kCosine>
                                          : knn_neighbours_kernel<kEuclidean>;
  kernel<<<grid, kThreads, 0, st>>>(rowptr, cols, vals, sq, means, crowptr, crows, cent, n_rows, n_cols, queries,
                                    pos_of_row, n_queries, K, out_ids, out_sims, out_cnt, scratch);
  const cudaError_t e = cudaGetLastError();
  QREC_CUDA(cudaFreeAsync(scratch, st));
  QREC_CUDA(e);
  count_launch();
  return QREC_OK;
}

}  // namespace

extern "C" {

int qrec_knn_neighbours_f64(int32_t metric, const int64_t* rowptr, const int32_t* cols, const double* vals,
                            const double* sq, const double* means, int32_t n_rows, int32_t n_cols,
                            const int64_t* col_rowptr, const int32_t* col_rows, const int64_t* col_entries,
                            const int32_t* queries, const int32_t* pos_of_row, int32_t n_queries, int32_t K,
                            int32_t* out_ids, double* out_sims, int32_t* out_cnt, int32_t max_ctas, void* stream) {
  return launch_neighbours(metric, (const long long*)rowptr, cols, vals, sq, means, n_rows, n_cols,
                           (const long long*)col_rowptr, col_rows, (const long long*)col_entries, queries, pos_of_row,
                           n_queries, K, out_ids, out_sims, out_cnt, max_ctas, (cudaStream_t)stream);
}

int qrec_knn_predict_f64(const int64_t* rowptr, const int32_t* sorted_cols, const double* sorted_vals,
                         const double* means, double global_mean, const int32_t* queries, int32_t K,
                         const int32_t* nbr_ids, const double* nbr_sims, const int32_t* nbr_cnt, int64_t n_lines,
                         const int32_t* line_qpos, const int32_t* line_probe, int32_t minus_one_unrated, double* pred,
                         int32_t* status, void* stream) {
  QREC_REQUIRE(n_lines >= 0 && K >= 0, "knn_predict: n_lines=%lld K=%d", (long long)n_lines, K);
  if (n_lines == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && means && queries && nbr_cnt && line_qpos && line_probe && pred && status &&
                   (K == 0 || (nbr_ids && nbr_sims)),
               "knn_predict: null pointer");
  knn_predict_kernel<<<capped_grid((n_lines + kThreads - 1) / kThreads, 8), kThreads, 0, (cudaStream_t)stream>>>(
      (const long long*)rowptr, sorted_cols, sorted_vals, means, global_mean, queries, K, nbr_ids, nbr_sims, nbr_cnt,
      n_lines, line_qpos, line_probe, minus_one_unrated, pred, status);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_knn_pair_similarity_f64(const int64_t* rowptr, const int32_t* cols, const double* vals, const double* sq,
                                  const double* means, const int32_t* sorted_cols, const double* sorted_vals,
                                  const double* sorted_sq, int64_t n_pairs, const int32_t* a, const int32_t* b,
                                  const double* w, double* out, void* stream) {
  QREC_REQUIRE(n_pairs >= 0, "knn_pair_similarity: n_pairs=%lld < 0", (long long)n_pairs);
  if (n_pairs == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && means && a && b && w && out, "knn_pair_similarity: null pointer");
  knn_pair_similarity_kernel<<<capped_grid((n_pairs + kThreads - 1) / kThreads, 8), kThreads, 0,
                               (cudaStream_t)stream>>>((const long long*)rowptr, cols, vals, sq, means, sorted_cols,
                                                       sorted_vals, sorted_sq, n_pairs, a, b, w, out);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_slopeone_predict_f64(const int64_t* item_rowptr, const int32_t* item_users, const double* item_vals,
                              const double* item_means, const int64_t* user_rowptr, const int32_t* user_items,
                              const double* user_vals, const double* user_means, double global_mean, int32_t n_items,
                              const int32_t* test_items, int32_t n_test_items, const int64_t* line_rowptr,
                              const int32_t* line_user, const int64_t* line_out, double* pred, int32_t* status,
                              int32_t max_ctas, void* stream) {
  QREC_REQUIRE(n_items >= 0 && n_test_items >= 0, "slopeone_predict: n_items=%d n_test_items=%d", n_items,
               n_test_items);
  QREC_REQUIRE(max_ctas >= 0, "slopeone_predict: max_ctas=%d < 0", max_ctas);
  if (n_test_items == 0) return QREC_OK;
  QREC_REQUIRE(item_rowptr && user_rowptr && test_items && line_rowptr && pred && status,
               "slopeone_predict: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_of(n_test_items, max_ctas);
  const size_t stride = slopeone_scratch_stride(n_items);
  unsigned char* scratch = nullptr;
  QREC_CUDA(cudaMallocAsync((void**)&scratch, stride * grid, st));
  QREC_CUDA(cudaMemsetAsync(scratch, 0, stride * grid, st));
  slopeone_predict_kernel<<<grid, kThreads, 0, st>>>((const long long*)item_rowptr, item_users, item_vals, item_means,
                                                     (const long long*)user_rowptr, user_items, user_vals, user_means,
                                                     global_mean, n_items, test_items, n_test_items,
                                                     (const long long*)line_rowptr, line_user,
                                                     (const long long*)line_out, pred, status, scratch);
  const cudaError_t e = cudaGetLastError();
  QREC_CUDA(cudaFreeAsync(scratch, st));
  QREC_CUDA(e);
  count_launch();
  return QREC_OK;
}

}  // extern "C"
