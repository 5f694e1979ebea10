// f-2: the normalised joint adjacency and its per-epoch edge-dropout rebuild as kernels.
//
// Reference: base/graphRecommender.py:10-29 (create_joint_sparse_adjaceny: A = R (+) R^T with duplicate lines
// summed, D^-1/2 A D^-1/2 in float32) and model/ranking/SGL.py:113-155 (_create_adj_mat with aug_type 1: a random
// subset of the interaction LINES is kept, the sub-graph is re-normalised with ITS OWN degrees and rebuilt on the
// host every epoch, twice).  On the device the structure of the full graph (CSR, sorted columns) is built once;
// what changes per epoch is which undirected edges survive, and dropping entries from a sorted CSR keeps it a
// sorted CSR, so a rebuild is: mask -> per-row kept counts and degrees -> exclusive scan -> ordered compaction with
// the new D^-1/2 scaling.  No sort, no host round trip.
//
//   pair id   every undirected edge (u,i) appears twice in the joint CSR (row u, row U+i); `pair` maps each stored
//             entry to its edge id so that both copies see the same keep flag and the same multiplicity.
//   weight    multiplicity of the edge = number of KEPT interaction lines that map to it (the reference's
//             csr_matrix constructor sums duplicates); an edge whose weight is 0 is dropped.
#include "common.h"
#include "philox.cuh"

namespace {

__device__ __forceinline__ float inv_sqrt_deg(float deg) {   // np.power(rowsum, -0.5) with inf -> 0
  return deg > 0.f ? (float)(1.0 / sqrt((double)deg)) : 0.f;
}

// one warp per row: deg[r] = sum of the row's weights, cnt[r] = number of entries with weight > 0
__global__ void __launch_bounds__(256)
adj_row_stats_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ pair,
                     const float* __restrict__ pair_w, float* __restrict__ deg, long long* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += nwarps) {
    const long long lo = __ldg(rowptr + r), hi = __ldg(rowptr + r + 1);
    float s = 0.f;
    int c = 0;
    for (long long e = lo + lane; e < hi; e += 32) {
      const float w = pair_w ? __ldg(pair_w + __ldg(pair + e)) : 1.f;
      s += w;
      c += w > 0.f;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
    if (lane == 0) { deg[r] = s; if (cnt) cnt[r + 1] = c; }
  }
}

// vals[e] = (d_r^-1/2 * w) * d_c^-1/2 in float32, the reference's operand order (scale.dot(adj).dot(scale))
__global__ void __launch_bounds__(256)
adj_normalize_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                     const int* __restrict__ pair, const float* __restrict__ pair_w, const float* __restrict__ deg,
                     float* __restrict__ vals) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += nwarps) {
    const long long lo = __ldg(rowptr + r), hi = __ldg(rowptr + r + 1);
    const float dr = inv_sqrt_deg(__ldg(deg + r));
    for (long long e = lo + lane; e < hi; e += 32) {
      const float w = pair_w ? __ldg(pair_w + __ldg(pair + e)) : 1.f;
      vals[e] = __fmul_rn(__fmul_rn(dr, w), inv_sqrt_deg(__ldg(deg + __ldg(cols + e))));
    }
  }
}

// ordered compaction of the surviving entries of every row into the new CSR, scaled with the sub-graph's degrees
__global__ void __launch_bounds__(256)
adj_compact_kernel(int n_rows, const long long* __restrict__ rowptr, const int* __restrict__ cols,
                   const int* __restrict__ pair, const float* __restrict__ pair_w, const float* __restrict__ deg,
                   const long long* __restrict__ new_rowptr, int* __restrict__ new_cols, float* __restrict__ new_vals) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < n_rows; r += nwarps) {
    const long long lo = __ldg(rowptr + r), hi = __ldg(rowptr + r + 1);
    long long out = __ldg(new_rowptr + r);
    const float dr = inv_sqrt_deg(__ldg(deg + r));
    for (long long base = lo; base < hi; base += 32) {
      const long long e = base + lane;
      float w = 0.f;
      int c = 0;
      if (e < hi) { w = __ldg(pair_w + __ldg(pair + e)); c = __ldg(cols + e); }
      const unsigned m = __ballot_sync(0xffffffffu, w > 0.f);
      if (w > 0.f) {
        const long long pos = out + __popc(m & ((1u << lane) - 1u));
        new_cols[pos] = c;
        new_vals[pos] = __fmul_rn(__fmul_rn(dr, w), inv_sqrt_deg(__ldg(deg + c)));
      }
      out += __popc(m);
    }
  }
}

// pair_w[p] += 1 for every kept interaction line (duplicate lines of one edge add up, like scipy's constructor)
__global__ void __launch_bounds__(256)
line_weights_kernel(long long n_lines, const int* __restrict__ line_pair, const unsigned char* __restrict__ keep,
                    float* __restrict__ pair_w) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n_lines; k += stride)
    if (keep == nullptr || keep[k]) atomicAdd(pair_w + __ldg(line_pair + k), 1.f);
}

// Bernoulli(1 - drop) keep flag per interaction line, Philox counter (line, tag, epoch)
__global__ void __launch_bounds__(256)
edge_keep_kernel(long long n_lines, float drop, uint32_t k0, uint32_t k1, uint32_t tag, uint32_t epoch,
                 unsigned char* __restrict__ keep) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n_lines; k += stride) {
    uint32_t w[4];
    qrec::philox4x32_10((uint32_t)k, (uint32_t)((unsigned long long)k >> 32), tag, epoch, k0, k1, w);
    keep[k] = ((float)(w[0] >> 8) * (1.0f / 16777216.0f)) >= drop;
  }
}

// exclusive scan of cnt[1..n] in place (cnt[0] = 0 on entry): three small kernels, 1024 elements per block
constexpr int SCAN_BLOCK = 1024;
__global__ void __launch_bounds__(SCAN_BLOCK)
scan_blocks_kernel(long long* __restrict__ x, long long n, long long* __restrict__ block_sums) {
  __shared__ long long sh[SCAN_BLOCK];
  const long long k = (long long)blockIdx.x * SCAN_BLOCK + threadIdx.x;
  sh[threadIdx.x] = k < n ? x[k] : 0;
  __syncthreads();
  for (int o = 1; o < SCAN_BLOCK; o <<= 1) {
    const long long v = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
    __syncthreads();
    sh[threadIdx.x] += v;
    __syncthreads();
  }
  if (k < n) x[k] = sh[threadIdx.x];
  if (threadIdx.x == SCAN_BLOCK - 1) block_sums[blockIdx.x] = sh[threadIdx.x];
}
__global__ void __launch_bounds__(SCAN_BLOCK)
scan_sums_kernel(long long* __restrict__ block_sums, int n_blocks) {     // one block, serial over chunks
  __shared__ long long sh[SCAN_BLOCK];
  __shared__ long long carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_blocks; base += SCAN_BLOCK) {
    const int k = base + threadIdx.x;
    sh[threadIdx.x] = k < n_blocks ? block_sums[k] : 0;
    __syncthreads();
    for (int o = 1; o < SCAN_BLOCK; o <<= 1) {
      const long long v = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += v;
      __syncthreads();
    }
    if (k < n_blocks) block_sums[k] = sh[threadIdx.x] + carry;
    __syncthreads();
    if (threadIdx.x == 0) carry += sh[SCAN_BLOCK - 1];
    __syncthreads();
  }
}
__global__ void __launch_bounds__(SCAN_BLOCK)
scan_add_kernel(long long* __restrict__ x, long long n, const long long* __restrict__ block_sums) {
  const long long k = (long long)blockIdx.x * SCAN_BLOCK + threadIdx.x;
  if (blockIdx.x > 0 && k < n) x[k] += block_sums[blockIdx.x - 1];
}

int grid_rows(long long n_rows) { return qrec::capped_grid((n_rows + 7) / 8, 8); }

}  // namespace

extern "C" {

int qrec_adj_normalize_f32(int32_t n_rows, const int64_t* rowptr, const int32_t* cols, const int32_t* pair,
                           const float* pair_w, float* deg, float* vals, void* stream) {
  QREC_REQUIRE(n_rows >= 0, "qrec_adj_normalize_f32: n_rows < 0");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && cols && deg && vals, "qrec_adj_normalize_f32: null pointer");
  QREC_REQUIRE((pair == nullptr) == (pair_w == nullptr), "qrec_adj_normalize_f32: pair and pair_w come together");
  cudaStream_t st = (cudaStream_t)stream;
  adj_row_stats_kernel<<<grid_rows(n_rows), 256, 0, st>>>(n_rows, reinterpret_cast<const long long*>(rowptr), pair, pair_w, deg, nullptr);
  QREC_LAUNCH_CHECK();
  adj_normalize_kernel<<<grid_rows(n_rows), 256, 0, st>>>(n_rows, reinterpret_cast<const long long*>(rowptr), cols, pair, pair_w, deg, vals);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_edge_keep_philox(int64_t n_lines, float drop_rate, uint64_t seed, uint32_t tag, uint32_t epoch, uint8_t* keep,
                          void* stream) {
  QREC_REQUIRE(n_lines >= 0 && drop_rate >= 0.f && drop_rate <= 1.f, "qrec_edge_keep_philox: bad argument");
  if (n_lines == 0) return QREC_OK;
  QREC_REQUIRE(keep != nullptr, "qrec_edge_keep_philox: null pointer");
  edge_keep_kernel<<<grid_rows((n_lines + 31) / 32), 256, 0, (cudaStream_t)stream>>>(n_lines, drop_rate, (uint32_t)seed,
                                                                                   (uint32_t)(seed >> 32), tag, epoch, keep);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_adj_line_weights_f32(int64_t n_lines, const int32_t* line_pair, const uint8_t* keep, int64_t n_pairs, float* pair_w,
                              void* stream) {
  QREC_REQUIRE(n_lines >= 0 && n_pairs >= 0, "qrec_adj_line_weights_f32: negative size");
  if (n_pairs == 0) return QREC_OK;
  QREC_REQUIRE(pair_w && (line_pair || n_lines == 0), "qrec_adj_line_weights_f32: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  QREC_CUDA(cudaMemsetAsync(pair_w, 0, (size_t)n_pairs * sizeof(float), st));
  if (n_lines == 0) return QREC_OK;
  line_weights_kernel<<<grid_rows((n_lines + 31) / 32), 256, 0, st>>>(n_lines, line_pair, keep, pair_w);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_adj_subgraph_count(int32_t n_rows, const int64_t* rowptr, const int32_t* pair, const float* pair_w, float* deg,
                            int64_t* new_rowptr, int64_t* scan_scratch, void* stream) {
  QREC_REQUIRE(n_rows >= 0, "qrec_adj_subgraph_count: n_rows < 0");
  QREC_REQUIRE(rowptr && pair && pair_w && deg && new_rowptr && scan_scratch, "qrec_adj_subgraph_count: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  QREC_CUDA(cudaMemsetAsync(new_rowptr, 0, sizeof(int64_t), st));
  if (n_rows == 0) return QREC_OK;
  long long* nr = reinterpret_cast<long long*>(new_rowptr);
  long long* sc = reinterpret_cast<long long*>(scan_scratch);
  adj_row_stats_kernel<<<grid_rows(n_rows), 256, 0, st>>>(n_rows, reinterpret_cast<const long long*>(rowptr), pair, pair_w, deg, nr);
  QREC_LAUNCH_CHECK();
  const long long n = (long long)n_rows + 1;
  const int blocks = (int)((n + SCAN_BLOCK - 1) / SCAN_BLOCK);
  scan_blocks_kernel<<<blocks, SCAN_BLOCK, 0, st>>>(nr, n, sc);        // inclusive scan of [0, c_0, c_1, ...] = rowptr
  QREC_LAUNCH_CHECK();
  if (blocks > 1) {
    scan_sums_kernel<<<1, SCAN_BLOCK, 0, st>>>(sc, blocks);
    QREC_LAUNCH_CHECK();
    scan_add_kernel<<<blocks, SCAN_BLOCK, 0, st>>>(nr, n, sc);
    QREC_LAUNCH_CHECK();
  }
  return QREC_OK;
}

int qrec_adj_subgraph_fill_f32(int32_t n_rows, const int64_t* rowptr, const int32_t* cols, const int32_t* pair,
                               const float* pair_w, const float* deg, const int64_t* new_rowptr, int32_t* new_cols,
                               float* new_vals, void* stream) {
  QREC_REQUIRE(n_rows >= 0, "qrec_adj_subgraph_fill_f32: n_rows < 0");
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(rowptr && cols && pair && pair_w && deg && new_rowptr && new_cols && new_vals, "qrec_adj_subgraph_fill_f32: null pointer");
  adj_compact_kernel<<<grid_rows(n_rows), 256, 0, (cudaStream_t)stream>>>(
      n_rows, reinterpret_cast<const long long*>(rowptr), cols, pair, pair_w, deg, reinterpret_cast<const long long*>(new_rowptr),
      new_cols, new_vals);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
