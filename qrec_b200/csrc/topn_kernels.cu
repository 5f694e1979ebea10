// K8: batched ranking evaluation in ONE kernel (SURVEY.md 8f-1).
//
// The reference ranks one test user at a time (base/recommender.py:143-152): candidates = Q.dot(P[u]), the
// user's rated items are overwritten with 0 (not removed: `candidates[item] = 0`), then a heap keeps the N
// best, replacing its minimum only on a strictly larger score (util/qmath.py:134-146), and the result is
// sorted by score, descending.  Here a block of 128 users is scored against the item table tile by tile
// (fp32 FMA, k ascending -- the same sums as the GEMV up to the order of the partial sums) and the scores
// never leave the SM: every score is compared in registers with its row's current N-th best, the rated test
// (binary search of the user's sorted rated row) runs only for the few that pass, survivors are appended to the
// row's candidate list (256 keys, L2-resident scratch) and a warp-level bitonic sort compacts a row back to N
// whenever its list could overflow.  Nothing of the [users x items] score matrix is written to memory.
//
// Ordering: (score descending, item id ascending), -0.0 and +0.0 one score -- a total order, so the result does
// not depend on the scan order.  It is not the reference heap's: at a tie across the cut the heap can keep later
// ids, and inside a tie it keeps heap order.  evaluate.batched_top_n asks for one key more than it needs and ranks
// the rows with equal scores again on the host, so `-eval gpu` returns the heap's lists on the device's fp32 scores.
#include "common.h"
#include "topn.cuh"

namespace {

using namespace qrec;

constexpr int CAP = 256;   // candidate slots per user (>= N_max + items per tile)
constexpr int NMAX = 101;  // base/recommender.py:131-134 clamps N to <= 100; evaluate.py asks for one key past the cut

// ---------------------------------------------------------------------------------------------------------------
// The kernel: 128 users x 128 items per tile, 8 x 8 register tile per thread, double-buffered k-chunks of 16
// (global -> registers while the previous chunk is multiplied, 4 LDS.128 per 64 FMA), 2 CTAs per SM.  The candidate
// lists (256 keys per user) live in a global workspace that stays in the L2 (a CTA only ever touches its 128 rows'
// 256 KB); the per-row count and cut-off sit in shared memory, where the hot compare happens.
// ---------------------------------------------------------------------------------------------------------------
constexpr int VM = 128, VN = 128, VK = 16;
constexpr int VAS = VM + 4, VBS = VN + 4;

__global__ void __launch_bounds__(256, 2)
score_topn_kernel(const float* __restrict__ U, const float* __restrict__ V, int d, int n_items,
                  const int* __restrict__ user_ids, int n_rows, const long long* __restrict__ rated_rowptr,
                  const int* __restrict__ rated_cols, float rated_value, int N, int* __restrict__ out_ids,
                  float* __restrict__ out_scores, unsigned long long* __restrict__ workspace) {
  __shared__ __align__(16) float tiles[2 * VK * VAS + 2 * VK * VBS];       // 33 KB: A and B chunks, two buffers each
  float (*As)[VK][VAS] = reinterpret_cast<float (*)[VK][VAS]>(tiles);
  float (*Bs)[VK][VBS] = reinterpret_cast<float (*)[VK][VBS]>(tiles + 2 * VK * VAS);
  // the sort buffers (one per warp, 16 KB) alias the tile memory: compaction and the final ordering run between
  // barriers that separate them from the multiply phase
  unsigned long long (*scratch)[CAP] = reinterpret_cast<unsigned long long (*)[CAP]>(tiles);
  __shared__ unsigned long long thr[VM];
  __shared__ int cnt[VM];
  __shared__ int uid[VM];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int row0 = blockIdx.x * VM;
  const int tx = tid & 15, ty = tid >> 4;                  // 16 x 16 threads: rows ty*8..+7, cols tx*4+{0..3} and 64+tx*4+{0..3}
  unsigned long long* cand = workspace + (size_t)blockIdx.x * VM * CAP;
  for (int r = tid; r < VM; r += 256) {
    cnt[r] = 0;
    thr[r] = 0ULL;
    uid[r] = (row0 + r < n_rows) ? user_ids[row0 + r] : -1;
  }
  __syncthreads();
  const unsigned long long rated_key_hi = (unsigned long long)ord_of(rated_value) << 32;
  // tile loaders: thread t stages row (t >> 1) of A and of B, 8 consecutive k starting at (t & 1) * 8
  const int lr = tid >> 1, lk = (tid & 1) * 8;
  const int nchunks = (d + VK - 1) / VK;

  for (int c0 = 0; c0 < n_items; c0 += VN) {
    // ---- compaction: a row that could overflow during this tile goes back to its N best
    for (int r = warp; r < VM; r += 8) {
      const int c = cnt[r];
      if (c > CAP - VN) {
        unsigned long long* k = scratch[warp];
        for (int t = lane; t < CAP; t += 32) k[t] = t < c ? __ldcg(cand + (size_t)r * CAP + t) : 0ULL;
        warp_sort_desc<CAP>(k, lane);
        for (int t = lane; t < N; t += 32) cand[(size_t)r * CAP + t] = k[t];
        if (lane == 0) { cnt[r] = N; thr[r] = k[N - 1]; }
        __syncwarp();
      }
    }
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float ra[8], rb[8];
    auto fetch = [&](int k0) {                              // global -> registers (chunk k0)
      const int u = uid[lr];
      const int item = c0 + lr;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int k = k0 + lk + q;
        ra[q] = (u >= 0 && k < d) ? __ldg(U + (size_t)u * d + k) : 0.f;
        rb[q] = (item < n_items && k < d) ? __ldg(V + (size_t)item * d + k) : 0.f;
      }
    };
    auto stage = [&](int buf) {                             // registers -> shared, transposed: [k][row]
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        As[buf][lk + q][lr] = ra[q];
        Bs[buf][lk + q][lr] = rb[q];
      }
    };
    __syncthreads();                                        // previous tile's selection is done with thr / cnt
    fetch(0);
    stage(0);
    __syncthreads();
    for (int ch = 0; ch < nchunks; ++ch) {
      const int buf = ch & 1;
      if (ch + 1 < nchunks) fetch((ch + 1) * VK);
#pragma unroll
      for (int k = 0; k < VK; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
        const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
        const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      if (ch + 1 < nchunks) {
        stage(buf ^ 1);                                     // the other buffer: nobody reads it during this chunk
        __syncthreads();
      }
    }
    // ---- selection in registers
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = ty * 8 + i;
      const int u = uid[r];
      if (u < 0) continue;
      const unsigned long long th = thr[r];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = c0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
        if (c >= n_items) continue;
        const unsigned long long low = (unsigned long long)(0xffffffffu - (uint32_t)c);
        unsigned long long key = ((unsigned long long)ord_of(acc[i][j]) << 32) | low;
        // a rated item scores `rated_value` whatever its dot product: it can pass even when the raw score does not
        if (key > th || (rated_key_hi | low) > th) {
          if (is_rated(rated_cols, __ldg(rated_rowptr + u), __ldg(rated_rowptr + u + 1), c)) key = rated_key_hi | low;
          if (key > th) {
            const int slot = atomicAdd(cnt + r, 1);
            cand[(size_t)r * CAP + slot] = key;             // slot < CAP by the compaction rule
          }
        }
      }
    }
    __syncthreads();                                        // appends (global) and counts visible to the compaction
  }
  // ---- final order and output
  for (int r = warp; r < VM; r += 8) {
    if (uid[r] < 0) continue;
    const int c = cnt[r];
    unsigned long long* k = scratch[warp];
    for (int t = lane; t < CAP; t += 32) k[t] = t < c ? __ldcg(cand + (size_t)r * CAP + t) : 0ULL;
    warp_sort_desc<CAP>(k, lane);
    for (int t = lane; t < N; t += 32) {
      const unsigned long long key = k[t];
      out_ids[(size_t)(row0 + r) * N + t] = (int)(0xffffffffu - (uint32_t)(key & 0xffffffffULL));
      out_scores[(size_t)(row0 + r) * N + t] = score_of((uint32_t)(key >> 32));
    }
    __syncwarp();
  }
}

}  // namespace

extern "C" int qrec_score_topn_f32(const float* dev_U, const float* dev_V, int32_t d, int32_t n_items,
                                   const int32_t* dev_user_ids, int32_t n_rows, const int64_t* dev_rated_rowptr,
                                   const int32_t* dev_rated_cols, float rated_value, int32_t N, int32_t* dev_out_ids,
                                   float* dev_out_scores, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && n_items >= 1 && d >= 1, "qrec_score_topn_f32: bad size");
  QREC_REQUIRE(N >= 1 && N <= NMAX && N <= n_items, "qrec_score_topn_f32: N=%d must be in 1..min(%d, n_items)", N, NMAX);
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(dev_U && dev_V && dev_user_ids && dev_rated_rowptr && dev_rated_cols && dev_out_ids && dev_out_scores,
               "qrec_score_topn_f32: null pointer");
  const int grid = (n_rows + VM - 1) / VM;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* ws = nullptr;                       // candidate lists: 2 KB per user, stream-ordered scratch
  QREC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&ws), (size_t)grid * VM * CAP * sizeof(unsigned long long), st));
  score_topn_kernel<<<grid, 256, 0, st>>>(
      dev_U, dev_V, d, n_items, dev_user_ids, n_rows, reinterpret_cast<const long long*>(dev_rated_rowptr), dev_rated_cols,
      rated_value, N, dev_out_ids, dev_out_scores, ws);
  const cudaError_t launch_err = cudaGetLastError();
  QREC_CUDA(cudaFreeAsync(ws, st));
  if (launch_err != cudaSuccess) return qrec::cuda_fail(launch_err, "kernel launch", __FILE__, __LINE__);
  qrec::count_launch();
  return QREC_OK;
}
