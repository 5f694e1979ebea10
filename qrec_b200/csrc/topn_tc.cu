// K8 on the tensor cores (SURVEY.md 8f-1: "tiled P_tile . Q^T on tensor cores -> rated positions := 0 -> per-row
// top-N").  Same contract and same selection rule as csrc/topn_kernels.cu (the reference flow of
// base/recommender.py:143-152 + util/qmath.py:134-146); what changes is where the scores come from:
//
//   * a CTA owns 128 users.  Their rows of U are split once into two TF32 operands, hi = to_tf32(x) and
//     lo = to_tf32(x - hi) (csrc/wgmma.cuh), stored K-major / SWIZZLE_128B in shared memory (the layout of csrc/tc_gemm.cu);
//   * the item table is split the same way ONCE per call by a small pre-pass (split_items_kernel) that writes each
//     128-item tile as one contiguous block already in the shared-memory layout; the main kernel streams those blocks
//     through a 2-stage ring with cp.async.bulk (one 64 KB bulk copy per tile, completion on an mbarrier) -- no
//     thread touches the item operands;
//   * two warpgroups each multiply 64 of the users against the tile with wgmma.mma_async m64n128k8 TF32
//     (csrc/wgmma.cuh) three times per k-step -- hi.hi + lo.hi + hi.lo, the classical 3xTF32 error-compensated
//     product: the dropped lo.lo term is 2^-22 relative, i.e. fp32-level scores, which is what keeps the index lists
//     equal to an fp32 GEMV's wherever scores are distinct (plain TF32's 10-bit mantissa reorders close scores) --
//     into 64 accumulator registers per thread, and park the 64 x 128 scores in the warpgroup's own shared-memory tile;
//   * every thread then owns one user row and one half of the tile (warps 4g + h and 4g + h + 2 of warpgroup g cover
//     rows 32 (2g + h) ..; one takes columns 0-63 of the tile, the other 64-127), each with its OWN candidate list and
//     cut-off (the N best overall are among the N best of the two halves; the lists are merged at the end) -- and runs
//     the selection of topn_kernels.cu with the count and cut-off in
//     REGISTERS: 16 scores are compared without a branch; the few that beat the cut-off look up the row's 512-bit
//     rated-set signature (built in shared memory when the kernel starts), run the exact rated test (bisection) only
//     on a signature hit, and are appended to the row's 512-key list (L2-resident scratch).  Whenever a list could
//     overflow, its warp finds the list's N-th largest key by a bit-wise search (16 keys per lane in registers, one
//     warp reduction per bit -- no sort) and keeps the N keys at or above it; rows are sorted once, at the end.
//     The operand stage is handed back to the copy engine as soon as both warpgroups' MMAs have retired, so the next
//     tile streams in during the selection.
// Nothing of the [users x items] matrix is written.  d <= 64, a multiple of 4 (one or two 128-byte k-blocks, zero-padded).
#include "common.h"
#include "device.cuh"
#include "topn.cuh"
#include "wgmma.cuh"

namespace {

using namespace qrec;
using wg::sw_off;
using wg::to_tf32;

constexpr int CAP = 320;   // candidate slots per half-row list (>= N_max + TRIG_EXTRA + the 64 items a tile can add)
constexpr int TRIG_EXTRA = 96;   // a list is cut back to its N best once it holds more than N + TRIG_EXTRA keys
constexpr int SORTN = 256; // keys of the final per-row sort (two lists of at most N_max keys)
constexpr int NT = 256;    // multiplying and selecting threads per CTA: two warpgroups (a 9th warp drives the bulk copies)
constexpr int SIGW = 16;   // 32-bit words of a row's rated-set signature (512 bits) kept in shared memory
constexpr int NMAX = 101;  // base/recommender.py:131-134 clamps N to <= 100; evaluate.py asks for one key past the cut
constexpr int TM = 128, TN = 128;
constexpr int KBLK = TM * 128;                       // bytes of one k-block (32 fp32 = 128 B per row) of a 128-row operand
constexpr int SP = TN + 4;                           // row pitch (floats) of a warpgroup's score tile: conflict-free row reads

// bulk copy global -> shared (TMA engine), completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void group_sync(int group) {     // the 128 threads of one warpgroup
  asm volatile("bar.sync %0, 128;" ::"r"(1 + group) : "memory");
}
// x = hi + lo with hi, lo representable in TF32 (up to 2^-22 |x|)
__device__ __forceinline__ void split_tf32(const float4 v, float4& hi, float4& lo) {
  hi = to_tf32(v);
  lo = to_tf32(make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w));
}

// Pre-pass: tile t of the item table (items [128 t, 128 t + 128), zero rows past the end, zero columns past d) as one
// block of 2 * KB * 16 KB in the workspace: hi operand, then lo operand, each K-major SWIZZLE_128B -- byte for byte what
// the main kernel wants in shared memory.
template <int KB>
__global__ void __launch_bounds__(128)
split_items_kernel(const float* __restrict__ V, int d, int n_items, uint8_t* __restrict__ blocks) {
  constexpr int D = KB * 32;
  constexpr int OPER = KB * KBLK;
  constexpr int VPT = TN * D / 4 / 128;
  const int c0 = blockIdx.x * TN;
  uint8_t* const out = blocks + (size_t)blockIdx.x * 2 * OPER;
#pragma unroll
  for (int p = 0; p < VPT; ++p) {
    const int q = threadIdx.x + 128 * p;
    const int row = q / (D / 4), c4 = (q % (D / 4)) * 4;
    const float4 v = (c0 + row < n_items && c4 < d) ? __ldg(reinterpret_cast<const float4*>(V + (size_t)(c0 + row) * d + c4))
                                                    : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 hi, lo;
    split_tf32(v, hi, lo);
    const uint32_t off = (uint32_t)(c4 >> 5) * KBLK + sw_off(row, c4 & 31);
    *reinterpret_cast<float4*>(out + off) = hi;
    *reinterpret_cast<float4*>(out + OPER + off) = lo;
  }
}

// KB = d / 32 k-blocks.  Shared memory: A hi | A lo (KB x 16 KB each), then NSB = 3 - KB operand stages (hi | lo,
// KB x 16 KB each), one 2 KB sort buffer per warp (8 warps), the 128 rows' 512-bit rated-set signatures (8 KB) and
// the two warpgroups' 64 x 128 score tiles (33 KB each).
template <int KB>
__global__ void __launch_bounds__(NT + 32, 1)
score_topn_tc_kernel(const float* __restrict__ U, const uint8_t* __restrict__ item_blocks, int d, int n_items,
                     const int* __restrict__ user_ids, int n_rows, const long long* __restrict__ rated_rowptr,
                     const int* __restrict__ rated_cols, float rated_value, int N, int* __restrict__ out_ids,
                     float* __restrict__ out_scores, unsigned long long* __restrict__ workspace) {
  constexpr int D = KB * 32;
  constexpr int OPER = KB * KBLK;                     // bytes of one 128-row operand (hi or lo)
  constexpr int APT = TM * D / 4 / NT;                // float4 per thread of the users' 128-row operand (4 or 8)
  constexpr int NSB = 3 - KB;                         // operand stages: two at d <= 32, one at d <= 64 (227 KB)
  extern __shared__ uint8_t smem_raw[];
  __shared__ int cnt_sh[2][TM];
  __shared__ uint64_t full[NSB];                      // operand stage s holds a whole tile (bulk-copy bytes counted)
  __shared__ uint64_t empty[NSB];                     // the 8 warps' MMAs that read stage s have retired
  // 1024-byte alignment by an offset from the array itself (not an integer round trip): the compiler keeps the
  // shared address space, so the sort / rated buffers are read with LDS / written with STS
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* const sA_hi = smem;
  uint8_t* const sA_lo = smem + OPER;
  uint8_t* const sB = smem + 2 * OPER;                // stage s: hi at sB + s * 2 * OPER, lo right behind it
  unsigned long long* const sort_buf = reinterpret_cast<unsigned long long*>(smem + (2 + 2 * NSB) * OPER);
  uint32_t* const sig = reinterpret_cast<uint32_t*>(smem + (2 + 2 * NSB) * OPER + 8 * SORTN * sizeof(unsigned long long));   // [SIGW][TM], word-major
  float* const scores_all = reinterpret_cast<float*>(sig + SIGW * TM);                 // [2][64][SP]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int grp = warp >> 2;                          // warpgroup: users 64 grp .. 64 grp + 63 of the CTA
  const bool selecting = warp < NT / 32;
  // the thread's 32-row quarter and which 64 columns of a tile it selects from (the 9th warp selects nothing)
  const int wq = selecting ? 2 * grp + (warp & 1) : 0, half = selecting ? (warp >> 1) & 1 : 2;
  const int rowl = wq * 32 + lane;                    // the thread's user row inside the CTA
  float* const scores = scores_all + (size_t)(grp & 1) * 64 * SP;                      // this warpgroup's score tile
  const int row0 = blockIdx.x * TM;
  const int my_row = row0 + rowl;
  const int u = (my_row < n_rows) ? __ldg(user_ids + my_row) : -1;
  unsigned long long* const cand = workspace + (size_t)blockIdx.x * TM * 2 * CAP;   // this CTA's 2 x 128 lists
  unsigned long long* const my_cand = cand + ((size_t)rowl * 2 + half) * CAP;
  unsigned long long* const my_sort = sort_buf + (size_t)warp * SORTN;
  long long rlo = 0, rhi = 0;
  if (u >= 0) { rlo = __ldg(rated_rowptr + u); rhi = __ldg(rated_rowptr + u + 1); }
  const unsigned long long rated_key_hi = (unsigned long long)ord_of(rated_value) << 32;
  // this row's rated-set signature: bit hash(item) of 512 (the owning thread is the only writer of its column)
  if (half == 0) {
#pragma unroll
    for (int w = 0; w < SIGW; ++w) sig[w * TM + rowl] = 0u;
    for (long long k = rlo; k < rhi; ++k) {
      const uint32_t h = ((uint32_t)__ldg(rated_cols + k) * 0x9E3779B1u) >> 23;
      sig[(h >> 5) * TM + rowl] |= 1u << (h & 31);
    }
  }

  if (tid == 0) {
    for (int b = 0; b < NSB; ++b) {
      mbar_init(&full[b], 1);
      mbar_init(&empty[b], NT / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // ---- the users' rows, split and stored once: float4 number q of the tile is (row q / (D/4), columns 4 * (q % (D/4)))
#pragma unroll
  for (int p = 0; p < APT; ++p) {
    if (tid >= NT) break;                             // the 9th warp stages nothing
    const int q = tid + NT * p;
    const int row = q / (D / 4), c4 = (q % (D / 4)) * 4;
    const int ur = (row0 + row < n_rows) ? __ldg(user_ids + row0 + row) : -1;
    const float4 v = (ur >= 0 && c4 < d) ? __ldg(reinterpret_cast<const float4*>(U + (size_t)ur * d + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 hi, lo;
    split_tf32(v, hi, lo);
    const uint32_t off = (uint32_t)(c4 >> 5) * KBLK + sw_off(row, c4 & 31);
    *reinterpret_cast<float4*>(sA_hi + off) = hi;
    *reinterpret_cast<float4*>(sA_lo + off) = lo;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // the A operands: generic-proxy writes -> async proxy (wgmma)
  __syncthreads();

  const int n_tiles = (n_items + TN - 1) / TN;
  int cnt = 0;                                        // this thread's row: candidates in its list, current cut-off
  unsigned long long thr = 0ULL;

  // Row `src` of this warp goes back to its N best: the N-th largest of its c keys by a bit-wise search on the keys
  // held in registers (keys are distinct: the item id is part of the key), then the keys at or above it move to the
  // front of the list.  The owner's count and cut-off are updated.
  auto compact_row = [&](int src) {
    const int c = __shfl_sync(0xffffffffu, cnt, src);
    unsigned long long* list = cand + ((size_t)(wq * 32 + src) * 2 + half) * CAP;
    unsigned long long k[CAP / 32];
#pragma unroll
    for (int i = 0; i < CAP / 32; ++i) k[i] = (lane + 32 * i < c) ? __ldcg(list + lane + 32 * i) : 0ULL;
    // high words first (the score): the largest T with at least N keys whose high word is >= T
    uint32_t th = 0;
#pragma unroll 1
    for (int b = 31; b >= 0; --b) {
      const uint32_t t1 = th | (1u << b);
      int n = 0;
#pragma unroll
      for (int i = 0; i < CAP / 32; ++i) n += ((uint32_t)(k[i] >> 32) >= t1) ? 1 : 0;
      if (__reduce_add_sync(0xffffffffu, n) >= N) th = t1;
    }
    int above = 0, equal = 0;
#pragma unroll
    for (int i = 0; i < CAP / 32; ++i) {
      above += ((uint32_t)(k[i] >> 32) > th) ? 1 : 0;
      equal += ((uint32_t)(k[i] >> 32) == th) ? 1 : 0;
    }
    above = __reduce_add_sync(0xffffffffu, above);
    equal = __reduce_add_sync(0xffffffffu, equal);
    uint32_t tl = 0;                                   // low word (inverted item id) of the N-th key among the ties
    if (equal > N - above) {                           // more keys tie on the score than fit: the smallest item ids win
#pragma unroll 1
      for (int b = 31; b >= 0; --b) {
        const uint32_t t1 = tl | (1u << b);
        int n = 0;
#pragma unroll
        for (int i = 0; i < CAP / 32; ++i) n += ((uint32_t)(k[i] >> 32) == th && (uint32_t)k[i] >= t1) ? 1 : 0;
        if (__reduce_add_sync(0xffffffffu, n) >= N - above) tl = t1;
      }
    }
    const unsigned long long cut = ((unsigned long long)th << 32) | tl;     // keys >= cut: exactly N of them
    unsigned long long low = ~0ULL;
    int base = 0;
    __syncwarp();
#pragma unroll
    for (int i = 0; i < CAP / 32; ++i) {
      const bool keep = k[i] >= cut && k[i] != 0ULL;
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        __stcg(list + base + __popc(m & ((1u << lane) - 1u)), k[i]);
        low = k[i] < low ? k[i] : low;
      }
      base += __popc(m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, low, o);
      low = other < low ? other : low;
    }
    if (lane == src) { cnt = base; thr = low; }        // base == N; low = the N-th best key
    __syncwarp();
  };
  // tile t: this warpgroup's 64 users x 128 items on the tensor cores, parked in its score tile, then the selection
  constexpr uint32_t TILE_BYTES = 2 * OPER;
  auto select_tile = [&](int t) {
    // a row that could overflow during this tile goes back to its N best first (its warp works on it together)
    unsigned need = __ballot_sync(0xffffffffu, cnt > N + TRIG_EXTRA);
    while (need) {
      const int src = __ffs(need) - 1;
      need &= need - 1;
      compact_row(src);
    }
    {
      const int s = t % NSB;
      mbar_wait(&full[s], (uint32_t)((t / NSB) & 1));                  // tile t has landed
      __syncwarp();                                                      // wgmma is warp-aligned: reconverge after the spin
      uint8_t* const sB_hi = sB + s * TILE_BYTES;
      uint8_t* const sB_lo = sB_hi + OPER;
      float acc[64];
      wg::fence();
      bool first = true;
#pragma unroll
      for (int kb = 0; kb < KB; ++kb) {
        const int a_off = kb * KBLK + grp * (KBLK / 2);                 // this warpgroup's 64 rows of the k-block
        const uint64_t a_hi = wg::desc_sw128(smem_u32(sA_hi + a_off)), a_lo = wg::desc_sw128(smem_u32(sA_lo + a_off));
        const uint64_t b_hi = wg::desc_sw128(smem_u32(sB_hi + kb * KBLK)), b_lo = wg::desc_sw128(smem_u32(sB_lo + kb * KBLK));
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4) {
          const uint64_t step = (uint64_t)(k4 * 2);   // +2 = 32 bytes (8 tf32) along K inside the 128-byte span
#pragma unroll
          for (int term = 0; term < 3; ++term) {      // small terms first: lo.hi, hi.lo, then hi.hi
            const uint64_t da = (term == 0 ? a_lo : a_hi) + step;
            const uint64_t db = (term == 1 ? b_lo : b_hi) + step;
            wg::mma_m64n128k8_tf32(acc, da, db, first ? 0u : 1u);
            first = false;
          }
        }
      }
      wg::commit();
      wg::wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      group_sync(grp);                                // every warp of the group is done reading the previous tile's scores
      const int w4 = warp & 3;
#pragma unroll
      for (int e = 0; e < 64; e += 2)
        *reinterpret_cast<float2*>(scores + wg::frag_row(w4, lane, e) * SP + wg::frag_col(lane, e)) = make_float2(acc[e], acc[e + 1]);
      group_sync(grp);
    }
    // pre-filter for the 128 scores of this tile (the cut-off only moves in the compaction above): a score below the
    // cut-off's score cannot pass, unless the list is not full yet or a rated item's fixed value could pass
    const bool open_row = thr == 0ULL || (uint32_t)(thr >> 32) <= (uint32_t)(rated_key_hi >> 32);
    const float thr_f = open_row ? -INFINITY : score_of((uint32_t)(thr >> 32));
    const int c0 = t * TN + half * 64;                                // first item of this thread's 64 columns
    const int valid = n_items - c0;                                    // columns of them that are items (may be <= 0 or > 64)
    const float* const my_scores = scores + (rowl - 64 * grp) * SP + half * 64;
#pragma unroll 1
    for (int cc = 0; cc < 64; cc += 16) {
      uint32_t r[16];
#pragma unroll
      for (int q = 0; q < 16; q += 4) {
        const float4 v = *reinterpret_cast<const float4*>(my_scores + cc + q);
        r[q] = __float_as_uint(v.x); r[q + 1] = __float_as_uint(v.y); r[q + 2] = __float_as_uint(v.z); r[q + 3] = __float_as_uint(v.w);
      }
      // 16 compares without a branch: bit q of `pass` <=> score q is at or above the cut-off's score
      uint32_t pass = 0;
#pragma unroll
      for (int q = 0; q < 16; ++q) pass |= (__uint_as_float(r[q]) >= thr_f ? 1u : 0u) << q;
      if (valid - cc < 16) pass &= (valid - cc) <= 0 ? 0u : ((1u << (valid - cc)) - 1u);
      if (u < 0) pass = 0;
      if (pass) {                                     // the few that pass: exact 64-bit test, rated test on a signature hit
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          if (pass & (1u << q)) {
            const int c = c0 + cc + q;
            const unsigned long long low = (unsigned long long)(0xffffffffu - (uint32_t)c);
            unsigned long long key = ((unsigned long long)ord_of(__uint_as_float(r[q])) << 32) | low;
            // a rated item scores `rated_value` whatever its dot product: it can pass even when the raw score does not
            if (key > thr || (rated_key_hi | low) > thr) {
              const uint32_t h = ((uint32_t)c * 0x9E3779B1u) >> 23;
              if (((sig[(h >> 5) * TM + rowl] >> (h & 31)) & 1u) && is_rated(rated_cols, rlo, rhi, c)) key = rated_key_hi | low;
              if (key > thr) {
                __stcg(my_cand + cnt, key);           // cnt < CAP by the compaction rule
                ++cnt;
              }
            }
          }
        }
      }
    }
    __syncwarp();
  };

  // ---- main loop.  The 9th warp's lane 0 streams the item tiles in (tile j into the operand stage that the MMAs of
  // tile j - NSB have released) and never selects; the two warpgroups follow at their own pace (no CTA-wide barrier
  // per tile: a warpgroup that compacts a list only holds back the stage its MMAs have not released yet).
  if (warp == NT / 32) {
    if (lane == 0) {
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j % NSB;
        if (j >= NSB) mbar_wait(&empty[s], (uint32_t)((j / NSB - 1) & 1));   // the MMAs of tile j - NSB have retired
        mbar_expect_tx(&full[s], TILE_BYTES);
        bulk_g2s(sB + s * TILE_BYTES, item_blocks + (size_t)j * TILE_BYTES, TILE_BYTES, &full[s]);
      }
    }
  } else {
    for (int t = 0; t < n_tiles; ++t) select_tile(t);
  }

  // ---- final: every list down to at most N keys, then the two lists of a row merged, sorted and written
  __syncwarp();
  if (warp < NT / 32) {
    unsigned need = __ballot_sync(0xffffffffu, cnt > N);
    while (need) {
      const int src = __ffs(need) - 1;
      need &= need - 1;
      compact_row(src);
    }
  }
  if (warp < NT / 32) cnt_sh[half][rowl] = cnt;
  __syncthreads();                                    // both halves' lists (global, st.cg) and counts are visible
  for (int src = half; src < 32 && warp < NT / 32; src += 2) {   // the two warps of a lane quarter share its 32 rows
    const int r = wq * 32 + src;
    const int ur = __shfl_sync(0xffffffffu, u, src);
    if (ur < 0) continue;
    const int ca = cnt_sh[0][r], cb = cnt_sh[1][r];   // <= N each
    const unsigned long long* la = cand + (size_t)r * 2 * CAP;
    const unsigned long long* lb = la + CAP;
    __syncwarp();
    for (int k = lane; k < SORTN; k += 32) my_sort[k] = k < ca ? __ldcg(la + k) : (k - ca < cb ? __ldcg(lb + (k - ca)) : 0ULL);
    warp_sort_desc<SORTN>(my_sort, lane);
    const size_t orow = (size_t)(row0 + r) * N;
    for (int k = lane; k < N; k += 32) {
      const unsigned long long key = my_sort[k];
      out_ids[orow + k] = (int)(0xffffffffu - (uint32_t)(key & 0xffffffffULL));
      out_scores[orow + k] = score_of((uint32_t)(key >> 32));
    }
    __syncwarp();
  }
}

template <int KB>
int launch_tc(const float* U, const float* V, int d, int n_items, const int* user_ids, int n_rows, const long long* rowptr,
              const int* cols, float rated_value, int N, int* out_ids, float* out_scores, cudaStream_t st) {
  constexpr int SMEM = (2 + 2 * (3 - KB)) * KB * KBLK + 8 * SORTN * (int)sizeof(unsigned long long) + SIGW * TM * (int)sizeof(uint32_t) +
                       2 * 64 * SP * (int)sizeof(float) + 1024;   // operands + sort buffers + signatures + score tiles + alignment
  QREC_CUDA(allow_dynamic_smem((const void*)score_topn_tc_kernel<KB>, SMEM));
  const int grid = (n_rows + TM - 1) / TM;
  const int n_tiles = (n_items + TN - 1) / TN;
  const size_t list_bytes = (size_t)grid * TM * 2 * CAP * sizeof(unsigned long long);   // candidate lists: 2 x 2.5 KB per user
  const size_t block_bytes = (size_t)n_tiles * 2 * KB * KBLK;                         // the split item table, tile by tile
  uint8_t* ws = nullptr;                                                              // stream-ordered scratch
  QREC_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&ws), list_bytes + block_bytes, st));
  uint8_t* const blocks = ws + list_bytes;                                            // (list_bytes is a multiple of 640 KB)
  split_items_kernel<KB><<<n_tiles, 128, 0, st>>>(V, d, n_items, blocks);
  score_topn_tc_kernel<KB><<<grid, NT + 32, SMEM, st>>>(U, blocks, d, n_items, user_ids, n_rows, rowptr, cols, rated_value, N, out_ids,
                                                    out_scores, reinterpret_cast<unsigned long long*>(ws));
  const cudaError_t launch_err = cudaGetLastError();
  QREC_CUDA(cudaFreeAsync(ws, st));
  if (launch_err != cudaSuccess) return qrec::cuda_fail(launch_err, "kernel launch", __FILE__, __LINE__);
  qrec::count_launch(2);
  return QREC_OK;
}

}  // namespace

extern "C" int qrec_score_topn_tc_f32(const float* dev_U, const float* dev_V, int32_t d, int32_t n_items,
                                      const int32_t* dev_user_ids, int32_t n_rows, const int64_t* dev_rated_rowptr,
                                      const int32_t* dev_rated_cols, float rated_value, int32_t N, int32_t* dev_out_ids,
                                      float* dev_out_scores, void* stream) {
  QREC_REQUIRE(n_rows >= 0 && n_items >= 1, "qrec_score_topn_tc_f32: bad size");
  QREC_REQUIRE(d >= 4 && d <= 64 && d % 4 == 0, "qrec_score_topn_tc_f32: d=%d unsupported (multiple of 4, <= 64; use qrec_score_topn_f32)", d);
  QREC_REQUIRE(N >= 1 && N <= NMAX && N <= n_items, "qrec_score_topn_tc_f32: N=%d must be in 1..min(%d, n_items)", N, NMAX);
  if (n_rows == 0) return QREC_OK;
  QREC_REQUIRE(dev_U && dev_V && dev_user_ids && dev_rated_rowptr && dev_rated_cols && dev_out_ids && dev_out_scores,
               "qrec_score_topn_tc_f32: null pointer");
  QREC_REQUIRE((reinterpret_cast<uintptr_t>(dev_U) & 15) == 0 && (reinterpret_cast<uintptr_t>(dev_V) & 15) == 0,
               "qrec_score_topn_tc_f32: tables must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long* rp = reinterpret_cast<const long long*>(dev_rated_rowptr);
  if (d <= 32)                                            // columns beyond d are zero-filled up to the 32-wide k-block
    return launch_tc<1>(dev_U, dev_V, d, n_items, dev_user_ids, n_rows, rp, dev_rated_cols, rated_value, N, dev_out_ids, dev_out_scores, st);
  return launch_tc<2>(dev_U, dev_V, d, n_items, dev_user_ids, n_rows, rp, dev_rated_cols, rated_value, N, dev_out_ids, dev_out_scores, st);
}
