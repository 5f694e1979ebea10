// Replicated item table, data-parallel BPR (SURVEY.md 8e: users range-partitioned, Q replicated): every
// rank trains on its own users and the ranks exchange the SUM of their item-row deltas.  These kernels
// make that exchange asynchronous and overlappable with the next K1 launch:
//
//   compute stream:  K1(wave k) -> delta_k: D = Q - B -> K1(wave k+1) ...
//   side stream   :                 [ exchange: S = sum over ranks of D ] -> merge_k: Q += S - D ; B += S
//
// B ("base") is the globally agreed table at the last exchange.  delta reads Q element-wise ONCE; every
// local update that lands after that read is, by construction, part of the next delta, and merge adds the
// other ranks' contribution with a float atomic (RED), which commutes with K1's own REDs on the same rows.
// So the invariant  Q_r - B = (local updates not yet exchanged)  holds for any interleaving, and K1 never
// waits for the exchange.  (reference: model/ranking/BPR.py:45-52 updates Q[i], Q[j] in place; summing the
// ranks' deltas is the data-parallel form of those in-place updates.)
//
// The exchange is either NCCL (all-reduce of S) or the two peer-memory kernels below: reduce-scatter by
// P2P loads over NVLink (each rank sums its slice of all ranks' D), all-gather fused with the merge (each
// rank reads the summed slices from their owners and applies them).  All kernels here are built to
// co-reside with K1 (128 threads, <= 32 registers: K1 leaves 4096 registers per SM free at 3 CTAs/SM).
#include "common.h"
#include "device.cuh"

namespace {

using qrec::red_add_v4;

constexpr int kMaxPeers = 16;
struct PeerPtrs { const float* p[kMaxPeers]; };

// peer data is written by another GPU between launches: bypass L1, read at system scope
__device__ __forceinline__ float4 ld_peer_v4(const float* p) {
  float4 v;
  asm volatile("ld.global.relaxed.sys.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(128, 16)
table_delta_kernel(const float4* __restrict__ Q, const float4* __restrict__ B, float4* __restrict__ D, float4* __restrict__ S,
                   long long n4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n4; k += stride) {
    const float4 q = __ldcg(Q + k);          // Q is being RED-updated in L2: read it there
    const float4 b = B[k];
    const float4 d = make_float4(q.x - b.x, q.y - b.y, q.z - b.z, q.w - b.w);
    D[k] = d;
    if (S != nullptr) S[k] = d;
  }
}

__global__ void __launch_bounds__(128, 16)
table_merge_kernel(float* __restrict__ Q, float4* __restrict__ B, const float4* __restrict__ D, const float4* __restrict__ S,
                   long long n4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n4; k += stride) {
    const float4 s = S[k], d = D[k];
    float4 b = B[k];
    red_add_v4(Q + 4 * k, make_float4(s.x - d.x, s.y - d.y, s.z - d.z, s.w - d.w));
    b.x += s.x; b.y += s.y; b.z += s.z; b.w += s.w;
    B[k] = b;
  }
}

// S_mine[lo4 .. hi4) = sum over ranks (fixed order 0..world-1, so every slice is summed the same way) of D_r
__global__ void __launch_bounds__(128, 16)
table_reduce_scatter_kernel(PeerPtrs peers_D, int world, float4* __restrict__ S, long long lo4, long long hi4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = lo4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; k < hi4; k += stride) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < world; ++r) {
      const float4 v = ld_peer_v4(peers_D.p[r] + 4 * k);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    S[k] = acc;
  }
}

// element k belongs to the slice of rank k / slice4; read its sum there, then merge as above
__global__ void __launch_bounds__(128, 16)
table_gather_merge_kernel(PeerPtrs peers_S, int world, long long slice4, float* __restrict__ Q, float4* __restrict__ B,
                          const float4* __restrict__ D, long long n4) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x; k < n4; k += stride) {
    int owner = (int)(k / slice4);
    if (owner >= world) owner = world - 1;
    const float4 s = ld_peer_v4(peers_S.p[owner] + 4 * k);
    const float4 d = D[k];
    float4 b = B[k];
    red_add_v4(Q + 4 * k, make_float4(s.x - d.x, s.y - d.y, s.z - d.z, s.w - d.w));
    b.x += s.x; b.y += s.y; b.z += s.z; b.w += s.w;
    B[k] = b;
  }
}

int grid_for(long long n4) { return qrec::capped_grid((n4 + 127) / 128, 4); }

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

extern "C" {

int qrec_table_delta_f32(const float* Q, const float* B, float* D, float* S, int64_t n, void* stream) {
  QREC_REQUIRE(n >= 0 && (n % 4) == 0, "qrec_table_delta_f32: n=%lld must be a non-negative multiple of 4", (long long)n);
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(Q && B && D, "qrec_table_delta_f32: null pointer");
  QREC_REQUIRE(aligned16(Q) && aligned16(B) && aligned16(D) && aligned16(S), "qrec_table_delta_f32: pointers must be 16-byte aligned");
  table_delta_kernel<<<grid_for(n / 4), 128, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(Q), reinterpret_cast<const float4*>(B), reinterpret_cast<float4*>(D),
      reinterpret_cast<float4*>(S), n / 4);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_table_merge_f32(float* Q, float* B, const float* D, const float* S, int64_t n, void* stream) {
  QREC_REQUIRE(n >= 0 && (n % 4) == 0, "qrec_table_merge_f32: n=%lld must be a non-negative multiple of 4", (long long)n);
  if (n == 0) return QREC_OK;
  QREC_REQUIRE(Q && B && D && S, "qrec_table_merge_f32: null pointer");
  QREC_REQUIRE(aligned16(Q) && aligned16(B) && aligned16(D) && aligned16(S), "qrec_table_merge_f32: pointers must be 16-byte aligned");
  table_merge_kernel<<<grid_for(n / 4), 128, 0, (cudaStream_t)stream>>>(Q, reinterpret_cast<float4*>(B),
                                                                        reinterpret_cast<const float4*>(D),
                                                                        reinterpret_cast<const float4*>(S), n / 4);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_table_reduce_scatter_p2p_f32(const float* const* peer_D, int32_t world, int32_t rank, float* S, int64_t n,
                                      void* stream) {
  QREC_REQUIRE(peer_D && S, "qrec_table_reduce_scatter_p2p_f32: null pointer");
  QREC_REQUIRE(world >= 1 && world <= kMaxPeers && rank >= 0 && rank < world, "qrec_table_reduce_scatter_p2p_f32: bad world/rank");
  QREC_REQUIRE(n >= 0 && (n % 4) == 0, "qrec_table_reduce_scatter_p2p_f32: n must be a multiple of 4");
  if (n == 0) return QREC_OK;
  PeerPtrs pp;
  for (int r = 0; r < world; ++r) {
    QREC_REQUIRE(peer_D[r] && aligned16(peer_D[r]), "qrec_table_reduce_scatter_p2p_f32: peer pointer %d null or unaligned", r);
    pp.p[r] = peer_D[r];
  }
  const long long n4 = n / 4, slice4 = (n4 + world - 1) / world;
  const long long lo4 = slice4 * rank < n4 ? slice4 * rank : n4;
  const long long hi4 = lo4 + slice4 < n4 ? lo4 + slice4 : n4;
  if (hi4 <= lo4) return QREC_OK;
  table_reduce_scatter_kernel<<<grid_for(hi4 - lo4), 128, 0, (cudaStream_t)stream>>>(pp, world, reinterpret_cast<float4*>(S), lo4, hi4);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

int qrec_table_gather_merge_p2p_f32(const float* const* peer_S, int32_t world, float* Q, float* B, const float* D, int64_t n,
                                    void* stream) {
  QREC_REQUIRE(peer_S && Q && B && D, "qrec_table_gather_merge_p2p_f32: null pointer");
  QREC_REQUIRE(world >= 1 && world <= kMaxPeers, "qrec_table_gather_merge_p2p_f32: bad world");
  QREC_REQUIRE(n >= 0 && (n % 4) == 0, "qrec_table_gather_merge_p2p_f32: n must be a multiple of 4");
  if (n == 0) return QREC_OK;
  PeerPtrs pp;
  for (int r = 0; r < world; ++r) {
    QREC_REQUIRE(peer_S[r] && aligned16(peer_S[r]), "qrec_table_gather_merge_p2p_f32: peer pointer %d null or unaligned", r);
    pp.p[r] = peer_S[r];
  }
  const long long n4 = n / 4, slice4 = (n4 + world - 1) / world;
  table_gather_merge_kernel<<<grid_for(n4), 128, 0, (cudaStream_t)stream>>>(pp, world, slice4, Q, reinterpret_cast<float4*>(B),
                                                                            reinterpret_cast<const float4*>(D), n4);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}

}  // extern "C"
