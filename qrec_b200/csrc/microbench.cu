// Measurement infrastructure for K1's roofline (bench.py "roofline.row_op_peak"): how many 256-byte
// embedding-row operations per second this GPU retires when NOTHING else is done -- the memory-system
// ceiling the fused BPR kernel (bpr_kernels.cu) is compared with.  K1 does, per triple, 2 row gathers
// (LDG.E.128 per lane) and 2 row scatter-adds (REDG.E.ADD.F32x4 per lane) into the item table
// (model/ranking/BPR.py:45-52 reads and writes Q[i], Q[j]); this kernel issues exactly those
// instructions against random rows of a table of the same shape with no arithmetic between them.
//   mode 0: gathers only            mode 1: reductions only          mode 2: one gather + one reduction
// A table that fits the L2 (100K x 64 fp32 = 25.6 MB) gives the L2 ceiling; a table much larger than
// the L2 (4M rows = 1 GB) gives the HBM ceiling of the same access pattern.
#include "common.h"

namespace {

__device__ __forceinline__ uint32_t mix32(uint32_t x) {   // lowbias32 hash: rows are uniform and independent
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

template <int MODE, int INFLIGHT>
__global__ void __launch_bounds__(256)
row_op_kernel(float* __restrict__ T, uint32_t rows, long long n_ops, uint32_t seed, float* sink) {
  // 16 lanes own one 64-float row (a float4 each), like K1 at d=64
  const int l = threadIdx.x & 15;
  const long long group = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
  const long long ngroups = ((long long)gridDim.x * blockDim.x) >> 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 delta = make_float4(1e-9f, -1e-9f, 1e-9f, -1e-9f);
  for (long long k = group * INFLIGHT; k < n_ops; k += ngroups * INFLIGHT) {
    uint32_t r[INFLIGHT];
    float4 v[INFLIGHT];
#pragma unroll
    for (int f = 0; f < INFLIGHT; ++f) {
      const uint32_t h = mix32((uint32_t)(k + f) * 0x9e3779b9U + seed);
      r[f] = (uint32_t)(((unsigned long long)h * rows) >> 32);
    }
    if (MODE != 1) {
#pragma unroll
      for (int f = 0; f < INFLIGHT; ++f) v[f] = *reinterpret_cast<const float4*>(T + (size_t)r[f] * 64 + l * 4);
#pragma unroll
      for (int f = 0; f < INFLIGHT; ++f) { acc.x += v[f].x; acc.y += v[f].y; acc.z += v[f].z; acc.w += v[f].w; }
    }
    if (MODE != 0) {
#pragma unroll
      for (int f = 0; f < INFLIGHT; ++f) {
        // mode 2 reduces into a DIFFERENT random row than it read (K1 reduces into the rows it read some
        // hundred cycles earlier; an unrelated row is the harder, hit-free case)
        const uint32_t rr = MODE == 2 ? (uint32_t)(((unsigned long long)mix32(r[f] + 0x5bd1e995U + seed) * rows) >> 32) : r[f];
        float* a = T + (size_t)rr * 64 + l * 4;
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(delta.x), "f"(delta.y),
                     "f"(delta.z), "f"(delta.w) : "memory");
      }
    }
  }
  if (acc.x + acc.y + acc.z + acc.w == 123.456f) *sink = acc.x;   // keeps the gathers alive
}

}  // namespace

extern "C" int qrec_ubench_row_ops_f32(float* dev_table, int64_t rows, int64_t n_ops, int32_t mode,
                                       uint32_t seed, float* dev_sink, void* stream) {
  QREC_REQUIRE(dev_table && dev_sink, "ubench_row_ops: null pointer");
  QREC_REQUIRE(rows > 0 && rows < (1LL << 32) && n_ops >= 0, "ubench_row_ops: bad sizes");
  QREC_REQUIRE(mode >= 0 && mode <= 2, "ubench_row_ops: mode must be 0 (gather), 1 (reduce) or 2 (both)");
  if (n_ops == 0) return QREC_OK;
  const int grid = qrec::sm_count() * 8;         // 8 CTAs of 256 threads per SM: full occupancy at <= 32 registers
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (mode == 0) row_op_kernel<0, 8><<<grid, 256, 0, st>>>(dev_table, (uint32_t)rows, n_ops, seed, dev_sink);
  else if (mode == 1) row_op_kernel<1, 8><<<grid, 256, 0, st>>>(dev_table, (uint32_t)rows, n_ops, seed, dev_sink);
  else row_op_kernel<2, 8><<<grid, 256, 0, st>>>(dev_table, (uint32_t)rows, n_ops, seed, dev_sink);
  QREC_LAUNCH_CHECK();
  return QREC_OK;
}
