// Hopper (sm_90a) warpgroup MMA, TF32 in / fp32 accumulate, for the tensor-core kernels (tc_gemm.cu, topn_tc.cu).
// Both operands are read from shared memory in the canonical K-major SWIZZLE_128B layout: rows of 32 fp32 (128 B),
// 8-row 1024 B atoms, 16-byte chunk index XOR row % 8 -- what sw_off() writes and what a TMA copy with
// CU_TENSOR_MAP_SWIZZLE_128B produces.  A 128 x K tile is two m64 halves 8 KB apart per 32-wide k-block.
//
// Accumulator fragment of one m64nN instruction (N / 2 floats per thread of the warpgroup): element e of thread
// (warp w of the warpgroup, lane l) is row 16 w + l / 4 + 8 ((e >> 1) & 1), column 8 (e >> 2) + 2 (l % 4) + (e & 1).
#pragma once
#include <cstdint>

namespace wg {

// byte offset of element (row, k) inside a K-major SWIZZLE_128B tile (k in [0,32) fp32)
__device__ __forceinline__ uint32_t sw_off(int row, int k) {
  const int chunk = (k >> 2) ^ (row & 7);
  return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + chunk * 16 + (k & 3) * 4);
}

// fp32 -> TF32, rounded to nearest (ties away).  The tensor cores read the top 19 bits of an fp32 operand, i.e.
// truncate; rounding while staging removes that systematic toward-zero bias (2^-11 unbiased instead of up to
// 2^-10 one-sided per operand).
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float4 to_tf32(float4 v) { return make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w)); }

// shared-memory matrix descriptor, K-major SWIZZLE_128B: start >> 4 | LBO 16 B (unused by this layout) | SBO 1024 B
// (one 8-row atom) | layout type 1 (128B swizzle).  The atom must be 1024-byte aligned; a step of 8 tf32 along K is
// +32 bytes of start address (+2 in the descriptor).
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// accumulator element e of this thread: row and column inside the m64 x N tile
__device__ __forceinline__ int frag_row(int warp_in_group, int lane, int e) { return 16 * warp_in_group + (lane >> 2) + 8 * ((e >> 1) & 1); }
__device__ __forceinline__ int frag_col(int lane, int e) { return 8 * (e >> 2) + 2 * (lane & 3) + (e & 1); }

// d (+)= A[64 x 8] * B[N x 8]^T; accumulate = 0 overwrites d
__device__ __forceinline__ void mma_m64n64k8_tf32(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void mma_m64n128k8_tf32(float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}

}  // namespace wg
