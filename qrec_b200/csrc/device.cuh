// Device building blocks shared by the kernels of libqrec.so: the vector scatter-add every hot kernel ends in,
// lane-group reductions, the SFU sigmoid / -ln of the throughput kernels, the ticket / wait / publish protocol of the
// in-order kernels, the per-block loss reduction and the mbarrier helpers of the bulk-copy (TMA) pipelines.
#pragma once
#include <cstdint>

namespace qrec {

// REDG.E.ADD.F32x4: adds v to the 16-byte aligned float4 at addr in one instruction
__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- L2 residency hints: tables that should stay in L2 are read and written under an evict_last policy, and loads
// that are not reused do not allocate in L1.  A policy is a 64-bit register made once per thread by createpolicy.
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
// a read-only load under policy `pol` that does not allocate in L1
__device__ __forceinline__ float4 ld_stream_v4(const float4* p, unsigned long long pol) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0, %1, %2, %3}, [%4], %5;"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ void st_hint_v4(float4* p, float4 v, unsigned long long pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w),
               "l"(pol) : "memory");
}
// a read-only float4 that is not allocated in L1 (no L2 policy)
__device__ __forceinline__ float4 ldg_no_l1_v4(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

// ---- Programmatic dependent launch (sm_90).  In a kernel launched with programmatic stream serialization,
// pdl_wait() returns once the previous kernel on the stream has completed and its memory operations are visible;
// everything before it may overlap that kernel.  pdl_launch_dependents() lets the next such kernel on the stream be
// launched before this one ends.  In a kernel launched normally both are no-ops.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }

// acc += s * x
__device__ __forceinline__ void fma4(float4& acc, float s, float4 x) {
  acc.x = fmaf(s, x.x, acc.x); acc.y = fmaf(s, x.y, acc.y);
  acc.z = fmaf(s, x.z, acc.z); acc.w = fmaf(s, x.w, acc.w);
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// sum over the LPR lanes of an aligned lane group (xor-shuffle butterfly); mask: the lanes taking part
template <int LPR>
__device__ __forceinline__ float group_sum(float v, unsigned mask = 0xffffffffu) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o);
  return v;
}

// Throughput kernels: sigmoid and -ln(s) on the SFU (ex2.approx / lg2.approx / rcp.approx).  The relative error
// (~2^-21) is far below the fp32 rounding of the row update it scales; parity mode keeps expf/logf.
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_neg_log(float s) { return -__logf(s); }

// Row versions of the parity kernels: a warp waits with acquire loads until its rows reach the version it needs
// and publishes its own update with a release add.
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ---- In-order kernels.  K1's, K9's and K16's ordered SGD kernels and K17's user pass replay a sequential loop with
// one warp per position; K12's item sweep does so with one CTA per item.  They share one protocol:
//   * positions are drawn from a global ticket in order (warp_next_ticket; K12 draws per CTA), so they go to running
//     warps in order;
//   * before it reads, a position polls the counters that earlier positions publish until they reach the values it
//     needs (spin_until with acquire loads);
//   * after it writes, every lane's stores are made visible (warp_fence) before the release adds that publish them.
// A position waits only on smaller ones, which running warps hold, and the smallest unfinished position waits on
// nobody, so the scheme cannot deadlock whatever the grid size.  A position waits for at most (#resident warps)
// predecessors, i.e. milliseconds; about 8.6 s (2^33 ns) of polling means its wait numbers do not describe the
// stream, and it traps (the host sees a launch failure) instead of hanging the GPU.

// the warp's next position: lane 0 draws it, every lane gets it
__device__ __forceinline__ unsigned long long warp_next_ticket(unsigned long long* ticket) {
  unsigned long long k = 0;
  if ((threadIdx.x & 31) == 0) k = atomicAdd(ticket, 1ULL);
  return __shfl_sync(0xffffffffu, k, 0);
}

// Polls until ready() is true, sleeping FIRST_NS after the first miss and doubling up to MAX_NS; traps after
// 2^33 / MAX_NS polls.  Warp kernels pass a ready() that votes with __all_sync, so the warp leaves together.
template <unsigned FIRST_NS, unsigned MAX_NS, typename F>
__device__ __forceinline__ void spin_until(F ready) {
  constexpr unsigned kMaxPolls = (unsigned)((1ULL << 33) / MAX_NS);
  unsigned backoff = FIRST_NS, polls = 0;
  while (!ready()) {
    __nanosleep(backoff);
    if (backoff < MAX_NS) backoff <<= 1;
    if (++polls > kMaxPolls) __trap();
  }
}

// every lane's row writes visible before any lane's release add
__device__ __forceinline__ void warp_fence() {
  __threadfence();
  __syncwarp();
}

// The block's per-thread fp32 loss terms summed into *loss with one double atomic (none when the sum is 0).
// Called by every thread of a block of at most 256 threads.
__device__ __forceinline__ void block_add_loss(float lsum, double* loss) {
  __shared__ float wsum[8];
  lsum = warp_sum(lsum);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += (double)wsum[w];
    if (t != 0.0) atomicAdd(loss, t);
  }
}

// ---- mbarriers (shared::cta) for the bulk-copy engine
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: after ~4M polls a protocol error traps (the launch fails with an error) instead of hanging the device.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spins = 0;; ++spins) {
    if (mbar_try_wait(bar, parity)) return;
    if (spins > (1u << 22)) __trap();
  }
}

}  // namespace qrec
