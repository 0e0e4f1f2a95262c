// Hand-written PTX wrappers for the Hopper data path: mbarrier, TMA (cp.async.bulk.tensor), wgmma and the
// shared-memory matrix descriptors.  Shared by conv_tcgen05.cu and fused_convnet.cu.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>

namespace pdt {
namespace ptx {

// ---------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
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
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}

__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// Ampere-style async copy with zero fill (src_bytes = 0 → 16 zero bytes)
__device__ __forceinline__ void cp_async_16(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------------------------------------------
// wgmma (sm_90a): one warpgroup (4 consecutive warps, the first a multiple of 4) issues the MMA; the fp32
// accumulator lives in the registers of its 128 threads.  TF32 operands come from shared memory through
// K-major matrix descriptors (TF32 wgmma has no MN-major form).
// ---------------------------------------------------------------------------------------------------
// Index of the calling thread's warpgroup, in a form the compiler knows to be warp-uniform: branching on it keeps the
// wgmma of the taken side out of a "divergent path", where ptxas would serialise them.
__device__ __forceinline__ int warpgroup_index() { return __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x) / 128, 0); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64×32] (+)= A[64×8] · B[32×8]ᵀ; accumulate = 0 overwrites D.
__device__ __forceinline__ void wgmma_m64n32k8_tf32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
// D[64×16] (+)= A[64×8] · B[16×8]ᵀ
__device__ __forceinline__ void wgmma_m64n16k8_tf32(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  static_assert(N == 16 || N == 32, "wgmma_tf32: N = 16 or 32");
  if constexpr (N == 32) wgmma_m64n32k8_tf32(d, adesc, bdesc, accumulate);
  else wgmma_m64n16k8_tf32(d, adesc, bdesc, accumulate);
}
// Accumulator fragment of an m64nN wgmma: element e of warpgroup thread wt (0..127) is D[frag_row][frag_col].
__device__ __forceinline__ int wgmma_frag_row(int wt, int e) { return 16 * (wt >> 5) + ((wt & 31) >> 2) + 8 * ((e >> 1) & 1); }
__device__ __forceinline__ int wgmma_frag_col(int wt, int e) { return 8 * (e >> 2) + 2 * (wt & 3) + (e & 1); }

// Store the fragment of rows [row0, row0 + 64) into a row-major fp32 tile (pitch in floats), so that one thread can then
// read a whole accumulator row.
template <int N>
__device__ __forceinline__ void wgmma_frag_store(const float (&d)[N / 2], float* tile, int pitch, int row0, int wt) {
#pragma unroll
  for (int e = 0; e < N / 2; ++e) tile[(row0 + wgmma_frag_row(wt, e)) * pitch + wgmma_frag_col(wt, e)] = d[e];
}

// K-major shared-memory matrix descriptor (sm_90 layout) for rows of ROWB bytes (128 → SWIZZLE_128B, 64 → SWIZZLE_64B):
//   start address >> 4 | LBO (unused for swizzled K-major: 1) << 16 | SBO = 8 rows >> 4 << 32 | layout << 62.
// The swizzle phase follows the absolute shared-memory address, so a descriptor may start at any row of a 1024-byte-aligned
// buffer (the window convolutions read filter taps as row-shifted views of one patch).  The start-address field is the low
// 14 bits, so descriptors are advanced by plain integer adds of (bytes >> 4).
template <int ROWB>
__device__ __forceinline__ uint64_t gmma_desc_kmajor(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((8 * ROWB) >> 4) << 32;
  d |= static_cast<uint64_t>(ROWB == 128 ? 1 : 2) << 62;
  return d;
}

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}

}  // namespace ptx
}  // namespace pdt
