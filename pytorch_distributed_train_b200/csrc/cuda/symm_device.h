// Host/device shared definitions for the symmetric-memory collectives, plus the device-side
// cross-GPU synchronisation primitives (compiled only under nvcc).
#pragma once
#include <cstddef>
#include <cstdint>

namespace pdt {

constexpr int kSymmMaxWorld = 8;       // one NVSwitch domain (single node, like the reference)
constexpr int kSymmChannels = 4;       // independent flag/staging sets: one per concurrent stream
constexpr int kSymmMaxBlocks = 160;    // >= the SM count (132 on an H100 SXM): every CTA of a collective owns a flag row
constexpr int kChanComm = 0;           // process-group collectives on the comm stream
constexpr int kChanInline = 1;         // collectives fused into compute kernels on the caller's stream
constexpr int kChanAux = 2;            // side uses (debug, tests)
constexpr int kChanBench = 3;

// Passed by value to every collective kernel.
struct SymmDev {
  char* peer[kSymmMaxWorld];   // this process's mapping of rank r's heap
  char* mc;                    // multicast mapping of the same heap (nullptr: no NVLS)
  uint32_t* flags;             // OFFSET-less: my signal pad for this channel = peer[rank] + flags_off
  size_t flags_off;            // byte offset of this channel's pad inside every heap
  uint32_t* epochs;            // local device memory: epochs[block]
  int* status;                 // host-mapped: written on timeout before trapping
  unsigned long long timeout_ns;
  int rank, world, channel;
};

}  // namespace pdt

#ifdef __CUDACC__
namespace pdt {

// ---- memory-model primitives (PTX, system scope) ----------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- NVLS (multimem) ---------------------------------------------------------------------------
__device__ __forceinline__ float4 multimem_ld_reduce_f32x4(const void* mc_ptr) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc_ptr)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f32x4(void* mc_ptr, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16x8(const void* mc_ptr) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc_ptr)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 multimem_ld_reduce_f16x8(const void* mc_ptr) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc_ptr)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_b32x4(void* mc_ptr, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// ---- block-level barrier across GPUs -----------------------------------------------------------
// Flag row of (channel, block): kSymmMaxWorld uint32 slots, slot r written by rank r.
// Epochs only grow; a waiter accepts any value >= its epoch (wrap-safe signed compare), so a
// fast peer that already entered the next barrier cannot be missed and nothing is ever reset.
// The epoch lives in device memory and is advanced by the kernel itself ⇒ CUDA-graph replays
// stay in lockstep across ranks.
//
// Call with all threads of the block.  `release`/`acquire` say whether data written before /
// read after the barrier must be ordered with it.
__device__ __forceinline__ uint32_t* symm_flag_row(const SymmDev& d, int r, int block) {
  return reinterpret_cast<uint32_t*>(d.peer[r] + d.flags_off) + static_cast<size_t>(block) * kSymmMaxWorld;
}

__device__ __forceinline__ void symm_trap_timeout(const SymmDev& d, int peer, uint32_t want, uint32_t got) {
  // code: 0x7D000000 | channel<<20 | peer<<16 | low 16 bits of the epoch we waited for
  *reinterpret_cast<volatile int*>(d.status) = 0x7D000000 | (d.channel << 20) | (peer << 16) | (want & 0xffff);
  (void)got;
  __threadfence_system();
  __trap();
}

// Returns the epoch used (for chained barriers pass the previous value + 1 via `epoch`).
__device__ __forceinline__ void symm_barrier_block(const SymmDev& d, int block, uint32_t epoch) {
  __syncthreads();  // every thread's prior global/peer stores are ordered before the signal below
  const int t = threadIdx.x;
  if (t < d.world) {
    // release: cumulativity covers the whole block's writes (ordered by bar.sync above)
    st_release_sys(symm_flag_row(d, t, block) + d.rank, epoch);
    const uint32_t* mine = symm_flag_row(d, d.rank, block) + t;
    uint32_t v = ld_acquire_sys(mine);
    if (static_cast<int32_t>(v - epoch) < 0) {
      const unsigned long long t0 = globaltimer_ns();
      int spins = 0;
      while (static_cast<int32_t>((v = ld_acquire_sys(mine)) - epoch) < 0) {
        if (++spins > 64) {
          __nanosleep(20);
          if ((spins & 1023) == 0 && globaltimer_ns() - t0 > d.timeout_ns) symm_trap_timeout(d, t, epoch, v);
        }
      }
    }
  }
  __syncthreads();  // acquire results become visible to the whole block
}

// Each block reads its current epoch, runs `n` barriers numbered epoch+1..epoch+n, and the last
// thread stores the new value on exit.
struct SymmEpoch {
  uint32_t base;
  int used;
  __device__ __forceinline__ SymmEpoch(const SymmDev& d, int block) : base(d.epochs[block]), used(0) {}
  __device__ __forceinline__ uint32_t next() { return base + static_cast<uint32_t>(++used); }
  __device__ __forceinline__ void commit(const SymmDev& d, int block) {
    __syncthreads();
    if (threadIdx.x == 0) d.epochs[block] = base + static_cast<uint32_t>(used);
  }
};

}  // namespace pdt
#endif  // __CUDACC__
