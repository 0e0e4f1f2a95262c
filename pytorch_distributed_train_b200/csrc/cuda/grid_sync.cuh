// Device-side grid barrier for cooperative kernels (all CTAs co-resident).  See GridBar.
#pragma once
#include <cuda_runtime.h>

namespace pdt {

// Device memory of the grid barrier shared by every cooperative kernel of a device (zero before first use):
// a monotonically increasing epoch word and an arrival counter.
struct GridSync {
  unsigned int* epoch;
  unsigned int* flags;   // [0] = arrival counter
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned int ld_acquire_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int ld_relaxed_gpu(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_gpu(unsigned int* p, unsigned int v) {
  asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_gpu(unsigned int* p, unsigned int v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Grid barrier: one arrival counter, one monotonically increasing epoch word.  Thread 0 of a CTA arrives with a fence +
// atomicAdd; the last arriver zeroes the counter and publishes the barrier's epoch; everybody else polls the epoch word
// with *relaxed* loads (one poller per CTA; an acquire per spin would invalidate L1 every iteration).  Everything read
// after the barrier comes from L2 (ld.global.cg), the GPU's coherence point, so no trailing fence is needed.  Each CTA
// tracks the epoch locally (read once at kernel start, +1 per barrier): no read of the word before arriving, nothing to
// reset between launches or CUDA-graph replays, any grid size.  A flag-per-CTA variant (every CTA polling every flag)
// puts ~10^4 pollers on four cache lines and is slower than the counter.
// Programmatic dependent launch: a grid launched while the kernel before it still runs touches no grid-barrier word — the
// constructor's epoch read included — before griddep_wait() (hopper_ptx.cuh).  That kernel may still be passing its own barriers on
// the same two words: a dependent that read the epoch early would start from a stale value and pass its first barrier on the other
// kernel's epoch store.
struct GridBar {
  unsigned int e;
  __device__ __forceinline__ explicit GridBar(GridSync gs) : e(gs.epoch ? *reinterpret_cast<volatile unsigned int*>(gs.epoch) : 0u) {}
  // NAMED > 0: only the first NAMED threads of the CTA take part (named barrier 1) — the kernel has extra warps with their own roles.
  template <int NAMED = 0>
  __device__ __forceinline__ void cta_sync() {
    if constexpr (NAMED > 0) asm volatile("bar.sync 1, %0;" ::"n"(NAMED) : "memory");
    else __syncthreads();
  }
  // Split form: arrive() publishes this CTA's contribution, wait() blocks until every CTA has arrived.  Work placed between
  // the two runs in the barrier's shadow (the barrier latency plus the skew between CTAs) — it must not depend on other CTAs.
  template <int NAMED = 0>
  __device__ __forceinline__ void arrive(GridSync gs) {
    ++e;
    cta_sync<NAMED>();   // the CTA's partial row is complete
    if (threadIdx.x == 0) {
      __threadfence();   // ... and performed at GPU scope before the arrival (bar.sync makes the fence cumulative over the CTA)
      const unsigned int prev = atomicAdd(gs.flags, 1u);
      if (prev == gridDim.x - 1) {
        st_relaxed_gpu(gs.flags, 0u);
        __threadfence();
        st_relaxed_gpu(gs.epoch, e);
      }
    }
  }
  template <int NAMED = 0>
  __device__ __forceinline__ void wait(GridSync gs) {
    if (threadIdx.x == 0) {
      unsigned int spins = 0;
      unsigned long long t0 = 0;
      while (static_cast<int>(ld_relaxed_gpu(gs.epoch) - e) < 0) {
        // a grid that is not fully resident (non-cooperative launch on a busy GPU) would spin forever: trap after 4 s instead
        if ((++spins & 0xFFFu) == 0) {
          unsigned long long t;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
          if (t0 == 0) t0 = t;
          else if (t - t0 > 4000000000ull) asm volatile("trap;");
        }
      }
    }
    cta_sync<NAMED>();
  }
  template <int NAMED = 0>
  __device__ __forceinline__ void sync(GridSync gs) {
    arrive<NAMED>(gs);
    wait<NAMED>(gs);
  }
  __device__ __forceinline__ void finish(GridSync) {}
};

#endif  // __CUDACC__

}  // namespace pdt
