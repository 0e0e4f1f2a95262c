// Deterministic grid-wide reduction of per-CTA partial vectors, without a second kernel.
//
// Two-level ticket tree: contributors (CTAs, or tiles of a persistent kernel) are grouped by 16; the
// last contributor of a group to arrive folds that group's partials (all participating threads in
// parallel, fixed row order) into a group partial; the last *group* to finish folds the
// ≤ ceil(n/16) group partials and calls fin(i, total) for every output i.  The longest dependent
// chain is ~16 + n/16 row loads split over width-wise thread groups, instead of n serial L2 round
// trips in one thread.  Summation order depends only on (n, width, thread count) ⇒ bit-reproducible.
// Counters are left at zero, so the same scratch serves the next launch / CUDA-graph replay.
#pragma once
#include <cuda_runtime.h>

#include "ops_kernels.h"

namespace pdt {

constexpr int kFoldGroup = 16;

struct CtaSync {
  __device__ __forceinline__ void operator()() const { __syncthreads(); }
};
// Sub-CTA barrier for warp-specialised kernels: `N` threads (multiple of 32) on named barrier `ID`.
template <int ID, int N>
struct NamedSync {
  __device__ __forceinline__ void operator()() const { asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory"); }
};

// Sum rows[0..nrows) of a row-major [nrows][width] matrix; the total of column i is returned to the
// threads with tid < width.  Every one of the `nthreads` participating threads must call it.
template <typename Sync>
__device__ __forceinline__ float fold_rows(const float* rows, int nrows, int width, float* s_tmp /* >= nthreads floats */, int tid,
                                           int nthreads, Sync sync) {
  int G = 1;
  while (G * 2 * width <= nthreads && G < 16) G *= 2;
  const int i = tid % width, g = tid / width;
  if (g < G) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int r = g;
    for (; r + 3 * G < nrows; r += 4 * G) {  // four independent loads in flight
      a0 += __ldcg(rows + static_cast<size_t>(r) * width + i);
      a1 += __ldcg(rows + static_cast<size_t>(r + G) * width + i);
      a2 += __ldcg(rows + static_cast<size_t>(r + 2 * G) * width + i);
      a3 += __ldcg(rows + static_cast<size_t>(r + 3 * G) * width + i);
    }
    for (; r < nrows; r += G) a0 += __ldcg(rows + static_cast<size_t>(r) * width + i);
    s_tmp[g * width + i] = (a0 + a1) + (a2 + a3);
  }
  sync();
  float tot = 0.f;
  if (tid < width)
    for (int k = 0; k < G; ++k) tot += s_tmp[k * width + tid];
  sync();
  return tot;
}

// blk_vals: this contributor's `width` partial values (visible to all participating threads).
// bid / nblk: linear id of this contributor and the number of contributors.
// scr.partials must hold (nblk + ceil(nblk/16)) * width floats; the fold region of scr.counter (ops_kernels.h: words
// [0, scr.fold_counters), which no fixed counter word shares) must hold 1 + ceil(nblk/16) zeroed uints.
// s_flag: one int of shared memory; s_tmp: ≥ nthreads floats of shared memory.
template <typename Sync, typename Fin>
__device__ __forceinline__ void grid_fold(const float* blk_vals, int width, int bid, int nblk, ReduceScratch scr, float* s_tmp, int* s_flag,
                                          int tid, int nthreads, Sync sync, Fin fin) {
  const int ngroups = (nblk + kFoldGroup - 1) / kFoldGroup;
  const int grp = bid / kFoldGroup;
  const int grp_size = min(kFoldGroup, nblk - grp * kFoldGroup);
  float* level1 = scr.partials + static_cast<size_t>(nblk) * width;
  for (int i = tid; i < width; i += nthreads) scr.partials[static_cast<size_t>(bid) * width + i] = blk_vals[i];
  __threadfence();
  sync();
  if (tid == 0) *s_flag = (atomicAdd(scr.counter + 1 + grp, 1u) == static_cast<unsigned>(grp_size - 1));
  sync();
  if (!*s_flag) return;
  __threadfence();
  const float gsum = fold_rows(scr.partials + static_cast<size_t>(grp) * kFoldGroup * width, grp_size, width, s_tmp, tid, nthreads, sync);
  if (tid < width) level1[static_cast<size_t>(grp) * width + tid] = gsum;
  __threadfence();
  sync();
  if (tid == 0) {
    scr.counter[1 + grp] = 0u;
    *s_flag = (atomicAdd(scr.counter, 1u) == static_cast<unsigned>(ngroups - 1));
  }
  sync();
  if (!*s_flag) return;
  __threadfence();
  const float total = fold_rows(level1, ngroups, width, s_tmp, tid, nthreads, sync);
  if (tid < width) fin(tid, total);
  if (tid == 0) *scr.counter = 0u;
}

}  // namespace pdt
