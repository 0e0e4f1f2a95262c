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

// Sum load(r, i) over rows r in [0, nrows) for every column i in [0, width); the total of column i is returned to the threads
// with tid < width.  Every one of the `nthreads` participating threads must call it.
template <typename Sync, typename Load>
__device__ __forceinline__ float fold_cols(int nrows, int width, float* s_tmp /* >= nthreads floats */, int tid, int nthreads, Sync sync,
                                           Load load) {
  int G = 1;
  while (G * 2 * width <= nthreads && G < 16) G *= 2;
  const int i = tid % width, g = tid / width;
  if (g < G) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int r = g;
    for (; r + 3 * G < nrows; r += 4 * G) {  // four independent loads in flight
      a0 += load(r, i);
      a1 += load(r + G, i);
      a2 += load(r + 2 * G, i);
      a3 += load(r + 3 * G, i);
    }
    for (; r < nrows; r += G) a0 += load(r, i);
    s_tmp[g * width + i] = (a0 + a1) + (a2 + a3);
  }
  sync();
  float tot = 0.f;
  if (tid < width)
    for (int k = 0; k < G; ++k) tot += s_tmp[k * width + tid];
  sync();
  return tot;
}

// Sum rows[0..nrows) of a row-major [nrows][width] matrix (written by other CTAs: read through L2).
template <typename Sync>
__device__ __forceinline__ float fold_rows(const float* rows, int nrows, int width, float* s_tmp /* >= nthreads floats */, int tid,
                                           int nthreads, Sync sync) {
  return fold_cols(nrows, width, s_tmp, tid, nthreads, sync,
                   [&](int r, int i) { return __ldcg(rows + static_cast<size_t>(r) * width + i); });
}

// Rows of [Σ (C) | M2 (C)], row r summarising cnt(r) elements per channel with M2 taken about the row's own mean, combined into
// the same pair for their union without cancellation (Chan, Golub & LeVeque):
//   Σ = Σ_r Σ_r,   M2 = Σ_r M2_r + Σ_r d_r² / cnt(r),   d_r = Σ_r − cnt(r)·mean,   mean = Σ / n,   n = Σ_r cnt(r),
// where Σy²/n − mean² in fp32 would lose the variance's digits in proportion to mean²/var.  Two passes over the rows, each in a
// fixed order: the sums, then the deviations d_r, whose sum also corrects Σ and the mean for the rounding of the first pass.
// Threads tid < C get channel tid's Σ, mean and M2.  s_tmp: >= nthreads + 2C floats.
template <typename Sync, typename Cnt>
__device__ __forceinline__ void fold_centred_rows(const float* rows, int nrows, int C, Cnt cnt, float n, float* s_tmp, int tid, int nthreads,
                                                  Sync sync, float* sum, float* mean, float* m2) {
  float* s_stat = s_tmp + nthreads;   // [mean (C) | Σ_r M2_r (C)]
  const float tot = fold_rows(rows, nrows, 2 * C, s_tmp, tid, nthreads, sync);
  if (tid < 2 * C) s_stat[tid] = tid < C ? tot / n : tot;
  sync();
  const float dev = fold_cols(nrows, 2 * C, s_tmp, tid, nthreads, sync, [&](int r, int i) {
    const int c = i < C ? i : i - C;
    const float k = cnt(r), d = fmaf(-k, s_stat[c], __ldcg(rows + static_cast<size_t>(r) * 2 * C + c));
    return i < C ? d : d * d / k;
  });
  if (tid >= C && tid < 2 * C) s_stat[tid] += dev;
  sync();
  if (tid < C) {
    *sum = tot + dev;
    *mean = s_stat[tid] + dev / n;
    *m2 = s_stat[C + tid];
  }
}

// The ticket tree.  fold(rows, nrows, first, span, out) combines `nrows` rows starting at row `first` of its level, each covering
// `span` contributors (level 1: its group's contributors, span 1; level 2: the group partials, span 16), and stores the result in
// out[0..width), or hands it to the caller's fin when out == nullptr (the last fold).
// blk_vals: this contributor's `width` partial values (visible to all participating threads).
// bid / nblk: linear id of this contributor and the number of contributors.
// scr.partials must hold (nblk + ceil(nblk/16)) * width floats; the fold region of scr.counter (ops_kernels.h: words
// [0, scr.fold_counters), which no fixed counter word shares) must hold 1 + ceil(nblk/16) zeroed uints.
// s_flag: one int of shared memory.
template <typename Sync, typename Fold>
__device__ __forceinline__ void grid_fold_tree(const float* blk_vals, int width, int bid, int nblk, ReduceScratch scr, int* s_flag, int tid,
                                               int nthreads, Sync sync, Fold fold) {
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
  fold(scr.partials + static_cast<size_t>(grp) * kFoldGroup * width, grp_size, grp * kFoldGroup, 1, level1 + static_cast<size_t>(grp) * width);
  __threadfence();
  sync();
  if (tid == 0) {
    scr.counter[1 + grp] = 0u;
    *s_flag = (atomicAdd(scr.counter, 1u) == static_cast<unsigned>(ngroups - 1));
  }
  sync();
  if (!*s_flag) return;
  __threadfence();
  fold(level1, ngroups, 0, kFoldGroup, static_cast<float*>(nullptr));
  if (tid == 0) *scr.counter = 0u;
}

// Column sums of the contributors' partials: fin(i, total) for every column i.  s_tmp: >= nthreads floats of shared memory.
template <typename Sync, typename Fin>
__device__ __forceinline__ void grid_fold(const float* blk_vals, int width, int bid, int nblk, ReduceScratch scr, float* s_tmp, int* s_flag,
                                          int tid, int nthreads, Sync sync, Fin fin) {
  grid_fold_tree(blk_vals, width, bid, nblk, scr, s_flag, tid, nthreads, sync, [&](const float* rows, int nrows, int, int, float* out) {
    const float tot = fold_rows(rows, nrows, width, s_tmp, tid, nthreads, sync);
    if (tid < width) {
      if (out) out[tid] = tot;
      else fin(tid, tot);
    }
  });
}

// The contributors' [Σ (C) | M2 (C)] partials (fold_centred_rows), contributor b covering min(per, total − b·per) elements per
// channel: fin(c, mean, M2) for every channel c.  s_tmp: >= nthreads + 2C floats of shared memory.
template <typename Sync, typename Fin>
__device__ __forceinline__ void grid_fold_centred(const float* blk_vals, int C, int per, int total, int bid, int nblk, ReduceScratch scr,
                                                  float* s_tmp, int* s_flag, int tid, int nthreads, Sync sync, Fin fin) {
  grid_fold_tree(blk_vals, 2 * C, bid, nblk, scr, s_flag, tid, nthreads, sync, [&](const float* rows, int nrows, int first, int span, float* out) {
    const int row_elems = per * span;   // elements per channel that one row of this level covers (the last row: the rest)
    auto cnt = [&](int r) { return static_cast<float>(min(row_elems, total - (first + r) * row_elems)); };
    const float n = static_cast<float>(min(nrows * row_elems, total - first * row_elems));
    float sum, mean, m2;
    fold_centred_rows(rows, nrows, C, cnt, n, s_tmp, tid, nthreads, sync, &sum, &mean, &m2);
    if (tid < C) {
      if (out) {
        out[tid] = sum;
        out[C + tid] = m2;
      } else {
        fin(tid, mean, m2);
      }
    }
  });
}

}  // namespace pdt
