// wgmma/TMA kernels (sm_90a): TF32 GEMM self-test and the implicit-GEMM 5x5 convolution.  The "tcgen05" names
// date from the project's first (Blackwell) version.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "grid_sync.cuh"
#include "ops_kernels.h"

namespace pdt {

// True for the shapes the tensor-core convolution handles (the ConvNet's conv2: 16→32 channels).
bool conv_tcgen05_supported(const ConvShape& s);

// y NHWC [B,H,W,32] = conv5x5(x NHWC [B,H,W,16], w [32,16,5,5]) + bias; stats as in launch_conv5x5_fwd.
void launch_conv5x5_fwd_tcgen05(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s,
                                ReduceScratch scr, cudaStream_t st);
// dx NHWC [B,H,W,16] = conv_transpose(dy NHWC [B,H,W,32], w [32,16,5,5])
void launch_conv5x5_dgrad_tcgen05(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// Same contracts, fully TMA-fed: every filter tap's A-tile is one cp.async.bulk.tensor im2col load
// (no producer warps); one warpgroup issues the wgmma and runs the epilogue.
void launch_conv5x5_fwd_tma(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s, ReduceScratch scr,
                            cudaStream_t st);
void launch_conv5x5_dgrad_tma(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// Opt-in (impl == "win"), not covered by the test suite: one tiled TMA load of the haloed patch per tile, the 25 taps
// as row-shifted wgmma descriptors into that single buffer (index math: tools/emulate_window_conv.py).
void launch_conv5x5_fwd_win(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s, ReduceScratch scr,
                            cudaStream_t st);
void launch_conv5x5_dgrad_win(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// dw [32,16,5,5], db [32] (nullable) from dy NHWC [B,H,W,32] and x NHWC [B,H,W,16]: persistent split-K over
// pixel tiles with MN-major operands (mma.sync), four register-resident accumulator tiles, deterministic fold of the per-CTA partials.
void launch_conv5x5_wgrad_tcgen05(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st);

// Window formulation for zero-haloed 18×18 frames (cooperative fused layers): dy_pad [B,18,18,32], x_pad [B,18,18,16], dysum [B,32]
// (per-image Σdy rows, folded into db).  All operands arrive by TMA: no im2col gather.
// With a grid-barrier descriptor the per-CTA partials are folded inside the same (cooperative) launch; without one a second
// kernel folds them.
// Tensor maps of the window weight gradient: tm_x = overlapping-row view of the x frame [B,18,18,16] (row pitch 64 B, row length
// 128 B, box 64 rows), tm_dy = the dy frame [B,18,18,32] as rows of 32 floats (box 128 rows); both SWIZZLE_128B.
void make_wgrad_win_tmaps(const float* x_pad, const float* dy_pad, int B, CUtensorMap* tm_x, CUtensorMap* tm_dy);
void launch_conv5x5_wgrad_win(const float* dy_pad, const float* x_pad, const float* dysum, float* dw, float* db, int B, ReduceScratch scr,
                              cudaStream_t st, GridSync gs = GridSync{nullptr, nullptr});

// D[M,N] = A[M,K] · B[N,K]^T, fp32 in/out, TF32 tensor-core math (K % 4 == 0, N % 16 == 0, N <= 256).
void launch_gemm_tf32_tcgen05(const float* a, const float* b, float* d, int M, int N, int K, cudaStream_t st);

// Hardware probe (tools/exp_rowshift.py): D[128,32] = A[shift:shift+128, :] · B[32, :]^T with A [256][rowb/4] loaded
// once into swizzled smem and the wgmma descriptor started `shift` rows in; mode 1 sets the descriptor base offset.
void launch_umma_rowshift_probe(const float* a, const float* b, float* d, int rowb, int shift, int mode, cudaStream_t st);

}  // namespace pdt
