// wgmma/TMA kernels (sm_90a): TF32 GEMM self-test and the implicit-GEMM 5x5 convolution.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "ops_kernels.h"

namespace pdt {

// True for the shapes the tensor-core convolution handles (the ConvNet's conv2: 16→32 channels).
bool conv_wgmma_supported(const ConvShape& s);

// y NHWC [B,H,W,32] = conv5x5(x NHWC [B,H,W,16], w [32,16,5,5]) + bias; stats as in launch_conv5x5_fwd.
// cp.async-gather kernel: four producer warps gather the im2col A-tile into swizzled smem.
void launch_conv5x5_fwd_gather(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s,
                               ReduceScratch scr, cudaStream_t st);
// dx NHWC [B,H,W,16] = conv_transpose(dy NHWC [B,H,W,32], w [32,16,5,5])
void launch_conv5x5_dgrad_gather(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// Same contracts, fully TMA-fed: every filter tap's A-tile is one cp.async.bulk.tensor im2col load
// (no producer warps); one warpgroup issues the wgmma and runs the epilogue.
void launch_conv5x5_fwd_im2col(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s, ReduceScratch scr,
                               cudaStream_t st);
void launch_conv5x5_dgrad_im2col(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// dw [32,16,5,5], db [32] (nullable) from dy NHWC [B,H,W,32] and x NHWC [B,H,W,16]: persistent split-K over
// pixel tiles with MN-major operands (mma.sync), four register-resident accumulator tiles, deterministic fold of the per-CTA partials.
void launch_conv5x5_wgrad_mma(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st);

// D[M,N] = A[M,K] · B[N,K]^T, fp32 in/out, TF32 tensor-core math (K % 4 == 0, N % 16 == 0, N <= 256).
void launch_gemm_tf32_wgmma(const float* a, const float* b, float* d, int M, int N, int K, cudaStream_t st);

}  // namespace pdt
