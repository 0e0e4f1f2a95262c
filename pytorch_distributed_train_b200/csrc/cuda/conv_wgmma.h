// wgmma/TMA kernels (sm_90a): the tensor-core 5x5 convolution of the ConvNet's conv2 (16→32 channels).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "ops_kernels.h"

namespace pdt {

// True for the shapes the tensor-core convolution handles (the ConvNet's conv2: 16→32 channels).
bool conv_wgmma_supported(const ConvShape& s);

// y NHWC [B,H,W,32] = conv5x5(x NHWC [B,H,W,16], w [32,16,5,5]) + bias; stats and form as in launch_conv5x5_fwd.
// Fully TMA-fed: every filter tap's A-tile is one cp.async.bulk.tensor im2col load; one warpgroup issues the wgmma and
// runs the epilogue.
void launch_conv5x5_fwd_im2col(const float* x, const float* w, const float* bias, float* y, void* stats, ConvStats form, ConvShape s,
                               ReduceScratch scr, cudaStream_t st);
// dx NHWC [B,H,W,16] = conv_transpose(dy NHWC [B,H,W,32], w [32,16,5,5]), same kernel.
void launch_conv5x5_dgrad_im2col(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// dw [32,16,5,5], db [32] (nullable) from dy NHWC [B,H,W,32] and x NHWC [B,H,W,16]: persistent split-K over
// pixel tiles with MN-major operands (mma.sync), four register-resident accumulator tiles, deterministic fold of the per-CTA partials.
void launch_conv5x5_wgrad_mma(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st);

}  // namespace pdt
