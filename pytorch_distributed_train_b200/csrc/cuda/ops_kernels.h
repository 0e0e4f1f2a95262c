// Host launchers for the sm_90a compute kernels (no torch types; raw pointers + stream).
// Activation layout between fused layers is NHWC (= torch channels_last), fp32.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "symm_device.h"  // count_kernel_launch()

namespace pdt {

struct ConvShape {
  int B, H, W, Cin, Cout;  // 5x5, stride 1, pad 2 ("same")
};

// Scratch for deterministic cross-CTA reductions: partials[max_blocks][width] + a ticket counter.
struct ReduceScratch {
  float* partials;
  unsigned int* counter;  // `counters` ticket words; zero before first use, kernels leave them at zero
  int capacity_floats;
  int counters;
};

// ---- SIMT direct convolution (conv1; conv2 fallback + oracle for the tensor-core kernels) -------------
// x NHWC [B,H,W,Cin], w torch layout [Cout,Cin,5,5], bias [Cout] (nullable) → y NHWC [B,H,W,Cout].
// stats (nullable): [2*Cout+1] = per-channel Σy, Σy², then the element count per channel.
void launch_conv5x5_fwd(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s,
                        ReduceScratch scr, cudaStream_t st);
// dx NHWC [B,H,W,Cin] = conv_transpose(dy NHWC [B,H,W,Cout], w)
void launch_conv5x5_dgrad(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);
// dw [Cout,Cin,5,5], db [Cout] (nullable) from dy NHWC and x NHWC.
void launch_conv5x5_wgrad(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st);

// ---- BatchNorm(train) + ReLU + MaxPool2x2, fused -----------------------------------------------------
// y NHWC [B,H,W,C]; stats [2C+1] (Σ, Σ², n — already all-reduced when SyncBN is on).
// out: pooled [B,H/2,W/2,C] NHWC, or NCHW when out_nchw. saved [2C] ← mean, invstd.
// running_mean/var (nullable) updated with `momentum` (unbiased var), nbt (nullable, int64) += 1.
void launch_bn_relu_pool_fwd(const float* y, const float* stats, const float* gamma, const float* beta, float* out, float* saved,
                             float* running_mean, float* running_var, long long* nbt, float momentum, float eps, int B, int H,
                             int W, int C, bool out_nchw, cudaStream_t st);
// Pass 1 of backward: sums [2C] ← Σdz, Σdz·x̂ over the *local* batch (dz = grad at the BN output,
// i.e. pooled grad routed to the arg-max position and masked by ReLU).  Also dγ = Σdz·x̂, dβ = Σdz.
void launch_bn_relu_pool_bwd_reduce(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta,
                                    float* sums, float* dgamma, float* dbeta, int B, int H, int W, int C, bool dout_nchw,
                                    ReduceScratch scr, cudaStream_t st);
// Pass 2: dy NHWC [B,H,W,C] from the (possibly all-reduced) sums and the global count n.
void launch_bn_relu_pool_bwd_apply(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta,
                                   const float* sums, const float* count, float* dy, int B, int H, int W, int C, bool dout_nchw,
                                   cudaStream_t st);

// ---- generic NCHW BatchNorm pieces (SyncBatchNorm on arbitrary models) ---------------------------------
void launch_bn_stats_nchw(const float* x, float* stats, int N, int C, int HW, ReduceScratch scr, cudaStream_t st);
// same sums accumulated and returned in fp64 (SyncBatchNorm forward: var = E[x²] − μ² needs the headroom)
// fp64 [2C+1(+pad)] all-reduced statistics → mean / invstd / count (fp32) + running-stat update (nullable), one launch
void launch_bn_finalize(const double* stats, int C, double eps, float momentum, float* mean, float* invstd, float* count_out,
                        float* running_mean, float* running_var, cudaStream_t st);
void launch_bn_stats_nchw_f64(const float* x, double* stats, int N, int C, int HW, ReduceScratch scr, cudaStream_t st);
void launch_bn_apply_nchw(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta, float* out,
                          int N, int C, int HW, cudaStream_t st);
void launch_bn_bwd_reduce_nchw(const float* dy, const float* x, const float* mean, const float* invstd, float* red4c, int N, int C,
                               int HW, ReduceScratch scr, cudaStream_t st);
void launch_bn_bwd_apply_nchw(const float* dy, const float* x, const float* mean, const float* invstd, const float* gamma,
                              const float* mean_dy, const float* mean_dy_xmu, float* dx, int N, int C, int HW, cudaStream_t st);

// ---- classifier head -----------------------------------------------------------------------------------
// out[B,N] = x[B,K] · w[N,K]^T + b
void launch_linear_fwd(const float* x, const float* w, const float* b, float* out, int B, int K, int N, cudaStream_t st);
// dx[B,K] = dout·w (nullable); dw[N,K] = dout^T·x; db[N] = Σ dout
void launch_linear_bwd(const float* dout, const float* x, const float* w, float* dx, float* dw, float* db, int B, int K, int N,
                       cudaStream_t st);
// loss (scalar, mean over B) and probs[B,C] (softmax, kept for backward)
// emit_grad: `probs` receives (softmax − onehot)/B instead (the backward of a mean loss with unit incoming gradient)
void launch_cross_entropy_fwd(const float* logits, const long long* target, float* loss, float* probs, int B, int C, cudaStream_t st,
                              bool emit_grad = false);
// dlogits = (probs - onehot) * (*dloss) / B
void launch_cross_entropy_bwd(const float* probs, const long long* target, const float* dloss, float* dlogits, int B, int C,
                              cudaStream_t st);

// ---- optimizer -------------------------------------------------------------------------------------------
struct SgdTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* m[kMax];
  int n[kMax];
  int count;
};
struct SgdHyper {
  float lr, momentum, dampening, weight_decay;
  int nesterov, maximize, first_step;
  const float* lr_dev;  // optional device-resident learning rate (graph-capturable schedules)
};
void launch_sgd_multi(const SgdTensorList& tl, SgdHyper h, cudaStream_t st);

}  // namespace pdt
