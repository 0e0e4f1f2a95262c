// Host launchers for the sm_90a compute kernels (no torch types; raw pointers + stream).
// Activation layout between fused layers is NHWC (= torch channels_last), fp32.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

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

// Adam / AdamW with torch's single-tensor arithmetic.  `step` is the per-parameter fp32 step count on the device (torch's
// capturable layout): the launch uses step + 1 for the bias corrections and leaves step + 1 behind, so a replayed CUDA graph
// advances it.
struct AdamTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* m[kMax];     // exp_avg
  float* v[kMax];     // exp_avg_sq
  float* step[kMax];
  int n[kMax];
  int count;
};
struct AdamHyper {
  double lr, beta1, beta2;   // double, as torch's host-side bias corrections are
  float eps, weight_decay;
  int decoupled, maximize;   // decoupled: AdamW (p *= 1 - lr·wd); else Adam (g += wd·p)
  const float* lr_dev;       // optional device-resident learning rate (graph-capturable schedules)
};
// ticket: one zeroed counter word; every block takes a ticket after it has read its step, the last one advances all steps and
// resets the word to zero.
void launch_adam_multi(const AdamTensorList& tl, AdamHyper h, unsigned int* ticket, cudaStream_t st);

// Gradient-norm clipping (torch.nn.utils.clip_grad_norm_ with norm_type 2 or inf) as two launches per table set: the norm, then
// the scale.  A set of more than kMax tensors is split into tables launched back to back; every block of every table writes one
// partial (fp32 Σg² or max |g|), and the block of the last table that takes the last ticket folds all partials of the set in
// index order in fp64, so the norm is the same bit for bit from run to run.
struct GradTensorList {
  static constexpr int kMax = 48;
  float* g[kMax];
  int n[kMax];
  int count;
};
struct GradNormArgs {
  float* partials;       // one float per block of every table of the set
  int part_base;         // index of this table's first partial
  int part_total;        // partials of the whole set
  int last;              // this is the set's last table: its last block folds
  int norm_inf;          // 1: max |g|, 0: Euclidean norm
  float max_norm;
  float* out;            // [0] total norm, [1] clip coefficient min(max_norm / (norm + 1e-6), 1) (NaN propagates)
  unsigned int* ticket;  // one zeroed counter word; the last block resets it
};
int grad_multi_blocks_x(const GradTensorList& tl);   // blockIdx.x extent of a table's launches
void launch_grad_norm_multi(const GradTensorList& tl, GradNormArgs a, cudaStream_t st);
// g *= *coef for every tensor of the table
void launch_grad_scale_multi(const GradTensorList& tl, const float* coef, cudaStream_t st);

#ifdef __CUDACC__
// max that keeps a NaN (fmaxf drops it), as torch's inf-norm does
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || a > b) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || a > b) ? a : b; }
// torch's clip coefficient, op for op in fp32: reciprocal(norm + 1e-6) · max_norm, then clamp(max=1), which keeps a NaN
__device__ __forceinline__ float clip_coef(float norm, float max_norm) {
  const float c = (1.f / (norm + 1e-6f)) * max_norm;
  return c > 1.f ? 1.f : c;
}
#endif

}  // namespace pdt
