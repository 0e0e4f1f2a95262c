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

// Scratch for deterministic cross-CTA reductions: partials[max_blocks][width] + ticket counters.
struct ReduceScratch {
  float* partials;
  unsigned int* counter;  // the per-device counter words laid out below; zero before first use, kernels leave them at zero
  int capacity_floats;
  int fold_counters;      // words of the fold region, counter[0, fold_counters)
};

// Per-device reduction scratch: kScratchFloats partial floats and kCounterWords counter words.  The counter words are:
//   [0, kFoldCounterWords)  the fold region: grid_fold's group counter [0] and one ticket [1 + g] per group of 16 contributors,
//                           or the single ticket [0] of a last-block fold.  Every per-op fold launch checks that its
//                           1 + ceil(blocks / 16) words fit; the region is large enough that the partials run out first.
//   kGridEpochWord          epoch of the cooperative kernels' grid barrier (GridBar): only ever increases, never reset
//   kGridArrivalWord        arrival count of that barrier
//   kCeCounterWord          arrival counter of the whole-forward kernel's cross-entropy mean
//   kAdamTicketWord         step hand-over ticket of adam_multi, nadam_multi, radam_multi, rmsprop_multi, adagrad_multi, adamax_multi,
//                           adadelta_multi, asgd_multi and rprop_multi
//   kClipTicketWord         fold ticket of grad_norm_clip
//   kAvgTicketWord          n_averaged hand-over ticket of avg_multi
// Each fixed word sits in a 32-byte sector of its own.  A ticket word serves one launch set at a time: the sets that use it are
// ordered by the device's compute stream, so no two of them (two adam_multi or two avg_multi sets) may run concurrently on
// different streams of one device.
constexpr int kScratchFloats = 4 << 20;                   // 16 MiB
constexpr int kFoldCounterWords = kScratchFloats / 64;    // a fold of width ≥ 4 fills the partials before it runs out of tickets
constexpr int kGridEpochWord = kFoldCounterWords;
constexpr int kGridArrivalWord = kFoldCounterWords + 8;
constexpr int kCeCounterWord = kFoldCounterWords + 16;
constexpr int kAdamTicketWord = kFoldCounterWords + 24;
constexpr int kClipTicketWord = kFoldCounterWords + 32;
constexpr int kAvgTicketWord = kFoldCounterWords + 40;
constexpr int kCounterWords = kFoldCounterWords + 48;

// ---- SIMT direct convolution (conv1: 1→16 channels; conv2 runs on the tensor-core kernels of conv_wgmma.h) ----
// x NHWC [B,H,W,Cin], w torch layout [Cout,Cin,5,5], bias [Cout] (nullable) → y NHWC [B,H,W,Cout].
// stats (nullable) in the form `form`.  The centred forms fold the mean and M2 (the sum of squared deviations from the mean)
// without cancellation (grid_fold.cuh), so they keep the variance's digits when |mean| ≫ std.
enum ConvStats : int {
  kConvSums = 0,      // fp32 [2C+1] Σy, Σy², then the element count per channel
  kConvCentred = 1,   // fp32 [2C+1] mean, M2, count
  kConvSums64 = 2,    // fp64 [2C+2] Σy = n·mean, Σy² = M2 + n·mean², count, 0: formed from the centred fold, summable across GPUs
                      // (SyncBatchNorm)
};
void launch_conv5x5_fwd(const float* x, const float* w, const float* bias, float* y, void* stats, ConvStats form, ConvShape s,
                        ReduceScratch scr, cudaStream_t st);
// dw [Cout,Cin,5,5], db [Cout] (nullable) from dy NHWC and x NHWC.
void launch_conv5x5_wgrad(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st);
// dx NHWC [B,H,W,1] from dy NHWC [B,H,W,16] and w [16,1,5,5] (conv1's input gradient): one thread per pixel, fp32 fmaf in a
// fixed order, so the result is deterministic at any B.
void launch_conv5x5_dgrad(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st);

// ---- BatchNorm(train) + ReLU + MaxPool2x2, fused -----------------------------------------------------
// Every bn_relu_pool launcher takes C ∈ {4, 8, 16, 32, 64} and even H, W.
// y NHWC [B,H,W,C]; stats in one of the BnStats forms below.
// out: pooled [B,H/2,W/2,C] NHWC, or NCHW when out_nchw. saved [2C] ← mean, invstd; kBnSums64: saved [2C+1], the count last.
// running_mean/var (nullable) updated with `momentum` (unbiased var), nbt (nullable, int64) += 1.
enum BnStats : int {
  kBnSums = 0,      // fp32 [2C+1] Σ, Σ², n (conv5x5_fwd kConvSums; Σ²/n − mean² loses digits when |mean| ≫ std)
  kBnCentred = 1,   // fp32 [2C+1] mean, M2, n (conv5x5_fwd kConvCentred: one GPU)
  kBnMeanVar = 2,   // fp32 [2C] mean, variance (eval mode: the running statistics, used as they are)
  kBnSums64 = 3,    // fp64 [2C+2] Σ, Σ², n, pad (conv5x5_fwd kConvSums64, all-reduced by SyncBatchNorm): mean and variance in fp64
};
void launch_bn_relu_pool_fwd(const float* y, const void* stats, const float* gamma, const float* beta, float* out, float* saved,
                             float* running_mean, float* running_var, long long* nbt, float momentum, float eps, int B, int H,
                             int W, int C, bool out_nchw, BnStats form, cudaStream_t st);
// Pass 1 of backward: sums [2C] ← Σdz, Σdz·x̂ over the *local* batch (dz = grad at the BN output,
// i.e. pooled grad routed to the arg-max position and masked by ReLU).  Also dγ = Σdz·x̂, dβ = Σdz.
void launch_bn_relu_pool_bwd_reduce(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta,
                                    float* sums, float* dgamma, float* dbeta, int B, int H, int W, int C, bool dout_nchw,
                                    ReduceScratch scr, cudaStream_t st);
// Pass 2: dy NHWC [B,H,W,C] from the (possibly all-reduced) sums and the global count n.  mean_var: the forward ran on kBnMeanVar
// statistics (eval), constants of the graph: dy = γ·invstd·dz at the arg-max and 0 elsewhere, and sums and count are not read.
void launch_bn_relu_pool_bwd_apply(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta,
                                   const float* sums, const float* count, float* dy, int B, int H, int W, int C, bool dout_nchw,
                                   bool mean_var, cudaStream_t st);

// ---- generic NCHW BatchNorm pieces (SyncBatchNorm on arbitrary models) ---------------------------------
// stats [2C+1] ← per-channel Σx, Σx², then the element count per channel, accumulated and returned in fp64 (SyncBatchNorm
// forward: var = E[x²] − μ² needs the headroom)
void launch_bn_stats_nchw_f64(const float* x, double* stats, int N, int C, int HW, ReduceScratch scr, cudaStream_t st);
// fp64 [2C+1(+pad)] all-reduced statistics → mean / invstd / count (fp32) + running-stat update (nullable), one launch
void launch_bn_finalize(const double* stats, int C, double eps, float momentum, float* mean, float* invstd, float* count_out,
                        float* running_mean, float* running_var, cudaStream_t st);
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
// Cross-entropy with torch's ignore_index semantics: a row whose target is outside [0, C) (ignore_index) adds nothing, the mean is
// over the n rows whose target is in [0, C), and with n = 0 the loss is NaN and every gradient zero.
// loss (scalar, mean over the n rows) and probs[B,C] (softmax, kept for backward)
// emit_grad: `probs` receives (softmax − onehot)/n instead, zero in ignored rows (the backward of a mean loss with unit incoming
// gradient)
void launch_cross_entropy_fwd(const float* logits, const long long* target, float* loss, float* probs, int B, int C, cudaStream_t st,
                              bool emit_grad = false);
// dlogits = (probs - onehot) * (*dloss) / n, zero in ignored rows
void launch_cross_entropy_bwd(const float* probs, const long long* target, const float* dloss, float* dlogits, int B, int C,
                              cudaStream_t st);

// torch's other cross-entropy options.  A row is counted when its target t lies in [0, C) and is not ignore_index; with class
// weights w (1 without), W = Σ_c w_c and ε = smoothing, a counted row adds
//   (1-ε)·w_t·(lse − l_t) + (ε/C)·Σ_c w_c·(lse − l_c)        with gradient   [(1-ε)·w_t·(p_c − [c=t]) + (ε/C)·(W·p_c − w_c)] / D
// and the loss is Σ terms / D: D = Σ_{counted} w_t for the mean (0 ⇒ NaN), 1 for the sum.  D and W are summed in a fixed order.
struct CeSpec {
  const float* weight = nullptr;   // [C] or null
  float smoothing = 0.f;
  long long ignore_index = -100;
  bool sum = false;                // reduction 'sum' (else 'mean')
  // the default spec is the plain mean above, which runs the kernels without the options
  bool is_default(int C) const { return weight == nullptr && smoothing == 0.f && !sum && (ignore_index < 0 || ignore_index >= C); }
};
void launch_cross_entropy_fwd(const float* logits, const long long* target, float* loss, float* probs, int B, int C, cudaStream_t st,
                              bool emit_grad, const CeSpec& spec);
void launch_cross_entropy_bwd(const float* probs, const long long* target, const float* dloss, float* dlogits, int B, int C,
                              cudaStream_t st, const CeSpec& spec);
// Class-probability targets q [B, C] (torch's floating-point target).  With q' = q·(1−ε) + ε/C, a_c = w_c·q'_c and S = Σ_c a_c,
// a row adds
//   Σ_c a_c·(lse − l_c)        with gradient   (p_c·S − a_c) / D
// and the loss is Σ terms / D: D = B for the mean whatever the weights (B = 0 ⇒ NaN), 1 for the sum.  Entries are not validated
// (negative ones, rows that do not sum to one), and spec.ignore_index plays no part: torch refuses any but −100 with such targets.
// One thread per row sums S in class order, and the forward's batch sum is in a fixed order.
void launch_cross_entropy_fwd_soft(const float* logits, const float* q, float* loss, float* probs, int B, int C, cudaStream_t st,
                                   bool emit_grad, const CeSpec& spec);
void launch_cross_entropy_bwd_soft(const float* probs, const float* q, const float* dloss, float* dlogits, int B, int C, cudaStream_t st,
                                   const CeSpec& spec);
// Evaluation metrics of logits[0:rows, C] (the first `rows` rows of the batch; the rest take no part), added to the fp64 acc[4] by
// one launch of the forward kernel that writes no loss or softmax:
//   acc[0] += Σ loss terms (the sum before the division by D)   acc[1] += D = Σ_{counted} w_t, whatever spec.sum says
//   acc[2] += counted rows whose argmax is the target             acc[3] += counted rows
// argmax is torch.argmax's: the first maximal index, a NaN counting as the maximum.  Plain adds, one block, stream-ordered: the
// totals are reproducible bit for bit.
void launch_cross_entropy_eval(const float* logits, const long long* target, double* acc, int rows, int C, cudaStream_t st,
                               const CeSpec& spec);

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
// AMSGrad (torch's amsgrad=True): the same update with the running maximum vmax = max(vmax, exp_avg_sq) (a NaN in either stays,
// as torch.maximum's) in the denominator.
struct AmsgradTensorList : AdamTensorList {
  float* vmax[kMax];  // max_exp_avg_sq
};
void launch_adam_multi(const AmsgradTensorList& tl, AdamHyper h, unsigned int* ticket, cudaStream_t st);

// NAdam with torch's single-tensor arithmetic (g' = ±g + wd·p, or AdamW's p *= 1 − lr·wd with decoupled): with t = step + 1,
//   μ_t = β1·(1 − ½·0.96^(t·ψ)), μ_{t+1} likewise (double);  Π_t = fp32(Π·fp32(μ_t)) (torch's fp32 mu_product *= μ_t)
//   m = lerp(m, g', 1 − β1);  v = β2·v + (1 − β2)·g'²;  d = sqrt(v / bc2) + eps
//   p −= (c_g·g' + c_m·m) / d,  c_g = lr·(1 − μ_t)/(1 − Π_t),  c_m = lr·μ_{t+1}/(1 − Π_t·μ_{t+1})   (c_g, c_m in double, rounded
//   to fp32; torch's two addcdiv terms over one division)
// The launch leaves t and Π_t behind (adam_multi's ticket hand-over), so a replayed CUDA graph advances both.
struct NadamTensorList : AdamTensorList {
  float* mu_product[kMax];
};
struct NadamHyper : AdamHyper {
  double momentum_decay;   // ψ
};
void launch_nadam_multi(const NadamTensorList& tl, NadamHyper h, unsigned int* ticket, cudaStream_t st);

// RAdam with torch's single-tensor arithmetic (weight decay as in NAdam): with t = step + 1, bc1 = 1 − β1^t, bc2 = 1 − β2^t,
// ρ∞ = 2/(1 − β2) − 1 and ρ_t = ρ∞ − 2t·β2^t / bc2 (double), m and v as in Adam, then
//   ρ_t > 5:  p −= lr·rect·sqrt(bc2)/bc1 · m / (sqrt(v) + eps),  rect = sqrt((ρ_t − 4)(ρ_t − 2)ρ∞ / ((ρ∞ − 4)(ρ∞ − 2)ρ_t))
//   else:     p −= lr/bc1 · m
// The branch is taken per tensor on the device from its step count; the launch leaves t behind (adam_multi's ticket hand-over).
void launch_radam_multi(const AdamTensorList& tl, AdamHyper h, unsigned int* ticket, cudaStream_t st);

// RMSprop with torch's single-tensor arithmetic (g' = ±g + wd·p):
//   sq = α·sq + (1 − α)·g'²;  centered: ga = lerp(ga, g', 1 − α), avg = sqrt(sq − ga²) + eps;  else avg = sqrt(sq) + eps
//   momentum: buf = momentum·buf + g'/avg, p −= lr·buf;  else p −= lr·g'/avg
// `step` does not enter the arithmetic; it is advanced as torch advances it, with adam_multi's ticket hand-over.
struct RmspropTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* sq[kMax];    // square_avg
  float* buf[kMax];   // momentum_buffer (nullptr: momentum == 0)
  float* ga[kMax];    // grad_avg (nullptr: not centered)
  float* step[kMax];
  int n[kMax];
  int count;
};
struct RmspropHyper {
  float lr, alpha, one_minus_alpha, eps, weight_decay, momentum;   // 1 − α formed in double, as torch's Python scalar is
  int maximize;
  const float* lr_dev;   // optional device-resident learning rate (graph-capturable schedules)
};
void launch_rmsprop_multi(const RmspropTensorList& tl, RmspropHyper h, unsigned int* ticket, cudaStream_t st);

// Adagrad with torch's single-tensor arithmetic (g' = ±g + wd·p): with s the step before this update,
//   clr = lr / (1 + s·lr_decay) (double, rounded to fp32 once per tensor);  sum += g'²;  p −= clr·g' / (sqrt(sum) + eps)
// The launch leaves step + 1 behind (adam_multi's ticket hand-over).
struct AdagradTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* sum[kMax];
  float* step[kMax];
  int n[kMax];
  int count;
};
struct AdagradHyper {
  double lr, lr_decay;   // double, as torch's host-side clr is
  float eps, weight_decay;
  int maximize;
  const float* lr_dev;   // optional device-resident learning rate (graph-capturable schedules)
};
void launch_adagrad_multi(const AdagradTensorList& tl, AdagradHyper h, unsigned int* ticket, cudaStream_t st);

// Adamax with torch's single-tensor arithmetic (optim_update.cuh: adamax_update; AdamHyper's decoupled is unused): with t = step + 1,
// clr = lr / (1 − β1^t) in double, rounded to fp32 once per tensor.  The tables are Adam's, v holding exp_inf; the launch leaves t
// behind (adam_multi's ticket hand-over).
void launch_adamax_multi(const AdamTensorList& tl, AdamHyper h, unsigned int* ticket, cudaStream_t st);

// Adadelta with torch's single-tensor arithmetic (optim_update.cuh: adadelta_update).  `step` does not enter the arithmetic; it is
// advanced with adam_multi's ticket hand-over.
struct AdadeltaTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* sq[kMax];    // square_avg
  float* acc[kMax];   // acc_delta
  float* step[kMax];
  int n[kMax];
  int count;
};
struct AdadeltaHyper {
  float lr, rho, one_minus_rho, eps, weight_decay;   // 1 − ρ formed in double, as torch's Python scalar is
  int maximize;
  const float* lr_dev;   // optional device-resident learning rate (graph-capturable schedules)
};
void launch_adadelta_multi(const AdadeltaTensorList& tl, AdadeltaHyper h, unsigned int* ticket, cudaStream_t st);

// ASGD with torch's single-tensor, non-capturable arithmetic (optim_update.cuh: asgd_update), from each tensor's fp32 eta and mu on
// the device.  The block that takes the last ticket stores, with t = step + 1, step = t, eta = fp32(lr / (1 + λ·lr·t)^α) and
// mu = fp32(1 / max(1, t − t0)) (double, from the device lr when there is one), so a replayed graph follows torch's schedules.
struct AsgdTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* ax[kMax];
  float* step[kMax];
  float* eta[kMax];
  float* mu[kMax];
  int n[kMax];
  int count;
};
struct AsgdHyper {
  double lr, lambd, alpha, t0;   // double, as torch's host-side eta and mu are
  float weight_decay;
  int maximize;
  const float* lr_dev;   // optional device-resident learning rate (graph-capturable schedules)
};
void launch_asgd_multi(const AsgdTensorList& tl, AsgdHyper h, unsigned int* ticket, cudaStream_t st);

// Rprop with torch's single-tensor arithmetic (optim_update.cuh: rprop_update); no learning rate (step_size starts at lr) and no
// weight decay.  `step` is advanced with adam_multi's ticket hand-over.
struct RpropTensorList {
  static constexpr int kMax = 48;
  float* p[kMax];
  const float* g[kMax];
  float* prev[kMax];
  float* step_size[kMax];
  float* step[kMax];
  int n[kMax];
  int count;
};
struct RpropHyper {
  float etaminus, etaplus, step_min, step_max;
  int maximize;
};
void launch_rprop_multi(const RpropTensorList& tl, RpropHyper h, unsigned int* ticket, cudaStream_t st);

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

// Weight averaging: torch.optim.swa_utils.AveragedModel.update_parameters with the EMA or SWA multi_avg_fn, one table of
// (averaged, model) tensor pairs per launch.  n = *n_averaged (int64 on the device).  An averaged pair takes the model's value
// when n == 0 and otherwise, in fp32, torch's CUDA lerp(avg, p, w) with w = fp32(1 − decay) (EMA) or 1 / fp32(n + 1) (SWA); an
// int64 pair follows torch's EMA branch for integers, fp32(avg)·fp32(decay) + fp32(p)·w truncated (torch's SWA raises there, so no
// caller sends one).  A copied pair (the buffers when use_buffers=False) takes the model's value on every update.
struct AvgTensorList {
  static constexpr int kMax = 48;
  enum Mode : unsigned char { kAvgF32, kCopyF32, kAvgI64, kCopyI64 };
  void* avg[kMax];
  const void* src[kMax];
  int n[kMax];
  unsigned char mode[kMax];
  int count;
};
struct AvgArgs {
  long long* n_averaged;   // read by every block of every table; the last table's last block stores n + 1
  int swa;                 // 1: SWA weight, 0: EMA
  float decay;             // EMA: fp32(decay), the integer branch's factor
  float weight;            // EMA: fp32(1 − decay)
  int last;                // this is the set's last table
  unsigned int* ticket;    // one zeroed counter word; the block that takes the last ticket resets it
};
void launch_avg_multi(const AvgTensorList& tl, AvgArgs a, cudaStream_t st);

// ---- data augmentation ---------------------------------------------------------------------------------
// The Philox seed and offset of one launch: torch's PhiloxCudaState without torch's types.  Under CUDA-graph capture the seed and
// the base offset are read from device memory (seed_ptr, offset_ptr + offset), which the graph's replay refreshes, so every replay
// draws new values; otherwise seed and offset are used as they are.
struct PhiloxSeed {
  unsigned long long seed, offset;
  const long long* seed_ptr;     // null unless captured
  const long long* offset_ptr;
};
// Every parameter is drawn as U[from, from + range) in fp32, torch's uniform_; a range of 0 gives `from` (1 for an absent scale,
// 0 for the others).  fill: the value of pixels whose source lies outside the image.
struct AffineSpec {
  float angle_from, angle_range;
  float tx_from, tx_range, ty_from, ty_range;   // before the rounding to whole pixels
  float scale_from, scale_range;
  float shear_x_from, shear_x_range, shear_y_from, shear_y_range;
  float fill;
  int bilinear;   // 0: nearest
};
// Philox values each image consumes (two curand_uniform4 from subsequence b): the generator's offset increment per launch
constexpr int kAffineOffsetIncrement = 8;
// torchvision's RandomAffine applied to each image of x [B, C, H, W] (fp32 contiguous NCHW) with its own parameters, into y of the
// same shape.  Image b draws (angle, tx, ty, scale, shear_x, shear_y) from Philox subsequence b, tx and ty rounded half to even,
// and stores them in params[b, 0:6] (fp32, nullable).  The inverse matrix is torchvision's _get_inverse_affine_matrix with
// center (0, 0) in double; output pixel (i, j) samples the source at
//   sx = m0·(j − cw) + m1·(i − ch) + m2 + cw,   sy = m3·(j − cw) + m4·(i − ch) + m5 + ch,   cw = (W − 1)/2, ch = (H − 1)/2
// (double): nearest rounds half to even and takes `fill` outside the image; bilinear reads 0 outside and returns
// (v − fill)·mask + fill, mask being the bilinear weight of the in-bounds taps.  One launch (none when B = 0).
void launch_random_affine(const float* x, float* y, float* params, int B, int C, int H, int W, const AffineSpec& s, PhiloxSeed rng,
                          cudaStream_t st);
// The blur weights and scales of one elastic launch.  weights (device, fp32): for dx, the k[0] x weights (kernel size k[0], sigma[0])
// then its k[0] y weights (k[0], sigma[1]); then the same for dy with k[1]; k[c] = 0: plane c is not blurred.
struct ElasticSpec {
  const float* weights;
  int k[2];
  float alpha_x, alpha_y;   // fp32(alpha[0]), fp32(alpha[1])
  float fill;
  int bilinear;   // 0: nearest
};
// Philox values each subsequence of an elastic launch consumes (one curand_uniform4): the generator's offset increment per launch
constexpr int kElasticOffsetIncrement = 4;
// Shared memory of one elastic CTA: the dx and dy noise planes and one scratch plane, fp32.
size_t elastic_smem_bytes(int H, int W);
// Throws std::invalid_argument (naming the limit) unless an H×W image's planes fit the current device's opt-in shared memory.
void check_elastic_size(int H, int W);
// torchvision's v2.ElasticTransform applied to each image of x [B, C, H, W] (fp32 contiguous NCHW) with its own field, into y of
// the same shape.  Image b draws dx0, dy0 ~ U[-1, 1) over H×W (torch.rand·2 − 1; Philox layout in augment.cu) and stores them in
// noise[b, 0:2] (fp32 [B, 2, H, W], nullable).  Plane c with k[c] > 0 is blurred separably in fp32 with reflect indexing (x pass,
// then y pass); then dx = fl(fl(blurred_dx · alpha_x) / W), dy = fl(fl(blurred_dy · alpha_y) / H), and output pixel (i, j)
// samples the source at (j + dx·W/2, i + dy·H/2) in double with random_affine's sampling (nearest: ties to even, `fill` outside;
// bilinear: (v − fill)·mask + fill).  Every channel shares the image's field.  One launch of B CTAs (none when B = 0).
void launch_elastic(const float* x, float* y, float* noise, int B, int C, int H, int W, const ElasticSpec& s, PhiloxSeed rng,
                    cudaStream_t st);
// Attempts each Gamma draw of mix_batch_kernel may make before it gives up (Marsaglia–Tsang rejects at most 4.9% of attempts for a
// shape ≥ 1, so a draw reaches the cap with probability below 0.049^16 ≈ 1e-21)
constexpr int kGammaMaxAttempts = 16;
// Philox values one mix_batch launch consumes at most, every CTA reading the same ones from subsequence 0: 4 for (r_x, r_y), then per
// Gamma draw 8 per attempt (a curand_normal2_double and a curand_uniform2_double), two draws.  The generator's offset increment per
// launch, so consecutive launches never read overlapping parts of the stream.
constexpr int kMixOffsetIncrement = 4 + 2 * kGammaMaxAttempts * 8;
// torchvision's MixUp (cutmix = 0) or CutMix (cutmix = 1) on the batch x [B, C, H, W] (fp32 contiguous NCHW), image i paired with
// image i − 1 (image 0 with image B − 1), into the new tensor y and the fp32 targets q [B, K].  The targets are int64 class
// indices `labels` [B] (one-hot over K classes; an index outside [0, K) adds no mass to its row) or, when `labels` is null, fp32
// probabilities `probs` [B, K].  λ ~ Beta(α, α) = G₁/(G₁ + G₂) from two Gamma(α) draws (Marsaglia–Tsang in double; for α < 1,
// Gamma(α + 1)·U^(1/α) in logarithms), λ = 1/(1 + exp(log G₂ − log G₁)).  CutMix draws r_x in {0..W−1} and r_y in {0..H−1} and
// forms torchvision's box (x1, y1, x2, y2) and λ_adj = 1 − (x2 − x1)(y2 − y1)/(W·H) in double; pixels in [y1:y2, x1:x2] come from
// the partner on every channel.  MixUp gives y = fl(fl(x[i−1]·fp32(1 − λ)) + fl(x[i]·fp32(λ))); the targets take the same formula
// with λ (MixUp) or λ_adj (CutMix).  record (fp64, nullable): (λ) for MixUp, (λ, r_x, r_y, x1, y1, x2, y2, λ_adj) for CutMix.  One
// launch of B CTAs (none when B = 0); every CTA draws the batch's parameters itself.
void launch_mix_batch(const float* x, const long long* labels, const float* probs, float* y, float* q, double* record, int B, int C, int H,
                      int W, int K, double alpha, bool cutmix, PhiloxSeed rng, cudaStream_t st);

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
