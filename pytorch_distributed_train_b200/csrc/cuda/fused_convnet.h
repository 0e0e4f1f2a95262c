// Cooperative fused layer kernels of the reference ConvNet (one CTA per image; see fused_convnet.cu).
#pragma once
#include <cuda_runtime.h>

#include "grid_sync.cuh"
#include "ops_kernels.h"

namespace pdt {

// One CTA per image, all co-resident: the batch must not exceed the number of SMs.
bool fused_convnet_supported(int B);
// Phase trace of the cooperative kernels (globaltimer stamps of thread 0 of every CTA): [kernel slot 0..3][CTA][phase], slots
// 0 forward, 1 layer-1 backward, 3 layer-2 backward.
void fused_convnet_trace_enable(bool on);
void fused_convnet_trace_read(unsigned long long* host);

// Activations between the two layers live in zero-haloed 18×18 NHWC frames ([B,18,18,C], interior = rows/cols 2..15): the
// kernels read the halo as the convolution's zero padding.

// Optional rider of the last backward kernel: the SGD update of every parameter of the model.  Parameters 0..5 (conv1.w, conv1.b,
// bn1.w, bn1.b, conv2.w, conv2.b) get their gradient inside this kernel — the thread that writes the folded gradient element applies
// the update with the value still in its register; parameters 6..9 (gradients complete before the launch: classifier, bn2) are updated
// in the shadow of the kernel's first grid barrier.  Same arithmetic as sgd_multi_kernel.
struct SgdRider {
  int on = 0;
  float* p[10] = {};
  float* m[10] = {};           // momentum buffers (nullptr: momentum == 0)
  const float* g_prev[4] = {}; // gradients of parameters 6..9
  int n_prev[4] = {};
  SgdHyper h{};
};
// The same rider with the Adam / AdamW update (the arithmetic of adam_multi_kernel).  Every CTA reads the ten step counts before
// the kernel's first grid barrier; one thread writes step + 1 after the last one.
struct AdamRider {
  int on = 0;
  float* p[10] = {};
  float* m[10] = {};           // exp_avg
  float* v[10] = {};           // exp_avg_sq
  float* step[10] = {};        // fp32 step counts on the device
  const float* g_prev[4] = {};
  int n_prev[4] = {};
  AdamHyper h{};
};
// The Adam rider with AMSGrad (the arithmetic of amsgrad_multi_kernel): vmax = max(vmax, exp_avg_sq), a NaN kept, is the denominator's.
struct AmsgradRider : AdamRider {
  float* vmax[10] = {};        // max_exp_avg_sq
};
// The Adam rider's state with the NAdam update (the arithmetic of nadam_multi_kernel).  Every CTA reads the ten step counts and
// mu_products before the kernel's first grid barrier; one thread writes step + 1 and the new mu_product after the last one.
struct NadamRider : AdamRider {
  float* mu_product[10] = {};  // fp32 scalars on the device
  double momentum_decay = 0.0;
};
// The Adam rider's state with the RAdam update (the arithmetic of radam_multi_kernel): every CTA decides from the step counts it
// reads before the first grid barrier which parameters take the rectified step.
struct RadamRider : AdamRider {};
// The same rider with the RMSprop update (the arithmetic of rmsprop_multi_kernel).  The step counts do not enter the update; one
// thread writes step + 1 after the kernel's last grid barrier.
struct RmspropRider {
  int on = 0;
  float* p[10] = {};
  float* sq[10] = {};          // square_avg
  float* buf[10] = {};         // momentum_buffer (nullptr: momentum == 0)
  float* ga[10] = {};          // grad_avg (nullptr: not centered)
  float* step[10] = {};        // fp32 step counts on the device
  const float* g_prev[4] = {};
  int n_prev[4] = {};
  RmspropHyper h{};
};
// The same rider with the Adagrad update (the arithmetic of adagrad_multi_kernel).  Every CTA reads the ten step counts before the
// kernel's first grid barrier (the decayed learning rates); one thread writes step + 1 after the last one.
struct AdagradRider {
  int on = 0;
  float* p[10] = {};
  float* sum[10] = {};
  float* step[10] = {};        // fp32 step counts on the device
  const float* g_prev[4] = {};
  int n_prev[4] = {};
  AdagradHyper h{};
};
// The Adam rider's state with the Adamax update (optim_update.cuh: adamax_update), v holding exp_inf: every CTA forms the ten
// bias-corrected learning rates from the step counts it reads before the first grid barrier; one thread writes step + 1 after the last.
struct AdamaxRider : AdamRider {};
// The rider with the Adadelta update (optim_update.cuh: adadelta_update).  The step counts do not enter the update; one thread
// writes step + 1 after the kernel's last grid barrier.
struct AdadeltaRider {
  int on = 0;
  float* p[10] = {};
  float* sq[10] = {};          // square_avg
  float* acc[10] = {};         // acc_delta
  float* step[10] = {};        // fp32 step counts on the device
  const float* g_prev[4] = {};
  int n_prev[4] = {};
  AdadeltaHyper h{};
};
// The rider with the ASGD update (optim_update.cuh: asgd_update).  Every CTA reads the ten step counts, etas and mus before the
// kernel's first grid barrier; one thread writes step + 1 and the next eta and mu after the last one.
struct AsgdRider {
  int on = 0;
  float* p[10] = {};
  float* ax[10] = {};
  float* step[10] = {};        // fp32 scalars on the device
  float* eta[10] = {};
  float* mu[10] = {};
  const float* g_prev[4] = {};
  int n_prev[4] = {};
  AsgdHyper h{};
};
// The rider with the Rprop update (optim_update.cuh: rprop_update).  The step counts do not enter the update; one thread writes
// step + 1 after the kernel's last grid barrier.
struct RpropRider {
  int on = 0;
  float* p[10] = {};
  float* prev[10] = {};
  float* step_size[10] = {};
  float* step[10] = {};        // fp32 step counts on the device
  const float* g_prev[4] = {};
  int n_prev[4] = {};
  RpropHyper h{};
};
// Any of the riders with gradient-norm clipping in front of the update (torch.nn.utils.clip_grad_norm_, norm_type 2 or inf).  Every CTA
// adds up the squares (or the max |g|) of the gradient elements it sees — those of parameters 6..9 in the shadow of the first
// grid barrier, those of 0..5 as it folds them (4, 5 in that shadow too) — and writes one partial; after one more grid barrier every CTA folds the B
// partials in the same order (fp64), derives the same coefficient, and in a grid-stride pass writes g·coef back to every
// gradient and applies the update with it.  CTA 0 stores the norm.
template <class Base>
struct ClipRider : Base {
  float max_norm = 0.f;
  int norm_inf = 0;            // 1: max |g|, 0: Euclidean norm
  float* norm_out = nullptr;   // the total norm (fp32 scalar)
  float* part = nullptr;       // [B] per-CTA partials
};

// conv2's weight gradient per image (wpart [B][400][32], rows (kh, kw, ci), the layout launch_convnet_l2_bwd_fc writes given x2) from
// given frames: dy2_pad [B,18,18,32] (zero halo), x2_pad [B,18,18,16].  One CTA per image, not cooperative.  No training step runs it:
// with the dy frame of launch_convnet_l2_bwd_fc without x2 it is the tests' bit-exact reference for the partials backward A computes.
void launch_conv2_wgrad_partials(const float* dy2_pad, const float* x2_pad, int B, float* wpart, cudaStream_t st);
// Layer-1 backward: dp [B,18,18,16] frame (interior read) → dgamma/dbeta [16], dw [16,1,5,5], db [16]; it also folds conv2's weight
// gradient: the per-image partials wpart and Σdy rows dysum2 [B,32] → dw2 [32,16,5,5], db2 [32], in the shadow of the kernel's first
// grid barrier.  partials: B·32, partials_w: B·512 floats.  Rider: SgdRider, AdamRider, AmsgradRider, NadamRider, RadamRider,
// RmspropRider, AdagradRider, AdamaxRider, AdadeltaRider, AsgdRider or RpropRider, or one of them in a ClipRider.
// accumulate: gradient accumulation — every gradient written (dgamma, dbeta, dw, db, dw2, db2) becomes g_old + this batch's value, and
// the rider updates with (and clips) the accumulated gradient.
// y: conv1's output [B,28,28,16] (conv1 + bias) as launch_convnet_fwd wrote it, or nullptr: then each CTA recomputes it from x and
// conv1's weights w1 [16,1,5,5] and bias b1 [16] (nullable) in the forward's order, bit for bit; w1 is required then.
template <class Rider = SgdRider>
void launch_convnet_l1_bwd_wgrad(const float* dp, const float* y, const float* w1, const float* b1, const float* x, const float* saved,
                                 const float* gamma, const float* beta, float* dgamma, float* dbeta, float* dw, float* db, const float* wpart,
                                 const float* dysum2, float* dw2, float* db2, int B, float* partials, float* partials_w, GridSync gs, cudaStream_t st,
                                 Rider rider = Rider{}, bool accumulate = false);
// Optional rider of the whole-forward kernel: the mean cross-entropy of the logits against `target` and its gradient
// (softmax − onehot)/n, computed by the CTA that owns the image; the batch mean is folded by the CTA that finishes last
// (arrival counter, fixed summation order).  n counts the images whose target is in [0, ncls); the others (ignore_index) add
// no term and get a zero gradient, and n = 0 gives a NaN loss, as in torch.  target == nullptr: off.
struct FusedCe {
  const long long* target = nullptr;   // [B]
  float* loss_parts = nullptr;         // [B + 1] scratch: one term per image, then n
  float* loss = nullptr;               // scalar; nullptr = the mean is folded later (launch_convnet_l2_bwd_fc)
  float* dlogits = nullptr;            // [B, ncls]
  unsigned int* counter = nullptr;     // zero before first use; reset by the kernel
};
// The same rider with a gradient scale: the loss is scale · (mean cross-entropy) and dlogits its gradient, i.e. the unscaled
// gradient times scale, rounded as autograd's grad · scale would be.  Gradient accumulation over k micro-batches uses 1/k (torch's
// loss / k convention).  The mean's divisor loss_parts[B] becomes n / scale, so a mean folded later carries the scale too.
struct ScaledCe : FusedCe {
  float scale = 1.f;
};
// The scaled rider with torch's other cross-entropy options (ops_kernels.h: CeSpec): class weights [ncls], label smoothing, any
// ignore_index, sum or mean.  A counted image has a target in [0, ncls) other than ignore_index; loss_parts[B] holds the divisor D
// (Σ_{counted} w_t for the mean, 1 for the sum) over the scale, so the later fold divides by it as it does by n / scale.
struct SmoothCe : ScaledCe {
  const float* weight = nullptr;   // [ncls] or null
  float smoothing = 0.f;
  long long ignore_index = -100;
  bool sum = false;                // reduction 'sum' (else 'mean')
  bool is_default(int ncls) const { return weight == nullptr && smoothing == 0.f && !sum && (ignore_index < 0 || ignore_index >= ncls); }
};
// The rider with class-probability targets q [B, ncls] in place of `target` (ops_kernels.h: launch_cross_entropy_fwd_soft): class
// weights, label smoothing, sum or mean; ignore_index plays no part.  Every image counts, so loss_parts[B] holds D = B (the mean)
// or 1 (the sum) over the scale, and nothing is summed before the image's term.
struct SoftCe : SmoothCe {
  const float* target_probs = nullptr;   // [B, ncls]; nullptr: `target` (class indices) or off
};

// The whole training forward in one launch: layer 1 and layer 2 (+ classifier, ncls ≤ 16) of an image in the same CTA; the
// pooled layer-1 activations go into conv2's shared-memory patch directly.  x [B,28,28] → y1 [B,28,28,16] (conv1 + bias; nullptr:
// not stored — the layer-1 backward recomputes it), p1 [B,18,18,16] frame (BN + ReLU + pool), saved1 [32] = mean, invstd; y2 [B,14,14,32], out [B,32,7,7] NCHW, saved2
// [64]; logits [B,ncls].  partials: B·(32 + 64) floats.
// With probability targets the SoftCe instantiation runs; with class-index targets a non-default spec runs the SmoothCe one, else
// ce.scale != 1 the ScaledCe one; otherwise the kernel without the scale.
void launch_convnet_fwd(const float* x, const float* w1, const float* b1, const float* g1, const float* be1, float* y1, float* p1, float* saved1,
                        float* rm1, float* rv1, long long* nbt1, float mom1, float eps1, const float* w2, const float* b2, const float* g2,
                        const float* be2, float* y2, float* out, float* saved2, float* rm2, float* rv2, long long* nbt2, float mom2, float eps2,
                        const float* fcw, const float* fcb, float* logits, int ncls, int B, float* partials, GridSync gs, cudaStream_t st,
                        SoftCe ce = SoftCe{});
// Layer-2 backward with the classifier's backward riding along: d(out) is computed from dlogits [B,ncls] and the fc weights
// [ncls,1568] inside the kernel; dfcw [ncls,1568] / dfcb [ncls] are produced from `pooled` = the forward's out [B,1568].  ncls ≤ 16.
// → dgamma/dbeta [32], dy [B,18,18,32] frame with zero halo (gradient at the conv2 output), dx [B,18,18,16] frame (data gradient,
// interior written), dysum [B,32] (per-image Σdy: the conv2 bias gradient is the sum of its rows).
// x2 != nullptr (conv2's input frame [B,18,18,16]): conv2's weight-gradient partials per image go to wpart [B][400][32] instead,
// and dy is not written.  The training step always passes x2; without it the kernel is the tests' reference (see
// launch_conv2_wgrad_partials).
void launch_convnet_l2_bwd_fc(const float* dlogits, const float* fcw, const float* pooled, float* dfcw, float* dfcb, int ncls, const float* y,
                              const float* saved, const float* gamma, const float* beta, const float* w, float* dgamma, float* dbeta, float* dy,
                              float* dx, float* dysum, int B, float* partials, GridSync gs, cudaStream_t st,
                              const float* loss_parts = nullptr, float* loss_out = nullptr,   // mean of the forward kernel's CE terms
                              const float* x2 = nullptr, float* wpart = nullptr,
                              bool accumulate = false);   // dfcw, dfcb, dgamma, dbeta, loss_out += this batch's values (needs x2)

}  // namespace pdt
