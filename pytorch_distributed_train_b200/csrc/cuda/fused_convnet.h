// Cooperative fused layer kernels of the reference ConvNet (one CTA per image; see fused_convnet.cu).
#pragma once
#include <cuda_runtime.h>

#include "grid_sync.cuh"
#include "ops_kernels.h"

namespace pdt {

// One CTA per image, all co-resident: the batch must not exceed the number of SMs.
bool fused_convnet_supported(int B);
// Phase trace of the cooperative kernels (globaltimer stamps of thread 0 of every CTA): [kernel 0..3][CTA][phase].
void fused_convnet_trace_enable(bool on);
void fused_convnet_trace_read(unsigned long long* host);

// Activations between the two layers live in zero-haloed 18×18 NHWC frames ([B,18,18,C], interior = rows/cols 2..15):
// layer 2 reads the halo as the convolution's zero padding (one TMA box per image, row-shifted descriptors per tap).
// x [B,28,28] → y [B,28,28,16] (conv1 + bias, kept for backward), out [B,18,18,16] frame (BN + ReLU + pool), saved [32] = mean, invstd.
// partials: B·32 floats of scratch.
void launch_convnet_l1_fwd(const float* x, const float* w, const float* bias, const float* gamma, const float* beta, float* y, float* out,
                           float* saved, float* running_mean, float* running_var, long long* nbt, float momentum, float eps, int B,
                           float* partials, GridSync gs, cudaStream_t st);
// dp [B,18,18,16] frame (interior read) → dgamma/dbeta [16], dw [16,1,5,5], db [16].  partials: B·32, partials_w: B·512 floats.
void launch_convnet_l1_bwd(const float* dp, const float* y, const float* x, const float* saved, const float* gamma, const float* beta,
                           float* dgamma, float* dbeta, float* dw, float* db, int B, float* partials, float* partials_w, GridSync gs,
                           cudaStream_t st);
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
// Either rider with gradient-norm clipping in front of the update (torch.nn.utils.clip_grad_norm_, norm_type 2 or inf).  Every CTA
// adds up the squares (or the max |g|) of the gradient elements it sees — those of parameters 6..9 in the shadow of the first
// grid barrier, those of 0..5 as it folds them — and writes one partial; after one more grid barrier every CTA folds the B
// partials in the same order (fp64), derives the same coefficient, and in a grid-stride pass writes g·coef back to every
// gradient and applies the update with it.  CTA 0 stores the norm.
template <class Base>
struct ClipRider : Base {
  float max_norm = 0.f;
  int norm_inf = 0;            // 1: max |g|, 0: Euclidean norm
  float* norm_out = nullptr;   // the total norm (fp32 scalar)
  float* part = nullptr;       // [B] per-CTA partials
};

// Layer-1 backward with the conv2 weight gradient of the same image running on the tensor cores next to it (two extra warps):
// dy2_pad [B,18,18,32] / x2_pad [B,18,18,16] frames and dysum2 [B,32] from layer-2 backward → dw2 [32,16,5,5], db2 [32].
// wpart: B·512·32 floats of scratch, disjoint from partials / partials_w.  Rider: SgdRider or AdamRider, or either one in a ClipRider.
template <class Rider = SgdRider>
void launch_convnet_l1_bwd_wgrad(const float* dp, const float* y, const float* x, const float* saved, const float* gamma, const float* beta,
                                 float* dgamma, float* dbeta, float* dw, float* db, const float* dy2_pad, const float* x2_pad, const float* dysum2,
                                 float* dw2, float* db2, int B, float* partials, float* partials_w, float* wpart, GridSync gs, cudaStream_t st,
                                 Rider rider = Rider{});
// x [B,18,18,16] frame → y [B,14,14,32], out [B,32,7,7] NCHW, saved [64]; logits [B,ncls] = fc(out) when logits != nullptr.
// partials: B·64 floats.
void launch_convnet_l2_fwd(const float* x, const float* w, const float* bias, const float* gamma, const float* beta, float* y, float* out,
                           float* saved, float* running_mean, float* running_var, long long* nbt, float momentum, float eps,
                           const float* fcw, const float* fcb, float* logits, int ncls, int B, float* partials, GridSync gs, cudaStream_t st);
// Optional rider of the whole-forward kernel: the mean cross-entropy of the logits against `target` and its gradient
// (softmax − onehot)/B, computed by the CTA that owns the image; the batch mean is folded by the CTA that finishes last
// (arrival counter, fixed summation order).  target == nullptr: off.
struct FusedCe {
  const long long* target = nullptr;   // [B]
  float* loss_parts = nullptr;         // [B] scratch
  float* loss = nullptr;               // scalar; nullptr = the mean is folded later (launch_convnet_l2_bwd_fc)
  float* dlogits = nullptr;            // [B, ncls]
  unsigned int* counter = nullptr;     // zero before first use; reset by the kernel
};

// The whole training forward in one launch: layer 1 and layer 2 (+ classifier, ncls ≤ 16) of an image in the same CTA; the
// pooled layer-1 activations go into conv2's shared-memory patch directly.  partials: B·(32 + 64) floats.
void launch_convnet_fwd(const float* x, const float* w1, const float* b1, const float* g1, const float* be1, float* y1, float* p1, float* saved1,
                        float* rm1, float* rv1, long long* nbt1, float mom1, float eps1, const float* w2, const float* b2, const float* g2,
                        const float* be2, float* y2, float* out, float* saved2, float* rm2, float* rv2, long long* nbt2, float mom2, float eps2,
                        const float* fcw, const float* fcb, float* logits, int ncls, int B, float* partials, GridSync gs, cudaStream_t st,
                        FusedCe ce = FusedCe{});
// dout [B,32,7,7] → dgamma/dbeta [32], dy [B,18,18,32] frame with zero halo (gradient at the conv2 output), dx [B,18,18,16] frame
// (data gradient, interior written), dysum [B,32] (per-image Σdy: the conv2 bias gradient is the sum of its rows).
void launch_convnet_l2_bwd(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta, const float* w,
                           float* dgamma, float* dbeta, float* dy, float* dx, float* dysum, int B, float* partials, GridSync gs, cudaStream_t st);
// The same with the classifier's backward riding along: d(out) is computed from dlogits [B,ncls] and the fc weights [ncls,1568]
// inside the kernel; dfcw [ncls,1568] / dfcb [ncls] are produced from `pooled` = the forward's out [B,1568].  ncls ≤ 16.
void launch_convnet_l2_bwd_fc(const float* dlogits, const float* fcw, const float* pooled, float* dfcw, float* dfcb, int ncls, const float* y,
                              const float* saved, const float* gamma, const float* beta, const float* w, float* dgamma, float* dbeta, float* dy,
                              float* dx, float* dysum, int B, float* partials, GridSync gs, cudaStream_t st,
                              const float* loss_parts = nullptr, float* loss_out = nullptr);   // batch mean of the forward kernel's CE terms

}  // namespace pdt
