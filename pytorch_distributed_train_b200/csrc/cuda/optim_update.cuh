// Per-element updates of Adamax, Adadelta, ASGD and Rprop, shared by their multi-tensor kernels (ops_simt.cu) and the riders of the
// ConvNet's last backward kernel (fused_convnet.cu), so that both compute the same bits.  Each follows torch's single-tensor
// (non-capturable) arithmetic; g is the gradient after maximize's negation, and the scalars are the per-launch values that torch forms
// on the host (ops_kernels.h), formed on the device.
#pragma once
#include <cuda_runtime.h>

#include "ops_kernels.h"

namespace pdt {

// Adamax: g' = g + wd·p;  m = lerp(m, g', 1 − β1);  u = max(β2·u, |g'| + eps) (torch.maximum: a NaN stays);  p −= clr·m/u
__device__ __forceinline__ void adamax_update(float* p, float g, float* m, float* u, float weight_decay, float omb1, float b2, float eps,
                                              float clr) {
  const float pv = *p;
  if (weight_decay != 0.f) g = fmaf(weight_decay, pv, g);
  const float mv = fmaf(omb1, g - *m, *m);
  const float uv = nan_max(b2 * *u, fabsf(g) + eps);
  *m = mv;
  *u = uv;
  *p = fmaf(-clr, mv / uv, pv);
}

// Adadelta: g' = g + wd·p;  sq = ρ·sq + (1 − ρ)·g'²;  δ = sqrt(acc + eps) / sqrt(sq + eps) · g';  acc = ρ·acc + (1 − ρ)·δ²;
// p −= lr·δ
__device__ __forceinline__ void adadelta_update(float* p, float g, float* sq, float* acc, float weight_decay, float rho, float omr, float eps,
                                                float lr) {
  const float pv = *p;
  if (weight_decay != 0.f) g = fmaf(weight_decay, pv, g);
  const float s = fmaf(omr * g, g, rho * *sq);
  *sq = s;
  const float a = *acc;
  const float d = sqrtf(a + eps) / sqrtf(s + eps) * g;
  *acc = fmaf(omr * d, d, rho * a);
  *p = fmaf(-lr, d, pv);
}

// ASGD: g' = g + wd·p (the parameter before the decay);  p = p·decay with decay = fp32(1 − λ·η);  p −= η·g';  then ax = p when
// mu == 1, else ax += (p − ax)·mu, each operation rounded as torch's separate tensor ops round it (no fused multiply-add)
__device__ __forceinline__ void asgd_update(float* p, float g, float* ax, float weight_decay, float eta, float decay, float mu) {
  float pv = *p;
  if (weight_decay != 0.f) g = fmaf(weight_decay, pv, g);
  pv = fmaf(-eta, g, __fmul_rn(pv, decay));
  *p = pv;
  if (mu == 1.f) {
    *ax = pv;
  } else {
    const float a = *ax;
    *ax = __fadd_rn(a, __fmul_rn(__fsub_rn(pv, a), mu));
  }
}

// ASGD's schedules for the step that leaves the count at t (torch's non-capturable branch, in double): eta = lr / (1 + λ·lr·t)^α and
// mu = 1 / max(1, t − t0), each rounded to fp32 as torch's copy into its fp32 state rounds it.
__device__ __forceinline__ float asgd_eta(double lr, double lambd, double alpha, double t) {
  return static_cast<float>(lr / pow(1.0 + lambd * lr * t, alpha));
}
__device__ __forceinline__ float asgd_mu(double t0, double t) { return static_cast<float>(1.0 / fmax(1.0, t - t0)); }

// torch.sign of an fp32 value: (0 < x) − (x < 0), so a NaN gives 0
__device__ __forceinline__ float torch_sign(float x) { return static_cast<float>((0.f < x) - (x < 0.f)); }

// Rprop: s = sign(fp32(g·prev));  f = η+ (s > 0), η− (s < 0), 1 (otherwise: a zero, an underflowed or a NaN product);
// step_size = clamp(step_size·f, min, max) (torch's clamp: a NaN stays);  g'' = 0 where f == η−, else g;  p −= sign(g'')·step_size;
// prev = g''.  Every operation is exact or rounds once, as torch's do.
__device__ __forceinline__ void rprop_update(float* p, float g, float* prev, float* step_size, float etaminus, float etaplus, float step_min,
                                             float step_max) {
  const float s = torch_sign(g * *prev);
  const float f = s > 0.f ? etaplus : s < 0.f ? etaminus : 1.f;
  float ss = *step_size * f;
  if (ss == ss) ss = fminf(fmaxf(ss, step_min), step_max);
  *step_size = ss;
  const float gg = f == etaminus ? 0.f : g;
  *p = fmaf(-torch_sign(gg), ss, *p);
  *prev = gg;
}

}  // namespace pdt
