// Per-image random affine augmentation (torchvision's RandomAffine on a batch, every image with its own parameters), one launch.
// One CTA per image, one thread per pixel up to 1024: thread 0 draws the image's parameters from Philox subsequence b and forms
// torchvision's inverse matrix in double into shared memory; then every thread maps its output pixels to source coordinates once
// and samples all channels there.
// Batch-level MixUp and CutMix (torchvision's v2 transforms), one launch: one CTA per image, each drawing the batch's λ (and box)
// from the same Philox values, then mixing its image with its roll-by-one partner and writing its target row.
// Per-image elastic deformation (torchvision's v2.ElasticTransform, every image with its own field), one launch: one CTA per image
// holds the image's two noise planes and one scratch plane in shared memory (12 B per pixel), draws the noise, blurs it
// separably and warps the image with the shared sampler.  Philox layout: the noise value of pixel p (p = 4q + e, e in 0..3) of
// plane c (0: dx0, 1: dy0) of image b is component e of the one curand_uniform4 drawn from subsequence (2b + c)·⌈HW/4⌉ + q at
// the launch's offset, so no two images, planes or pixels share a value, and each subsequence consumes 4 values: the launch's
// offset increment (kElasticOffsetIncrement).
#include <cuda_runtime.h>
#include <curand_kernel.h>

#include <algorithm>
#include <stdexcept>
#include <string>

#include "cuda_utils.h"
#include "ops_kernels.h"

namespace pdt {

namespace {

// one thread per output pixel up to 1024 (a 28×28 image in one pass: each thread's source loads are the kernel's latency)
constexpr int kAffineMaxThreads = 1024;

// Philox subsequence `subsequence` at the launch's offset.  Captured: the graph's replay writes seed and base offset before it
// launches us.
__device__ __forceinline__ void philox_init(const PhiloxSeed& rng, unsigned long long subsequence, curandStatePhilox4_32_10_t* st) {
  unsigned long long seed = rng.seed, offset = rng.offset;
  if (rng.seed_ptr != nullptr) {
    seed = static_cast<unsigned long long>(*rng.seed_ptr);
    offset = static_cast<unsigned long long>(*rng.offset_ptr) + rng.offset;
  }
  curand_init(seed, subsequence, offset, st);
}

// torch's CUDA uniform_: curand's (0, 1] with 1 mapped to 0, then u·range + from in fp32: U[from, to)
__device__ __forceinline__ float draw(float r, float from, float range) { return (r == 1.f ? 0.f : r) * range + from; }

// Output pixel p of every channel of one image (src, dst: its first plane, C planes of H·W) from the source coordinate (sx, sy):
// grid_sample(align_corners=False, padding_mode="zeros") unnormalised.  Nearest rounds half to even and writes `fill` outside the
// image; bilinear reads 0 outside and returns torchvision's (v − fill)·mask + fill.
__device__ __forceinline__ void sample_pixel(const float* __restrict__ src, float* __restrict__ dst, int C, int H, int W, int p,
                                             double sxp, double syp, int bilinear, float fill) {
  const int hw = H * W;
  if (!bilinear) {
    const double rx = rint(sxp), ry = rint(syp);   // ties to even, as grid_sample's nearbyint
    const bool in = rx >= 0.0 && rx <= W - 1 && ry >= 0.0 && ry <= H - 1;   // false for NaN
    const int o = in ? static_cast<int>(ry) * W + static_cast<int>(rx) : 0;
    for (int ci = 0; ci < C; ++ci) dst[ci * hw + p] = in ? __ldg(src + ci * hw + o) : fill;
    return;
  }
  const double x0 = floor(sxp), y0 = floor(syp);
  const double fx = sxp - x0, fy = syp - y0;
  const bool vx0 = x0 >= 0.0 && x0 <= W - 1, vx1 = x0 >= -1.0 && x0 <= W - 2;
  const bool vy0 = y0 >= 0.0 && y0 <= H - 1, vy1 = y0 >= -1.0 && y0 <= H - 2;
  // taps nw, ne, sw, se; out-of-bounds taps read 0 and add nothing to the mask
  const bool v[4] = {vx0 && vy0, vx1 && vy0, vx0 && vy1, vx1 && vy1};
  const float w[4] = {static_cast<float>((1.0 - fx) * (1.0 - fy)), static_cast<float>(fx * (1.0 - fy)),
                      static_cast<float>((1.0 - fx) * fy), static_cast<float>(fx * fy)};
  int o[4];
  const int ix = vx0 || vx1 ? static_cast<int>(x0) : 0, iy = vy0 || vy1 ? static_cast<int>(y0) : 0;
  o[0] = iy * W + ix, o[1] = o[0] + 1, o[2] = o[0] + W, o[3] = o[0] + W + 1;
  float mask = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) mask += v[k] ? w[k] : 0.f;
  for (int ci = 0; ci < C; ++ci) {
    const float* __restrict__ plane = src + ci * hw;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (v[k]) acc += w[k] * __ldg(plane + o[k]);
    // torchvision's fill: (img − fill)·mask + fill, the mask being grid_sample's bilinear weight of the in-bounds taps
    dst[ci * hw + p] = (acc - fill) * mask + fill;
  }
}

__global__ void __launch_bounds__(kAffineMaxThreads) random_affine_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                        float* __restrict__ params, int C, int H, int W, AffineSpec s,
                                                                        PhiloxSeed rng) {
  __shared__ double m[6];
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    curandStatePhilox4_32_10_t st;
    philox_init(rng, b, &st);
    const float4 r0 = curand_uniform4(&st);
    const float4 r1 = curand_uniform4(&st);
    const float angle = draw(r0.x, s.angle_from, s.angle_range);
    const float tx = rintf(draw(r0.y, s.tx_from, s.tx_range));   // round half to even, as Python's round
    const float ty = rintf(draw(r0.z, s.ty_from, s.ty_range));
    const float scale = draw(r0.w, s.scale_from, s.scale_range);
    const float shear_x = draw(r1.x, s.shear_x_from, s.shear_x_range);
    const float shear_y = draw(r1.y, s.shear_y_from, s.shear_y_range);
    if (params != nullptr) {
      float* p = params + 6 * static_cast<long long>(b);
      p[0] = angle, p[1] = tx, p[2] = ty, p[3] = scale, p[4] = shear_x, p[5] = shear_y;
    }
    // torchvision's _get_inverse_affine_matrix(center=[0, 0], angle, (tx, ty), scale, (shear_x, shear_y)), in double
    constexpr double kRad = 3.14159265358979323846 / 180.0;
    const double rot = angle * kRad, sx = shear_x * kRad, sy = shear_y * kRad;
    const double a = cos(rot - sy) / cos(sy);
    const double bb = -cos(rot - sy) * tan(sx) / cos(sy) - sin(rot);
    const double c = sin(rot - sy) / cos(sy);
    const double d = -sin(rot - sy) * tan(sx) / cos(sy) + cos(rot);
    const double sc = scale;
    m[0] = d / sc, m[1] = -bb / sc, m[3] = -c / sc, m[4] = a / sc;
    m[2] = m[0] * -static_cast<double>(tx) + m[1] * -static_cast<double>(ty);
    m[5] = m[3] * -static_cast<double>(tx) + m[4] * -static_cast<double>(ty);
  }
  __syncthreads();
  const double m0 = m[0], m1 = m[1], m2 = m[2], m3 = m[3], m4 = m[4], m5 = m[5];
  const double cw = 0.5 * (W - 1), ch = 0.5 * (H - 1);
  const int hw = H * W;
  const float* __restrict__ src = x + static_cast<long long>(b) * C * hw;
  float* __restrict__ dst = y + static_cast<long long>(b) * C * hw;
  const float fill = s.fill;
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    const int i = p / W, j = p - (p / W) * W;
    // the source coordinate of output pixel (i, j): torchvision's _affine_grid + grid_sample(align_corners=False), unnormalised
    const double xj = j - cw, yi = i - ch;
    sample_pixel(src, dst, C, H, W, p, m0 * xj + m1 * yi + m2 + cw, m3 * xj + m4 * yi + m5 + ch, s.bilinear, fill);
  }
}

// one thread per pixel up to 1024, as random_affine_kernel
constexpr int kElasticMaxThreads = 1024;

// torch's reflect padding of an index in [−(n − 1), 2(n − 1)]
__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i : (i > n - 1 ? 2 * (n - 1) - i : i); }

// out = blur(in) with weights w (k taps, centred) along x (step 1, extent W) or y (step W, extent H), in fp32
__device__ __forceinline__ void blur_pass(const float* in, float* out, const float* __restrict__ w, int k, int H, int W, bool along_x) {
  const int r = k / 2;
  for (int p = threadIdx.x; p < H * W; p += blockDim.x) {
    const int i = p / W, j = p - i * W;
    float acc = 0.f;
    if (along_x) {
      for (int t = 0; t < k; ++t) acc += __ldg(w + t) * in[i * W + reflect(j + t - r, W)];
    } else {
      for (int t = 0; t < k; ++t) acc += __ldg(w + t) * in[reflect(i + t - r, H) * W + j];
    }
    out[p] = acc;
  }
}

// One CTA per image b: draws the two noise planes into shared memory (and into noise[b] when recording), blurs each (x pass into
// the scratch plane, y pass back), scales it to the displacement and warps all channels of the image through it.
__global__ void __launch_bounds__(kElasticMaxThreads) elastic_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                     float* __restrict__ noise, int C, int H, int W, ElasticSpec s,
                                                                     PhiloxSeed rng) {
  extern __shared__ float sm[];   // dx plane, dy plane, scratch: 3·H·W
  const int b = blockIdx.x;
  const int hw = H * W, groups = (hw + 3) / 4;
  for (int g = threadIdx.x; g < 2 * groups; g += blockDim.x) {
    const int c = g < groups ? 0 : 1, q = g - c * groups;
    curandStatePhilox4_32_10_t st;
    philox_init(rng, (2ull * b + c) * groups + q, &st);
    const float4 r = curand_uniform4(&st);
    const float v[4] = {draw(r.x, -1.f, 2.f), draw(r.y, -1.f, 2.f), draw(r.z, -1.f, 2.f), draw(r.w, -1.f, 2.f)};   // torch.rand·2 − 1
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int p = 4 * q + e;
      if (p >= hw) break;
      sm[c * hw + p] = v[e];
      if (noise != nullptr) noise[(2ll * b + c) * hw + p] = v[e];
    }
  }
  __syncthreads();
  float* tmp = sm + 2 * hw;
  const float* w = s.weights;
  for (int c = 0; c < 2; ++c) {
    const int k = s.k[c];
    if (k == 0) continue;   // the same for the whole CTA
    // plane c: x weights (k, sigma[0]), then y weights (k, sigma[1])
    blur_pass(sm + c * hw, tmp, w, k, H, W, true);
    __syncthreads();
    blur_pass(tmp, sm + c * hw, w + k, k, H, W, false);
    __syncthreads();
    w += 2 * k;
  }
  const float* __restrict__ src = x + static_cast<long long>(b) * C * hw;
  float* __restrict__ dst = y + static_cast<long long>(b) * C * hw;
  const float fw = static_cast<float>(W), fh = static_cast<float>(H);
  for (int p = threadIdx.x; p < hw; p += blockDim.x) {
    const int i = p / W, j = p - i * W;
    // torchvision's dx = blurred · alpha[0] / W in fp32 (dy likewise with H); the grid's identity plus displacement, unnormalised
    const float dx = __fdiv_rn(__fmul_rn(sm[p], s.alpha_x), fw), dy = __fdiv_rn(__fmul_rn(sm[hw + p], s.alpha_y), fh);
    sample_pixel(src, dst, C, H, W, p, j + 0.5 * W * static_cast<double>(dx), i + 0.5 * H * static_cast<double>(dy), s.bilinear, s.fill);
  }
}

constexpr int kMixThreads = 256;

// log of one Gamma(alpha) draw: Marsaglia & Tsang (2000) in double, for alpha < 1 boosted as Gamma(alpha + 1)·U^(1/alpha) with the
// power kept as a logarithm (at small alpha the draw itself underflows).  Every attempt consumes 8 Philox values whether it is
// accepted or not, so a draw never reads past its kGammaMaxAttempts · 8; a draw that exhausts them (probability < 1e-21) returns
// log d, the distribution's mode region.
__device__ double log_gamma_draw(curandStatePhilox4_32_10_t* st, double alpha) {
  const bool boost = alpha < 1.0;
  const double d = (boost ? alpha + 1.0 : alpha) - 1.0 / 3.0;
  const double c = 1.0 / sqrt(9.0 * d);
  const double log_d = log(d);
  for (int k = 0; k < kGammaMaxAttempts; ++k) {
    const double2 n = curand_normal2_double(st);
    const double2 u = curand_uniform2_double(st);   // (0, 1): u.x decides, u.y is the boost's U
    const double t = 1.0 + c * n.x;
    if (t <= 0.0) continue;
    const double log_v = 3.0 * log(t);
    if (log(u.x) < 0.5 * n.x * n.x + d - d * (t * t * t) + d * log_v) return log_d + log_v + (boost ? log(u.y) / alpha : 0.0);
  }
  return log_d;
}

// One CTA per image i: thread 0 draws the batch's parameters (every CTA draws the same ones, from Philox subsequence 0), then the
// CTA writes image i and target row i.
__global__ void __launch_bounds__(kMixThreads, 1) mix_batch_kernel(const float* __restrict__ x, const long long* __restrict__ labels,
                                                                const float* __restrict__ probs, float* __restrict__ y,
                                                                float* __restrict__ q, double* __restrict__ record, int B, int C, int H,
                                                                int W, int K, double alpha, int cutmix, PhiloxSeed rng) {
  __shared__ double s_lam;
  __shared__ int s_box[4];
  const int i = blockIdx.x;
  if (threadIdx.x == 0) {
    curandStatePhilox4_32_10_t st;
    philox_init(rng, 0, &st);
    const double2 r = curand_uniform2_double(&st);   // (0, 1), drawn by MixUp too so that both modes read the stream alike
    const double lg1 = log_gamma_draw(&st, alpha);
    const double lg2 = log_gamma_draw(&st, alpha);
    // λ = G₁/(G₁ + G₂), never 0/0 when both draws underflow
    const double lam = 1.0 / (1.0 + exp(lg2 - lg1));
    double lam_mix = lam;
    int x1 = 0, y1 = 0, x2 = 0, y2 = 0;
    if (cutmix) {
      // torchvision's CutMix.make_params from (λ, r_x, r_y), in double
      const int rx = min(static_cast<int>((1.0 - r.x) * W), W - 1), ry = min(static_cast<int>((1.0 - r.y) * H), H - 1);
      const double rr = 0.5 * sqrt(1.0 - lam);
      const int rw_half = static_cast<int>(rr * W), rh_half = static_cast<int>(rr * H);
      x1 = max(rx - rw_half, 0), y1 = max(ry - rh_half, 0), x2 = min(rx + rw_half, W), y2 = min(ry + rh_half, H);
      lam_mix = 1.0 - static_cast<double>(static_cast<long long>(x2 - x1) * (y2 - y1)) / static_cast<double>(static_cast<long long>(W) * H);
      if (record != nullptr && i == 0) {
        record[0] = lam, record[1] = rx, record[2] = ry, record[3] = x1, record[4] = y1, record[5] = x2, record[6] = y2;
        record[7] = lam_mix;
      }
    } else if (record != nullptr && i == 0) {
      record[0] = lam;
    }
    s_lam = lam_mix;
    s_box[0] = x1, s_box[1] = y1, s_box[2] = x2, s_box[3] = y2;
  }
  __syncthreads();
  const double lam = s_lam;
  // torchvision's tensor ops: the Python float λ and 1 − λ (formed in double) each rounded to fp32 as a scalar operand
  const float lf = static_cast<float>(lam), omf = static_cast<float>(1.0 - lam);
  const int prev = i == 0 ? B - 1 : i - 1;
  float* __restrict__ qi = q + static_cast<long long>(i) * K;
  if (labels != nullptr) {
    const long long li = labels[i], lp = labels[prev];
    for (int k = threadIdx.x; k < K; k += blockDim.x) qi[k] = __fadd_rn(k == lp ? omf : 0.f, k == li ? lf : 0.f);
  } else {
    const float* __restrict__ pi = probs + static_cast<long long>(i) * K;
    const float* __restrict__ pp = probs + static_cast<long long>(prev) * K;
    for (int k = threadIdx.x; k < K; k += blockDim.x) qi[k] = __fadd_rn(__fmul_rn(__ldg(pp + k), omf), __fmul_rn(__ldg(pi + k), lf));
  }
  const int hw = H * W, n = C * hw;
  const float* __restrict__ xi = x + static_cast<long long>(i) * n;
  const float* __restrict__ xp = x + static_cast<long long>(prev) * n;
  float* __restrict__ yi = y + static_cast<long long>(i) * n;
  if (cutmix) {
    const int x1 = s_box[0], y1 = s_box[1], x2 = s_box[2], y2 = s_box[3];
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      const int p = e % hw, h = p / W, w = p - h * W;
      const bool inside = h >= y1 && h < y2 && w >= x1 && w < x2;
      yi[e] = __ldg((inside ? xp : xi) + e);
    }
  } else {
    // two roundings, no FMA: fl(fl(x[i−1]·(1 − λ)) + fl(x[i]·λ))
    for (int e = threadIdx.x; e < n; e += blockDim.x) yi[e] = __fadd_rn(__fmul_rn(__ldg(xp + e), omf), __fmul_rn(__ldg(xi + e), lf));
  }
}

}  // namespace

void launch_random_affine(const float* x, float* y, float* params, int B, int C, int H, int W, const AffineSpec& s, PhiloxSeed rng,
                          cudaStream_t st) {
  if (B < 0 || C < 1 || H < 1 || W < 1) throw std::invalid_argument("random_affine: bad shape");
  if (static_cast<long long>(C) * H * W >= (1LL << 31)) throw std::invalid_argument("random_affine: an image must have fewer than 2^31 elements");
  if (B == 0) return;
  const int threads = static_cast<int>(std::min<long long>(kAffineMaxThreads, (static_cast<long long>(H) * W + 31) / 32 * 32));
  random_affine_kernel<<<B, threads, 0, st>>>(x, y, params, C, H, W, s, rng);
  check_launch("random_affine");
}

void launch_mix_batch(const float* x, const long long* labels, const float* probs, float* y, float* q, double* record, int B, int C, int H,
                      int W, int K, double alpha, bool cutmix, PhiloxSeed rng, cudaStream_t st) {
  if (B < 0 || C < 1 || H < 1 || W < 1 || K < 1) throw std::invalid_argument("mix_batch: bad shape");
  if (static_cast<long long>(C) * H * W >= (1LL << 31)) throw std::invalid_argument("mix_batch: an image must have fewer than 2^31 elements");
  if (!(alpha > 0.0)) throw std::invalid_argument("mix_batch: alpha must be positive");
  if (B == 0) return;
  mix_batch_kernel<<<B, kMixThreads, 0, st>>>(x, labels, probs, y, q, record, B, C, H, W, K, alpha, cutmix ? 1 : 0, rng);
  check_launch("mix_batch");
}

size_t elastic_smem_bytes(int H, int W) { return 3 * sizeof(float) * static_cast<size_t>(H) * W; }

void check_elastic_size(int H, int W) {
  if (H < 1 || W < 1) throw std::invalid_argument("elastic: bad shape");
  const size_t need = elastic_smem_bytes(H, W), limit = smem_optin_limit();
  if (need > limit)
    throw std::invalid_argument("elastic: a " + std::to_string(H) + "x" + std::to_string(W) + " image needs " + std::to_string(need) +
                                " bytes of shared memory (12 per pixel), above the device's opt-in limit of " + std::to_string(limit) +
                                " bytes per block");
}

void launch_elastic(const float* x, float* y, float* noise, int B, int C, int H, int W, const ElasticSpec& s, PhiloxSeed rng,
                    cudaStream_t st) {
  if (B < 0 || C < 1) throw std::invalid_argument("elastic: bad shape");
  if (static_cast<long long>(C) * H * W >= (1LL << 31)) throw std::invalid_argument("elastic: an image must have fewer than 2^31 elements");
  check_elastic_size(H, W);
  for (int c = 0; c < 2; ++c)
    if (s.k[c] != 0 && (s.k[c] < 1 || s.k[c] % 2 == 0 || s.k[c] / 2 >= H || s.k[c] / 2 >= W))
      throw std::invalid_argument("elastic: the blur needs an odd kernel size whose half is below the image's height and width");
  if (B == 0) return;
  const size_t smem = elastic_smem_bytes(H, W);
  opt_in_smem(elastic_kernel, smem);
  const int threads = static_cast<int>(std::min<long long>(kElasticMaxThreads, (static_cast<long long>(H) * W + 31) / 32 * 32));
  elastic_kernel<<<B, threads, smem, st>>>(x, y, noise, C, H, W, s, rng);
  check_launch("elastic");
}

}  // namespace pdt
