// sm_90a SIMT kernels for the ConvNet hot path (ref model: ddp_example.py:22-41) and the generic
// BatchNorm pieces behind SyncBatchNorm.  They replace what the reference dispatches to
// cuDNN/ATen: conv + bias + BN-statistics in one pass, BN-apply + ReLU +
// MaxPool in one pass (no int64 pool indices: the arg-max is recomputed in backward), fused
// log-softmax/NLL, one multi-tensor SGD launch.  All cross-CTA reductions are deterministic
// (per-CTA partials + last-CTA fold in fixed order), so runs are bit-reproducible.
// The SIMT convolution serves conv1 (1→16 channels); conv2 (16→32, 88% of the FLOPs) runs on the
// tensor-core kernels of conv_wgmma.cu.
#include <cuda_runtime.h>

#include <algorithm>
#include <stdexcept>
#include <string>

#include "cuda_utils.h"
#include "grid_fold.cuh"
#include "ops_kernels.h"

namespace pdt {

namespace {

// deterministic grid-wide fold: see grid_fold.cuh (two-level ticket tree, parallel row folds)

// =====================================================================================================
// Direct 5x5 "same" convolution, NHWC, one CTA = TH output rows of one image, all output channels.
//   thread = (pixel, group of CPT output channels); input patch planar in smem, weights [tap][ci][co].
// =====================================================================================================
template <int CIN, int COUT, int CPT, int TH, bool STATS>
__global__ void __launch_bounds__(448) conv5x5_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                      float* __restrict__ y, void* stats, ConvStats form, ReduceScratch scr, int B, int H,
                                                      int W) {
  constexpr int G = COUT / CPT;
  extern __shared__ __align__(16) float smem[];
  const int PW = W + 4, PH = TH + 4;
  float* xs = smem;                              // [CIN][PH][PW]
  float* ws = smem + CIN * PH * PW;              // [25][CIN][COUT]   (16B aligned: host pads)
  ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 15) & ~uintptr_t(15));
  float* red = ws + 25 * CIN * COUT;             // [warps][2*COUT] + [2*COUT]
  const int tiles = H / TH;
  const int n = blockIdx.x / tiles, tile = blockIdx.x % tiles;
  const int tid = threadIdx.x;

  for (int i = tid; i < 25 * CIN * COUT; i += blockDim.x) {
    const int tap = i / (CIN * COUT), ci = (i / COUT) % CIN, co = i % COUT;
    ws[i] = w[(co * CIN + ci) * 25 + tap];
  }
  for (int i = tid; i < CIN * PH * PW; i += blockDim.x) {
    const int ci = i % CIN, c = (i / CIN) % PW, r = i / (CIN * PW);
    const int ih = tile * TH + r - 2, iw = c - 2;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = x[((static_cast<size_t>(n) * H + ih) * W + iw) * CIN + ci];
    xs[(ci * PH + r) * PW + c] = v;
  }
  __syncthreads();

  const int npix = TH * W;
  const int pix = tid / G, cg = tid % G;
  const bool valid = pix < npix;
  const int py = valid ? pix / W : 0, px = valid ? pix % W : 0;
  float acc[CPT];
#pragma unroll
  for (int j = 0; j < CPT; ++j) acc[j] = bias ? bias[cg * CPT + j] : 0.f;
#pragma unroll 1
  for (int kh = 0; kh < 5; ++kh) {
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      const float* wt = ws + ((kh * 5 + kw) * CIN) * COUT + cg * CPT;
      const float* xp = xs + (py + kh) * PW + (px + kw);
#pragma unroll 4
      for (int ci = 0; ci < CIN; ++ci) {
        const float xv = xp[ci * PH * PW];
#pragma unroll
        for (int j4 = 0; j4 < CPT / 4; ++j4) {
          const float4 wv = *reinterpret_cast<const float4*>(wt + ci * COUT + j4 * 4);
          acc[j4 * 4 + 0] = fmaf(xv, wv.x, acc[j4 * 4 + 0]);
          acc[j4 * 4 + 1] = fmaf(xv, wv.y, acc[j4 * 4 + 1]);
          acc[j4 * 4 + 2] = fmaf(xv, wv.z, acc[j4 * 4 + 2]);
          acc[j4 * 4 + 3] = fmaf(xv, wv.w, acc[j4 * 4 + 3]);
        }
      }
    }
  }
  if (valid) {
    float* yp = y + ((static_cast<size_t>(n) * H + tile * TH + py) * W + px) * COUT + cg * CPT;
#pragma unroll
    for (int j4 = 0; j4 < CPT / 4; ++j4)
      *reinterpret_cast<float4*>(yp + j4 * 4) = make_float4(acc[j4 * 4], acc[j4 * 4 + 1], acc[j4 * 4 + 2], acc[j4 * 4 + 3]);
  }
  if constexpr (STATS) {
    // the CTA's per-channel sums of d = y − K and d²: K = 0 gives Σy and Σy².  Centred, K is the CTA's first pixel, and the
    // CTA's M2 = Σd² − (Σd)²/n then cancels only in proportion to ((mean − K)/std)², whatever the size of the mean
    const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    const bool centred = form != kConvSums;
    float* blk = red + nwarps * 2 * COUT;
    __shared__ float s_k[COUT];
    if (centred) {
      if (pix == 0)
#pragma unroll
        for (int j = 0; j < CPT; ++j) s_k[cg * CPT + j] = acc[j];
      __syncthreads();
    }
#pragma unroll
    for (int j = 0; j < CPT; ++j) {
      const float d = centred ? acc[j] - s_k[cg * CPT + j] : acc[j];
      float s = valid ? d : 0.f, q = valid ? d * d : 0.f;
#pragma unroll
      for (int off = G; off < 32; off <<= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, off);
        q += __shfl_xor_sync(0xffffffffu, q, off);
      }
      if (lane < G) {
        red[warp * 2 * COUT + cg * CPT + j] = s;
        red[warp * 2 * COUT + COUT + cg * CPT + j] = q;
      }
    }
    __syncthreads();
    if (tid < 2 * COUT) {
      float s = 0.f;
      for (int wi = 0; wi < nwarps; ++wi) s += red[wi * 2 * COUT + tid];
      blk[tid] = s;
    }
    __syncthreads();
    if (centred) {
      if (tid < COUT) {   // [Σd, Σd²] → [Σy, M2]
        const float sd = blk[tid], n = static_cast<float>(npix);
        blk[COUT + tid] = fmaxf(blk[COUT + tid] - sd * sd / n, 0.f);
        blk[tid] = fmaf(n, s_k[tid], sd);
      }
      __syncthreads();
    }
    const float cnt = static_cast<float>(B) * H * W;
    __shared__ float s_tmp[1024];
    __shared__ int s_flag;
    if (centred) {
      grid_fold_centred(blk, COUT, npix, B * H * W, blockIdx.x, gridDim.x, scr, s_tmp, &s_flag, tid, blockDim.x, CtaSync{},
                        [&](int i, float mean, float m2) { store_centred_stats(stats, form, COUT, i, mean, m2, cnt); });
    } else {
      float* sums = static_cast<float*>(stats);
      grid_fold(blk, 2 * COUT, blockIdx.x, gridDim.x, scr, s_tmp, &s_flag, tid, blockDim.x, CtaSync{}, [&](int i, float v) {
        sums[i] = v;
        if (i == 0) sums[2 * COUT] = cnt;
      });
    }
  }
}

// =====================================================================================================
// Weight gradient: one CTA = TH rows of one image; a lane owns one (tap,ci) pair × all COUT, the warps split the
// pixels and smem folds the warps.
// Partials [CTA][25*CIN*COUT + COUT] are folded by a second kernel (too large for a last-CTA fold).
// =====================================================================================================
template <int CIN, int COUT, int TH>
__global__ void __launch_bounds__(256) conv5x5_wgrad_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                            float* __restrict__ partials, int B, int H, int W) {
  extern __shared__ __align__(16) float smem[];
  const int PW = W + 4, PH = TH + 4, npix = TH * W;
  float* xs = smem;  // [CIN][PH][PW]
  float* dys = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(smem + CIN * PH * PW) + 15) & ~uintptr_t(15));  // [npix][COUT]
  const int tiles = H / TH;
  const int n = blockIdx.x / tiles, tile = blockIdx.x % tiles, tid = threadIdx.x;
  for (int i = tid; i < CIN * PH * PW; i += blockDim.x) {
    const int ci = i % CIN, c = (i / CIN) % PW, r = i / (CIN * PW);
    const int ih = tile * TH + r - 2, iw = c - 2;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = x[((static_cast<size_t>(n) * H + ih) * W + iw) * CIN + ci];
    xs[(ci * PH + r) * PW + c] = v;
  }
  const float* dyg = dy + (static_cast<size_t>(n) * H + tile * TH) * W * COUT;
  for (int i = tid; i < npix * COUT / 4; i += blockDim.x)
    reinterpret_cast<float4*>(dys)[i] = reinterpret_cast<const float4*>(dyg)[i];
  __syncthreads();
  constexpr int P = 25 * CIN;
  const int width = P * COUT + COUT;
  float* out = partials + static_cast<size_t>(blockIdx.x) * width;
  static_assert(P <= 32, "conv5x5_wgrad_kernel: one lane per (tap, ci) pair");
  const int lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  float acc[COUT];
#pragma unroll
  for (int j = 0; j < COUT; ++j) acc[j] = 0.f;
  if (lane < P) {
    const int tap = lane / CIN, ci = lane % CIN, kh = tap / 5, kw = tap % 5;
    for (int pix = warp; pix < npix; pix += nwarps) {
      const int py = pix / W, px = pix % W;
      const float xv = xs[(ci * PH + py + kh) * PW + px + kw];
      const float4* d4 = reinterpret_cast<const float4*>(dys + pix * COUT);
#pragma unroll
      for (int j4 = 0; j4 < COUT / 4; ++j4) {
        const float4 d = d4[j4];
        acc[j4 * 4 + 0] = fmaf(xv, d.x, acc[j4 * 4 + 0]);
        acc[j4 * 4 + 1] = fmaf(xv, d.y, acc[j4 * 4 + 1]);
        acc[j4 * 4 + 2] = fmaf(xv, d.z, acc[j4 * 4 + 2]);
        acc[j4 * 4 + 3] = fmaf(xv, d.w, acc[j4 * 4 + 3]);
      }
    }
  }
  float* fold = dys + npix * COUT;  // [nwarps][P*COUT], sized by the host
  if (lane < P)
#pragma unroll
    for (int co = 0; co < COUT; ++co) fold[(warp * P + lane) * COUT + co] = acc[co];
  __syncthreads();
  for (int i = tid; i < P * COUT; i += blockDim.x) {
    const int p = i / COUT, co = i % COUT;
    float s = 0.f;
    for (int wi = 0; wi < nwarps; ++wi) s += fold[(wi * P + p) * COUT + co];
    const int tap = p / CIN, ci = p % CIN;
    out[(co * CIN + ci) * 25 + tap] = s;
  }
  // bias gradient partial: Σ_pixels dy[:, co] — 256/COUT pixel slices in parallel, folded in slice order
  {
    __shared__ float s_db[256];
    constexpr int SL = 256 / COUT;
    const int co = tid % COUT, sl = tid / COUT;
    float s = 0.f;
    if (tid < 256)
      for (int pix = sl; pix < npix; pix += SL) s += dys[pix * COUT + co];
    __syncthreads();
    if (tid < 256) s_db[tid] = s;
    __syncthreads();
    if (tid < COUT) {
      float tot = 0.f;
      for (int k = 0; k < SL; ++k) tot += s_db[k * COUT + tid];
      out[P * COUT + tid] = tot;
    }
  }
}

// =====================================================================================================
// conv1's data gradient (COUT→1), the transposed 5x5 convolution dx[h][w] = Σ_{kh,kw,co} dy[h+2−kh][w+2−kw][co]·w[co][kh][kw].
// One CTA = TH rows of one image, one thread per dx pixel; the dy patch planar in smem (zero halo), the flipped filter [tap][co].
// A pixel is one thread's chain of 25·COUT fmaf in a fixed order (taps row-major, channels inner), with no reduction across
// threads or CTAs: the result does not depend on B or the launch, and repeats bit for bit.
// =====================================================================================================
template <int COUT, int TH>
__global__ void __launch_bounds__(448) conv5x5_dgrad_cin1_kernel(const float* __restrict__ dy, const float* __restrict__ w,
                                                                 float* __restrict__ dx, int H, int W) {
  extern __shared__ __align__(16) float smem[];
  const int PW = W + 4, PH = TH + 4;
  float* ds = smem;                    // [COUT][PH][PW]: patch row r is dy row tile·TH + r − 2
  float* ws = smem + COUT * PH * PW;   // [25][COUT]: ws[(fh·5 + fw)·COUT + co] = w[co][4−fh][4−fw]
  const int tiles = H / TH;
  const int n = blockIdx.x / tiles, tile = blockIdx.x % tiles, tid = threadIdx.x;
  for (int i = tid; i < 25 * COUT; i += blockDim.x) {
    const int tap = i / COUT, co = i % COUT;
    ws[i] = w[co * 25 + 24 - tap];
  }
  for (int i = tid; i < COUT * PH * PW; i += blockDim.x) {
    const int co = i % COUT, c = (i / COUT) % PW, r = i / (COUT * PW);
    const int ih = tile * TH + r - 2, iw = c - 2;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = dy[((static_cast<size_t>(n) * H + ih) * W + iw) * COUT + co];
    ds[(co * PH + r) * PW + c] = v;
  }
  __syncthreads();
  if (tid >= TH * W) return;
  const int py = tid / W, px = tid % W;
  float acc = 0.f;
#pragma unroll 1
  for (int fh = 0; fh < 5; ++fh) {
#pragma unroll
    for (int fw = 0; fw < 5; ++fw) {
      const float* wt = ws + (fh * 5 + fw) * COUT;
      const float* dp = ds + (py + fh) * PW + px + fw;   // dy row tile·TH + py + 2 − kh with kh = 4 − fh
#pragma unroll
      for (int co = 0; co < COUT; ++co) acc = fmaf(dp[co * PH * PW], wt[co], acc);
    }
  }
  dx[(static_cast<size_t>(n) * H + tile * TH + py) * W + px] = acc;
}

// out[i] = Σ_b partials[b][i] in a fixed order: a CTA owns 32 outputs (lane = output), its 8 warps
// stride over the partial rows (coalesced 128-byte reads), then the 8 sub-sums are added in warp order.
__global__ void __launch_bounds__(256) fold_partials_kernel(const float* __restrict__ partials, int nblk, int width, int split,
                                                            float* out_a, float* out_b) {
  __shared__ float s_sub[8][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + lane;
  float s0 = 0.f, s1 = 0.f;
  if (i < width) {
    int b = warp;
    for (; b + 8 < nblk; b += 16) {
      s0 += partials[static_cast<size_t>(b) * width + i];
      s1 += partials[static_cast<size_t>(b + 8) * width + i];
    }
    if (b < nblk) s0 += partials[static_cast<size_t>(b) * width + i];
  }
  s_sub[warp][lane] = s0 + s1;
  __syncthreads();
  if (warp == 0 && i < width) {
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) s += s_sub[w8][lane];
    if (i < split) out_a[i] = s;
    else if (out_b) out_b[i - split] = s;
  }
}

// =====================================================================================================
// BatchNorm(train) + ReLU + MaxPool 2x2
// =====================================================================================================
// The batch mean and variance (biased) of channel c from stats in the form `form` (BnStats).  kBnSums' E[y²] − mean² in fp32
// cancels the variance's digits when |mean| ≫ std; it stays as the plain-sums form of the kernels.  The centred form (M2 about the
// mean), the eval form (the running statistics as they are) and SyncBatchNorm's fp64 sums, whose E[y²] − mean² in fp64 keeps the
// variance to about 1e-16·mean²/var, have no such cancellation.
__device__ __forceinline__ void bn_mean_var(const void* stats, int C, int c, int form, float* mean, float* var) {
  if (form == kBnSums64) {
    const double* s = static_cast<const double*>(stats);
    const double n = fmax(s[2 * C], 1.0), m = s[c] / n;
    *mean = static_cast<float>(m);
    *var = static_cast<float>(fmax(s[C + c] / n - m * m, 0.0));
    return;
  }
  const float* s = static_cast<const float*>(stats);
  if (form == kBnMeanVar) {
    *mean = s[c];
    *var = s[C + c];
    return;
  }
  const float n = fmaxf(s[2 * C], 1.f);
  *mean = form == kBnSums ? s[c] / n : s[c];
  *var = form == kBnCentred ? s[C + c] / n : fmaxf(s[C + c] / n - *mean * *mean, 0.f);
}

// the element count per channel (every form but kBnMeanVar)
__device__ __forceinline__ float bn_stats_count(const void* stats, int C, int form) {
  return form == kBnSums64 ? static_cast<float>(static_cast<const double*>(stats)[2 * C]) : static_cast<const float*>(stats)[2 * C];
}

__device__ __forceinline__ void bn_coeffs(const void* stats, const float* gamma, const float* beta, float eps, int C, int form,
                                          float* s_scale, float* s_shift, float* s_mean, float* s_invstd) {
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float mean, var;
    bn_mean_var(stats, C, c, form, &mean, &var);
    const float invstd = rsqrtf(var + eps);
    const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
    s_mean[c] = mean;
    s_invstd[c] = invstd;
    s_scale[c] = g * invstd;
    s_shift[c] = b - mean * g * invstd;
  }
}

__global__ void __launch_bounds__(256) bn_relu_pool_fwd_kernel(const float* __restrict__ y, const void* __restrict__ stats,
                                                               const float* __restrict__ gamma, const float* __restrict__ beta,
                                                               float* __restrict__ out, float* saved, float* running_mean,
                                                               float* running_var, long long* nbt, float momentum, float eps, int B,
                                                               int H, int W, int C, int out_nchw, int form) {
  __shared__ float s_scale[64], s_shift[64], s_mean[64], s_invstd[64];
  bn_coeffs(stats, gamma, beta, eps, C, form, s_scale, s_shift, s_mean, s_invstd);
  __syncthreads();
  if (blockIdx.x == 0) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      saved[c] = s_mean[c];
      saved[C + c] = s_invstd[c];
      if (running_mean) {
        const float n = fmaxf(bn_stats_count(stats, C, form), 1.f);
        float mean, var;
        bn_mean_var(stats, C, c, form, &mean, &var);
        const float unbiased = var * (n / fmaxf(n - 1.f, 1.f));
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * s_mean[c];
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
      }
    }
    if (threadIdx.x == 0) {
      if (nbt) *nbt += 1;
      if (form == kBnSums64) saved[2 * C] = bn_stats_count(stats, C, form);   // the group's count, for the backward
    }
  }
  const int Q = C / 4, PH = H / 2, PW = W / 2;
  const long long total = static_cast<long long>(B) * PH * PW * Q;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int cq = static_cast<int>(idx % Q);
  const long long pp = idx / Q;
  const int pw = static_cast<int>(pp % PW), ph = static_cast<int>((pp / PW) % PH), n = static_cast<int>(pp / (static_cast<long long>(PW) * PH));
  const float4 sc = *reinterpret_cast<const float4*>(s_scale + cq * 4), sh = *reinterpret_cast<const float4*>(s_shift + cq * 4);
  float4 m = make_float4(0.f, 0.f, 0.f, 0.f);  // relu floor doubles as the max identity
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const int ih = 2 * ph + (d >> 1), iw = 2 * pw + (d & 1);
    const float4 v = *reinterpret_cast<const float4*>(y + ((static_cast<size_t>(n) * H + ih) * W + iw) * C + cq * 4);
    m.x = fmaxf(m.x, fmaf(v.x, sc.x, sh.x));
    m.y = fmaxf(m.y, fmaf(v.y, sc.y, sh.y));
    m.z = fmaxf(m.z, fmaf(v.z, sc.z, sh.z));
    m.w = fmaxf(m.w, fmaf(v.w, sc.w, sh.w));
  }
  if (out_nchw) {
    const size_t plane = static_cast<size_t>(PH) * PW;
    float* o = out + (static_cast<size_t>(n) * C + cq * 4) * plane + static_cast<size_t>(ph) * PW + pw;
    o[0] = m.x; o[plane] = m.y; o[2 * plane] = m.z; o[3 * plane] = m.w;
  } else {
    *reinterpret_cast<float4*>(out + pp * C + cq * 4) = m;
  }
}

// arg-max of the four BN outputs of one channel (first maximum wins, like torch's max_pool2d);
// returns the routed gradient (0 when ReLU clipped) and x̂ at the arg-max.
__device__ __forceinline__ void route(const float v[4], float scale, float shift, float mean, float invstd, float g, int* arg, float* dz,
                                      float* xhat) {
  float best = fmaf(v[0], scale, shift);
  int a = 0;
#pragma unroll
  for (int d = 1; d < 4; ++d) {
    const float z = fmaf(v[d], scale, shift);
    if (z > best) { best = z; a = d; }
  }
  *arg = a;
  *dz = best > 0.f ? g : 0.f;
  *xhat = (v[a] - mean) * invstd;
}

// MEAN_VAR (APPLY only): the forward normalised with kBnMeanVar statistics, which are constants of the graph, so the apply pass has
// no batch-mean terms and reads neither sums nor count.
template <bool APPLY, bool MEAN_VAR = false>
__global__ void __launch_bounds__(256) bn_relu_pool_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ y,
                                                               const float* __restrict__ saved, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float* sums, float* dgamma,
                                                               float* dbeta, const float* count, float* __restrict__ dy, int B, int H,
                                                               int W, int C, int dout_nchw, ReduceScratch scr) {
  __shared__ float s_scale[64], s_shift[64], s_mean[64], s_invstd[64], s_m1[64], s_m2[64];
  __shared__ float s_red[8 * 128 + 128];
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float mean = saved[c], invstd = saved[C + c];
    const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
    s_mean[c] = mean;
    s_invstd[c] = invstd;
    s_scale[c] = g * invstd;
    s_shift[c] = b - mean * g * invstd;
    if (APPLY && !MEAN_VAR) {
      const float n = fmaxf(*count, 1.f);
      s_m1[c] = sums[c] / n;
      s_m2[c] = sums[C + c] / n;
    }
  }
  __syncthreads();
  const int Q = C / 4, PH = H / 2, PW = W / 2;
  const long long total = static_cast<long long>(B) * PH * PW * Q;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool valid = idx < total;
  const int cq = static_cast<int>(threadIdx.x % Q);  // blockDim % Q == 0 ⇒ equals idx % Q
  float a1[4] = {0.f, 0.f, 0.f, 0.f}, a2[4] = {0.f, 0.f, 0.f, 0.f};
  if (valid) {
    const long long pp = idx / Q;
    const int pw = static_cast<int>(pp % PW), ph = static_cast<int>((pp / PW) % PH), n = static_cast<int>(pp / (static_cast<long long>(PW) * PH));
    float g4[4];
    if (dout_nchw) {
      const size_t plane = static_cast<size_t>(PH) * PW;
      const float* o = dout + (static_cast<size_t>(n) * C + cq * 4) * plane + static_cast<size_t>(ph) * PW + pw;
      g4[0] = o[0]; g4[1] = o[plane]; g4[2] = o[2 * plane]; g4[3] = o[3 * plane];
    } else {
      const float4 t = *reinterpret_cast<const float4*>(dout + pp * C + cq * 4);
      g4[0] = t.x; g4[1] = t.y; g4[2] = t.z; g4[3] = t.w;
    }
    float4 v4[4];
    size_t off[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      off[d] = ((static_cast<size_t>(n) * H + 2 * ph + (d >> 1)) * W + 2 * pw + (d & 1)) * C + cq * 4;
      v4[d] = *reinterpret_cast<const float4*>(y + off[d]);
    }
    float4 o4[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = cq * 4 + k;
      const float v[4] = {reinterpret_cast<const float*>(&v4[0])[k], reinterpret_cast<const float*>(&v4[1])[k],
                          reinterpret_cast<const float*>(&v4[2])[k], reinterpret_cast<const float*>(&v4[3])[k]};
      int arg;
      float dz, xhat;
      route(v, s_scale[c], s_shift[c], s_mean[c], s_invstd[c], g4[k], &arg, &dz, &xhat);
      if constexpr (!APPLY) {
        a1[k] = dz;
        a2[k] = dz * xhat;
      } else if constexpr (MEAN_VAR) {
        // dy = γ·invstd·dz at the arg-max, 0 at the window's other positions
#pragma unroll
        for (int d = 0; d < 4; ++d) reinterpret_cast<float*>(&o4[d])[k] = d == arg ? s_scale[c] * dz : 0.f;
      } else {
        // dy = γ·invstd·(dz_pos − mean(dz) − x̂_pos·mean(dz·x̂)) at every position of the window
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          const float xh = (v[d] - s_mean[c]) * s_invstd[c];
          const float dzp = (d == arg) ? dz : 0.f;
          reinterpret_cast<float*>(&o4[d])[k] = s_scale[c] * (dzp - s_m1[c] - xh * s_m2[c]);
        }
      }
    }
    if constexpr (APPLY) {
#pragma unroll
      for (int d = 0; d < 4; ++d) *reinterpret_cast<float4*>(dy + off[d]) = o4[d];
    }
  }
  if constexpr (!APPLY) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float s = a1[k], q = a2[k];
      for (int off = Q; off < 32; off <<= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, off);
        q += __shfl_xor_sync(0xffffffffu, q, off);
      }
      if (lane < Q) {
        s_red[warp * 2 * C + cq * 4 + k] = s;
        s_red[warp * 2 * C + C + cq * 4 + k] = q;
      }
    }
    __syncthreads();
    float* blk = s_red + nwarps * 2 * C;
    if (threadIdx.x < 2 * C) {
      float s = 0.f;
      for (int wi = 0; wi < nwarps; ++wi) s += s_red[wi * 2 * C + threadIdx.x];
      blk[threadIdx.x] = s;
    }
    __syncthreads();
    __shared__ float s_tmp[256];
    __shared__ int s_flag;
    grid_fold(blk, 2 * C, blockIdx.x, gridDim.x, scr, s_tmp, &s_flag, threadIdx.x, blockDim.x, CtaSync{}, [&](int i, float v) {
      sums[i] = v;
      if (i < C) { if (dbeta) dbeta[i] = v; }
      else if (dgamma) dgamma[i - C] = v;
    });
  }
}

// =====================================================================================================
// Generic NCHW BatchNorm pieces
// =====================================================================================================
__global__ void __launch_bounds__(256) bn_bwd_reduce_nchw_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                 const float* __restrict__ mean, const float* __restrict__ invstd,
                                                                 float* out, int N, int C, int HW, int S, ReduceScratch scr) {
  // Σdy, Σdy·(x-μ) of channel c over slice s
  const int c = blockIdx.x / S, s = blockIdx.x % S;
  const long long total = static_cast<long long>(N) * HW;
  const long long chunk = (total + S - 1) / S;
  const long long lo = chunk * s, hi = min(total, lo + chunk);
  const float mu = mean[c];
  float s1 = 0.f, s2 = 0.f;
  for (long long e = lo + threadIdx.x; e < hi; e += blockDim.x) {
    const long long n = e / HW, hw = e % HW;
    const size_t off = (static_cast<size_t>(n) * C + c) * HW + hw;
    const float d = dy[off];
    s1 += d;
    s2 += d * (x[off] - mu);
  }
  __shared__ float r1[8], r2[8], blk[2];
  for (int off = 16; off > 0; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  if ((threadIdx.x & 31) == 0) { r1[threadIdx.x >> 5] = s1; r2[threadIdx.x >> 5] = s2; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float t1 = 0.f, t2 = 0.f;
    for (int wi = 0; wi < (blockDim.x >> 5); ++wi) { t1 += r1[wi]; t2 += r2[wi]; }
    blk[0] = t1; blk[1] = t2;
  }
  __syncthreads();
  // fold: partial index = block → (c, s); the last CTA folds per channel in slice order
  __shared__ int s_last;
  if (threadIdx.x < 2) scr.partials[static_cast<size_t>(blockIdx.x) * 2 + threadIdx.x] = blk[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(scr.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    float t1 = 0.f, t2 = 0.f;
    for (int k = 0; k < S; ++k) {
      t1 += __ldcg(&scr.partials[(static_cast<size_t>(ch) * S + k) * 2]);
      t2 += __ldcg(&scr.partials[(static_cast<size_t>(ch) * S + k) * 2 + 1]);
    }
    out[ch] = t1;                        // Σdy
    out[C + ch] = t2;                    // Σdy·(x-μ)
    out[2 * C + ch] = t2 * invstd[ch];   // dγ
    out[3 * C + ch] = t1;                // dβ
  }
  if (threadIdx.x == 0) *scr.counter = 0u;
}

// Forward statistics in fp64: Σx, Σx² of channel c.  Downstream computes var = E[x²] − μ², which
// amplifies the rounding of the two sums by μ²/σ²; fp32 sums made first-step gradients of a
// SyncBN ResNet-18 differ from torch's (Welford) by up to 1 %, fp64 sums
// (and an fp64 exchange between ranks) bring that to 1e-5.  The kernel is bandwidth-bound either way.
__global__ void __launch_bounds__(256) bn_stats_nchw_f64_kernel(const float* __restrict__ x, double* out, int N, int C, int HW, int S,
                                                                ReduceScratch scr) {
  const int c = blockIdx.x / S, s = blockIdx.x % S;
  const long long total = static_cast<long long>(N) * HW;
  const long long chunk = (total + S - 1) / S;
  const long long lo = chunk * s, hi = min(total, lo + chunk);
  double s1 = 0.0, s2 = 0.0;
  for (long long e = lo + threadIdx.x; e < hi; e += blockDim.x) {
    const long long n = e / HW, hw = e % HW;
    const double v = static_cast<double>(x[(static_cast<size_t>(n) * C + c) * HW + hw]);
    s1 += v;
    s2 = fma(v, v, s2);
  }
  __shared__ double r1[8], r2[8];
  for (int off = 16; off > 0; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  if ((threadIdx.x & 31) == 0) { r1[threadIdx.x >> 5] = s1; r2[threadIdx.x >> 5] = s2; }
  __syncthreads();
  double* parts = reinterpret_cast<double*>(scr.partials);
  if (threadIdx.x == 0) {
    double t1 = 0.0, t2 = 0.0;
    for (int wi = 0; wi < (blockDim.x >> 5); ++wi) { t1 += r1[wi]; t2 += r2[wi]; }
    parts[static_cast<size_t>(blockIdx.x) * 2] = t1;
    parts[static_cast<size_t>(blockIdx.x) * 2 + 1] = t2;
  }
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(scr.counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int ch = threadIdx.x; ch < C; ch += blockDim.x) {
    double t1 = 0.0, t2 = 0.0;
    for (int k = 0; k < S; ++k) {
      t1 += __ldcg(&parts[(static_cast<size_t>(ch) * S + k) * 2]);
      t2 += __ldcg(&parts[(static_cast<size_t>(ch) * S + k) * 2 + 1]);
    }
    out[ch] = t1;
    out[C + ch] = t2;
    if (ch == 0) out[2 * C] = static_cast<double>(total);
  }
  if (threadIdx.x == 0) *scr.counter = 0u;
}

// All-reduced fp64 statistics → mean, invstd (fp32) and the running-statistics update, in one launch instead of the
// ≈15 elementwise ATen kernels the same arithmetic costs in Python (generic SyncBatchNorm forward; opt-in for now).
__global__ void bn_finalize_kernel(const double* __restrict__ stats, int C, double eps, float momentum, float* __restrict__ mean,
                                   float* __restrict__ invstd, float* __restrict__ count_out, float* running_mean, float* running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = fmax(stats[2 * C], 1.0);
  const double m = stats[c] / n;
  const double var = fmax(stats[C + c] / n - m * m, 0.0);
  mean[c] = static_cast<float>(m);
  invstd[c] = static_cast<float>(rsqrt(var + eps));
  if (c == 0) count_out[0] = static_cast<float>(stats[2 * C]);
  if (running_mean) {
    const double unbiased = var * (n / fmax(n - 1.0, 1.0));
    running_mean[c] = running_mean[c] * (1.f - momentum) + static_cast<float>(m) * momentum;
    running_var[c] = running_var[c] * (1.f - momentum) + static_cast<float>(unbiased) * momentum;
  }
}

__global__ void bn_apply_nchw_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ invstd,
                                     const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ out,
                                     long long total, int C, int HW) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>((i / HW) % C);
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  out[i] = (x[i] - mean[c]) * invstd[c] * g + b;
}

__global__ void bn_bwd_apply_nchw_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                         const float* __restrict__ invstd, const float* __restrict__ gamma,
                                         const float* __restrict__ mean_dy, const float* __restrict__ mean_dy_xmu, float* __restrict__ dx,
                                         long long total, int C, int HW) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>((i / HW) % C);
  const float is = invstd[c], g = gamma ? gamma[c] : 1.f;
  dx[i] = (dy[i] - mean_dy[c] - (x[i] - mean[c]) * is * is * mean_dy_xmu[c]) * is * g;
}

// =====================================================================================================
// Linear + cross entropy
// =====================================================================================================
// out[row, n] = Σ_k x[row, k] w[n, k] + b[n].  A CTA owns R rows so every weight element it loads is
// reused R times (25 CTAs re-read the 62 KB weight matrix instead of 100), threads split K.
template <int NMAX, int R>
__global__ void __launch_bounds__(256) linear_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ b, float* __restrict__ out, int B, int K, int N) {
  const int row0 = blockIdx.x * R;
  float acc[R][NMAX];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int n = 0; n < NMAX; ++n) acc[r][n] = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float wv[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) wv[n] = n < N ? w[static_cast<size_t>(n) * K + k] : 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float xv = (row0 + r < B) ? x[static_cast<size_t>(row0 + r) * K + k] : 0.f;
#pragma unroll
      for (int n = 0; n < NMAX; ++n) acc[r][n] = fmaf(xv, wv[n], acc[r][n]);
    }
  }
  __shared__ float red[8][R * NMAX];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int n = 0; n < NMAX; ++n) {
      float v = acc[r][n];
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) red[warp][r * NMAX + n] = v;
    }
  __syncthreads();
  if (threadIdx.x < R * NMAX) {
    const int r = threadIdx.x / NMAX, n = threadIdx.x % NMAX;
    if (n < N && row0 + r < B) {
      float s = b ? b[n] : 0.f;
      for (int wi = 0; wi < (blockDim.x >> 5); ++wi) s += red[wi][threadIdx.x];
      out[static_cast<size_t>(row0 + r) * N + n] = s;
    }
  }
}

template <int NMAX>
__global__ void __launch_bounds__(256) linear_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ x,
                                                         const float* __restrict__ w, float* __restrict__ dx, float* __restrict__ dw,
                                                         float* __restrict__ db, int B, int K, int N, int dx_blocks) {
  if (static_cast<int>(blockIdx.x) < dx_blocks) {
    // dx[row, k] = Σ_n dout[row, n] w[n, k]
    if (!dx) return;
    const int row = blockIdx.x;
    float d[NMAX];
#pragma unroll
    for (int n = 0; n < NMAX; ++n) d[n] = n < N ? dout[static_cast<size_t>(row) * N + n] : 0.f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
      float s = 0.f;
#pragma unroll
      for (int n = 0; n < NMAX; ++n)
        if (n < N) s = fmaf(d[n], w[static_cast<size_t>(n) * K + k], s);
      dx[static_cast<size_t>(row) * K + k] = s;
    }
    return;
  }
  // dw[n, k] = Σ_b dout[b, n] x[b, k]: a CTA owns a slab of 32 k-columns (lane = column); its 8 warps
  // split the batch rows (8-way shorter dependency chain than one thread per column), the 8 sub-sums
  // are folded in warp order.  Batch is staged through smem in chunks of BC rows.
  extern __shared__ float s_d[];  // [BC][N]
  __shared__ float s_fold[8][NMAX][32];  // lane-contiguous: conflict-free stores and loads
  constexpr int BC = 128;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int k = (blockIdx.x - dx_blocks) * 32 + lane;
  float acc[NMAX];
#pragma unroll
  for (int n = 0; n < NMAX; ++n) acc[n] = 0.f;
  float bsum = 0.f;  // used by the first dw CTA for db
  for (int b0 = 0; b0 < B; b0 += BC) {
    const int nb = min(BC, B - b0);
    __syncthreads();
    for (int i = threadIdx.x; i < nb * N; i += blockDim.x) s_d[i] = dout[static_cast<size_t>(b0) * N + i];
    __syncthreads();
    if (k < K) {
      float xv[BC / 8];   // this warp's rows of the chunk: every load is issued before the first FMA needs one
#pragma unroll
      for (int j = 0; j < BC / 8; ++j) {
        const int b = warp + 8 * j;
        xv[j] = b < nb ? x[static_cast<size_t>(b0 + b) * K + k] : 0.f;
      }
#pragma unroll
      for (int j = 0; j < BC / 8; ++j) {
        const int b = warp + 8 * j;
        if (b < nb) {
#pragma unroll
          for (int n = 0; n < NMAX; ++n)
            if (n < N) acc[n] = fmaf(xv[j], s_d[b * N + n], acc[n]);
        }
      }
    }
    if (static_cast<int>(blockIdx.x) == dx_blocks && threadIdx.x < N)
      for (int b = 0; b < nb; ++b) bsum += s_d[b * N + threadIdx.x];
  }
#pragma unroll
  for (int n = 0; n < NMAX; ++n) s_fold[warp][n][lane] = acc[n];
  __syncthreads();
  // 32 columns × N outputs folded by the CTA's threads
  for (int i = threadIdx.x; i < 32 * N; i += blockDim.x) {
    const int n = i / 32, l = i % 32;
    const int kk = (blockIdx.x - dx_blocks) * 32 + l;
    if (kk < K) {
      float s = 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) s += s_fold[w8][n][l];
      dw[static_cast<size_t>(n) * K + kk] = s;
    }
  }
  if (db && static_cast<int>(blockIdx.x) == dx_blocks && threadIdx.x < N) db[threadIdx.x] = bsum;
}

// Rows whose target lies in [0, C), counted by every thread of the block (ignore_index: torch's mean is over these rows only).
__device__ __forceinline__ int ce_counted_rows(const long long* __restrict__ target, int B, int C) {
  int n = 0;
  for (int r0 = 0; r0 < B; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    const long long t = r < B ? target[r] : -1;
    n += __syncthreads_count(t >= 0 && t < C);
  }
  return n;
}

// emit_grad: write d(loss)/d(logits) = (softmax − onehot)/n instead of the softmax — the whole backward of a mean
// cross-entropy whose incoming gradient is 1, produced by the forward launch (the backward kernel disappears).
// Ignored rows (target outside [0, C)) add no loss term and get a zero gradient; n counts the others (0 ⇒ NaN loss, as torch).
__global__ void __launch_bounds__(256) cross_entropy_fwd_kernel(const float* __restrict__ logits, const long long* __restrict__ target,
                                                                float* loss, float* __restrict__ probs, int B, int C, int emit_grad) {
  float local = 0.f;
  const int counted = ce_counted_rows(target, B, C);
  const float invN = 1.f / static_cast<float>(counted);
  for (int r = threadIdx.x; r < B; r += blockDim.x) {
    const float* l = logits + static_cast<size_t>(r) * C;
    float m = l[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, l[c]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += __expf(l[c] - m);
    const float inv = 1.f / s, lse = m + __logf(s);
    const long long t = target[r];
    const bool counted_row = t >= 0 && t < C;
    for (int c = 0; c < C; ++c) {
      const float p = __expf(l[c] - m) * inv;
      probs[static_cast<size_t>(r) * C + c] = !emit_grad ? p : counted_row ? (p - (t == c ? 1.f : 0.f)) * invN : 0.f;
    }
    if (counted_row) local += lse - l[t];
  }
  // fixed-order block reduction (deterministic)
  __shared__ float red[256];
  red[threadIdx.x] = local;
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss = red[0] / static_cast<float>(counted);
}

__global__ void __launch_bounds__(256) cross_entropy_bwd_kernel(const float* __restrict__ probs, const long long* __restrict__ target,
                                                                const float* __restrict__ dloss, float* __restrict__ dlogits, int B, int C) {
  const int counted = ce_counted_rows(target, B, C);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int r = i / C, c = i % C;
  const long long t = target[r];
  const float g = (dloss ? *dloss : 1.f) / static_cast<float>(counted);
  dlogits[i] = (t >= 0 && t < C) ? (probs[i] - (t == c ? 1.f : 0.f)) * g : 0.f;
}

// ---- the same with a CeSpec (class weights, label smoothing, any ignore_index, sum or mean) ------------------------------------
__device__ __forceinline__ bool ce_spec_counted(long long t, int C, const CeSpec& s) { return t >= 0 && t < C && t != s.ignore_index; }

// Σ of v over the 256 threads of the block in a fixed order (every thread gets the same bits); red: 256 floats of shared memory
__device__ float ce_block_sum(float v, float* red) {
  __syncthreads();
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const float r = red[0];
  __syncthreads();
  return r;
}

// The divisor D (Σ_{counted} w_t for the mean, 1 for the sum) and W = Σ_c w_c, the same bits in every block and in both kernels
__device__ __forceinline__ void ce_spec_sums(const long long* __restrict__ target, int B, int C, const CeSpec& s, float* red, float& D,
                                             float& W) {
  float d = 0.f, w = 0.f;
  if (!s.sum) {
    for (int r = threadIdx.x; r < B; r += blockDim.x) {
      const long long t = target[r];
      if (ce_spec_counted(t, C, s)) d += s.weight ? s.weight[t] : 1.f;
    }
  }
  if (s.weight)
    for (int c = threadIdx.x; c < C; c += blockDim.x) w += s.weight[c];
  D = s.sum ? 1.f : ce_block_sum(d, red);
  W = s.weight ? ce_block_sum(w, red) : static_cast<float>(C);
}

// acc (accumulate mode, probs == nullptr, a mean spec): instead of the loss, thread 0 adds the block's Σ loss terms, D, the
// counted rows whose argmax (torch.argmax's: the first maximal index, a NaN counting as the maximum) is the target, and the
// counted rows to acc[0..3]: plain fp64 adds, ordered by the stream, so the totals are the same bits from run to run.
__global__ void __launch_bounds__(256) cross_entropy_fwd_spec_kernel(const float* __restrict__ logits, const long long* __restrict__ target,
                                                                     float* loss, float* __restrict__ probs, int B, int C, int emit_grad,
                                                                     CeSpec s, double* acc) {
  __shared__ float red[256];
  __shared__ int s_counts[2];   // hits, counted rows (accumulate mode)
  float D, W;
  ce_spec_sums(target, B, C, s, red, D, W);
  const float keep = 1.f - s.smoothing, eps_c = s.smoothing / static_cast<float>(C);
  float local = 0.f;
  int hits = 0, counted = 0;
  for (int r = threadIdx.x; r < B; r += blockDim.x) {
    const float* l = logits + static_cast<size_t>(r) * C;
    float m = l[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, l[c]);
    float sx = 0.f;
    for (int c = 0; c < C; ++c) sx += __expf(l[c] - m);
    const float inv = 1.f / sx, lse = m + __logf(sx);
    const long long t = target[r];
    const bool counted_row = ce_spec_counted(t, C, s);
    const float wt = counted_row ? (s.weight ? s.weight[t] : 1.f) : 0.f;
    float smooth = 0.f;   // Σ_c w_c·(lse − l_c): every term non-negative
    for (int c = 0; c < C; ++c) {
      const float lc = l[c], wc = s.weight ? s.weight[c] : 1.f;
      const float p = __expf(lc - m) * inv;
      smooth += wc * (lse - lc);
      if (probs)
        probs[static_cast<size_t>(r) * C + c] =
            !emit_grad ? p : counted_row ? (keep * wt * (p - (t == c ? 1.f : 0.f)) + eps_c * (W * p - wc)) / D : 0.f;
    }
    if (counted_row) local += keep * wt * (lse - l[t]) + eps_c * smooth;
    if (acc && counted_row) {
      int top = 0;
      float best = l[0];
      for (int c = 1; c < C; ++c)
        if (l[c] > best || (isnan(l[c]) && !isnan(best))) best = l[c], top = c;
      hits += top == t;
      ++counted;
    }
  }
  const float total = ce_block_sum(local, red);
  if (acc) {
    if (threadIdx.x == 0) s_counts[0] = s_counts[1] = 0;
    __syncthreads();
    atomicAdd(&s_counts[0], hits);   // integer sums: the same whatever the order
    atomicAdd(&s_counts[1], counted);
    __syncthreads();
    if (threadIdx.x == 0) {
      acc[0] += static_cast<double>(total);
      acc[1] += static_cast<double>(D);
      acc[2] += static_cast<double>(s_counts[0]);
      acc[3] += static_cast<double>(s_counts[1]);
    }
    return;
  }
  // a mean over zero total weight is NaN, as torch's, also when the smoothing terms of zero-weight rows make the sum positive
  if (threadIdx.x == 0) *loss = (D == 0.f ? 0.f : total) / D;
}

__global__ void __launch_bounds__(256) cross_entropy_bwd_spec_kernel(const float* __restrict__ probs, const long long* __restrict__ target,
                                                                     const float* __restrict__ dloss, float* __restrict__ dlogits, int B, int C,
                                                                     CeSpec s) {
  __shared__ float red[256];
  float D, W;
  ce_spec_sums(target, B, C, s, red, D, W);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * C) return;
  const int r = i / C, c = i % C;
  const long long t = target[r];
  if (!ce_spec_counted(t, C, s)) {
    dlogits[i] = 0.f;
    return;
  }
  const float keep = 1.f - s.smoothing, eps_c = s.smoothing / static_cast<float>(C);
  const float wt = s.weight ? s.weight[t] : 1.f, wc = s.weight ? s.weight[c] : 1.f, p = probs[i];
  const float g = (dloss ? *dloss : 1.f) / D;
  dlogits[i] = (keep * wt * (p - (t == c ? 1.f : 0.f)) + eps_c * (W * p - wc)) * g;
}

// ---- class-probability targets (ops_kernels.h: launch_cross_entropy_fwd_soft) ---------------------------------------------------
// w_c·q'_c with q' = q·(1−ε) + ε/C, torch's smoothing of a probability target
__device__ __forceinline__ float ce_soft_a(const float* __restrict__ qr, int c, const CeSpec& s, float keep, float eps_c) {
  return (s.weight ? s.weight[c] : 1.f) * (qr[c] * keep + eps_c);
}

// One thread per row: the row's term Σ_c a_c·(lse − l_c), a_c = w_c·q'_c, and S = Σ_c a_c in class order; emit_grad as in
// cross_entropy_fwd_kernel, with the gradient (p_c·S − a_c) / D.
__global__ void __launch_bounds__(256) cross_entropy_fwd_soft_kernel(const float* __restrict__ logits, const float* __restrict__ q,
                                                                     float* loss, float* __restrict__ probs, int B, int C, int emit_grad,
                                                                     CeSpec s) {
  __shared__ float red[256];
  const float D = s.sum ? 1.f : static_cast<float>(B);
  const float keep = 1.f - s.smoothing, eps_c = s.smoothing / static_cast<float>(C);
  float local = 0.f;
  for (int r = threadIdx.x; r < B; r += blockDim.x) {
    const float* l = logits + static_cast<size_t>(r) * C;
    const float* qr = q + static_cast<size_t>(r) * C;
    float m = l[0];
    for (int c = 1; c < C; ++c) m = fmaxf(m, l[c]);
    float sx = 0.f;
    for (int c = 0; c < C; ++c) sx += __expf(l[c] - m);
    const float inv = 1.f / sx, lse = m + __logf(sx);
    float S = 0.f, term = 0.f;
    for (int c = 0; c < C; ++c) {
      const float a = ce_soft_a(qr, c, s, keep, eps_c);
      S += a;
      term += a * (lse - l[c]);
    }
    for (int c = 0; c < C; ++c) {
      const float p = __expf(l[c] - m) * inv;
      probs[static_cast<size_t>(r) * C + c] = !emit_grad ? p : (p * S - ce_soft_a(qr, c, s, keep, eps_c)) / D;
    }
    local += term;
  }
  const float total = ce_block_sum(local, red);
  if (threadIdx.x == 0) *loss = total / D;   // an empty batch's mean is 0 / 0 = NaN, as torch's
}

// One thread per row: S in the forward kernel's order, then dlogits = (p_c·S − a_c) · dloss / D
__global__ void __launch_bounds__(256) cross_entropy_bwd_soft_kernel(const float* __restrict__ probs, const float* __restrict__ q,
                                                                     const float* __restrict__ dloss, float* __restrict__ dlogits, int B, int C,
                                                                     CeSpec s) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B) return;
  const float keep = 1.f - s.smoothing, eps_c = s.smoothing / static_cast<float>(C);
  const float* qr = q + static_cast<size_t>(r) * C;
  float S = 0.f;
  for (int c = 0; c < C; ++c) S += ce_soft_a(qr, c, s, keep, eps_c);
  const float g = (dloss ? *dloss : 1.f) / (s.sum ? 1.f : static_cast<float>(B));
  for (int c = 0; c < C; ++c) {
    const size_t i = static_cast<size_t>(r) * C + c;
    dlogits[i] = (probs[i] * S - ce_soft_a(qr, c, s, keep, eps_c)) * g;
  }
}

// =====================================================================================================
// Multi-tensor SGD: blockIdx.y = tensor, blockIdx.x strides its elements
// =====================================================================================================
__global__ void __launch_bounds__(256) sgd_multi_kernel(SgdTensorList tl, SgdHyper h) {
  const int t = blockIdx.y;
  const int n = tl.n[t];
  float* __restrict__ p = tl.p[t];
  const float* __restrict__ g = tl.g[t];
  float* __restrict__ m = tl.m[t];
  const float lr = h.lr_dev ? *h.lr_dev : h.lr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float gv = h.maximize ? -g[i] : g[i];
    const float pv = p[i];
    if (h.weight_decay != 0.f) gv = fmaf(h.weight_decay, pv, gv);
    if (h.momentum != 0.f) {
      float b = h.first_step ? gv : fmaf(h.momentum, m[i], (1.f - h.dampening) * gv);
      m[i] = b;
      gv = h.nesterov ? fmaf(h.momentum, b, gv) : b;
    }
    p[i] = fmaf(-lr, gv, pv);
  }
}

// =====================================================================================================
// Multi-tensor Adam / AdamW: same layout as sgd_multi_kernel.  Thread 0 of every block reads its tensor's step s and forms
// the bias corrections of step s + 1 in double; the block that takes the last ticket writes s + 1 back for every tensor
// (no block reads a step after it has taken its ticket) and resets the ticket word for the next launch.  AMS (AMSGrad):
// vmax = max(vmax, v) keeping a NaN, and the denominator is formed from vmax instead of v.
// =====================================================================================================
template <bool AMS, class TL>
__device__ __forceinline__ void adam_multi_body(const TL& tl, const AdamHyper& h, unsigned int* ticket) {
  const int t = blockIdx.y;
  __shared__ float s_f[3];
  if (threadIdx.x == 0) {
    const double lr = h.lr_dev ? static_cast<double>(*h.lr_dev) : h.lr;
    const double s = static_cast<double>(*tl.step[t] + 1.f);
    s_f[0] = static_cast<float>(lr / (1.0 - pow(h.beta1, s)));   // step size lr / bc1
    s_f[1] = static_cast<float>(sqrt(1.0 - pow(h.beta2, s)));    // sqrt(bc2)
    s_f[2] = static_cast<float>(1.0 - lr * h.weight_decay);      // AdamW's decay factor
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1) {
      __threadfence();
      for (int i = 0; i < tl.count; ++i) *tl.step[i] += 1.f;
      atomicExch(ticket, 0u);
    }
  }
  __syncthreads();
  const int n = tl.n[t];
  float* __restrict__ p = tl.p[t];
  const float* __restrict__ g = tl.g[t];
  float* __restrict__ m = tl.m[t];
  float* __restrict__ v = tl.v[t];
  float* __restrict__ vmax = nullptr;
  if constexpr (AMS) vmax = tl.vmax[t];
  const float step_size = s_f[0], bc2s = s_f[1], decay = s_f[2];
  const float omb1 = static_cast<float>(1.0 - h.beta1), b2 = static_cast<float>(h.beta2), omb2 = static_cast<float>(1.0 - h.beta2);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float gv = h.maximize ? -g[i] : g[i];
    float pv = p[i];
    if (h.weight_decay != 0.f) {
      if (h.decoupled) pv *= decay;
      else gv = fmaf(h.weight_decay, pv, gv);
    }
    const float mv = fmaf(omb1, gv - m[i], m[i]);
    const float vv = fmaf(omb2 * gv, gv, b2 * v[i]);
    m[i] = mv;
    v[i] = vv;
    float den = vv;
    if constexpr (AMS) {
      den = nan_max(vmax[i], vv);
      vmax[i] = den;
    }
    p[i] = fmaf(-step_size, mv / (sqrtf(den) / bc2s + h.eps), pv);
  }
}
__global__ void __launch_bounds__(256) adam_multi_kernel(AdamTensorList tl, AdamHyper h, unsigned int* ticket) {
  adam_multi_body<false>(tl, h, ticket);
}
__global__ void __launch_bounds__(256) amsgrad_multi_kernel(AmsgradTensorList tl, AdamHyper h, unsigned int* ticket) {
  adam_multi_body<true>(tl, h, ticket);
}
// a kernel's parameters take at most 4 KiB
static_assert(sizeof(AmsgradTensorList) + sizeof(AdamHyper) + sizeof(unsigned int*) <= 4096, "amsgrad_multi_kernel: parameters too large");

// The step hand-over of adam_multi_kernel for the tables of rmsprop / adagrad (thread 0 of every block, after it has read its step):
// the block that takes the last ticket writes s + 1 back for every tensor and resets the ticket word.
template <class TL>
__device__ __forceinline__ void advance_steps_last(const TL& tl, unsigned int* ticket) {
  __threadfence();
  if (atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1) {
    __threadfence();
    for (int i = 0; i < tl.count; ++i) *tl.step[i] += 1.f;
    atomicExch(ticket, 0u);
  }
}

// =====================================================================================================
// Multi-tensor RMSprop: same layout as sgd_multi_kernel.  The step count does not enter the update; thread 0 of every block takes a
// ticket, and the block that takes the last one advances every step.  buf / ga of a tensor are null when momentum == 0 / not
// centered: one kernel for the four combinations.
// =====================================================================================================
__global__ void __launch_bounds__(256) rmsprop_multi_kernel(RmspropTensorList tl, RmspropHyper h, unsigned int* ticket) {
  const int t = blockIdx.y;
  if (threadIdx.x == 0) advance_steps_last(tl, ticket);
  const int n = tl.n[t];
  float* __restrict__ p = tl.p[t];
  const float* __restrict__ g = tl.g[t];
  float* __restrict__ sq = tl.sq[t];
  float* __restrict__ buf = tl.buf[t];
  float* __restrict__ ga = tl.ga[t];
  const float lr = h.lr_dev ? *h.lr_dev : h.lr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float gv = h.maximize ? -g[i] : g[i];
    const float pv = p[i];
    if (h.weight_decay != 0.f) gv = fmaf(h.weight_decay, pv, gv);
    const float sv = fmaf(h.one_minus_alpha * gv, gv, h.alpha * sq[i]);
    sq[i] = sv;
    float var = sv;
    if (ga) {
      const float a = fmaf(h.one_minus_alpha, gv - ga[i], ga[i]);
      ga[i] = a;
      var = fmaf(-a, a, sv);
    }
    const float u = gv / (sqrtf(var) + h.eps);
    if (buf) {
      const float b = fmaf(h.momentum, buf[i], u);
      buf[i] = b;
      p[i] = fmaf(-lr, b, pv);
    } else {
      p[i] = fmaf(-lr, u, pv);
    }
  }
}
static_assert(sizeof(RmspropTensorList) + sizeof(RmspropHyper) + sizeof(unsigned int*) <= 4096, "rmsprop_multi_kernel: parameters too large");

// =====================================================================================================
// Multi-tensor Adagrad: same layout as sgd_multi_kernel.  Thread 0 of every block reads its tensor's step s and forms
// clr = lr / (1 + s·lr_decay) in double; the step hand-over is adam_multi_kernel's.
// =====================================================================================================
__global__ void __launch_bounds__(256) adagrad_multi_kernel(AdagradTensorList tl, AdagradHyper h, unsigned int* ticket) {
  const int t = blockIdx.y;
  __shared__ float s_clr;
  if (threadIdx.x == 0) {
    const double lr = h.lr_dev ? static_cast<double>(*h.lr_dev) : h.lr;
    s_clr = static_cast<float>(lr / (1.0 + static_cast<double>(*tl.step[t]) * h.lr_decay));
    advance_steps_last(tl, ticket);
  }
  __syncthreads();
  const int n = tl.n[t];
  float* __restrict__ p = tl.p[t];
  const float* __restrict__ g = tl.g[t];
  float* __restrict__ sum = tl.sum[t];
  const float clr = s_clr;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    float gv = h.maximize ? -g[i] : g[i];
    const float pv = p[i];
    if (h.weight_decay != 0.f) gv = fmaf(h.weight_decay, pv, gv);
    const float s = fmaf(gv, gv, sum[i]);
    sum[i] = s;
    p[i] = fmaf(-clr, gv / (sqrtf(s) + h.eps), pv);
  }
}
static_assert(sizeof(AdagradTensorList) + sizeof(AdagradHyper) + sizeof(unsigned int*) <= 4096, "adagrad_multi_kernel: parameters too large");

// =====================================================================================================
// Gradient-norm clipping: same layout as sgd_multi_kernel.  grad_norm_multi_kernel: every block writes one partial (fp32 Σg² or
// max |g| of the elements it strides over, reduced over the block in a fixed order); on the set's last table, the block that
// takes the last ticket folds the partials of every table in index order in fp64 and stores the norm and torch's clip
// coefficient.  grad_scale_multi_kernel multiplies every gradient by that coefficient, read from device memory.
// =====================================================================================================
__global__ void __launch_bounds__(256) grad_norm_multi_kernel(GradTensorList tl, GradNormArgs a) {
  const int t = blockIdx.y;
  const int n = tl.n[t];
  const float* __restrict__ g = tl.g[t];
  float acc = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = g[i];
    acc = a.norm_inf ? nan_max(fabsf(v), acc) : fmaf(v, v, acc);
  }
  __shared__ float s_w[8];
  __shared__ double s_d[256];
  __shared__ bool s_last;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const float o = __shfl_xor_sync(0xffffffffu, acc, off);
    acc = a.norm_inf ? nan_max(acc, o) : acc + o;
  }
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = s_w[0];
    for (int w = 1; w < 8; ++w) s = a.norm_inf ? nan_max(s, s_w[w]) : s + s_w[w];
    a.partials[a.part_base + t * gridDim.x + blockIdx.x] = s;
    bool last = false;
    if (a.last) {
      __threadfence();
      last = atomicAdd(a.ticket, 1u) == gridDim.x * gridDim.y - 1;
    }
    s_last = last;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double d = 0.0;
  for (int i = threadIdx.x; i < a.part_total; i += blockDim.x) {
    const double v = static_cast<double>(__ldcg(a.partials + i));
    d = a.norm_inf ? nan_max(d, v) : d + v;
  }
  s_d[threadIdx.x] = d;
  __syncthreads();
  for (int h = 128; h >= 1; h >>= 1) {
    if (threadIdx.x < h) s_d[threadIdx.x] = a.norm_inf ? nan_max(s_d[threadIdx.x], s_d[threadIdx.x + h]) : s_d[threadIdx.x] + s_d[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float norm = static_cast<float>(a.norm_inf ? s_d[0] : sqrt(s_d[0]));
    a.out[0] = norm;
    a.out[1] = clip_coef(norm, a.max_norm);
    atomicExch(a.ticket, 0u);
  }
}

__global__ void __launch_bounds__(256) grad_scale_multi_kernel(GradTensorList tl, const float* coef) {
  const int t = blockIdx.y;
  const int n = tl.n[t];
  float* __restrict__ g = tl.g[t];
  const float c = *coef;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) g[i] *= c;
}

// torch's CUDA lerp (ATen/native/Lerp.h) as nvcc contracts it: a + w·(b − a) for |w| < 0.5, else b − (b − a)·(1 − w)
__device__ __forceinline__ float torch_lerp(float a, float b, float w) {
  const float d = b - a;
  return fabsf(w) < 0.5f ? fmaf(w, d, a) : fmaf(-d, 1.f - w, b);
}

// =====================================================================================================
// Weight averaging: same layout as sgd_multi_kernel.  Thread 0 of every block reads n_averaged; on the set's last table it then
// takes a ticket, and the block that takes the last one stores n + 1 (every block has read n by then) and resets the ticket word.
// =====================================================================================================
__global__ void __launch_bounds__(256) avg_multi_kernel(AvgTensorList tl, AvgArgs a) {
  const int t = blockIdx.y;
  __shared__ long long s_n;
  if (threadIdx.x == 0) {
    const long long na = *a.n_averaged;
    s_n = na;
    if (a.last) {
      __threadfence();
      if (atomicAdd(a.ticket, 1u) == gridDim.x * gridDim.y - 1) {
        __threadfence();
        *a.n_averaged = na + 1;
        atomicExch(a.ticket, 0u);
      }
    }
  }
  __syncthreads();
  const long long na = s_n;
  const int n = tl.n[t], mode = tl.mode[t];
  const int i0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
  if (mode == AvgTensorList::kAvgF32 || mode == AvgTensorList::kCopyF32) {
    float* __restrict__ d = static_cast<float*>(tl.avg[t]);
    const float* __restrict__ s = static_cast<const float*>(tl.src[t]);
    if (na == 0 || mode == AvgTensorList::kCopyF32) {
      for (int i = i0; i < n; i += stride) d[i] = s[i];
      return;
    }
    const float w = a.swa ? 1.f / static_cast<float>(na + 1) : a.weight;
    for (int i = i0; i < n; i += stride) d[i] = torch_lerp(d[i], s[i], w);
  } else {
    long long* __restrict__ d = static_cast<long long*>(tl.avg[t]);
    const long long* __restrict__ s = static_cast<const long long*>(tl.src[t]);
    if (na == 0 || mode == AvgTensorList::kCopyI64) {
      for (int i = i0; i < n; i += stride) d[i] = s[i];
      return;
    }
    // p_ema * decay + p_model * (1 - decay): three separate fp32 ops in torch, then copy_ truncates to int64
    for (int i = i0; i < n; i += stride)
      d[i] = static_cast<long long>(__fadd_rn(__fmul_rn(static_cast<float>(d[i]), a.decay), __fmul_rn(static_cast<float>(s[i]), a.weight)));
  }
}

size_t conv_smem(int cin, int cout, int th, int w, int threads) {
  return (static_cast<size_t>(cin) * (th + 4) * (w + 4) + 4 + 25 * cin * cout + (threads / 32 + 1) * 2 * cout) * sizeof(float);
}

}  // namespace

// ---- launchers ---------------------------------------------------------------------------------------
void launch_conv5x5_fwd(const float* x, const float* w, const float* bias, float* y, void* stats, ConvStats form, ConvShape s,
                        ReduceScratch scr, cudaStream_t st) {
  constexpr int TH = 7;
  if (!(s.Cin == 1 && s.Cout == 16)) throw std::invalid_argument("conv5x5_fwd: supported channel config is 1→16");
  if (s.H % TH != 0) throw std::invalid_argument("conv5x5_fwd: H must be a multiple of 7");
  const int blocks = s.B * (s.H / TH);
  if (stats && (static_cast<long long>(blocks + blocks / kFoldGroup + 1) * 2 * s.Cout > scr.capacity_floats || blocks / kFoldGroup + 2 > scr.fold_counters))
    throw std::invalid_argument("conv5x5_fwd: reduction scratch too small");
  const int threads = (TH * s.W + 31) / 32 * 32;
  const size_t sm = conv_smem(1, 16, TH, s.W, threads);
  if (stats) conv5x5_kernel<1, 16, 16, TH, true><<<blocks, threads, sm, st>>>(x, w, bias, y, stats, form, scr, s.B, s.H, s.W);
  else conv5x5_kernel<1, 16, 16, TH, false><<<blocks, threads, sm, st>>>(x, w, bias, y, stats, kConvSums, scr, s.B, s.H, s.W);
  check_launch("conv5x5_fwd");
}

void launch_conv5x5_wgrad(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st) {
  constexpr int TH = 7;
  if (!(s.Cin == 1 && s.Cout == 16)) throw std::invalid_argument("conv5x5_wgrad: supported channel config is 1→16");
  if (s.H % TH != 0) throw std::invalid_argument("conv5x5_wgrad: H must be a multiple of 7");
  const int blocks = s.B * (s.H / TH);
  const int width = 25 * s.Cin * s.Cout + s.Cout;
  if (static_cast<long long>(blocks) * width > scr.capacity_floats) throw std::invalid_argument("conv5x5_wgrad: reduction scratch too small");
  const size_t xs_f = static_cast<size_t>(s.Cin) * (TH + 4) * (s.W + 4);
  const size_t fold_f = static_cast<size_t>(8) * 25 * 16;  // [warps][P*COUT] after dys
  const size_t sm = (xs_f + 4 + static_cast<size_t>(TH) * s.W * s.Cout + fold_f) * sizeof(float);
  conv5x5_wgrad_kernel<1, 16, TH><<<blocks, 256, sm, st>>>(dy, x, scr.partials, s.B, s.H, s.W);
  check_launch("conv5x5_wgrad");
  fold_partials_kernel<<<(width + 31) / 32, 256, 0, st>>>(scr.partials, blocks, width, 25 * s.Cin * s.Cout, dw, db);
  check_launch("fold_partials");
}

void launch_conv5x5_dgrad(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st) {
  constexpr int TH = 7;
  if (!(s.Cin == 1 && s.Cout == 16)) throw std::invalid_argument("conv5x5_dgrad: supported channel configs are 16→32 and 1→16");
  if (s.H % TH != 0) throw std::invalid_argument("conv5x5_dgrad: H must be a multiple of 7");
  const size_t sm = (static_cast<size_t>(s.Cout) * (TH + 4) * (s.W + 4) + 25 * s.Cout) * sizeof(float);
  if (TH * s.W > 448 || sm > 48 * 1024) throw std::invalid_argument("conv5x5_dgrad: W must be at most 63");
  const int blocks = s.B * (s.H / TH);
  if (blocks == 0) return;
  conv5x5_dgrad_cin1_kernel<16, TH><<<blocks, (TH * s.W + 31) / 32 * 32, sm, st>>>(dy, w, dx, s.H, s.W);
  check_launch("conv5x5_dgrad");
}

// The backward kernel takes a thread's channel quad from threadIdx.x % (C/4), which needs 256 % (C/4) == 0, and reduces the
// quads of a warp with a shuffle tree over C/4 lanes, which needs a power of two: C ∈ {4, 8, 16, 32, 64}.  Pooling takes even H, W.
static void check_bn_relu_pool_shape(int C, int H, int W, const char* what) {
  if (!(C == 4 || C == 8 || C == 16 || C == 32 || C == 64) || H % 2 || W % 2)
    throw std::invalid_argument(std::string(what) + ": C must be 4, 8, 16, 32 or 64, and H and W even");
}

void launch_bn_relu_pool_fwd(const float* y, const void* stats, const float* gamma, const float* beta, float* out, float* saved,
                             float* running_mean, float* running_var, long long* nbt, float momentum, float eps, int B, int H, int W,
                             int C, bool out_nchw, BnStats form, cudaStream_t st) {
  check_bn_relu_pool_shape(C, H, W, "bn_relu_pool_fwd");
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 4);
  bn_relu_pool_fwd_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, st>>>(y, stats, gamma, beta, out, saved, running_mean, running_var,
                                                                                 nbt, momentum, eps, B, H, W, C, out_nchw ? 1 : 0,
                                                                                 static_cast<int>(form));
  check_launch("bn_relu_pool_fwd");
}

void launch_bn_relu_pool_bwd_reduce(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta, float* sums,
                                    float* dgamma, float* dbeta, int B, int H, int W, int C, bool dout_nchw, ReduceScratch scr,
                                    cudaStream_t st) {
  check_bn_relu_pool_shape(C, H, W, "bn_relu_pool_bwd_reduce");
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 4);
  const int blocks = static_cast<int>((total + 255) / 256);
  if (static_cast<long long>(blocks + blocks / kFoldGroup + 1) * 2 * C > scr.capacity_floats || blocks / kFoldGroup + 2 > scr.fold_counters)
    throw std::invalid_argument("bn_relu_pool_bwd: reduction scratch too small");
  bn_relu_pool_bwd_kernel<false><<<blocks, 256, 0, st>>>(dout, y, saved, gamma, beta, sums, dgamma, dbeta, nullptr, nullptr, B, H, W, C,
                                                         dout_nchw ? 1 : 0, scr);
  check_launch("bn_relu_pool_bwd_reduce");
}

void launch_bn_relu_pool_bwd_apply(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta,
                                   const float* sums, const float* count, float* dy, int B, int H, int W, int C, bool dout_nchw,
                                   bool mean_var, cudaStream_t st) {
  check_bn_relu_pool_shape(C, H, W, "bn_relu_pool_bwd_apply");
  const long long total = static_cast<long long>(B) * (H / 2) * (W / 2) * (C / 4);
  auto kern = mean_var ? bn_relu_pool_bwd_kernel<true, true> : bn_relu_pool_bwd_kernel<true, false>;
  kern<<<static_cast<int>((total + 255) / 256), 256, 0, st>>>(dout, y, saved, gamma, beta, const_cast<float*>(sums), nullptr, nullptr, count, dy,
                                                              B, H, W, C, dout_nchw ? 1 : 0, ReduceScratch{});
  check_launch("bn_relu_pool_bwd_apply");
}

static int bn_slices(int N, int C, int HW) {
  const long long total = static_cast<long long>(N) * HW;
  int S = static_cast<int>(std::min<long long>(std::max<long long>(1, total / 2048), std::max(1, 592 / std::max(1, C))));
  return std::max(1, S);
}

void launch_bn_stats_nchw_f64(const float* x, double* stats, int N, int C, int HW, ReduceScratch scr, cudaStream_t st) {
  const int S = bn_slices(N, C, HW);
  if (static_cast<long long>(C) * S * 4 > scr.capacity_floats) throw std::invalid_argument("bn_stats: reduction scratch too small");
  bn_stats_nchw_f64_kernel<<<C * S, 256, 0, st>>>(x, stats, N, C, HW, S, scr);
  check_launch("bn_stats_nchw_f64");
}
void launch_bn_finalize(const double* stats, int C, double eps, float momentum, float* mean, float* invstd, float* count_out,
                        float* running_mean, float* running_var, cudaStream_t st) {
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(stats, C, eps, momentum, mean, invstd, count_out, running_mean, running_var);
  check_launch("bn_finalize");
}
void launch_bn_apply_nchw(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta, float* out, int N,
                          int C, int HW, cudaStream_t st) {
  const long long total = static_cast<long long>(N) * C * HW;
  bn_apply_nchw_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, st>>>(x, mean, invstd, gamma, beta, out, total, C, HW);
  check_launch("bn_apply_nchw");
}
void launch_bn_bwd_reduce_nchw(const float* dy, const float* x, const float* mean, const float* invstd, float* red4c, int N, int C, int HW,
                               ReduceScratch scr, cudaStream_t st) {
  const int S = bn_slices(N, C, HW);
  if (static_cast<long long>(C) * S * 2 > scr.capacity_floats) throw std::invalid_argument("bn_bwd_reduce: reduction scratch too small");
  bn_bwd_reduce_nchw_kernel<<<C * S, 256, 0, st>>>(dy, x, mean, invstd, red4c, N, C, HW, S, scr);
  check_launch("bn_bwd_reduce_nchw");
}
void launch_bn_bwd_apply_nchw(const float* dy, const float* x, const float* mean, const float* invstd, const float* gamma,
                              const float* mean_dy, const float* mean_dy_xmu, float* dx, int N, int C, int HW, cudaStream_t st) {
  const long long total = static_cast<long long>(N) * C * HW;
  bn_bwd_apply_nchw_kernel<<<static_cast<int>((total + 255) / 256), 256, 0, st>>>(dy, x, mean, invstd, gamma, mean_dy, mean_dy_xmu, dx, total, C, HW);
  check_launch("bn_bwd_apply_nchw");
}

void launch_linear_fwd(const float* x, const float* w, const float* b, float* out, int B, int K, int N, cudaStream_t st) {
  if (N > 16) throw std::invalid_argument("linear_fwd (fused head): N <= 16 supported; wider layers use the GEMM path");
  linear_fwd_kernel<16, 4><<<(B + 3) / 4, 256, 0, st>>>(x, w, b, out, B, K, N);
  check_launch("linear_fwd");
}
void launch_linear_bwd(const float* dout, const float* x, const float* w, float* dx, float* dw, float* db, int B, int K, int N,
                       cudaStream_t st) {
  if (N > 16) throw std::invalid_argument("linear_bwd (fused head): N <= 16 supported");
  const int dw_blocks = (K + 31) / 32;
  linear_bwd_kernel<16><<<B + dw_blocks, 256, 128 * N * sizeof(float), st>>>(dout, x, w, dx, dw, db, B, K, N, B);
  check_launch("linear_bwd");
}
void launch_cross_entropy_fwd(const float* logits, const long long* target, float* loss, float* probs, int B, int C, cudaStream_t st,
                              bool emit_grad) {
  cross_entropy_fwd_kernel<<<1, 256, 0, st>>>(logits, target, loss, probs, B, C, emit_grad ? 1 : 0);
  check_launch("cross_entropy_fwd");
}
void launch_cross_entropy_bwd(const float* probs, const long long* target, const float* dloss, float* dlogits, int B, int C,
                              cudaStream_t st) {
  cross_entropy_bwd_kernel<<<(B * C + 255) / 256, 256, 0, st>>>(probs, target, dloss, dlogits, B, C);
  check_launch("cross_entropy_bwd");
}
void launch_cross_entropy_fwd(const float* logits, const long long* target, float* loss, float* probs, int B, int C, cudaStream_t st,
                              bool emit_grad, const CeSpec& spec) {
  if (spec.is_default(C)) return launch_cross_entropy_fwd(logits, target, loss, probs, B, C, st, emit_grad);
  cross_entropy_fwd_spec_kernel<<<1, 256, 0, st>>>(logits, target, loss, probs, B, C, emit_grad ? 1 : 0, spec, nullptr);
  check_launch("cross_entropy_fwd");
}
void launch_cross_entropy_eval(const float* logits, const long long* target, double* acc, int rows, int C, cudaStream_t st,
                               const CeSpec& spec) {
  CeSpec mean = spec;
  mean.sum = false;   // acc takes the sum of the terms and the mean's divisor D whatever the reduction
  cross_entropy_fwd_spec_kernel<<<1, 256, 0, st>>>(logits, target, nullptr, nullptr, rows, C, 0, mean, acc);
  check_launch("cross_entropy_eval");
}
void launch_cross_entropy_bwd(const float* probs, const long long* target, const float* dloss, float* dlogits, int B, int C,
                              cudaStream_t st, const CeSpec& spec) {
  if (spec.is_default(C)) return launch_cross_entropy_bwd(probs, target, dloss, dlogits, B, C, st);
  cross_entropy_bwd_spec_kernel<<<(B * C + 255) / 256, 256, 0, st>>>(probs, target, dloss, dlogits, B, C, spec);
  check_launch("cross_entropy_bwd");
}
void launch_cross_entropy_fwd_soft(const float* logits, const float* q, float* loss, float* probs, int B, int C, cudaStream_t st,
                                   bool emit_grad, const CeSpec& spec) {
  cross_entropy_fwd_soft_kernel<<<1, 256, 0, st>>>(logits, q, loss, probs, B, C, emit_grad ? 1 : 0, spec);
  check_launch("cross_entropy_fwd");
}
void launch_cross_entropy_bwd_soft(const float* probs, const float* q, const float* dloss, float* dlogits, int B, int C, cudaStream_t st,
                                   const CeSpec& spec) {
  if (B == 0) return;
  cross_entropy_bwd_soft_kernel<<<(B + 255) / 256, 256, 0, st>>>(probs, q, dloss, dlogits, B, C, spec);
  check_launch("cross_entropy_bwd");
}

void launch_sgd_multi(const SgdTensorList& tl, SgdHyper h, cudaStream_t st) {
  if (tl.count == 0) return;
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  const int bx = std::max(1, std::min(64, (maxn + 1023) / 1024));
  sgd_multi_kernel<<<dim3(bx, tl.count), 256, 0, st>>>(tl, h);
  check_launch("sgd_multi");
}

void launch_adam_multi(const AdamTensorList& tl, AdamHyper h, unsigned int* ticket, cudaStream_t st) {
  if (tl.count == 0) return;
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  const int bx = std::max(1, std::min(64, (maxn + 1023) / 1024));
  adam_multi_kernel<<<dim3(bx, tl.count), 256, 0, st>>>(tl, h, ticket);
  check_launch("adam_multi");
}
void launch_adam_multi(const AmsgradTensorList& tl, AdamHyper h, unsigned int* ticket, cudaStream_t st) {
  if (tl.count == 0) return;
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  const int bx = std::max(1, std::min(64, (maxn + 1023) / 1024));
  amsgrad_multi_kernel<<<dim3(bx, tl.count), 256, 0, st>>>(tl, h, ticket);
  check_launch("adam_multi");
}
void launch_rmsprop_multi(const RmspropTensorList& tl, RmspropHyper h, unsigned int* ticket, cudaStream_t st) {
  if (tl.count == 0) return;
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  const int bx = std::max(1, std::min(64, (maxn + 1023) / 1024));
  rmsprop_multi_kernel<<<dim3(bx, tl.count), 256, 0, st>>>(tl, h, ticket);
  check_launch("rmsprop_multi");
}
void launch_adagrad_multi(const AdagradTensorList& tl, AdagradHyper h, unsigned int* ticket, cudaStream_t st) {
  if (tl.count == 0) return;
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  const int bx = std::max(1, std::min(64, (maxn + 1023) / 1024));
  adagrad_multi_kernel<<<dim3(bx, tl.count), 256, 0, st>>>(tl, h, ticket);
  check_launch("adagrad_multi");
}

int grad_multi_blocks_x(const GradTensorList& tl) {
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  return std::max(1, std::min(64, (maxn + 1023) / 1024));
}

void launch_grad_norm_multi(const GradTensorList& tl, GradNormArgs a, cudaStream_t st) {
  if (tl.count == 0) return;
  grad_norm_multi_kernel<<<dim3(grad_multi_blocks_x(tl), tl.count), 256, 0, st>>>(tl, a);
  check_launch("grad_norm_multi");
}

void launch_grad_scale_multi(const GradTensorList& tl, const float* coef, cudaStream_t st) {
  if (tl.count == 0) return;
  grad_scale_multi_kernel<<<dim3(grad_multi_blocks_x(tl), tl.count), 256, 0, st>>>(tl, coef);
  check_launch("grad_scale_multi");
}

void launch_avg_multi(const AvgTensorList& tl, AvgArgs a, cudaStream_t st) {
  if (tl.count == 0) return;
  int maxn = 0;
  for (int i = 0; i < tl.count; ++i) maxn = std::max(maxn, tl.n[i]);
  const int bx = std::max(1, std::min(64, (maxn + 1023) / 1024));
  avg_multi_kernel<<<dim3(bx, tl.count), 256, 0, st>>>(tl, a);
  check_launch("avg_multi");
}

}  // namespace pdt
