// Cooperative fused kernels for the reference ConvNet (ref: ddp_example.py:22-41) — one CTA per image.
//
// A ConvNet step is a few µs of arithmetic spread over dependent kernel boundaries and every per-op kernel
// pays launch + ramp + drain + a grid-wide reduction.  Here everything that belongs to an image stays inside its CTA
// (registers / shared memory), and the only grid-wide dependencies — the BatchNorm batch statistics (forward), the
// Σdz, Σdz·x̂ sums (backward) and the folds of the weight gradients — are device-side grid barriers in the middle of a
// kernel instead of kernel boundaries.  A training step is three launches:
//
//   convnet_fwd_kernel         conv1 5x5 (1→16) ──barrier (Σy, Σy²)── BN + ReLU + MaxPool2 written straight into conv2's
//                              swizzled smem patch ── conv2 5x5 (16→32) on wgmma (the 25 taps are row-shifted descriptors
//                              into that patch; accumulators in registers) ──barrier── BN + ReLU + MaxPool2 + classifier
//                              (+ cross-entropy term and d(loss)/d(logits) when the targets are known)           (ref :25-34,40)
//   convnet_l2_bwd_kernel<FC>  classifier backward + MaxPool/ReLU/BN backward ──barrier (Σdz, Σdz·x̂)── dy → conv2 data
//                              gradient on wgmma
//   convnet_l1_bwd_kernel<WG>  MaxPool/ReLU/BN backward ──barrier── conv1 weight gradient (mma.sync) ──barrier── folds,
//                              while conv2's weight gradient is computed on mma.sync (MN-major window) and — on one
//                              GPU — the threads that write the folded gradients apply the SGD update (SgdRider)
//
// convnet_l1_fwd_kernel / convnet_l2_fwd_kernel (one kernel per layer) and the <false> instantiations are the variants without
// the riders (PDT_FUSED_WHOLE_FWD / PDT_FC_MERGED / PDT_WGRAD_MERGED = 0); all of them are exercised by tests/test_gpu_kernels.py.
//
// All cross-CTA sums are "every CTA writes one partial row, barrier, every CTA folds the rows in the same fixed order",
// so results are bit-reproducible and identical in every CTA.  The kernels are launched cooperatively (all CTAs
// co-resident: one per image, at most one per SM); grid barriers are split into arrive / wait so that independent work
// (stores nobody in the kernel waits for, cp.async staging, gradient slices) runs in their shadow (grid_sync.cuh).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <type_traits>

#include "cuda_utils.h"
#include "conv_wgmma.h"
#include "fused_convnet.h"
#include "grid_sync.cuh"
#include "hopper_ptx.cuh"
#include "wgrad_win.cuh"

namespace pdt {

namespace {

using namespace ptx;

// ---- optional phase trace (PDT_FUSED_TRACE=1): globaltimer stamps of thread 0 of every CTA, read back by tools ----------
__device__ unsigned long long g_trace[4][160][12];
__device__ int g_trace_on = 0;
// The switch is read ONCE per kernel (TRACE_INIT, one global load whose latency overlaps the prologue); a stamp is then a predicated
// branch on a register — a load of the switch per stamp would put a global-memory latency on the critical path at every stamp.
#define TRACE_INIT() const bool trace_on_ = (threadIdx.x == 0) && (*reinterpret_cast<volatile int*>(&g_trace_on) != 0)
__device__ __forceinline__ void trace_stamp(bool on, int kernel, int phase) {
  if (on) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_trace[kernel][blockIdx.x][phase] = t;
  }
}
#define trace(kernel, phase) trace_stamp(trace_on_, kernel, phase)

// CTA-wide sync of the first NAMED threads (named barrier 1) or of the whole CTA (NAMED = 0): kernels with extra
// role warps keep their "main" threads in step without involving the others.
template <int NAMED>
__device__ __forceinline__ void cta_sync() {
  if constexpr (NAMED > 0) asm volatile("bar.sync 1, %0;" ::"n"(NAMED) : "memory");
  else __syncthreads();
}

// Sum `rows` partial rows of `W` floats (written by other CTAs before a grid barrier) in a fixed order.
// Called by all (main) threads; the totals land in s_out[0..W).  s_tmp: [4][W] floats.  Needs >= 4*W threads.
template <int W, int NAMED = 0>
__device__ __forceinline__ void fold_rows(const float* __restrict__ partials, int rows, float* s_tmp, float* s_out) {
  const int tid = threadIdx.x;
  if (tid < 4 * W) {
    const int col = tid % W, grp = tid / W;
    float s = 0.f;
    for (int r = grp; r < rows; r += 32) {   // eight independent L2 loads in flight, summed in a fixed order
      float t[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t[j] = (r + 4 * j < rows) ? __ldcg(partials + static_cast<size_t>(r + 4 * j) * W + col) : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += t[j];
    }
    s_tmp[grp * W + col] = s;
  }
  cta_sync<NAMED>();
  if (tid < W) s_out[tid] = (s_tmp[tid] + s_tmp[W + tid]) + (s_tmp[2 * W + tid] + s_tmp[3 * W + tid]);
  cta_sync<NAMED>();
}

// The same with every thread of a THREADS-wide CTA loading: G = THREADS / W row classes, one L2 round trip for up to 8·G rows.
// s_tmp: [G][W] floats.
template <int W, int THREADS, int NAMED = 0>
__device__ __forceinline__ void fold_rows_wide(const float* __restrict__ partials, int rows, float* s_tmp, float* s_out) {
  constexpr int G = THREADS / W;
  const int tid = threadIdx.x;
  if (tid < G * W) {
    const int col = tid % W, grp = tid / W;
    float s = 0.f;
    for (int r = grp; r < rows; r += 8 * G) {
      float t[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) t[j] = (r + G * j < rows) ? __ldcg(partials + static_cast<size_t>(r + G * j) * W + col) : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) s += t[j];
    }
    s_tmp[grp * W + col] = s;
  }
  cta_sync<NAMED>();
  if (tid < W) {
    float tot = 0.f;
#pragma unroll
    for (int g = 0; g < G; ++g) tot += s_tmp[g * W + tid];
    s_out[tid] = tot;
  }
  cta_sync<NAMED>();
}

// Warp-level reduction of 32 per-thread values with 31 shuffles: after the call lane l holds Σ_lanes v[l] in v[0].
__device__ __forceinline__ void warp_transpose_reduce32(float (&v)[32], int lane) {
#pragma unroll
  for (int off = 16, half = 16; off >= 1; off >>= 1, half >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      const float send = upper ? v[i] : v[i + half];
      const float keep = upper ? v[i + half] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
}

// =====================================================================================================================
// Layer 1 — conv1 is 1→16 channels on a 28×28 image: K = 25 per output, 31 MFLOP per batch of 100.  One thread per
// output pixel, 16 accumulators in registers that *stay* in registers across the grid barrier.  Threads are ordered
// by pooling window (4 consecutive lanes = one 2×2 window), so max-pooling is two shuffles and the y / pooled
// stores are fully coalesced.
// =====================================================================================================================
constexpr int kL1Threads = 800;  // 784 pixels rounded up to whole warps
constexpr int kL1Warps = kL1Threads / 32;

struct L1Map {
  int win, d, ph, pw, r, c;
  bool valid;
  __device__ __forceinline__ explicit L1Map(int tid) {
    valid = tid < 784;
    const int t = valid ? tid : 0;
    win = t >> 2;
    d = t & 3;
    ph = win / 14;
    pw = win - ph * 14;
    r = 2 * ph + (d >> 1);
    c = 2 * pw + (d & 1);
  }
};

template <int NAMED = 0>
__device__ __forceinline__ void l1_load_image(const float* __restrict__ x, float* xs /*[32][32]*/, int tid) {
  for (int i = tid; i < 1024; i += kL1Threads) xs[i] = 0.f;
  cta_sync<NAMED>();
  if (tid < 784) {
    const int rr = tid / 28, cc = tid - rr * 28;
    xs[(rr + 2) * 32 + cc + 2] = x[tid];
  }
}

__global__ void __launch_bounds__(kL1Threads, 1)
convnet_l1_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ out,
                      float* saved, float* running_mean, float* running_var, long long* nbt, float momentum, float eps,
                      float* partials, GridSync gs) {
  __shared__ float xs[32 * 32];
  __shared__ __align__(16) float ws[25 * 16];
  __shared__ float red[kL1Warps * 32];
  __shared__ float s_tmp[4 * 32];
  __shared__ float s_tot[32];
  __shared__ float s_scale[16], s_shift[16];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;
  const L1Map m(tid);
  GridBar bar(gs);
  TRACE_INIT();
  trace(0, 0);

  l1_load_image(x + static_cast<size_t>(n) * 784, xs, tid);
  if (tid < 400) {
    const int tap = tid >> 4, co = tid & 15;
    ws[tid] = w[co * 25 + tap];
  }
  __syncthreads();

  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = bias ? __ldg(bias + j) : 0.f;
#pragma unroll 1
  for (int kh = 0; kh < 5; ++kh) {
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      const float xv = xs[(m.r + kh) * 32 + m.c + kw];
      const float4* wt = reinterpret_cast<const float4*>(ws + (kh * 5 + kw) * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 wv = wt[q];
        acc[4 * q + 0] = fmaf(xv, wv.x, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(xv, wv.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(xv, wv.z, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(xv, wv.w, acc[4 * q + 3]);
      }
    }
  }
  trace(0, 1);
  {
    float v[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      v[j] = m.valid ? acc[j] : 0.f;
      v[16 + j] = m.valid ? acc[j] * acc[j] : 0.f;
    }
    warp_transpose_reduce32(v, lane);
    red[warp * 32 + lane] = v[0];
  }
  __syncthreads();
  if (tid < 32) {
    float s = 0.f;
#pragma unroll 5
    for (int wi = 0; wi < kL1Warps; ++wi) s += red[wi * 32 + tid];
    partials[static_cast<size_t>(n) * 32 + tid] = s;
  }
  trace(0, 2);
  bar.sync(gs);
  trace(0, 3);
  fold_rows<32>(partials, B, s_tmp, s_tot);
  trace(0, 4);
  if (tid < 16) {
    const float cnt = static_cast<float>(B) * 784.f;
    const float mean = s_tot[tid] / cnt;
    const float var = fmaxf(s_tot[16 + tid] / cnt - mean * mean, 0.f);
    const float invstd = rsqrtf(var + eps);
    const float g = gamma ? gamma[tid] : 1.f, b = beta ? beta[tid] : 0.f;
    s_scale[tid] = g * invstd;
    s_shift[tid] = b - mean * g * invstd;
    if (n == 0) {
      saved[tid] = mean;
      saved[16 + tid] = invstd;
      if (running_mean) {
        const float unbiased = var * (cnt / fmaxf(cnt - 1.f, 1.f));
        running_mean[tid] = (1.f - momentum) * running_mean[tid] + momentum * mean;
        running_var[tid] = (1.f - momentum) * running_var[tid] + momentum * unbiased;
      }
      if (nbt && tid == 0) *nbt += 1;
    }
  }
  __syncthreads();
  float z[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    float t = fmaxf(fmaf(acc[j], s_scale[j], s_shift[j]), 0.f);
    t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 1));
    t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 2));
    z[j] = t;
  }
  if (m.valid) {  // lane d of the window writes channels 4d..4d+3: one 64-byte row per window
    float4 o;
    if (m.d == 0) o = make_float4(z[0], z[1], z[2], z[3]);
    else if (m.d == 1) o = make_float4(z[4], z[5], z[6], z[7]);
    else if (m.d == 2) o = make_float4(z[8], z[9], z[10], z[11]);
    else o = make_float4(z[12], z[13], z[14], z[15]);
    reinterpret_cast<float4*>(out + ((static_cast<size_t>(n) * 18 + m.ph + 2) * 18 + m.pw + 2) * 16)[m.d] = o;
  }
  // the 2-position halo of the frame is zero: layer 2 reads it as the convolution's zero padding (forward: one TMA box
  // per image; weight gradient: overlapping-row TMA view), so nobody has to special-case the image border
  for (int i = tid; i < 324 * 4; i += kL1Threads) {
    const int P = i >> 2, pr = P / 18, pc = P - pr * 18;
    if (pr < 2 || pr >= 16 || pc < 2 || pc >= 16) reinterpret_cast<float4*>(out + (static_cast<size_t>(n) * 324 + P) * 16)[i & 3] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (m.valid) {  // conv output is kept for the backward pass (BatchNorm needs x̂ at every position); stored last: nothing
                  // in this kernel waits for these 50 KB per CTA, least of all the fence in front of the grid barrier
    float4* yp = reinterpret_cast<float4*>(y + ((static_cast<size_t>(n) * 28 + m.r) * 28 + m.c) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) yp[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
  }
  bar.finish(gs);
  trace(0, 5);
}

// ---- layer 1 backward (+ conv2 weight gradient riding along) ---------------------------------------------------------------
// dynamic smem: dys [784][16] | fold [25 warps][16 co][32 taps]   (+ WG: the tensor-core weight-gradient pipeline, below)
constexpr int kL1BwdSmem = (784 * 16 + kL1Warps * 512) * 4;

// The conv2 weight gradient of an image needs nothing from layer-1 backward — only the dy / x frames that layer-2 backward
// left in global memory.  With WG the CTA carries one extra warp that TMA-loads both operands of the same image while the 25
// layer-1 warps do their SIMT work, and 15 of those warps compute dW2ᵀ[(kh, kw, ci)][co] = Σ_P xpad[P + (kh−2)·18 + (kw−2)][ci] ·
// dypad[P][co] on the tensor cores (wgrad_win.cuh) just before the kernel's second grid barrier; it is folded after it, next to
// the conv1 gradient:
//   * B (dy): the 256 positions starting at the first interior one, two TMA boxes.
//   * A (x): the whole image's overlapping-row view (pitch 64 B, length 128 B: row r = positions r and r+1 = two horizontally
//     adjacent taps × 16 channels), loaded ONCE (384 rows, 48 KB); the 32-row atom of tap pair (kh, kw/2) for position P is the
//     same buffer read (kh−2)·18 + (kw−2) rows further down.  The per-CTA partial has 512 rows in four groups of four atoms:
//     group kw/2 ∈ {0,1,2} stacks kh = 0..3 (stride 18 rows), group 3 holds kh = 4 with kw/2 = 0..2 (stride 2 rows; its fourth
//     atom is unused).  The stand-alone kernel (conv_wgmma.cu) orders the atoms by (kh, kw/2) instead.
// One launch and one grid barrier less than running the two kernels back to back.
struct L1WgCfg {
  static constexpr int kThreads = kL1Threads + 32;        // + one warp: the TMA loads
  static constexpr int kFrame = 18 * 18, kFirst = 2 * 18 + 2;
  // A window: rows [0, 384) of the image's overlapping-row view (row r = positions r, r+1 × 16 channels = 128 B), six 64-row boxes
  static constexpr int kABoxes = 6, kABytes = kABoxes * 64 * 128;
  static constexpr int kBBytes = 2 * 128 * 128;                    // both 128-position dy tiles of the image
  static constexpr int kOff = (kL1BwdSmem + 1023) / 1024 * 1024;   // window starts 1024-aligned behind the layer-1 buffers
  static constexpr size_t kSmem = 1024 + kOff + kABytes + kBBytes + 256;
};

// One SGD update (the arithmetic of sgd_multi_kernel, ops_simt.cu) of element *p with gradient g.
__device__ __forceinline__ void sgd_apply(float* p, float g, float* m, const SgdHyper& h, float lr) {
  float gv = h.maximize ? -g : g;
  const float pv = *p;
  if (h.weight_decay != 0.f) gv = fmaf(h.weight_decay, pv, gv);
  if (h.momentum != 0.f) {
    const float b = h.first_step ? gv : fmaf(h.momentum, *m, (1.f - h.dampening) * gv);
    *m = b;
    gv = h.nesterov ? fmaf(h.momentum, b, gv) : b;
  }
  *p = fmaf(-lr, gv, pv);
}

// Per-launch factors of the Adam rider, formed once per CTA before the first grid barrier (kAdamLr: index of the first
// non-parameter entry): step size lr/bc1 [10], sqrt(bc2) [10], AdamW decay 1 − lr·wd, 1 − β1, β2, 1 − β2.
constexpr int kAdamLr = 20, kAdamFactors = 24;
__device__ __forceinline__ void adam_factors(const AdamRider& r, float* f, int tid) {
  if (tid < 10 && r.step[tid]) {
    const double lr = r.h.lr_dev ? static_cast<double>(__ldg(r.h.lr_dev)) : r.h.lr;
    const double s = static_cast<double>(*r.step[tid] + 1.f);
    f[tid] = static_cast<float>(lr / (1.0 - pow(r.h.beta1, s)));
    f[10 + tid] = static_cast<float>(sqrt(1.0 - pow(r.h.beta2, s)));
    if (tid == 0) {
      f[kAdamLr] = static_cast<float>(1.0 - lr * r.h.weight_decay);
      f[kAdamLr + 1] = static_cast<float>(1.0 - r.h.beta1);
      f[kAdamLr + 2] = static_cast<float>(r.h.beta2);
      f[kAdamLr + 3] = static_cast<float>(1.0 - r.h.beta2);
    }
  }
}

// One Adam update (the arithmetic of adam_multi_kernel, ops_simt.cu) of element i of parameter k with gradient g.
__device__ __forceinline__ void adam_apply(const AdamRider& r, int k, int i, float g, const float* f) {
  float gv = r.h.maximize ? -g : g;
  float* p = r.p[k] + i;
  float* m = r.m[k] + i;
  float* v = r.v[k] + i;
  float pv = *p;
  if (r.h.weight_decay != 0.f) {
    if (r.h.decoupled) pv *= f[kAdamLr];
    else gv = fmaf(r.h.weight_decay, pv, gv);
  }
  const float mv = fmaf(f[kAdamLr + 1], gv - *m, *m);
  const float vv = fmaf(f[kAdamLr + 3] * gv, gv, f[kAdamLr + 2] * *v);
  *m = mv;
  *v = vv;
  *p = fmaf(-f[k], mv / (sqrtf(vv) / f[10 + k] + r.h.eps), pv);
}

// Gradient-norm clipping (ClipRider): one gradient element g into a thread's accumulator — Σg², or max |g| keeping a NaN.
template <class R>
__device__ __forceinline__ float clip_acc(const R& r, float acc, float g) { return r.norm_inf ? nan_max(fabsf(g), acc) : fmaf(g, g, acc); }
template <class R>
__device__ __forceinline__ float clip_comb(const R& r, float a, float b) { return r.norm_inf ? nan_max(a, b) : a + b; }

template <bool WG, class Rider = SgdRider>
__global__ void __launch_bounds__(WG ? L1WgCfg::kThreads : kL1Threads, 1)
convnet_l1_bwd_kernel(const float* __restrict__ dp, const float* __restrict__ y, const float* __restrict__ x, const float* __restrict__ saved,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float* dgamma, float* dbeta, float* dw, float* db,
                      float* partials, float* partials_w, GridSync gs,
                      // WG only: conv2 weight gradient of the same image
                      const __grid_constant__ CUtensorMap tm_x2, const __grid_constant__ CUtensorMap tm_dy2, float* __restrict__ wpart,
                      const float* __restrict__ dysum2, float* dw2, float* db2, const __grid_constant__ Rider sr) {
  constexpr bool kClip = std::is_same_v<Rider, ClipRider<SgdRider>> || std::is_same_v<Rider, ClipRider<AdamRider>>;
  constexpr bool kAdam = std::is_same_v<Rider, AdamRider> || std::is_same_v<Rider, ClipRider<AdamRider>>;
  static_assert(kAdam || std::is_base_of_v<SgdRider, Rider>, "convnet_l1_bwd_kernel: SgdRider or AdamRider, or either in a ClipRider");
  static_assert(WG || !(kAdam || kClip), "the Adam and clipping riders ride on the kernel with the conv2 weight gradient");
  constexpr int NAMED = WG ? kL1Threads : 0;
  extern __shared__ __align__(16) uint8_t dsm_raw[];
  // WG: everything is placed relative to a 1024-aligned base (the swizzled TMA tiles need it)
  uint8_t* dsm_b = WG ? reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(dsm_raw) + 1023) & ~uintptr_t(1023)) : dsm_raw;
  float* dsm = reinterpret_cast<float*>(dsm_b);
  float* dys = dsm;                  // [784][16]
  float* fold = dsm + 784 * 16;      // [25 warps][16][32]
  uint8_t* sa = dsm_b + L1WgCfg::kOff;                              // WG: A window
  uint8_t* sb = sa + L1WgCfg::kABytes;                              // WG: dy tiles
  uint64_t* ld_full = reinterpret_cast<uint64_t*>(sb + L1WgCfg::kBBytes);
  float* adam_f = reinterpret_cast<float*>(sb + L1WgCfg::kBBytes + 64);   // Adam rider: kAdamFactors floats behind the barrier word
  static_assert(64 + kAdamFactors * sizeof(float) <= 256, "Adam rider factors must fit the tail of the dynamic shared memory");
  __shared__ float xs[32 * 32];
  __shared__ float red[kL1Warps * 32];
  __shared__ float s_tmp[kL1Warps * 32];
  __shared__ float s_tot[32];
  __shared__ float s_scale[16], s_shift[16], s_mean[16], s_invstd[16];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;
  float* s_clip = red + 512;   // ClipRider: per-warp norm partials + the coefficient (s_db below takes red[0, 512) only)

  if constexpr (WG) {
    if (warp == kL1Warps) {
      // ================= operands of the conv2 weight gradient of image n: one warp loads them by TMA =================
      using Cfg = L1WgCfg;
      if (lane == 0) {
        tma_prefetch_desc(&tm_x2);
        tma_prefetch_desc(&tm_dy2);
        mbar_init(ld_full, 1);
        fence_mbar_init();
      }
      __syncwarp();
      asm volatile("bar.arrive 0, %0;" ::"n"(L1WgCfg::kThreads) : "memory");   // (1) the layer-1 warps sync on barrier 0 before they wait on ld_full
      const int frame0 = n * Cfg::kFrame;
      // let the layer-1 warps have the L2 → SM path for their opening loads first
      asm volatile("bar.sync 4, %0;" ::"n"(L1WgCfg::kThreads) : "memory");
      if (elect_one()) {
        mbar_arrive_expect_tx(ld_full, Cfg::kABytes + Cfg::kBBytes);
        for (int bx = 0; bx < Cfg::kABoxes; ++bx) tma_load_2d(sa + bx * 8192, &tm_x2, ld_full, 0, frame0 + 64 * bx);   // rows past the tensor are zero-filled
        tma_load_2d(sb, &tm_dy2, ld_full, 0, frame0 + Cfg::kFirst);
        tma_load_2d(sb + 128 * 128, &tm_dy2, ld_full, 0, frame0 + Cfg::kFirst + 128);
      }
      __syncwarp();
      return;
    }
  }

  const L1Map m(tid);
  GridBar bar(gs);
  TRACE_INIT();
  trace(1, 0);

  l1_load_image<NAMED>(x + static_cast<size_t>(n) * 784, xs, tid);
  if (tid < 16) {
    const float mean = saved[tid], invstd = saved[16 + tid];
    const float g = gamma ? gamma[tid] : 1.f, b = beta ? beta[tid] : 0.f;
    s_mean[tid] = mean;
    s_invstd[tid] = invstd;
    s_scale[tid] = g * invstd;
    s_shift[tid] = b - mean * g * invstd;
  }
  if constexpr (kAdam) {
    if (sr.on) adam_factors(sr, adam_f, tid);   // reads the step counts: before the first grid barrier
  }
  cta_sync<NAMED>();

  float yv[16], dz[16];
  {
    const float4* yp = reinterpret_cast<const float4*>(y + ((static_cast<size_t>(n) * 28 + m.r) * 28 + m.c) * 16);
    const float4* gp = reinterpret_cast<const float4*>(dp + ((static_cast<size_t>(n) * 18 + m.ph + 2) * 18 + m.pw + 2) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 a = m.valid ? yp[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 g4 = m.valid ? gp[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      yv[4 * q] = a.x; yv[4 * q + 1] = a.y; yv[4 * q + 2] = a.z; yv[4 * q + 3] = a.w;
      dz[4 * q] = g4.x; dz[4 * q + 1] = g4.y; dz[4 * q + 2] = g4.z; dz[4 * q + 3] = g4.w;
    }
  }
  // route the pooled gradient to the arg-max of the window (first maximum wins, like torch) and through the ReLU
  unsigned int mine = 0;
  float zmax[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float z = fmaf(yv[j], s_scale[j], s_shift[j]);
    float t = fmaxf(z, __shfl_xor_sync(0xffffffffu, z, 1));
    t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 2));
    zmax[j] = t;
    mine |= (z == t ? 1u : 0u) << j;
  }
  if constexpr (WG) asm volatile("bar.arrive 4, %0;" ::"n"(L1WgCfg::kThreads) : "memory");   // y / dp have arrived: the tensor-core warp may load
  unsigned int lower = 0;  // positions of the window that come before this one
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const unsigned int other = __shfl_sync(0xffffffffu, mine, (lane & ~3) + k);
    if (k < m.d) lower |= other;
  }
  const unsigned int win = mine & ~lower;
  {
    float v[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const bool take = m.valid && ((win >> j) & 1u) && zmax[j] > 0.f;
      dz[j] = take ? dz[j] : 0.f;
      const float xhat = (yv[j] - s_mean[j]) * s_invstd[j];
      yv[j] = xhat;  // from here on yv holds x̂
      v[j] = dz[j];
      v[16 + j] = dz[j] * xhat;
    }
    warp_transpose_reduce32(v, lane);
    red[warp * 32 + lane] = v[0];
  }
  cta_sync<NAMED>();
  if (tid < 32) {
    float s = 0.f;
#pragma unroll 5
    for (int wi = 0; wi < kL1Warps; ++wi) s += red[wi * 32 + tid];
    partials[static_cast<size_t>(n) * 32 + tid] = s;
  }
  trace(1, 1);
  bar.arrive<NAMED>(gs);
  // (each update below is spelled out for both riders: the SGD instantiation keeps the code it had before the Adam rider existed)
  const float sgd_lr = sr.on ? (sr.h.lr_dev ? __ldg(sr.h.lr_dev) : static_cast<float>(sr.h.lr)) : 0.f;
  if constexpr (kClip) {
    // in the barrier's shadow: the norm partial of the parameters whose gradients were complete before this kernel started
    // (classifier, bn2); their update waits for the coefficient
    float ca = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (sr.p[6 + t])
        for (int i = n * kL1Threads + tid; i < sr.n_prev[t]; i += B * kL1Threads) ca = clip_acc(sr, ca, __ldg(sr.g_prev[t] + i));
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) ca = clip_comb(sr, ca, __shfl_xor_sync(0xffffffffu, ca, off));
    if (lane == 0) s_clip[warp] = ca;
  } else if (sr.on) {
    // in the barrier's shadow: the optimizer step of the parameters whose gradients were complete before this kernel started
    // (classifier, bn2) — nothing in this kernel reads them
#pragma unroll
    for (int t = 0; t < 4; ++t)
      for (int i = n * kL1Threads + tid; i < sr.n_prev[t]; i += B * kL1Threads)
        if constexpr (kAdam) adam_apply(sr, 6 + t, i, __ldg(sr.g_prev[t] + i), adam_f);
        else sgd_apply(sr.p[6 + t] + i, __ldg(sr.g_prev[t] + i), sr.m[6 + t] ? sr.m[6 + t] + i : nullptr, sr.h, sgd_lr);
  }
  bar.wait<NAMED>(gs);
  trace(1, 2);
  fold_rows_wide<32, kL1Threads, NAMED>(partials, B, s_tmp, s_tot);  // [0..16) Σdz, [16..32) Σdz·x̂
  trace(1, 3);
  if (n == 0 && tid < 16) {
    if (dbeta) dbeta[tid] = s_tot[tid];
    if (dgamma) dgamma[tid] = s_tot[16 + tid];
  }
  const float inv_cnt = 1.f / (static_cast<float>(B) * 784.f);
  if (m.valid) {
    float4* dst = reinterpret_cast<float4*>(dys + (m.r * 28 + m.c) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * q + e;
        o[e] = s_scale[j] * (dz[j] - s_tot[j] * inv_cnt - yv[j] * (s_tot[16 + j] * inv_cnt));
      }
      dst[q] = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
  cta_sync<NAMED>();
  // conv1 weight gradient of this image on the tensor cores: dW[co][tap] = Σ_px dy[px][co] · x[px + tap] is a
  // 16 × 32 × 784 GEMM (taps 25..31 padded; tap 25 multiplies a column of ones → the bias gradient).  M = 16 is below
  // the 64-row wgmma tile, so this is warp-level mma.sync m16n8k8 (TF32 in, fp32 accumulate): a warp takes every
  // 25th group of 8 pixels, builds the A fragment from the staged dy and the four B fragments (8 taps each) straight
  // from the haloed image — no im2col buffer — and the 25 per-warp 16×32 accumulators are folded through smem.
  {
    const int g = lane >> 2, t4 = lane & 3;
    float c[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) c[j][e] = 0.f;
    int toff[4];   // offset of tap 8j + g inside the 32-wide haloed image; < 0: padding tap (25 = ones column)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int tap = 8 * j + g;
      toff[j] = tap < 25 ? (tap / 5) * 32 + tap % 5 : (tap == 25 ? -1 : -2);
    }
    for (int ks = warp; ks < 98; ks += kL1Warps) {
      const int pa = ks * 8 + t4, pb = pa + 4;          // the two pixels (K indices) this lane touches
      const int ia = (pa / 28) * 32 + pa % 28, ib = (pb / 28) * 32 + pb % 28;
      uint32_t af[4];
      af[0] = f32_to_tf32(dys[pa * 16 + g]);
      af[1] = f32_to_tf32(dys[pa * 16 + g + 8]);
      af[2] = f32_to_tf32(dys[pb * 16 + g]);
      af[3] = f32_to_tf32(dys[pb * 16 + g + 8]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xa = toff[j] >= 0 ? xs[ia + toff[j]] : (toff[j] == -1 ? 1.f : 0.f);
        const float xb = toff[j] >= 0 ? xs[ib + toff[j]] : (toff[j] == -1 ? 1.f : 0.f);
        mma_m16n8k8_tf32(c[j], af, f32_to_tf32(xa), f32_to_tf32(xb));
      }
    }
    // C fragment: c[j][0..1] = (co g, taps 8j + 2·t4 + {0,1}), c[j][2..3] = (co g + 8, same taps)
    float* wf = fold + warp * 512;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      *reinterpret_cast<float2*>(wf + g * 32 + 8 * j + 2 * t4) = make_float2(c[j][0], c[j][1]);
      *reinterpret_cast<float2*>(wf + (g + 8) * 32 + 8 * j + 2 * t4) = make_float2(c[j][2], c[j][3]);
    }
  }
  // bias gradient in full fp32 (its true value behind a BatchNorm is zero: TF32-rounded dy would leave 1e-4 of noise):
  // thread = (channel, one of 32 pixel classes), partial sums parked in the unused tap columns 26..31 of warp 0's tile
  float dbp = 0.f;
  if (tid < 512) {
    const int co = tid & 15, part = tid >> 4;
    for (int p = part; p < 784; p += 32) dbp += dys[p * 16 + co];
  }
  cta_sync<NAMED>();
  float* s_db = red;   // [32 parts][16]  (the statistics scratch is free again)
  if (tid < 512) s_db[tid] = dbp;
  cta_sync<NAMED>();
  if (tid < 512) {
    float sacc = 0.f;
    if ((tid & 31) == 25) {
      const int co = tid >> 5;
#pragma unroll 8
      for (int part = 0; part < 32; ++part) sacc += s_db[part * 16 + co];
    } else {
#pragma unroll 5
      for (int wi = 0; wi < kL1Warps; ++wi) sacc += fold[wi * 512 + tid];
    }
    partials_w[static_cast<size_t>(n) * 512 + tid] = sacc;   // index = co·32 + tap  (tap 25 = bias, 26..31 unused)
  }
  trace(1, 4);
  if constexpr (WG) {
    // the operands have been loading since the kernel started: 15 warps take one 32-row atom each and write this image's
    // partial [512][32]
    asm volatile("bar.sync 0, %0;" ::"n"(L1WgCfg::kThreads) : "memory");   // (1) ld_full initialised (long ago)
    if (warp < 15) {
      mbar_wait(ld_full, 0);
      const int mt = warp >> 2, a = warp & 3;   // atom a of group mt (group 3 has three)
      const int shift0 = mt < 3 ? (0 - 2) * 18 + 2 * mt - 2 : 2 * 18 - 2;
      const int stride = mt < 3 ? 18 : 2;

      float acc[2][4][4];
#pragma unroll
      for (int j2 = 0; j2 < 2; ++j2)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[j2][nt][e] = 0.f;
      wgrad_win_atom<256, 32, 1>(acc, reinterpret_cast<const float*>(sa), L1WgCfg::kFirst + shift0 + a * stride, 0, reinterpret_cast<const float*>(sb), 0,
                     lane);
      wgrad_win_atom_store(acc, wpart + (static_cast<size_t>(n) * 512 + mt * 128 + a * 32) * 32, lane);
    }
    trace(1, 7);
  }
  bar.sync<NAMED>(gs);
  trace(1, 5);
  float ca = 0.f;   // ClipRider: this thread's share of the norm of the gradients folded from here on
  // every CTA folds a few of the 16 × 26 outputs over the B partial rows: one warp per output, fixed order
  for (int j = n + warp * B; j < 512; j += kL1Warps * B) {
    const int co = j >> 5, tap = j & 31;
    if (tap > 25) continue;
    float s = 0.f;
    for (int r = lane; r < B; r += 32) s += __ldcg(partials_w + static_cast<size_t>(r) * 512 + j);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) {
      if (tap < 25) {
        dw[co * 25 + tap] = s;
        if constexpr (kClip) ca = clip_acc(sr, ca, s);
        else if constexpr (kAdam) { if (sr.on) adam_apply(sr, 0, co * 25 + tap, s, adam_f); }
        else if (sr.on) sgd_apply(sr.p[0] + co * 25 + tap, s, sr.m[0] ? sr.m[0] + co * 25 + tap : nullptr, sr.h, sgd_lr);
      } else if (db) {
        db[co] = s;
        if constexpr (kClip) { if (sr.p[1]) ca = clip_acc(sr, ca, s); }
        else if constexpr (kAdam) { if (sr.on && sr.p[1]) adam_apply(sr, 1, co, s, adam_f); }
        else if (sr.on && sr.p[1]) sgd_apply(sr.p[1] + co, s, sr.m[1] ? sr.m[1] + co : nullptr, sr.h, sgd_lr);
      }
    }
  }
  if (sr.on && n == 0 && tid < 16) {
    // BatchNorm-1 affine parameters: their gradients are the totals this CTA folded after the first barrier.  Every CTA read
    // gamma / beta before that barrier, so updating them here (after the second one) races with nobody.
    if constexpr (kClip) {
      if (sr.p[3]) ca = clip_acc(sr, ca, s_tot[tid]);
      if (sr.p[2]) ca = clip_acc(sr, ca, s_tot[16 + tid]);
    } else if constexpr (kAdam) {
      if (sr.p[3]) adam_apply(sr, 3, tid, s_tot[tid], adam_f);
      if (sr.p[2]) adam_apply(sr, 2, tid, s_tot[16 + tid], adam_f);
    } else {
      if (sr.p[3]) sgd_apply(sr.p[3] + tid, s_tot[tid], sr.m[3] ? sr.m[3] + tid : nullptr, sr.h, sgd_lr);
      if (sr.p[2]) sgd_apply(sr.p[2] + tid, s_tot[16 + tid], sr.m[2] ? sr.m[2] + tid : nullptr, sr.h, sgd_lr);
    }
  }
  if constexpr (kAdam && !kClip) {
    // every CTA read the step counts before the first grid barrier and this is after the last one
    if (sr.on && n == 0 && tid == 0)
      for (int k = 0; k < 10; ++k)
        if (sr.step[k]) *sr.step[k] += 1.f;
  }
  if constexpr (WG) {
    // conv2 weight gradient: CTA n folds outputs n, n + B, … of the 400 (tap, ci) rows × 32 co (+ row 400: the bias, from the
    // per-image Σdy rows) over the B per-image partials — warp = one of 25 partial classes, lane = co, classes combined
    // through smem in a fixed order, up to five outputs per round so that ~20 L2 loads per thread are in flight
    float* s_f = fold;   // [5][25][32]
    constexpr size_t kStride = 512 * 32;
    for (int base = n; base < 401; base += 5 * B) {
      float acc[5];
      const float* src[5];
      size_t stride[5];
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        const int i = base + u * B;
        if (i < 400) {
          const int tap = i >> 4, ci = i & 15, kh = tap / 5, kw = tap - kh * 5;
          // accumulator row of (kh, kw, ci): tiles 0-2 = kw/2 with kh 0..3 stacked, tile 3 = kh 4 with kw/2 stacked
          const int mrow = (kh < 4 ? (kw >> 1) * 128 + kh * 32 : 384 + (kw >> 1) * 32) + (kw & 1) * 16 + ci;
          src[u] = wpart + static_cast<size_t>(mrow) * 32 + lane;
          stride[u] = kStride;
        } else {
          src[u] = i == 400 ? dysum2 + lane : nullptr;   // row 400: the bias gradient from the per-image Σdy rows
          stride[u] = 32;
        }
        acc[u] = 0.f;
      }
      for (int c0 = warp; c0 < B; c0 += 4 * kL1Warps) {   // 5 outputs × 4 rows = 20 independent L2 loads in flight per thread
        float t[5][4];
#pragma unroll
        for (int u = 0; u < 5; ++u)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = c0 + j * kL1Warps;
            t[u][j] = (src[u] != nullptr && c < B) ? __ldcg(src[u] + static_cast<size_t>(c) * stride[u]) : 0.f;
          }
#pragma unroll
        for (int u = 0; u < 5; ++u)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[u] += t[u][j];
      }
      cta_sync<NAMED>();
#pragma unroll
      for (int u = 0; u < 5; ++u) s_f[(u * kL1Warps + warp) * 32 + lane] = acc[u];
      cta_sync<NAMED>();
      if (tid < 160) {
        const int u = tid >> 5, i = base + u * B;
        if (i <= 400) {
          float tot = 0.f;
#pragma unroll 5
          for (int wi = 0; wi < kL1Warps; ++wi) tot += s_f[(u * kL1Warps + wi) * 32 + lane];
          if (i < 400) {
            const int e = (lane * 16 + (i & 15)) * 25 + (i >> 4);
            dw2[e] = tot;
            if constexpr (kClip) ca = clip_acc(sr, ca, tot);
            else if constexpr (kAdam) { if (sr.on) adam_apply(sr, 4, e, tot, adam_f); }
            else if (sr.on) sgd_apply(sr.p[4] + e, tot, sr.m[4] ? sr.m[4] + e : nullptr, sr.h, sgd_lr);
          } else if (db2) {
            db2[lane] = tot;
            if constexpr (kClip) { if (sr.p[5]) ca = clip_acc(sr, ca, tot); }
            else if constexpr (kAdam) { if (sr.on && sr.p[5]) adam_apply(sr, 5, lane, tot, adam_f); }
            else if (sr.on && sr.p[5]) sgd_apply(sr.p[5] + lane, tot, sr.m[5] ? sr.m[5] + lane : nullptr, sr.h, sgd_lr);
          }
        }
      }
    }
  }
  if constexpr (kClip) {
    // every gradient has been seen: one partial per CTA, one more grid barrier, then every CTA folds the B partials in the same
    // order and derives the same coefficient bit for bit
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) ca = clip_comb(sr, ca, __shfl_xor_sync(0xffffffffu, ca, off));
    if (lane == 0) s_clip[warp] = clip_comb(sr, s_clip[warp], ca);
    cta_sync<NAMED>();
    if (tid == 0) {
      float s = s_clip[0];
      for (int w = 1; w < kL1Warps; ++w) s = clip_comb(sr, s, s_clip[w]);
      sr.part[n] = s;
    }
    bar.sync<NAMED>(gs);
    if (warp == 0) {
      double d = 0.0;
      for (int r = lane; r < B; r += 32) {
        const double v = static_cast<double>(__ldcg(sr.part + r));
        d = sr.norm_inf ? nan_max(d, v) : d + v;
      }
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, d, off);
        d = sr.norm_inf ? nan_max(d, o) : d + o;
      }
      if (lane == 0) {
        const float norm = static_cast<float>(sr.norm_inf ? d : sqrt(d));
        s_clip[kL1Warps] = clip_coef(norm, sr.max_norm);
        if (n == 0) *sr.norm_out = norm;
      }
    }
    cta_sync<NAMED>();
    const float coef = s_clip[kL1Warps];
    // grid-stride pass over the ten gradients (read from L2: other CTAs wrote them): .grad becomes the clipped gradient, as after
    // clip_grad_norm_, and the update takes it
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      float* gk = k == 0 ? dw : k == 1 ? db : k == 2 ? dgamma : k == 3 ? dbeta : k == 4 ? dw2 : k == 5 ? db2 : const_cast<float*>(sr.g_prev[k - 6]);
      const int nk = k == 0 ? 400 : k == 4 ? 12800 : k == 5 ? 32 : k < 6 ? 16 : sr.n_prev[k - 6];
      if (!sr.p[k] || !gk) continue;
      for (int i = n * kL1Threads + tid; i < nk; i += B * kL1Threads) {
        const float gv = __ldcg(gk + i) * coef;
        gk[i] = gv;
        if constexpr (kAdam) adam_apply(sr, k, i, gv, adam_f);
        else sgd_apply(sr.p[k] + i, gv, sr.m[k] ? sr.m[k] + i : nullptr, sr.h, sgd_lr);
      }
    }
    if constexpr (kAdam) {
      // every CTA read the step counts before the first grid barrier and this is after the last one
      if (n == 0 && tid == 0)
        for (int k = 0; k < 10; ++k)
          if (sr.step[k]) *sr.step[k] += 1.f;
    }
  }
  bar.finish(gs);
  trace(1, 6);
}

// =====================================================================================================================
// Layer 2 — conv2 (16→32, 5x5) is 88 % of the model's FLOPs: wgmma.  One CTA = one 14×14 image.
// The zero-haloed input (18×18 positions × 128-byte rows, channels 16..31 zero-filled by TMA) is loaded ONCE; output
// pixel (oh, ow) is MMA row p = oh·18 + ow of one of two M = 128 tiles (rows 0..125 ↔ oh 0..6, 126..251 ↔ oh 7..13;
// ow ≥ 14 rows are padding), and filter tap (kh, kw) is the same buffer read through a K-major SWIZZLE_128B descriptor
// that starts (kh·18 + kw) rows further in (the swizzle phase follows the absolute address; the bit-exact
// tests/test_gpu_kernels.py::test_cooperative_layer2_exact_on_small_integers guards this).  Weights are swizzled into
// shared memory by the CTA itself.
// =====================================================================================================================
constexpr int kL2Threads = 256;
constexpr int kPW = 18;                          // padded width
constexpr int kPatchRows = 18 * 18;              // 324 positions
constexpr int kPatchBytes = kPatchRows * 128;    // 41,472
constexpr int kPatchAlloc = 43008;               // + slack rows read by the padding rows of tile 1 (multiple of 1024)

__device__ __forceinline__ uint32_t sw128_off(int row, int chunk16) { return static_cast<uint32_t>(row) * 128u + (static_cast<uint32_t>(chunk16 ^ (row & 7)) << 4); }

// conv2 of one image on the tensor cores, issued by the warpgroup of warps 4..7 (wt = thread index inside it): per output
// tile t, 25 taps × 2 K-steps of wgmma m64n32k8 per 64-row half, the A descriptors row-shifted into the haloed patch.  The
// accumulators go straight into ys [pixel][32] (bias added; 16-byte chunks rotated by the pixel index, as the column reads
// that follow expect).
__device__ __forceinline__ void l2_conv_wgmma(const uint8_t* sa, const uint8_t* sb, const float* __restrict__ bias, float* ys, int wt) {
  const uint64_t ad0 = gmma_desc_kmajor<128>(smem_u32(sa)), bd0 = gmma_desc_kmajor<128>(smem_u32(sb));
#pragma unroll 1
  for (int t = 0; t < 2; ++t) {
    float acc[2][16];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 16; ++e) acc[h][e] = 0.f;
    wgmma_fence();
#pragma unroll 1
    for (int kh = 0; kh < 5; ++kh) {
      const uint64_t ad = ad0 + static_cast<uint64_t>(((7 * t + kh) * kPW * 128) >> 4);
      const uint64_t bd = bd0 + static_cast<uint64_t>((kh * 5 * 4096) >> 4);
#pragma unroll
      for (int kw = 0; kw < 5; ++kw) {
#pragma unroll
        for (int k = 0; k < 2; ++k)   // K = 16 input channels = two K=8 steps; the zero upper half is never multiplied
#pragma unroll
          for (int h = 0; h < 2; ++h)
            wgmma_m64n32k8_tf32(acc[h], ad + ((h * 64 * 128 + kw * 128 + k * 32) >> 4), bd + ((kw * 4096 + k * 32) >> 4), (kh | kw | k) != 0);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int rr = 64 * h + wgmma_frag_row(wt, e), c = wgmma_frag_col(wt, e);
        const int orow = rr / kPW, ow = rr - orow * kPW;
        if (rr < 126 && ow < 14) {
          const int pix = (7 * t + orow) * 14 + ow;
          ys[pix * 32 + ((((c >> 2) + pix) & 7) << 2) + (c & 3)] = acc[h][e] + (bias ? __ldg(bias + c) : 0.f);
        }
      }
    }
  }
}

struct L2FwdSmem {
  static constexpr int kB = 25 * 32 * 128;       // weights: [tap][32 co][128 B] (ci 0..15 used)            102,400
  static constexpr int kYs = 196 * 32 * 4;       // conv output of the image, [pixel][32]                     25,088
  static constexpr int kTotal = 1024 + kPatchAlloc + kB + kYs + 8192;
};

__global__ void __launch_bounds__(kL2Threads, 1)
convnet_l2_fwd_kernel(const __grid_constant__ CUtensorMap tm_x, const float* __restrict__ w, const float* __restrict__ bias,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y, float* __restrict__ out,
                      float* saved, float* running_mean, float* running_var, long long* nbt, float momentum, float eps,
                      const float* __restrict__ fcw, const float* __restrict__ fcb, float* __restrict__ logits, int ncls,
                      float* partials, GridSync gs) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                  // input patch (TMA, SWIZZLE_128B)
  uint8_t* sb = sa + kPatchAlloc;                      // weights
  float* ys = reinterpret_cast<float*>(sb + L2FwdSmem::kB);
  float* misc = ys + 196 * 32;                         // 2048 floats
  float* s_part = misc;                                // [4][64]
  float* s_tmp = misc + 256;                           // [4][64]
  float* s_tot = misc + 512;                           // [64]
  float* s_scale = misc + 576;                         // [32]
  float* s_shift = misc + 608;                         // [32]

  __shared__ uint64_t bar_x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;

  GridBar bar(gs);
  TRACE_INIT();
  trace(2, 0);
  if (tid == 0) {
    tma_prefetch_desc(&tm_x);
    mbar_init(&bar_x, 1);
    fence_mbar_init();
  }
  // zero the slack behind the patch (read only by padding rows, but keep NaNs out of the accumulators)
  for (int i = tid; i < (kPatchAlloc - kPatchBytes) / 16; i += kL2Threads) reinterpret_cast<float4*>(sa + kPatchBytes)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bar_x, kPatchBytes);
    tma_load_4d(sa, &tm_x, &bar_x, 0, 0, 0, n);        // the frame carries its zero halo; channels ≥ 16: out-of-bounds zero fill
  }
  // B[tap][co][ci] = w[co][ci][tap], K-major rows of 128 B, SWIZZLE_128B
  {
    // thread = two (co, ci) pairs; a pair's 25 taps are contiguous in w (a warp reads 3,200 contiguous bytes) and land
    // 4,096 B apart in smem (one swizzled K-major tile per tap): all 50 loads are in flight before the first store
    float wv[2][25];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float* src = w + (tid + j * kL2Threads) * 25;
#pragma unroll
      for (int tap = 0; tap < 25; ++tap) wv[j][tap] = __ldg(src + tap);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int pair = tid + j * kL2Threads, co = pair >> 4, ci = pair & 15;
      uint8_t* dst = sb + sw128_off(co, ci >> 2) + (ci & 3) * 4;
#pragma unroll
      for (int tap = 0; tap < 25; ++tap) *reinterpret_cast<float*>(dst + tap * 4096) = wv[j][tap];
    }
  }
  fence_proxy_async_smem();   // generic-proxy writes of B → visible to the tensor core
  __syncthreads();
  trace(2, 1);
  // ---- conv2 + epilogue: the warpgroup of warps 4..7 ------------------------------------------------------------------------
  if (warpgroup_index() == 1) {
    mbar_wait(&bar_x, 0);
    l2_conv_wgmma(sa, sb, bias, ys, tid - 128);
  }
  __syncthreads();
  trace(2, 2);
  // ---- per-channel Σy, Σy² of this image: thread = (channel, quarter of the pixels) --------------------------------------
  if (tid < 128) {
    const int c = tid & 31, part = tid >> 5;
    float s1 = 0.f, s2 = 0.f;
    for (int p = part * 49; p < part * 49 + 49; ++p) {
      const float val = ys[p * 32 + ((((c >> 2) + p) & 7) << 2) + (c & 3)];
      s1 += val;
      s2 = fmaf(val, val, s2);
    }
    s_part[part * 64 + c] = s1;
    s_part[part * 64 + 32 + c] = s2;
  }
  __syncthreads();
  if (tid < 64) partials[static_cast<size_t>(n) * 64 + tid] = (s_part[tid] + s_part[64 + tid]) + (s_part[128 + tid] + s_part[192 + tid]);
  trace(2, 3);
  bar.sync(gs);
  trace(2, 4);
  // conv output → global (kept for backward), after the barrier: un-rotate the 16-byte chunks on the way out
  for (int i = tid; i < 196 * 8; i += kL2Threads) {
    const int pix = i >> 3, q = i & 7;
    reinterpret_cast<float4*>(y + (static_cast<size_t>(n) * 196 + pix) * 32)[q] = reinterpret_cast<const float4*>(ys + pix * 32)[(q + pix) & 7];
  }
  fold_rows<64>(partials, B, s_tmp, s_tot);
  trace(2, 5);
  if (tid < 32) {
    const float cnt = static_cast<float>(B) * 196.f;
    const float mean = s_tot[tid] / cnt;
    const float var = fmaxf(s_tot[32 + tid] / cnt - mean * mean, 0.f);
    const float invstd = rsqrtf(var + eps);
    const float g = gamma ? gamma[tid] : 1.f, b = beta ? beta[tid] : 0.f;
    s_scale[tid] = g * invstd;
    s_shift[tid] = b - mean * g * invstd;
    if (n == 0) {
      saved[tid] = mean;
      saved[32 + tid] = invstd;
      if (running_mean) {
        const float unbiased = var * (cnt / fmaxf(cnt - 1.f, 1.f));
        running_mean[tid] = (1.f - momentum) * running_mean[tid] + momentum * mean;
        running_var[tid] = (1.f - momentum) * running_var[tid] + momentum * unbiased;
      }
      if (nbt && tid == 0) *nbt += 1;
    }
  }
  __syncthreads();
  // ---- BN + ReLU + MaxPool 2×2 → NCHW [32][7][7] (the flatten order of the classifier, ref :39) ------------------------
  float* pool = reinterpret_cast<float*>(sb);   // the weights are dead after the MMAs: reuse their space
  for (int i = tid; i < 1568; i += kL2Threads) {
    const int c = i & 31, pp = i >> 5, ph = pp / 7, pw = pp - ph * 7;
    const float sc = s_scale[c], sh = s_shift[c];
    float mx = 0.f;   // the ReLU floor doubles as the identity of max
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int p = (2 * ph + (d >> 1)) * 14 + 2 * pw + (d & 1);
      mx = fmaxf(mx, fmaf(ys[p * 32 + ((((c >> 2) + p) & 7) << 2) + (c & 3)], sc, sh));
    }
    pool[c * 49 + pp] = mx;
  }
  __syncthreads();
  for (int i = tid; i < 1568; i += kL2Threads) out[static_cast<size_t>(n) * 1568 + i] = pool[i];
  trace(2, 6);
  // ---- classifier head riding on the pooled activations still in shared memory: logits = fc(pool) ----------------------
  if (logits != nullptr && ncls <= 16) {
    // thread t owns features t, t+256, … (≤ 7) for every class: all weight loads are independent and in flight together
    float pv[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) pv[j] = (tid + j * kL2Threads < 1568) ? pool[tid + j * kL2Threads] : 0.f;
    float accv[16];
#pragma unroll
    for (int c16 = 0; c16 < 16; ++c16) {
      float sacc = 0.f;
      if (c16 < ncls) {
        const float* wr = fcw + static_cast<size_t>(c16) * 1568 + tid;
#pragma unroll
        for (int j = 0; j < 7; ++j)
          if (tid + j * kL2Threads < 1568) sacc = fmaf(pv[j], __ldg(wr + j * kL2Threads), sacc);
      }
      accv[c16] = sacc;
    }
#pragma unroll
    for (int c16 = 0; c16 < 16; ++c16) {
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) accv[c16] += __shfl_xor_sync(0xffffffffu, accv[c16], off);
    }
    float* s_fc = s_part;   // [8 warps][16]
    if (lane == 0) {
#pragma unroll
      for (int c16 = 0; c16 < 16; ++c16) s_fc[warp * 16 + c16] = accv[c16];
    }
    __syncthreads();
    if (tid < ncls) {
      float sfin = fcb ? fcb[tid] : 0.f;
#pragma unroll
      for (int w8 = 0; w8 < 8; ++w8) sfin += s_fc[w8 * 16 + tid];
      logits[static_cast<size_t>(n) * ncls + tid] = sfin;
    }
  } else if (logits != nullptr) {
    // warp k computes classes k, k+8, ...: 1568-long dot products, lanes stride the features
    for (int cls = warp; cls < ncls; cls += kL2Threads / 32) {
      const float* wr = fcw + static_cast<size_t>(cls) * 1568;
      float s = 0.f;
      for (int k = lane; k < 1568; k += 32) s = fmaf(pool[k], __ldg(wr + k), s);
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
      if (lane == 0) logits[static_cast<size_t>(n) * ncls + cls] = s + (fcb ? fcb[cls] : 0.f);
    }
  }

  __syncthreads();
  bar.finish(gs);
  trace(2, 7);
}

// =====================================================================================================================
// Whole forward pass in ONE kernel: layer 1 and layer 2 (+ classifier) of an image run in the same CTA, so the pooled
// layer-1 activations never leave the SM on their way into conv2 — they are written straight into the swizzled,
// zero-haloed shared-memory patch the wgmma descriptors read (the global copy is still written: backward needs it) —
// and the conv2 weights are staged while conv1 computes.  Two grid barriers (BN1 and BN2 batch statistics), one launch.
// =====================================================================================================================
__global__ void __launch_bounds__(kL1Threads, 1)
convnet_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ g1,
                   const float* __restrict__ be1, float* __restrict__ y1, float* __restrict__ p1, float* saved1, float* rm1, float* rv1,
                   long long* nbt1, float mom1, float eps1, const float* __restrict__ w2, const float* __restrict__ b2,
                   const float* __restrict__ g2, const float* __restrict__ be2, float* __restrict__ y2, float* __restrict__ out, float* saved2,
                   float* rm2, float* rv2, long long* nbt2, float mom2, float eps2, const float* __restrict__ fcw,
                   const float* __restrict__ fcb, float* __restrict__ logits, int ncls, float* partials, GridSync gs, FusedCe ce) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                  // conv2 input patch, written by this CTA's layer-1 epilogue
  uint8_t* sb = sa + kPatchAlloc;                      // conv2 weights
  float* ys = reinterpret_cast<float*>(sb + L2FwdSmem::kB);
  float* misc = ys + 196 * 32;                         // 2048 floats
  float* s_part = misc;                                // [4][64] / [25 warps][16]
  float* s_tmp2 = misc + 1024;                         // [12][64]
  float* s_tot2 = misc + 768;                          // [64]
  float* s_scale2 = misc + 832;                        // [32]
  float* s_shift2 = misc + 864;                        // [32]
  __shared__ float xs[32 * 32];
  __shared__ __align__(16) float ws[25 * 16];
  __shared__ float red[kL1Warps * 32];
  __shared__ float s_tmp[kL1Warps * 32];
  __shared__ float s_tot[32];
  __shared__ float s_scale[16], s_shift[16];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;
  const L1Map m(tid);
  GridBar bar(gs);
  TRACE_INIT();
  trace(0, 0);

  for (int i = tid; i < kPatchAlloc / 16; i += kL1Threads) reinterpret_cast<float4*>(sa)[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // halo = 0
  l1_load_image(x + static_cast<size_t>(n) * 784, xs, tid);
  if (tid < 400) {
    const int tap = tid >> 4, co = tid & 15;
    ws[tid] = w1[co * 25 + tap];
  }
  // conv2 weights: one (co, ci) pair per thread, 25 taps contiguous in global, 4 KiB apart in smem (SWIZZLE_128B K-major tiles);
  // the loads fly while conv1 computes
  float wv[25];
  if (tid < 512) {
#pragma unroll
    for (int tap = 0; tap < 25; ++tap) wv[tap] = __ldg(w2 + tid * 25 + tap);
  }
  __syncthreads();
  trace(0, 11);

  // ---- layer 1 ------------------------------------------------------------------------------------------------------
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = b1 ? __ldg(b1 + j) : 0.f;
#pragma unroll 1
  for (int kh = 0; kh < 5; ++kh) {
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      const float xv = xs[(m.r + kh) * 32 + m.c + kw];
      const float4* wt = reinterpret_cast<const float4*>(ws + (kh * 5 + kw) * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 wq = wt[q];
        acc[4 * q + 0] = fmaf(xv, wq.x, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(xv, wq.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(xv, wq.z, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(xv, wq.w, acc[4 * q + 3]);
      }
    }
  }
  trace(0, 1);
  if (tid < 512) {
    const int co = tid >> 4, ci = tid & 15;
    uint8_t* dst = sb + sw128_off(co, ci >> 2) + (ci & 3) * 4;
#pragma unroll
    for (int tap = 0; tap < 25; ++tap) *reinterpret_cast<float*>(dst + tap * 4096) = wv[tap];
  }
  {
    float v[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      v[j] = m.valid ? acc[j] : 0.f;
      v[16 + j] = m.valid ? acc[j] * acc[j] : 0.f;
    }
    warp_transpose_reduce32(v, lane);
    red[warp * 32 + lane] = v[0];
  }
  __syncthreads();
  if (tid < 32) {
    float s = 0.f;
#pragma unroll 5
    for (int wi = 0; wi < kL1Warps; ++wi) s += red[wi * 32 + tid];
    partials[static_cast<size_t>(n) * 32 + tid] = s;
  }
  trace(0, 2);
  bar.arrive(gs);
  // in the barrier's shadow: everything layer 1 owes to global memory (backward reads it; nothing in this kernel does)
  if (m.valid) {
    float4* yp = reinterpret_cast<float4*>(y1 + ((static_cast<size_t>(n) * 28 + m.r) * 28 + m.c) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) yp[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
  }
  for (int i = tid; i < 324 * 4; i += kL1Threads) {
    const int P = i >> 2, pr = P / 18, pc = P - pr * 18;
    if (pr < 2 || pr >= 16 || pc < 2 || pc >= 16) reinterpret_cast<float4*>(p1 + (static_cast<size_t>(n) * 324 + P) * 16)[i & 3] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  bar.wait(gs);
  trace(0, 3);
  fold_rows_wide<32, kL1Threads>(partials, B, s_tmp, s_tot);
  if (tid < 16) {
    const float cnt = static_cast<float>(B) * 784.f;
    const float mean = s_tot[tid] / cnt;
    const float var = fmaxf(s_tot[16 + tid] / cnt - mean * mean, 0.f);
    const float invstd = rsqrtf(var + eps1);
    const float g = g1 ? g1[tid] : 1.f, b = be1 ? be1[tid] : 0.f;
    s_scale[tid] = g * invstd;
    s_shift[tid] = b - mean * g * invstd;
    if (n == 0) {
      saved1[tid] = mean;
      saved1[16 + tid] = invstd;
      if (rm1) {
        const float unbiased = var * (cnt / fmaxf(cnt - 1.f, 1.f));
        rm1[tid] = (1.f - mom1) * rm1[tid] + mom1 * mean;
        rv1[tid] = (1.f - mom1) * rv1[tid] + mom1 * unbiased;
      }
      if (nbt1 && tid == 0) *nbt1 += 1;
    }
  }
  __syncthreads();
  {
    float z[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float t = fmaxf(fmaf(acc[j], s_scale[j], s_shift[j]), 0.f);
      t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 1));
      t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, 2));
      z[j] = t;
    }
    if (m.valid) {  // lane d of the window owns channels 4d..4d+3 = one 16-byte chunk of the 128-byte patch row
      float4 o;
      if (m.d == 0) o = make_float4(z[0], z[1], z[2], z[3]);
      else if (m.d == 1) o = make_float4(z[4], z[5], z[6], z[7]);
      else if (m.d == 2) o = make_float4(z[8], z[9], z[10], z[11]);
      else o = make_float4(z[12], z[13], z[14], z[15]);
      const int P = (m.ph + 2) * kPW + m.pw + 2;
      *reinterpret_cast<float4*>(sa + sw128_off(P, m.d)) = o;                                   // conv2 reads this one
      reinterpret_cast<float4*>(p1 + (static_cast<size_t>(n) * 324 + P) * 16)[m.d] = o;         // backward (conv2 wgrad) reads this one
    }
  }
  fence_proxy_async_smem();   // generic-proxy writes of the patch and of the weights → visible to the tensor core
  __syncthreads();
  trace(0, 4);
  // ---- layer 2: 200 wgmma (K = 8, M = 64 each) by the warpgroup of warps 4..7 --------------------------------------------
  if (warpgroup_index() == 1) l2_conv_wgmma(sa, sb, b2, ys, tid - 128);
  __syncthreads();
  trace(0, 5);
  if (tid < 128) {
    const int c = tid & 31, part = tid >> 5;
    float s1 = 0.f, s2 = 0.f;
    for (int p = part * 49; p < part * 49 + 49; ++p) {
      const float val = ys[p * 32 + ((((c >> 2) + p) & 7) << 2) + (c & 3)];
      s1 += val;
      s2 = fmaf(val, val, s2);
    }
    s_part[part * 64 + c] = s1;
    s_part[part * 64 + 32 + c] = s2;
  }
  __syncthreads();
  float* partials2 = partials + static_cast<size_t>(B) * 32;
  if (tid < 64) partials2[static_cast<size_t>(n) * 64 + tid] = (s_part[tid] + s_part[64 + tid]) + (s_part[128 + tid] + s_part[192 + tid]);
  trace(0, 6);
  bar.arrive(gs);
  float* fcs = reinterpret_cast<float*>(sb + 8192);   // classifier weights, staged behind the pooled activations (conv2's weights are dead)
  const bool fc_staged = logits != nullptr && (reinterpret_cast<uintptr_t>(fcw) & 15) == 0;
  if (fc_staged) {
    for (int i = tid; i < ncls * 392; i += kL1Threads) cp_async_16(smem_u32(fcs + 4 * i), fcw + 4 * i, 16);
    cp_async_commit();
  }
  for (int i = tid; i < 196 * 8; i += kL1Threads) {   // in the barrier's shadow: conv2's output for the backward pass
    const int pix = i >> 3, q = i & 7;
    reinterpret_cast<float4*>(y2 + (static_cast<size_t>(n) * 196 + pix) * 32)[q] = reinterpret_cast<const float4*>(ys + pix * 32)[(q + pix) & 7];
  }
  bar.wait(gs);
  trace(0, 7);
  fold_rows_wide<64, kL1Threads>(partials2, B, s_tmp2, s_tot2);
  if (tid < 32) {
    const float cnt = static_cast<float>(B) * 196.f;
    const float mean = s_tot2[tid] / cnt;
    const float var = fmaxf(s_tot2[32 + tid] / cnt - mean * mean, 0.f);
    const float invstd = rsqrtf(var + eps2);
    const float g = g2 ? g2[tid] : 1.f, b = be2 ? be2[tid] : 0.f;
    s_scale2[tid] = g * invstd;
    s_shift2[tid] = b - mean * g * invstd;
    if (n == 0) {
      saved2[tid] = mean;
      saved2[32 + tid] = invstd;
      if (rm2) {
        const float unbiased = var * (cnt / fmaxf(cnt - 1.f, 1.f));
        rm2[tid] = (1.f - mom2) * rm2[tid] + mom2 * mean;
        rv2[tid] = (1.f - mom2) * rv2[tid] + mom2 * unbiased;
      }
      if (nbt2 && tid == 0) *nbt2 += 1;
    }
  }
  __syncthreads();
  float* pool = reinterpret_cast<float*>(sb);   // the weights are dead after the MMAs
  for (int i = tid; i < 1568; i += kL1Threads) {
    const int c = i & 31, pp = i >> 5, ph = pp / 7, pw = pp - ph * 7;
    const float sc = s_scale2[c], sh = s_shift2[c];
    float mx = 0.f;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      const int p = (2 * ph + (d >> 1)) * 14 + 2 * pw + (d & 1);
      mx = fmaxf(mx, fmaf(ys[p * 32 + ((((c >> 2) + p) & 7) << 2) + (c & 3)], sc, sh));
    }
    pool[c * 49 + pp] = mx;
  }
  cp_async_wait<0>();
  __syncthreads();
  trace(0, 8);
  for (int i = tid; i < 1568; i += kL1Threads) out[static_cast<size_t>(n) * 1568 + i] = pool[i];
  if (logits != nullptr) {
    // classifier: thread t owns features t and t + 800 for every class (≤ 16): all weight loads independent
    float accv[16];
    const float pv0 = pool[tid], pv1 = (tid + kL1Threads < 1568) ? pool[tid + kL1Threads] : 0.f;
#pragma unroll
    for (int c16 = 0; c16 < 16; ++c16) {
      float sacc = 0.f;
      if (c16 < ncls) {
        const float* wr = (fc_staged ? fcs : fcw) + static_cast<size_t>(c16) * 1568 + tid;
        sacc = pv0 * wr[0];
        if (tid + kL1Threads < 1568) sacc = fmaf(pv1, wr[kL1Threads], sacc);
      }
      accv[c16] = sacc;
    }
#pragma unroll
    for (int c16 = 0; c16 < 16; ++c16) {
#pragma unroll
      for (int off = 16; off >= 1; off >>= 1) accv[c16] += __shfl_xor_sync(0xffffffffu, accv[c16], off);
    }
    if (lane == 0) {
#pragma unroll
      for (int c16 = 0; c16 < 16; ++c16) s_part[warp * 16 + c16] = accv[c16];
    }
    __syncthreads();
    if (warp == 0) {
      float lg = -INFINITY;   // lanes < ncls: this image's logits
      if (lane < ncls) {
        lg = fcb ? fcb[lane] : 0.f;
#pragma unroll 5
        for (int wi = 0; wi < kL1Warps; ++wi) lg += s_part[wi * 16 + lane];
        logits[static_cast<size_t>(n) * ncls + lane] = lg;
      }
      trace(0, 9);
      if (ce.target != nullptr) {
        // cross-entropy of this image and its gradient for a unit incoming gradient
        float mx = lg;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        const float e = lane < ncls ? __expf(lg - mx) : 0.f;
        float ssum = e;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, off);
        const long long t = ce.target[n];
        const bool t_ok = t >= 0 && t < ncls;
        const float lt = __shfl_sync(0xffffffffu, lg, t_ok ? static_cast<int>(t) : 0);
        if (lane < ncls) ce.dlogits[static_cast<size_t>(n) * ncls + lane] = (e / ssum - (t == lane ? 1.f : 0.f)) / static_cast<float>(B);
        if (lane == 0) ce.loss_parts[n] = t_ok ? mx + __logf(ssum) - lt : 0.f;
        if (ce.loss != nullptr) {   // batch mean now (otherwise layer-2 backward folds it: ce.loss == nullptr)
          int last = 0;
          if (lane == 0) {
            __threadfence();
            last = atomicAdd(ce.counter, 1u) == static_cast<unsigned int>(B) - 1u;
          }
          last = __shfl_sync(0xffffffffu, last, 0);
          if (last) {   // every image's term is in L2: the CTA that finished last folds the batch mean in a fixed order
            __threadfence();
            float sl = 0.f;
            for (int r = lane; r < B; r += 32) sl += __ldcg(ce.loss_parts + r);
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) sl += __shfl_xor_sync(0xffffffffu, sl, off);
            if (lane == 0) {
              *ce.loss = sl / static_cast<float>(B);
              *ce.counter = 0u;
            }
          }
        }
      }
    }
  }
  trace(0, 10);
}

// ---- layer 2 backward: pool/ReLU/BN backward + conv2 data gradient ---------------------------------------------------------
struct L2BwdSmem {
  static constexpr int kB = 25 * 16 * 128;       // dgrad weights: [tap][16 ci][128 B = 32 co]                  51,200
  static constexpr int kTotal = 1024 + kPatchAlloc + kB + 4096;
  // FC (the classifier's backward rides along): fc weights [16][1568] | dlogits [B ≤ 160][16] | pooled slice [B ≤ 160][16]
  static constexpr int kFcW = 16 * 1568 * 4, kFcDl = 160 * 16 * 4, kFcP = 160 * 16 * 4;
  static constexpr int kTotalFc = kTotal + kFcW + kFcDl + kFcP;
};

// FC: the classifier's backward rides along.  The gradient of the pooled activations is not read from `dout` but computed
// on the fly, d(out)[n][k] = Σ_j dlogits[n][j] · Wfc[j][k] (fc weights staged in smem once per CTA); the classifier's weight
// gradient dWfc[j][k] = Σ_n dlogits[n][j] · out[n][k] is produced in 16-column slices, one slice per CTA (all images, fixed
// order: deterministic, no partials), the bias gradient by the CTA that owns "slice 98".  One kernel less per step.
template <bool FC>
__global__ void __launch_bounds__(kL2Threads, 1)
convnet_l2_bwd_kernel(const float* __restrict__ dout /*[B,32,7,7]*/, const float* __restrict__ y /*[B,14,14,32]*/,
                      const float* __restrict__ saved, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ w, float* dgamma, float* dbeta, float* __restrict__ dy /*[B,18,18,32] zero-haloed frame*/,
                      float* __restrict__ dx /*[B,18,18,16] frame, interior written*/, float* __restrict__ dysum /*[B,32]*/,
                      float* partials, GridSync gs,
                      // FC only
                      const float* __restrict__ dlogits /*[B,ncls]*/, const float* __restrict__ fcw /*[ncls,1568]*/,
                      const float* __restrict__ pooled /*[B,1568] = forward's out*/, float* dfcw /*[ncls,1568]*/, float* dfcb /*[ncls]*/,
                      int ncls, const float* __restrict__ loss_parts /*[B] or null*/, float* loss_out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                  // dy patch, written by the CTA in the TMA/wgmma SWIZZLE_128B layout
  uint8_t* sb = sa + kPatchAlloc;
  float* misc = reinterpret_cast<float*>(sb + L2BwdSmem::kB);   // 1024 floats
  float* s_part = misc;                                // [8][64]
  float* s_tmp = misc + 512;                           // [4][64]
  float* s_tot = misc + 768;                           // [64]
  float* s_scale = misc + 832;
  float* s_shift = misc + 864;
  float* s_mean = misc + 896;
  float* s_invstd = misc + 928;
  float* s_fcw = misc + 1024;                                   // FC: [ncls][1568]
  float* s_dl = s_fcw + L2BwdSmem::kFcW / 4;                    // FC: [B][16] (columns >= ncls zero)
  float* s_pool = s_dl + L2BwdSmem::kFcDl / 4;                  // FC: [B][16] slice of the pooled activations
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;

  GridBar bar(gs);
  TRACE_INIT();
  trace(3, 0);
  if constexpr (FC) {
    // stage the classifier weights (cp.async, no registers, lands while the dgrad weights are built), every image's dlogits and this
    // CTA's first 16-column slice of the pooled activations (loads batched in registers: one L2 latency, not one per element)
    for (int i = tid; i < ncls * 392; i += kL2Threads) cp_async_16(smem_u32(s_fcw + 4 * i), fcw + 4 * i, 16);
    cp_async_commit();
    float tdl[10], tp[10];
#pragma unroll
    for (int q = 0; q < 10; ++q) {
      const int i = tid + q * kL2Threads, r = i >> 4, j = i & 15;
      tdl[q] = (i < B * 16 && j < ncls) ? __ldg(dlogits + static_cast<size_t>(r) * ncls + j) : 0.f;
      tp[q] = (i < B * 16 && n < 98) ? __ldg(pooled + static_cast<size_t>(r) * 1568 + n * 16 + j) : 0.f;
    }
#pragma unroll
    for (int q = 0; q < 10; ++q) {
      const int i = tid + q * kL2Threads;
      if (i < B * 16) {
        s_dl[i] = tdl[q];
        s_pool[i] = tp[q];
      }
    }
  }
  for (int i = tid; i < kPatchAlloc / 16; i += kL2Threads) reinterpret_cast<float4*>(sa)[i] = make_float4(0.f, 0.f, 0.f, 0.f);   // halo = 0
  if (tid < 32) {
    const float mean = saved[tid], invstd = saved[32 + tid];
    const float g = gamma ? gamma[tid] : 1.f, b = beta ? beta[tid] : 0.f;
    s_mean[tid] = mean;
    s_invstd[tid] = invstd;
    s_scale[tid] = g * invstd;
    s_shift[tid] = b - mean * g * invstd;
  }
  // Bd[tap][ci][co] = w[co][ci][24 − tap]: the data gradient is a correlation with the flipped filter
  {
    float wv[2][25];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float* src = w + (tid + j * kL2Threads) * 25;
#pragma unroll
      for (int tap = 0; tap < 25; ++tap) wv[j][tap] = __ldg(src + tap);
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int pair = tid + j * kL2Threads, co = pair >> 4, ci = pair & 15;
      uint8_t* dst = sb + sw128_off(ci, co >> 2) + (co & 3) * 4;
#pragma unroll
      for (int tap = 0; tap < 25; ++tap) *reinterpret_cast<float*>(dst + (24 - tap) * 2048) = wv[j][tap];
    }
  }
  if constexpr (FC) cp_async_wait<0>();
  __syncthreads();
  trace(3, 1);

  // thread = (channel c, window group g): windows pp = g, g+8, ... (≤ 7 per thread); y values stay in registers
  const int c = tid & 31, g = tid >> 5;
  float yv[7][4], dzv[7];
  int arg[7];
  float s1 = 0.f, s2 = 0.f;
  const float sc = s_scale[c], sh = s_shift[c], mu = s_mean[c], is = s_invstd[c];
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const int pp = g + 8 * k;
    dzv[k] = 0.f;
    arg[k] = 0;
    if (pp < 49) {
      const int ph = pp / 7, pw = pp - ph * 7;
      float best = -INFINITY;
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        const int p = (2 * ph + (d >> 1)) * 14 + 2 * pw + (d & 1);
        yv[k][d] = y[(static_cast<size_t>(n) * 196 + p) * 32 + c];
        const float z = fmaf(yv[k][d], sc, sh);
        if (z > best) { best = z; arg[k] = d; }
      }
      float go;
      if constexpr (FC) {
        const float* wk = s_fcw + c * 49 + pp;       // bank = (17·c + pp) mod 32: conflict-free across the warp's 32 channels
        const float* dl = s_dl + n * 16;
        float g0 = 0.f, g1 = 0.f;
#pragma unroll
        for (int j = 0; j < 16; j += 2) {            // independent smem loads (classes >= ncls: dlogits column is zero, weight not read)
          g0 = fmaf(dl[j], j < ncls ? wk[j * 1568] : 0.f, g0);
          g1 = fmaf(dl[j + 1], j + 1 < ncls ? wk[(j + 1) * 1568] : 0.f, g1);
        }
        go = g0 + g1;
      } else {
        go = dout[static_cast<size_t>(n) * 1568 + c * 49 + pp];
      }
      dzv[k] = best > 0.f ? go : 0.f;
      float xh = 0.f;
#pragma unroll
      for (int d = 0; d < 4; ++d) if (d == arg[k]) xh = (yv[k][d] - mu) * is;
      s1 += dzv[k];
      s2 = fmaf(dzv[k], xh, s2);
    }
  }
  s_part[g * 64 + c] = s1;
  s_part[g * 64 + 32 + c] = s2;
  __syncthreads();
  if (tid < 64) {
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += s_part[q * 64 + tid];
    partials[static_cast<size_t>(n) * 64 + tid] = s;
  }
  trace(3, 2);
  bar.arrive(gs);
  // ---- in the shadow of the grid barrier: work that no other CTA waits for ----
  // zero halo of the global dy frame (the weight gradient sums over all 324 positions)
  for (int i = tid; i < 324 * 8; i += kL2Threads) {
    const int P = i >> 3, pr = P / 18, pc = P - pr * 18;
    if (pr < 2 || pr >= 16 || pc < 2 || pc >= 16) reinterpret_cast<float4*>(dy + (static_cast<size_t>(n) * 324 + P) * 32)[i & 7] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if constexpr (FC) {
    // classifier weight gradient, slice = 16 consecutive columns (98 slices; "slice 98" = the bias): thread = (column, class).
    // The first slice of this CTA (slice n) was staged at kernel start.
    const int kl = tid & 15, j = tid >> 4;
    for (int slice = n; slice < 99; slice += B) {
      if (slice < 98) {
        if (slice != n) {
          __syncthreads();   // s_pool free (previous slice consumed)
          float tp[10];
#pragma unroll
          for (int q = 0; q < 10; ++q) {
            const int i = tid + q * kL2Threads;
            tp[q] = i < B * 16 ? __ldg(pooled + static_cast<size_t>(i >> 4) * 1568 + slice * 16 + (i & 15)) : 0.f;
          }
#pragma unroll
          for (int q = 0; q < 10; ++q) {
            const int i = tid + q * kL2Threads;
            if (i < B * 16) s_pool[i] = tp[q];
          }
          __syncthreads();
        }
        if (j < ncls) {
          float a[4] = {0.f, 0.f, 0.f, 0.f};
          int r = 0;
          for (; r + 3 < B; r += 4) {
#pragma unroll
            for (int u = 0; u < 4; ++u) a[u] = fmaf(s_dl[(r + u) * 16 + j], s_pool[(r + u) * 16 + kl], a[u]);
          }
          for (; r < B; ++r) a[0] = fmaf(s_dl[r * 16 + j], s_pool[r * 16 + kl], a[0]);
          dfcw[static_cast<size_t>(j) * 1568 + slice * 16 + kl] = (a[0] + a[1]) + (a[2] + a[3]);
        }
      } else {
        if (dfcb != nullptr && tid < ncls) {
          float a = 0.f;
          for (int r = 0; r < B; ++r) a += s_dl[r * 16 + tid];
          dfcb[tid] = a;
        }
        if (loss_parts != nullptr && warp == 7) {   // the forward kernel left one cross-entropy term per image: batch mean, fixed order
          float sl = 0.f;
          for (int r = lane; r < B; r += 32) sl += __ldg(loss_parts + r);
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) sl += __shfl_xor_sync(0xffffffffu, sl, off);
          if (lane == 0) *loss_out = sl / static_cast<float>(B);
        }
      }
    }
  }
  bar.wait(gs);
  trace(3, 3);
  fold_rows<64>(partials, B, s_tmp, s_tot);
  trace(3, 4);
  if (n == 0 && tid < 32) {
    if (dbeta) dbeta[tid] = s_tot[tid];
    if (dgamma) dgamma[tid] = s_tot[32 + tid];
  }
  {
    const float inv_cnt = 1.f / (static_cast<float>(B) * 196.f);
    const float m1 = s_tot[c] * inv_cnt, m2 = s_tot[32 + c] * inv_cnt;
    float dsum = 0.f;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const int pp = g + 8 * k;
      if (pp < 49) {
        const int ph = pp / 7, pw = pp - ph * 7;
#pragma unroll
        for (int d = 0; d < 4; ++d) {
          const int oh = 2 * ph + (d >> 1), ow = 2 * pw + (d & 1);
          const float xh = (yv[k][d] - mu) * is;
          const float v = sc * ((d == arg[k] ? dzv[k] : 0.f) - m1 - xh * m2);
          const int P = (oh + 2) * kPW + ow + 2;
          dy[(static_cast<size_t>(n) * 324 + P) * 32 + c] = v;                      // frame for the weight-gradient kernel (TMA)
          *reinterpret_cast<float*>(sa + sw128_off(P, c >> 2) + (c & 3) * 4) = v;   // same frame in smem for the data-gradient MMAs
          dsum += v;
        }
      }
    }
    s_part[g * 64 + c] = dsum;
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid < 32) {   // Σdy of this image per channel: the conv2 bias gradient is the sum of these rows
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) s += s_part[q * 64 + tid];
    dysum[static_cast<size_t>(n) * 32 + tid] = s;
  }
  trace(3, 5);
  // ---- conv2 data gradient: 400 wgmma m64n16k8 by the warpgroup of warps 4..7, accumulators straight to the dx frame -------
  if (warpgroup_index() == 1) {
    const int wt = tid - 128;
    const uint64_t ad0 = gmma_desc_kmajor<128>(smem_u32(sa)), bd0 = gmma_desc_kmajor<128>(smem_u32(sb));
#pragma unroll 1
    for (int t = 0; t < 2; ++t) {
      float acc[2][8];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[h][e] = 0.f;
      wgmma_fence();
#pragma unroll 1
      for (int kh = 0; kh < 5; ++kh) {
        const uint64_t ad = ad0 + static_cast<uint64_t>(((7 * t + kh) * kPW * 128) >> 4);
        const uint64_t bd = bd0 + static_cast<uint64_t>((kh * 5 * 2048) >> 4);
#pragma unroll
        for (int kw = 0; kw < 5; ++kw) {
#pragma unroll
          for (int k = 0; k < 4; ++k)   // K = 32 output channels = four K=8 steps
#pragma unroll
            for (int h = 0; h < 2; ++h)
              wgmma_m64n16k8_tf32(acc[h], ad + ((h * 64 * 128 + kw * 128 + k * 32) >> 4), bd + ((kw * 2048 + k * 32) >> 4), (kh | kw | k) != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int rr = 64 * h + wgmma_frag_row(wt, e), ci = wgmma_frag_col(wt, e);
          const int orow = rr / kPW, ow = rr - orow * kPW;
          if (rr < 126 && ow < 14) dx[(static_cast<size_t>(n) * 324 + (7 * t + orow + 2) * 18 + ow + 2) * 16 + ci] = acc[h][e];
        }
      }
    }
  }
  __syncthreads();
  bar.finish(gs);
  trace(3, 6);
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
CUtensorMap make_patch_map(const float* base, int C, int W, int H, int N) {
  CUtensorMap m;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * 4, static_cast<cuuint64_t>(W) * C * 4, static_cast<cuuint64_t>(H) * W * C * 4};
  cuuint32_t box[4] = {32, static_cast<cuuint32_t>(W), static_cast<cuuint32_t>(H), 1};   // the whole (already haloed) frame
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = driver().cuTensorMapEncodeTiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, estr,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(fused conv2 patch) failed: " + cu_error(r));
  return m;
}

}  // namespace

bool fused_convnet_supported(int B) { return B >= 1 && B <= sm_count(); }

void fused_convnet_trace_enable(bool on) {
  const int v = on ? 1 : 0;
  PDT_CUDA_CHECK(cudaMemcpyToSymbol(g_trace_on, &v, sizeof(v)));
  if (on) {
    void* p = nullptr;
    PDT_CUDA_CHECK(cudaGetSymbolAddress(&p, g_trace));
    PDT_CUDA_CHECK(cudaMemset(p, 0, sizeof(unsigned long long) * 4 * 160 * 12));
  }
}
void fused_convnet_trace_read(unsigned long long* host /*[4][160][12]*/) {
  PDT_CUDA_CHECK(cudaDeviceSynchronize());
  PDT_CUDA_CHECK(cudaMemcpyFromSymbol(host, g_trace, sizeof(unsigned long long) * 4 * 160 * 12));
}

void launch_convnet_l1_fwd(const float* x, const float* w, const float* bias, const float* gamma, const float* beta, float* y, float* out,
                           float* saved, float* running_mean, float* running_var, long long* nbt, float momentum, float eps, int B,
                           float* partials, GridSync gs, cudaStream_t st) {
  launch_cooperative(convnet_l1_fwd_kernel, B, kL1Threads, 0, st, "convnet_l1_fwd", x, w, bias, gamma, beta, y, out, saved, running_mean, running_var, nbt,
                     momentum, eps, partials, gs);
}

void launch_convnet_l1_bwd(const float* dp, const float* y, const float* x, const float* saved, const float* gamma, const float* beta,
                           float* dgamma, float* dbeta, float* dw, float* db, int B, float* partials, float* partials_w, GridSync gs,
                           cudaStream_t st) {
  CUtensorMap none{};
  launch_cooperative(convnet_l1_bwd_kernel<false>, B, kL1Threads, static_cast<size_t>(kL1BwdSmem), st, "convnet_l1_bwd", dp, y, x, saved, gamma, beta, dgamma,
                     dbeta, dw, db, partials, partials_w, gs, none, none, static_cast<float*>(nullptr), static_cast<const float*>(nullptr),
                     static_cast<float*>(nullptr), static_cast<float*>(nullptr), SgdRider{});
}

template <class Rider>
void launch_convnet_l1_bwd_wgrad(const float* dp, const float* y, const float* x, const float* saved, const float* gamma, const float* beta,
                                 float* dgamma, float* dbeta, float* dw, float* db, const float* dy2_pad, const float* x2_pad, const float* dysum2,
                                 float* dw2, float* db2, int B, float* partials, float* partials_w, float* wpart, GridSync gs, cudaStream_t st,
                                 Rider rider) {
  CUtensorMap tm_x, tm_dy;
  make_wgrad_win_tmaps(x2_pad, dy2_pad, B, &tm_x, &tm_dy);
  launch_cooperative(convnet_l1_bwd_kernel<true, Rider>, B, L1WgCfg::kThreads, L1WgCfg::kSmem, st, "convnet_l1_bwd_wgrad", dp, y, x, saved, gamma, beta,
                     dgamma, dbeta, dw, db, partials, partials_w, gs, tm_x, tm_dy, wpart, dysum2, dw2, db2, rider);
}
template void launch_convnet_l1_bwd_wgrad<SgdRider>(const float*, const float*, const float*, const float*, const float*, const float*, float*,
                                                    float*, float*, float*, const float*, const float*, const float*, float*, float*, int, float*,
                                                    float*, float*, GridSync, cudaStream_t, SgdRider);
template void launch_convnet_l1_bwd_wgrad<AdamRider>(const float*, const float*, const float*, const float*, const float*, const float*, float*,
                                                     float*, float*, float*, const float*, const float*, const float*, float*, float*, int, float*,
                                                     float*, float*, GridSync, cudaStream_t, AdamRider);
template void launch_convnet_l1_bwd_wgrad<ClipRider<SgdRider>>(const float*, const float*, const float*, const float*, const float*,
                                                               const float*, float*, float*, float*, float*, const float*, const float*,
                                                               const float*, float*, float*, int, float*, float*, float*, GridSync, cudaStream_t,
                                                               ClipRider<SgdRider>);
template void launch_convnet_l1_bwd_wgrad<ClipRider<AdamRider>>(const float*, const float*, const float*, const float*, const float*,
                                                                const float*, float*, float*, float*, float*, const float*, const float*,
                                                                const float*, float*, float*, int, float*, float*, float*, GridSync, cudaStream_t,
                                                                ClipRider<AdamRider>);

void launch_convnet_l2_fwd(const float* x, const float* w, const float* bias, const float* gamma, const float* beta, float* y, float* out,
                           float* saved, float* running_mean, float* running_var, long long* nbt, float momentum, float eps,
                           const float* fcw, const float* fcb, float* logits, int ncls, int B, float* partials, GridSync gs, cudaStream_t st) {
  CUtensorMap tm_x = make_patch_map(x, 16, 18, 18, B);
  launch_cooperative(convnet_l2_fwd_kernel, B, kL2Threads, static_cast<size_t>(L2FwdSmem::kTotal), st, "convnet_l2_fwd", tm_x, w, bias, gamma, beta, y, out,
                     saved, running_mean, running_var, nbt, momentum, eps, fcw, fcb, logits, ncls, partials, gs);
}

void launch_convnet_fwd(const float* x, const float* w1, const float* b1, const float* g1, const float* be1, float* y1, float* p1, float* saved1,
                        float* rm1, float* rv1, long long* nbt1, float mom1, float eps1, const float* w2, const float* b2, const float* g2,
                        const float* be2, float* y2, float* out, float* saved2, float* rm2, float* rv2, long long* nbt2, float mom2, float eps2,
                        const float* fcw, const float* fcb, float* logits, int ncls, int B, float* partials, GridSync gs, cudaStream_t st,
                        FusedCe ce) {
  if (logits != nullptr && ncls > 16) throw std::invalid_argument("convnet_fwd: the fused classifier handles at most 16 classes");
  if (ce.target != nullptr && logits == nullptr) throw std::invalid_argument("convnet_fwd: the fused cross-entropy needs the fused classifier");
  launch_cooperative(convnet_fwd_kernel, B, kL1Threads, static_cast<size_t>(L2FwdSmem::kTotal), st, "convnet_fwd", x, w1, b1, g1, be1, y1, p1, saved1, rm1, rv1,
                     nbt1, mom1, eps1, w2, b2, g2, be2, y2, out, saved2, rm2, rv2, nbt2, mom2, eps2, fcw, fcb, logits, ncls, partials, gs, ce);
}

void launch_convnet_l2_bwd(const float* dout, const float* y, const float* saved, const float* gamma, const float* beta, const float* w,
                           float* dgamma, float* dbeta, float* dy, float* dx, float* dysum, int B, float* partials, GridSync gs,
                           cudaStream_t st) {
  launch_cooperative(convnet_l2_bwd_kernel<false>, B, kL2Threads, static_cast<size_t>(L2BwdSmem::kTotal), st, "convnet_l2_bwd", dout, y, saved, gamma, beta, w,
                     dgamma, dbeta, dy, dx, dysum, partials, gs, static_cast<const float*>(nullptr), static_cast<const float*>(nullptr),
                     static_cast<const float*>(nullptr), static_cast<float*>(nullptr), static_cast<float*>(nullptr), 0, static_cast<const float*>(nullptr),
                     static_cast<float*>(nullptr));
}

void launch_convnet_l2_bwd_fc(const float* dlogits, const float* fcw, const float* pooled, float* dfcw, float* dfcb, int ncls, const float* y,
                              const float* saved, const float* gamma, const float* beta, const float* w, float* dgamma, float* dbeta, float* dy,
                              float* dx, float* dysum, int B, float* partials, GridSync gs, cudaStream_t st, const float* loss_parts, float* loss_out) {
  if (ncls < 1 || ncls > 16) throw std::invalid_argument("convnet_l2_bwd_fc: 1..16 classes");
  if (B > 160) throw std::invalid_argument("convnet_l2_bwd_fc: batch too large for the staged dlogits");
  launch_cooperative(convnet_l2_bwd_kernel<true>, B, kL2Threads, static_cast<size_t>(L2BwdSmem::kTotalFc), st, "convnet_l2_bwd_fc",
                     static_cast<const float*>(nullptr), y, saved, gamma, beta, w, dgamma, dbeta, dy, dx, dysum, partials, gs, dlogits, fcw, pooled, dfcw,
                     dfcb, ncls, loss_parts, loss_out);
}

}  // namespace pdt
