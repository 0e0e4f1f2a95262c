// Cooperative fused kernels for the reference ConvNet (ref: ddp_example.py:22-41) — one CTA per image.
//
// A ConvNet step is a few µs of arithmetic spread over dependent kernel boundaries and every per-op kernel
// pays launch + ramp + drain + a grid-wide reduction.  Here everything that belongs to an image stays inside its CTA
// (registers / shared memory), and the only grid-wide dependencies — the BatchNorm batch statistics (forward), the
// Σdz, Σdz·x̂ sums (backward) and the folds of the weight gradients — are device-side grid barriers in the middle of a
// kernel instead of kernel boundaries.  A training step is three launches:
//
//   convnet_fwd_kernel         conv1 5x5 (1→16) ──barrier (Σy, M2)── BN + ReLU + MaxPool2 written straight into conv2's
//                              swizzled smem patch ── conv2 5x5 (16→32) on wgmma (the 25 taps are row-shifted descriptors
//                              into that patch; accumulators in registers) ──barrier── BN + ReLU + MaxPool2 + classifier
//                              (+ cross-entropy term and d(loss)/d(logits) when the targets are known)           (ref :25-34,40)
//   convnet_l2_bwd_kernel<WG>  classifier backward + MaxPool/ReLU/BN backward ──barrier (Σdz, Σdz·x̂)── dy → conv2 data
//                              gradient on wgmma (warps 4..7), next to it conv2's weight-gradient partial of the image on
//                              wgmma (warps 0..3; K-major copies of x, written in the barrier's shadow, and of dy)
//   convnet_l1_bwd_kernel      conv1 recomputed (the forward stores no conv1 output: the same FMA order gives the same bits)
//                              MaxPool/ReLU/BN backward ──barrier── conv1 weight gradient (mma.sync) ──barrier── conv1 fold;
//                              conv2's weight gradient is folded in the shadow of the first barrier, and — on one GPU — the
//                              threads that write the folded gradients apply the optimizer update (SgdRider / AdamRider / AmsgradRider /
//                              RmspropRider / AdagradRider)
//
// All cross-CTA sums are "every CTA writes one partial row, barrier, every CTA folds the rows in the same fixed order",
// so results are bit-reproducible and identical in every CTA.  The kernels are launched cooperatively (all CTAs
// co-resident: one per image, at most one per SM); grid barriers are split into arrive / wait so that independent work
// (stores nobody in the kernel waits for, cp.async staging, gradient slices) runs in their shadow (grid_sync.cuh).
// The two backward kernels are programmatic dependent launches: each grid is set up once every CTA of the kernel before it has
// passed its last grid barrier (griddep_launch_dependents), and waits for that kernel's completion at its top (griddep_wait).
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
// Kernel slots: 0 forward, 1 layer-1 backward, 3 layer-2 backward (slot 2 is unused).
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

// Sum `rows` partial rows of `W` floats (written by other CTAs before a grid barrier) in a fixed order.
// Called by all threads; the totals land in s_out[0..W).  s_tmp: [4][W] floats.  Needs >= 4*W threads.
template <int W>
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
  __syncthreads();
  if (tid < W) s_out[tid] = (s_tmp[tid] + s_tmp[W + tid]) + (s_tmp[2 * W + tid] + s_tmp[3 * W + tid]);
  __syncthreads();
}

// The same with every thread of a THREADS-wide CTA loading: G = THREADS / W row classes, one L2 round trip for up to 8·G rows.
// s_tmp: [G][W] floats.
template <int W, int THREADS>
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
  __syncthreads();
  if (tid < W) {
    float tot = 0.f;
#pragma unroll
    for (int g = 0; g < G; ++g) tot += s_tmp[g * W + tid];
    s_out[tid] = tot;
  }
  __syncthreads();
}

// Warp-level reduction of 32 per-thread values with 31 shuffles: after the call lane l holds Σ_lanes v[l] in v[0].  One step per
// template instance, so that every index into v is a constant and v stays in registers.
template <int HALF>
__device__ __forceinline__ void warp_transpose_reduce_step(float (&v)[32], int lane) {
  const bool upper = (lane & HALF) != 0;
#pragma unroll
  for (int i = 0; i < HALF; ++i) {
    const float send = upper ? v[i] : v[i + HALF];
    const float keep = upper ? v[i + HALF] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, HALF);
  }
}
__device__ __forceinline__ void warp_transpose_reduce32(float (&v)[32], int lane) {
  warp_transpose_reduce_step<16>(v, lane);
  warp_transpose_reduce_step<8>(v, lane);
  warp_transpose_reduce_step<4>(v, lane);
  warp_transpose_reduce_step<2>(v, lane);
  warp_transpose_reduce_step<1>(v, lane);
}
// The same for 16 values (v[16..32) are not read): lanes l and l + 16 both end with Σ_lanes v[l & 15] in v[0].
__device__ __forceinline__ void warp_transpose_reduce16(float (&v)[32], int lane) {
  warp_transpose_reduce_step<8>(v, lane);
  warp_transpose_reduce_step<4>(v, lane);
  warp_transpose_reduce_step<2>(v, lane);
  warp_transpose_reduce_step<1>(v, lane);
  v[0] += __shfl_xor_sync(0xffffffffu, v[0], 16);
}

// Batch statistics without cancellation.  Each CTA publishes, per channel, the sum of its n_img elements and M2_img, their squared
// deviations about the CTA's own mean.  The batch's M2 is then exact in form (Chan, Golub & LeVeque):
//   M2 = Σ_img M2_img + Σ_img d_img² / n_img,   d_img = Σ_img − n_img·mean,   mean = Σ_img Σ_img / (B·n_img),
// where Σy²/n − mean² in fp32 would lose the variance's digits in proportion to mean²/var (a channel whose mean is 1000 times
// its spread keeps none).  After the grid barrier every CTA folds the rows [Σ (C) | M2 (C)] in the same fixed order: thread
// (c, g) sums rows g, g + G, ... of channel c, keeping the first R row sums in registers, so that the deviations d_img from the
// batch mean need no second trip to L2 for B ≤ R·G (all the rows the cooperative launch can have on an H100).  Σ_img d_img also
// corrects the mean for the rounding of the first sum, which at large means is worth an ulp.  Leaves the mean in s_stat[0..C)
// and the biased variance in s_stat[C..2C); s_a, s_b: [THREADS] floats each.
template <int C, int THREADS, int R>
__device__ __forceinline__ void fold_centred_stats(const float* __restrict__ partials, int rows, float n_img, float* s_a, float* s_b,
                                                   float* s_stat) {
  constexpr int G = THREADS / C;
  const int tid = threadIdx.x, c = tid % C, g = tid / C;
  const bool folds = tid < G * C;
  float sv[R];
  {
    float s = 0.f, m = 0.f;
    if (folds) {
      float mv[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {   // R independent pairs of L2 loads in flight
        const bool in = g + G * j < rows;
        sv[j] = in ? __ldcg(partials + static_cast<size_t>(g + G * j) * 2 * C + c) : 0.f;
        mv[j] = in ? __ldcg(partials + static_cast<size_t>(g + G * j) * 2 * C + C + c) : 0.f;
      }
#pragma unroll
      for (int j = 0; j < R; ++j) {
        s += sv[j];
        m += mv[j];
      }
      for (int r = g + G * R; r < rows; r += G) {
        s += __ldcg(partials + static_cast<size_t>(r) * 2 * C + c);
        m += __ldcg(partials + static_cast<size_t>(r) * 2 * C + C + c);
      }
      s_a[tid] = s;
      s_b[tid] = m;
    }
  }
  __syncthreads();
  const float cnt = static_cast<float>(rows) * n_img;
  float m2_rows = 0.f;
  if (tid < C) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < G; ++k) {
      s += s_a[k * C + tid];
      m2_rows += s_b[k * C + tid];
    }
    s_stat[tid] = s / cnt;
  }
  __syncthreads();
  if (folds) {
    const float mean = s_stat[c];
    float ds = 0.f, dq = 0.f;
#pragma unroll
    for (int j = 0; j < R; ++j) {
      const float d = g + G * j < rows ? fmaf(-n_img, mean, sv[j]) : 0.f;
      ds += d;
      dq = fmaf(d, d, dq);
    }
    for (int r = g + G * R; r < rows; r += G) {
      const float d = fmaf(-n_img, mean, __ldcg(partials + static_cast<size_t>(r) * 2 * C + c));
      ds += d;
      dq = fmaf(d, d, dq);
    }
    s_a[tid] = ds;
    s_b[tid] = dq;
  }
  __syncthreads();
  if (tid < C) {
    float ds = 0.f, dq = 0.f;
#pragma unroll
    for (int k = 0; k < G; ++k) {
      ds += s_a[k * C + tid];
      dq += s_b[k * C + tid];
    }
    s_stat[tid] += ds / cnt;
    s_stat[C + tid] = (m2_rows + dq / n_img) / cnt;
  }
  __syncthreads();
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

// The zero-haloed image by the NT threads of the CTA, in two halves: load() requests this thread's pixels, so that their latency
// overlaps the other prologue loads (conv1's weights) instead of following them; store() zeroes the frame, waits for the CTA and
// writes them (the caller syncs before reading xs).
template <int NT>
struct L1Image {
  static constexpr int kPer = (784 + NT - 1) / NT;
  float v[kPer];
  __device__ __forceinline__ void load(const float* __restrict__ x, int tid) {
#pragma unroll
    for (int u = 0; u < kPer; ++u) v[u] = tid + u * NT < 784 ? x[tid + u * NT] : 0.f;
  }
  __device__ __forceinline__ void store(float* xs /*[32][32]*/, int tid) const {
    for (int i = tid; i < 1024; i += NT) xs[i] = 0.f;
    __syncthreads();
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int i = tid + u * NT, rr = i / 28, cc = i - rr * 28;
      if (i < 784) xs[(rr + 2) * 32 + cc + 2] = v[u];
    }
  }
};

// conv1 of P pixels of one image, channels c0 .. c0 + C of them: pixel i at xoff[i] = r·32 + c in the haloed image xs, ws = the weights
// [25 taps][16 co] in shared memory + c0, b1 = the bias + c0 (or null).  acc[i][j] = b1[j], then one fmaf per tap, kh outer, kw inner.
// Every caller accumulates in this one order whatever its CTA shape or channel split, so the forward's y1 and backward B's recompute
// of it are the same bits.
template <int P, int C>
__device__ __forceinline__ void conv1_pixels(const float* xs, const float* ws, const float* b1, const int (&xoff)[P], float (&acc)[P][C]) {
  static_assert(C % 4 == 0, "conv1_pixels: whole float4 weight groups");
#pragma unroll
  for (int j = 0; j < C; ++j) {
    const float b = b1 ? __ldg(b1 + j) : 0.f;
#pragma unroll
    for (int i = 0; i < P; ++i) acc[i][j] = b;
  }
#pragma unroll 1
  for (int kh = 0; kh < 5; ++kh) {
#pragma unroll
    for (int kw = 0; kw < 5; ++kw) {
      float xv[P];
#pragma unroll
      for (int i = 0; i < P; ++i) xv[i] = xs[xoff[i] + kh * 32 + kw];
      const float4* wt = reinterpret_cast<const float4*>(ws + (kh * 5 + kw) * 16);
#pragma unroll
      for (int q = 0; q < C / 4; ++q) {
        const float4 wq = wt[q];
#pragma unroll
        for (int i = 0; i < P; ++i) {
          acc[i][4 * q + 0] = fmaf(xv[i], wq.x, acc[i][4 * q + 0]);
          acc[i][4 * q + 1] = fmaf(xv[i], wq.y, acc[i][4 * q + 1]);
          acc[i][4 * q + 2] = fmaf(xv[i], wq.z, acc[i][4 * q + 2]);
          acc[i][4 * q + 3] = fmaf(xv[i], wq.w, acc[i][4 * q + 3]);
        }
      }
    }
  }
}

// One butterfly stage of a 4 × 4 block transpose over the four lanes of a pooling window (lanes 4w .. 4w + 3): lanes S apart swap
// the blocks whose index differs from theirs in bit S.  Constant indices only, so a stays in registers.
template <int S>
__device__ __forceinline__ void window_transpose_step(float (&a)[4][4], int lane) {
  const bool upper = (lane & S) != 0;
#pragma unroll
  for (int i0 = 0; i0 < 4; ++i0) {
    if (i0 & S) continue;
    const int i1 = i0 | S;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float got = __shfl_xor_sync(0xffffffffu, upper ? a[i0][j] : a[i1][j], S);
      a[i0][j] = upper ? got : a[i0][j];
      a[i1][j] = upper ? a[i1][j] : got;
    }
  }
}

// ---- layer 1 backward (+ the fold of conv2's weight gradient riding along) ---------------------------------------------------
// dynamic smem: dys [784][16] | fold [25 warps][16 co][32 taps]
constexpr int kL1BwdSmem = (784 * 16 + kL1Warps * 512) * 4;

// conv2's weight gradient of one image on wgmma: dW2ᵀ[(kh, kw, ci)][co] = Σ_P x[P + 18·kh + kw][ci] · dy[kFirst + P][co] over the
// 256 positions P ∈ [0, 256) of the zero-haloed 18 × 18 frames from the first interior one (kFirst; x index 0 is tap (0, 0) of
// position kFirst).  M = (tap, ci), N = co, K = P.  TF32 wgmma wants both operands K-major, i.e. with positions innermost, while
// the NHWC frames have channels innermost, so both are written transposed into shared memory, in the no-swizzle canonical layout
// (core matrix = 8 rows × 4 positions, 128 contiguous bytes), already rounded by cvt.rna — the tensor core then reads them exactly.
//   * A: four residue copies X_r of the x frame.  X_r holds block (cg, q) = x[4q + r + i][8·cg + row] (row 0..7, i 0..3) in
//     128-byte slot 2q + 9·cg.  Tap (kh, kw) with off = 18·kh + kw reads copy off mod 4 from block q = off / 4; taps kh, kh + 2,
//     kh + 4, kh + 6 are 36 positions = 18 slots apart, so with M-group g = 2j + cg one descriptor (LBO = 256, SBO = 1152) covers
//     an M = 64 tile of four kh × 16 channels.  Per kw two tiles: kh ∈ {0, 2, 4, 6} and {1, 3, 5, 7}; kh > 4 are pad rows,
//     computed from whatever lies there and not stored.  Positions ≥ 324 are written as zeros (they meet dy = 0, and 0 × NaN
//     would poison real rows).
//   * B: dyᵀ, block (co-group, K-chunk kc of four positions) at kc·512 + cog·128 (LBO = 512, SBO = 128).
// 10 tiles × 32 K-steps = 320 wgmma m64n32k8 per image; the partial is [400][32], rows in (kh, kw, ci) order.
struct Conv2Wg {
  static constexpr int kFrame = 18 * 18, kFirst = 2 * 18 + 2;
  static constexpr int kXBlocks = 83;                       // q = 0..82: covers every real tap (off ≤ 76) over 64 K-chunks
  static constexpr int kXCopy = (2 * (kXBlocks - 1) + 9 + 1) * 128;   // 175 slots, 22,400 B
  static constexpr int kLbo = 256, kSbo = 1152;
  // bytes from the first copy up to the end of the farthest pad-row read: copy 3, tile kh ∈ {1, 3, 5, 7} at kw = 1 (off 19, block
  // 4), M-group 7, K-step 31, second core matrix
  static constexpr int kXReach = 3 * kXCopy + 2 * 4 * 128 + 7 * kSbo + 31 * 512 + kLbo + 128;
  static constexpr int kXBytes = (kXReach + 1023) / 1024 * 1024;
  static constexpr int kDyT = 64 * 512;                     // dyᵀ: 32 co × 256 positions
};

// Byte offset of dy[kFirst + p][co] in dyᵀ (p < 256).
__device__ __forceinline__ uint32_t conv2_dyt_off(int co, int p) {
  return static_cast<uint32_t>((p >> 2) * 512 + (co >> 3) * 128 + (co & 7) * 16 + (p & 3) * 4);
}
__device__ __forceinline__ float tf32_round(float v) { return __uint_as_float(f32_to_tf32(v)); }

// The four residue copies of one image's x frame (frame = its [324][16] floats, read-only in this kernel) by the NT threads of the
// CTA, in two halves so that the loads can be issued long before the copies' region is free: task (ci, q) loads positions
// 4q .. 4q + 6 of channel ci (zero past the frame) and writes one 16-byte core-matrix row into each copy.
template <int NT>
struct Conv2WgX {
  static constexpr int kTasks = 16 * Conv2Wg::kXBlocks, kPer = (kTasks + NT - 1) / NT;
  float v[kPer][7];
  __device__ __forceinline__ void load(const float* __restrict__ frame, int tid) {
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int i = tid + u * NT, ci = i & 15, q = i >> 4;
#pragma unroll
      for (int k = 0; k < 7; ++k) {
        const int pos = 4 * q + k;
        v[u][k] = (i < kTasks && pos < Conv2Wg::kFrame) ? __ldg(frame + pos * 16 + ci) : 0.f;   // rounded in store(): no wait here
      }
    }
  }
  __device__ __forceinline__ void store(uint8_t* xt, int tid) const {
#pragma unroll
    for (int u = 0; u < kPer; ++u) {
      const int i = tid + u * NT, ci = i & 15, q = i >> 4;
      if (i < kTasks) {
        uint8_t* dst = xt + (2 * q + 9 * (ci >> 3)) * 128 + (ci & 7) * 16;
        float t[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) t[k] = tf32_round(v[u][k]);
#pragma unroll
        for (int r = 0; r < 4; ++r) *reinterpret_cast<float4*>(dst + r * Conv2Wg::kXCopy) = make_float4(t[r], t[r + 1], t[r + 2], t[r + 3]);
      }
    }
  }
};

// The 64 wgmma of column kw (its two tiles, 32 K-steps each) into a, as one commit group.  A loop, not unrolled code: the kernel
// runs it once per launch, and every SM would fetch straight-line code from L2 at the same time.
__device__ __forceinline__ void conv2_wgrad_issue(float (&a)[2][16], uint32_t xt, uint64_t bd, int kw) {
  uint64_t ad[2];
#pragma unroll
  for (int par = 0; par < 2; ++par) {
    const int off = 18 * par + kw;
    ad[par] = gmma_desc_kmajor_noswz<Conv2Wg::kLbo, Conv2Wg::kSbo>(xt + (off & 3) * Conv2Wg::kXCopy + (off >> 2) * 256);
  }
  wgmma_fence();
#pragma unroll 4
  for (int s = 0; s < 32; ++s)
#pragma unroll
    for (int par = 0; par < 2; ++par) wgmma_m64n32k8_tf32(a[par], ad[par] + s * (512 >> 4), bd + s * (1024 >> 4), s != 0);
  wgmma_commit();
}
// Rows kh ≤ 4 of column kw's accumulators to the image's partial.
__device__ __forceinline__ void conv2_wgrad_store(const float (&a)[2][16], float* __restrict__ wpart_n, int kw, int wt) {
#pragma unroll
  for (int par = 0; par < 2; ++par)
#pragma unroll
    for (int e = 0; e < 16; e += 2) {
      const int row = wgmma_frag_row(wt, e), g = row >> 3, kh = par + 2 * (g >> 1);
      if (kh < 5) {
        const int prow = (kh * 5 + kw) * 16 + 8 * (g & 1) + (row & 7);
        *reinterpret_cast<float2*>(wpart_n + prow * 32 + wgmma_frag_col(wt, e)) = make_float2(a[par][e], a[par][e + 1]);
      }
    }
}

// The per-image partial from the K-major operands (xt, dyt: shared addresses), issued by one warpgroup (wt = thread index in it):
// column kw + 1 is in flight while the accumulators of column kw are stored.  The same instructions in the same order wherever
// it runs, so the stand-alone kernel reproduces the layer-2 backward kernel bit for bit.
__device__ __forceinline__ void conv2_wgrad_wgmma(uint32_t xt, uint32_t dyt, float* __restrict__ wpart_n, int wt) {
  const uint64_t bd = gmma_desc_kmajor_noswz<512, 128>(dyt);
  float acc0[2][16], acc1[2][16];
  conv2_wgrad_issue(acc0, xt, bd, 0);
#pragma unroll 1
  for (int kw = 1; kw < 5; kw += 2) {
    conv2_wgrad_issue(acc1, xt, bd, kw);
    wgmma_wait<1>();
    conv2_wgrad_store(acc0, wpart_n, kw - 1, wt);
    conv2_wgrad_issue(acc0, xt, bd, kw + 1);
    wgmma_wait<1>();
    conv2_wgrad_store(acc1, wpart_n, kw, wt);
  }
  wgmma_wait<0>();
  conv2_wgrad_store(acc0, wpart_n, 4, wt);
}

// The per-image partials from given dy / x frames (the layer-1 backward binding's stand-alone form): one CTA = one warpgroup per
// image writes the operands from the frames and runs conv2_wgrad_wgmma.
constexpr size_t kConv2WgSmem = Conv2Wg::kXBytes + Conv2Wg::kDyT;
__global__ void __launch_bounds__(128, 1)
conv2_wgrad_partials_kernel(const float* __restrict__ dy2_pad, const float* __restrict__ x2_pad, float* __restrict__ wpart) {
  extern __shared__ __align__(1024) uint8_t smem_wg[];
  uint8_t* dyt = smem_wg + Conv2Wg::kXBytes;
  const int n = blockIdx.x, tid = threadIdx.x;
  {
    Conv2WgX<128> xr;
    xr.load(x2_pad + static_cast<size_t>(n) * Conv2Wg::kFrame * 16, tid);
    xr.store(smem_wg, tid);
  }
  const float* dyf = dy2_pad + (static_cast<size_t>(n) * Conv2Wg::kFrame + Conv2Wg::kFirst) * 32;
  for (int i = tid; i < 32 * 64; i += 128) {   // task (co, kc): positions 4kc .. 4kc + 3 of channel co, one 16-byte row
    const int co = i & 31, kc = i >> 5;
    const float* src = dyf + 4 * kc * 32 + co;
    *reinterpret_cast<float4*>(dyt + conv2_dyt_off(co, 4 * kc)) =
        make_float4(tf32_round(__ldg(src)), tf32_round(__ldg(src + 32)), tf32_round(__ldg(src + 64)), tf32_round(__ldg(src + 96)));
  }
  fence_proxy_async_smem();
  __syncthreads();
  conv2_wgrad_wgmma(smem_u32(smem_wg), smem_u32(dyt), wpart + static_cast<size_t>(n) * 400 * 32, tid);
}

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

// One Adam update (the arithmetic of adam_multi_kernel / amsgrad_multi_kernel, ops_simt.cu) of element i of parameter k with
// gradient g.  R: AdamRider or AmsgradRider, possibly in a ClipRider.
template <class R>
__device__ __forceinline__ void adam_apply(const R& r, int k, int i, float g, const float* f) {
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
  float den = vv;
  if constexpr (std::is_base_of_v<AmsgradRider, R>) {
    float* vm = r.vmax[k] + i;
    den = nan_max(*vm, vv);
    *vm = den;
  }
  *p = fmaf(-f[k], mv / (sqrtf(den) / f[10 + k] + r.h.eps), pv);
}

// One RMSprop update (the arithmetic of rmsprop_multi_kernel, ops_simt.cu) of element i of parameter k with gradient g.
// R: RmspropRider, possibly in a ClipRider.
template <class R>
__device__ __forceinline__ void rmsprop_apply(const R& r, int k, int i, float g, float lr) {
  float gv = r.h.maximize ? -g : g;
  float* p = r.p[k] + i;
  float* sq = r.sq[k] + i;
  const float pv = *p;
  if (r.h.weight_decay != 0.f) gv = fmaf(r.h.weight_decay, pv, gv);
  const float sv = fmaf(r.h.one_minus_alpha * gv, gv, r.h.alpha * *sq);
  *sq = sv;
  float var = sv;
  if (r.ga[k]) {
    float* ga = r.ga[k] + i;
    const float a = fmaf(r.h.one_minus_alpha, gv - *ga, *ga);
    *ga = a;
    var = fmaf(-a, a, sv);
  }
  const float u = gv / (sqrtf(var) + r.h.eps);
  if (r.buf[k]) {
    float* buf = r.buf[k] + i;
    const float b = fmaf(r.h.momentum, *buf, u);
    *buf = b;
    *p = fmaf(-lr, b, pv);
  } else {
    *p = fmaf(-lr, u, pv);
  }
}

// The Adagrad rider's decayed learning rates clr = lr / (1 + s·lr_decay) of the ten parameters (s: the step before this update),
// formed in double once per CTA before the first grid barrier.
__device__ __forceinline__ void adagrad_factors(const AdagradRider& r, float* f, int tid) {
  if (tid < 10 && r.step[tid]) {
    const double lr = r.h.lr_dev ? static_cast<double>(__ldg(r.h.lr_dev)) : r.h.lr;
    f[tid] = static_cast<float>(lr / (1.0 + static_cast<double>(*r.step[tid]) * r.h.lr_decay));
  }
}

// One Adagrad update (the arithmetic of adagrad_multi_kernel, ops_simt.cu) of element i of parameter k with gradient g; f: the
// factors of adagrad_factors.  R: AdagradRider, possibly in a ClipRider.
template <class R>
__device__ __forceinline__ void adagrad_apply(const R& r, int k, int i, float g, const float* f) {
  float gv = r.h.maximize ? -g : g;
  float* p = r.p[k] + i;
  float* sum = r.sum[k] + i;
  const float pv = *p;
  if (r.h.weight_decay != 0.f) gv = fmaf(r.h.weight_decay, pv, gv);
  const float s = fmaf(gv, gv, *sum);
  *sum = s;
  *p = fmaf(-f[k], gv / (sqrtf(s) + r.h.eps), pv);
}

// Gradient-norm clipping (ClipRider): one gradient element g into a thread's accumulator — Σg², or max |g| keeping a NaN.
template <class R>
__device__ __forceinline__ float clip_acc(const R& r, float acc, float g) { return r.norm_inf ? nan_max(fabsf(g), acc) : fmaf(g, g, acc); }
template <class R>
__device__ __forceinline__ float clip_comb(const R& r, float a, float b) { return r.norm_inf ? nan_max(a, b) : a + b; }

template <class R>
constexpr bool kClipRider =
    std::is_same_v<R, ClipRider<SgdRider>> || std::is_same_v<R, ClipRider<AdamRider>> || std::is_same_v<R, ClipRider<AmsgradRider>> ||
    std::is_same_v<R, ClipRider<RmspropRider>> || std::is_same_v<R, ClipRider<AdagradRider>>;
template <class R>
constexpr bool kAdamRider = std::is_same_v<R, AdamRider> || std::is_same_v<R, ClipRider<AdamRider>> || std::is_same_v<R, AmsgradRider> ||
                            std::is_same_v<R, ClipRider<AmsgradRider>>;
template <class R>
constexpr bool kRmspropRider = std::is_same_v<R, RmspropRider> || std::is_same_v<R, ClipRider<RmspropRider>>;
template <class R>
constexpr bool kAdagradRider = std::is_same_v<R, AdagradRider> || std::is_same_v<R, ClipRider<AdagradRider>>;

// Element i of parameter k's gradient is final with value g: a ClipRider adds it to this thread's share ca of the norm (the update
// waits for the coefficient), the others apply their update.  The caller tests whether the rider is on and the parameter takes part.
// adam_f: the per-launch factors of the Adam or Adagrad rider; sgd_lr: the learning rate of the SGD or RMSprop rider.
template <class Rider>
__device__ __forceinline__ void ride(const Rider& sr, float& ca, int k, int i, float g, const float* adam_f, float sgd_lr) {
  if constexpr (kClipRider<Rider>) ca = clip_acc(sr, ca, g);
  else if constexpr (kAdamRider<Rider>) adam_apply(sr, k, i, g, adam_f);
  else if constexpr (kRmspropRider<Rider>) rmsprop_apply(sr, k, i, g, sgd_lr);
  else if constexpr (kAdagradRider<Rider>) adagrad_apply(sr, k, i, g, adam_f);
  else sgd_apply(sr.p[k] + i, g, sr.m[k] ? sr.m[k] + i : nullptr, sr.h, sgd_lr);
}

// ACC (accumulate mode, gradient accumulation over micro-batches): every gradient this kernel writes — dgamma, dbeta, the conv1 fold
// dw / db and the conv2 fold dw2 / db2 — becomes g = g_old + v, and the rider updates with (and clips) that accumulated value.
// y: conv1's output [B][28][28][16], or null: then the CTA recomputes its pixel's values from the image and w1 / b1 (conv1_pixels, the
// forward's order, so the same bits) instead of loading 50 KB per image that the forward would have had to store.
template <class Rider = SgdRider, bool ACC = false>
__global__ void __launch_bounds__(kL1Threads, 1)
convnet_l1_bwd_kernel(const float* __restrict__ dp, const float* __restrict__ y, const float* w1, const float* b1, const float* __restrict__ x,
                      const float* __restrict__ saved,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float* dgamma, float* dbeta, float* dw, float* db,
                      float* partials, float* partials_w, GridSync gs,
                      // conv2's weight gradient, folded from the per-image partials [B][400][32] and Σdy rows [B][32]
                      const float* __restrict__ wpart, const float* __restrict__ dysum2, float* dw2, float* db2, const __grid_constant__ Rider sr) {
  constexpr bool kClip = kClipRider<Rider>, kAdam = kAdamRider<Rider>, kRmsprop = kRmspropRider<Rider>, kAdagrad = kAdagradRider<Rider>;
  static_assert(kAdam || kRmsprop || kAdagrad || std::is_base_of_v<SgdRider, Rider>,
                "convnet_l1_bwd_kernel: SgdRider, AdamRider, AmsgradRider, RmspropRider or AdagradRider, or one of them in a ClipRider");
  extern __shared__ __align__(16) float dsm[];
  float* dys = dsm;                  // [784][16]
  float* fold = dsm + 784 * 16;      // [25 warps][16][32]
  // Adam rider: the per-launch factors; Adagrad rider: the ten decayed learning rates
  __shared__ float adam_f[kAdam ? kAdamFactors : kAdagrad ? 10 : 1];
  __shared__ float xs[32 * 32];
  __shared__ __align__(16) float ws[25 * 16];   // conv1's weights [tap][co] when y is recomputed
  __shared__ float red[kL1Warps * 32];
  __shared__ float s_tmp[kL1Warps * 32];
  __shared__ float s_tot[32];
  __shared__ float s_scale[16], s_shift[16], s_mean[16], s_invstd[16];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;
  float* s_clip = red + 512;   // ClipRider: per-warp norm partials + the coefficient (s_db below takes red[0, 512) only)

  const L1Map m(tid);
  griddep_wait();   // programmatic launch behind the layer-2 backward: everything below reads its outputs or the grid-barrier words
  GridBar bar(gs);
  TRACE_INIT();
  trace(1, 0);

  // the image and conv1's weights are requested together (one round trip, not two in a row), then the pooled gradient, whose loads
  // are in flight while the image is staged and y is loaded or recomputed.  conv1's weights and bias (here and in conv1_pixels) are
  // read before the first grid barrier, and the rider updates them (parameters 0 and 1) only after the second one, so no CTA reads an
  // updated weight
  L1Image<kL1Threads> img;
  img.load(x + static_cast<size_t>(n) * 784, tid);
  const float w1v = y == nullptr && tid < 400 ? w1[(tid & 15) * 25 + (tid >> 4)] : 0.f;
  float dz[16];
  {
    const float4* gp = reinterpret_cast<const float4*>(dp + ((static_cast<size_t>(n) * 18 + m.ph + 2) * 18 + m.pw + 2) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 g4 = m.valid ? gp[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      dz[4 * q] = g4.x; dz[4 * q + 1] = g4.y; dz[4 * q + 2] = g4.z; dz[4 * q + 3] = g4.w;
    }
  }
  img.store(xs, tid);
  if (y == nullptr && tid < 400) ws[tid] = w1v;
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
  } else if constexpr (kAdagrad) {
    if (sr.on) adagrad_factors(sr, adam_f, tid);
  }
  __syncthreads();

  float yv[16];
  if (y != nullptr) {
    const float4* yp = reinterpret_cast<const float4*>(y + ((static_cast<size_t>(n) * 28 + m.r) * 28 + m.c) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 a = m.valid ? yp[q] : make_float4(0.f, 0.f, 0.f, 0.f);
      yv[4 * q] = a.x; yv[4 * q + 1] = a.y; yv[4 * q + 2] = a.z; yv[4 * q + 3] = a.w;
    }
  } else {
    // the window's four lanes share the recompute: lane d computes channels 4d .. 4d + 3 of the window's four pixels, so that every
    // weight read from shared memory serves four pixels, then the lanes transpose the 4 × 4 blocks: lane d gets its pixel's 16
    const int x0 = 2 * m.ph * 32 + 2 * m.pw;
    const int xoff[4] = {x0, x0 + 1, x0 + 32, x0 + 33};   // pixel d of the window: row 2·ph + (d >> 1), column 2·pw + (d & 1)
    float blk[4][4];
    conv1_pixels<4, 4>(xs, ws + 4 * m.d, b1 ? b1 + 4 * m.d : nullptr, xoff, blk);
    window_transpose_step<2>(blk, lane);
    window_transpose_step<1>(blk, lane);
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
      for (int j = 0; j < 4; ++j) yv[4 * e + j] = m.valid ? blk[e][j] : 0.f;   // the padding threads hold zeros, as when y is loaded
  }
  trace(1, 8);
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
  __syncthreads();
  if (tid < 32) {
    float s = 0.f;
#pragma unroll 5
    for (int wi = 0; wi < kL1Warps; ++wi) s += red[wi * 32 + tid];
    partials[static_cast<size_t>(n) * 32 + tid] = s;
  }
  trace(1, 1);
  bar.arrive(gs);
  const float sgd_lr = sr.on ? (sr.h.lr_dev ? __ldg(sr.h.lr_dev) : static_cast<float>(sr.h.lr)) : 0.f;
  float ca = 0.f;   // ClipRider: this thread's share of the gradient norm
  if (kClip || sr.on) {   // (a ClipRider is only made around a rider that is on)
    // in the barrier's shadow: the parameters whose gradients were complete before this kernel started (classifier, bn2, and
    // below conv2) — nothing in this kernel reads them
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (!kClip || sr.p[6 + t])
        for (int i = n * kL1Threads + tid; i < sr.n_prev[t]; i += B * kL1Threads) ride(sr, ca, 6 + t, i, __ldg(sr.g_prev[t] + i), adam_f, sgd_lr);
  }
  {
    // in the barrier's shadow: conv2's weight gradient, complete before this kernel started (the layer-2 backward kernel wrote the
    // per-image partials), and its optimizer step — nothing in this kernel reads conv2's parameters.  CTA n folds outputs n, n + B,
    // … of the 400 (tap, ci) rows × 32 co (+ row 400: the bias, from the per-image Σdy rows) over the B per-image partials [400][32],
    // whose row i is that output row — warp =
    // one of 25 partial classes, lane = co, classes combined through smem in a fixed order, up to five outputs per round so that
    // ~20 L2 loads per thread are in flight
    float* s_f = fold;   // [5][25][32]
    constexpr size_t kStride = 400 * 32;
    for (int base = n; base < 401; base += 5 * B) {
      float acc[5];
      const float* src[5];
      size_t stride[5];
#pragma unroll
      for (int u = 0; u < 5; ++u) {
        const int i = base + u * B;
        if (i < 400) {
          src[u] = wpart + static_cast<size_t>(i) * 32 + lane;
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
      __syncthreads();
#pragma unroll
      for (int u = 0; u < 5; ++u) s_f[(u * kL1Warps + warp) * 32 + lane] = acc[u];
      __syncthreads();
      if (tid < 160) {
        const int u = tid >> 5, i = base + u * B;
        if (i <= 400) {
          float tot = 0.f;
#pragma unroll 5
          for (int wi = 0; wi < kL1Warps; ++wi) tot += s_f[(u * kL1Warps + wi) * 32 + lane];
          if (i < 400) {
            const int e = (lane * 16 + (i & 15)) * 25 + (i >> 4);
            if constexpr (ACC) tot = dw2[e] + tot;
            dw2[e] = tot;
            if (kClip || sr.on) ride(sr, ca, 4, e, tot, adam_f, sgd_lr);
          } else if (db2) {
            if constexpr (ACC) tot = db2[lane] + tot;
            db2[lane] = tot;
            if ((kClip || sr.on) && sr.p[5]) ride(sr, ca, 5, lane, tot, adam_f, sgd_lr);
          }
        }
      }
    }
    trace(1, 7);
  }
  if constexpr (kClip) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) ca = clip_comb(sr, ca, __shfl_xor_sync(0xffffffffu, ca, off));
    if (lane == 0) s_clip[warp] = ca;
    ca = 0.f;
  }
  bar.wait(gs);
  trace(1, 2);
  fold_rows_wide<32, kL1Threads>(partials, B, s_tmp, s_tot);  // [0..16) Σdz, [16..32) Σdz·x̂
  trace(1, 3);
  if (n == 0 && tid < 16) {
    if constexpr (ACC) {   // s_tot keeps this batch's sums: the data gradient below needs them
      if (dbeta) dbeta[tid] = dbeta[tid] + s_tot[tid];
      if (dgamma) dgamma[tid] = dgamma[tid] + s_tot[16 + tid];
    } else {
      if (dbeta) dbeta[tid] = s_tot[tid];
      if (dgamma) dgamma[tid] = s_tot[16 + tid];
    }
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
  __syncthreads();
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
  __syncthreads();
  float* s_db = red;   // [32 parts][16]  (the statistics scratch is free again)
  if (tid < 512) s_db[tid] = dbp;
  __syncthreads();
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
  bar.sync(gs);
  trace(1, 5);
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
        if constexpr (ACC) s = dw[co * 25 + tap] + s;
        dw[co * 25 + tap] = s;
        if (kClip || sr.on) ride(sr, ca, 0, co * 25 + tap, s, adam_f, sgd_lr);
      } else if (db) {
        if constexpr (ACC) s = db[co] + s;
        db[co] = s;
        if ((kClip || sr.on) && sr.p[1]) ride(sr, ca, 1, co, s, adam_f, sgd_lr);
      }
    }
  }
  if (sr.on && n == 0 && tid < 16) {
    // BatchNorm-1 affine parameters: their gradients are the totals this CTA folded after the first barrier (in accumulate mode,
    // what this thread wrote above: those added to the earlier micro-batches').  Every CTA read gamma / beta before that barrier,
    // so updating them here (after the second one) races with nobody.
    const float gbeta = ACC && dbeta ? dbeta[tid] : 0.f, ggamma = ACC && dgamma ? dgamma[tid] : 0.f;
    if (sr.p[3]) ride(sr, ca, 3, tid, ACC ? gbeta : s_tot[tid], adam_f, sgd_lr);
    if (sr.p[2]) ride(sr, ca, 2, tid, ACC ? ggamma : s_tot[16 + tid], adam_f, sgd_lr);
  }
  if constexpr (kClip) {
    // every gradient has been seen: one partial per CTA, one more grid barrier, then every CTA folds the B partials in the same
    // order and derives the same coefficient bit for bit
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) ca = clip_comb(sr, ca, __shfl_xor_sync(0xffffffffu, ca, off));
    if (lane == 0) s_clip[warp] = clip_comb(sr, s_clip[warp], ca);
    __syncthreads();
    if (tid == 0) {
      float s = s_clip[0];
      for (int w = 1; w < kL1Warps; ++w) s = clip_comb(sr, s, s_clip[w]);
      sr.part[n] = s;
    }
    bar.sync(gs);
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
    __syncthreads();
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
        else if constexpr (kRmsprop) rmsprop_apply(sr, k, i, gv, sgd_lr);
        else if constexpr (kAdagrad) adagrad_apply(sr, k, i, gv, adam_f);
        else sgd_apply(sr.p[k] + i, gv, sr.m[k] ? sr.m[k] + i : nullptr, sr.h, sgd_lr);
      }
    }
  }
  if constexpr (kAdam || kRmsprop || kAdagrad) {
    // every CTA read the step counts before the first grid barrier and this is after the last one
    if ((kClip || sr.on) && n == 0 && tid == 0)
      for (int k = 0; k < 10; ++k)
        if (sr.step[k]) *sr.step[k] += 1.f;
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

// Row P of the 128 halo rows of the 18 × 18 patch (h < 128): the top two rows, the two side columns on each side of rows 2..15,
// the bottom two rows.
__device__ __forceinline__ int patch_halo_row(int h) {
  if (h < 36) return h;
  if (h >= 92) return 16 * kPW + (h - 92);
  const int s = h - 36, side = s & 3;
  return (2 + (s >> 2)) * kPW + (side < 2 ? side : 14 + side);
}

// Output tile t of conv2 of one image on the tensor cores, issued by one warpgroup (wt = thread index inside it; the two tiles run
// on two warpgroups at once): 25 taps × 2 K-steps of wgmma m64n32k8 per 64-row half, the two halves independent accumulator
// chains, the A descriptors row-shifted into the haloed patch.  The accumulators go straight into ys [pixel][32] (bias added;
// 16-byte chunks rotated by the pixel index, as the column reads that follow expect), and the BatchNorm sums of the kept elements
// are taken while they are still in registers: s_stat[8 warps][32] gets this warp's Σy.
__device__ __forceinline__ void l2_conv_wgmma(const uint8_t* sa, const uint8_t* sb, const float* __restrict__ bias, float* ys, float* s_stat,
                                              int t, int wt) {
  const uint64_t ad0 = gmma_desc_kmajor<128>(smem_u32(sa)), bd0 = gmma_desc_kmajor<128>(smem_u32(sb));
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
  // a thread holds 8 columns, c = 8·(e >> 2) + 2·(wt & 3) + (e & 1): sums slot k = 2·(e >> 2) + (e & 1)
  float s1[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) s1[k] = 0.f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int e = 0; e < 16; ++e) {
      const int rr = 64 * h + wgmma_frag_row(wt, e), c = wgmma_frag_col(wt, e), k = 2 * (e >> 2) + (e & 1);
      const int orow = rr / kPW, ow = rr - orow * kPW;
      if (rr < 126 && ow < 14) {
        const int pix = (7 * t + orow) * 14 + ow;
        const float v = acc[h][e] + (bias ? __ldg(bias + c) : 0.f);
        ys[pix * 32 + ((((c >> 2) + pix) & 7) << 2) + (c & 3)] = v;
        s1[k] += v;
      }
    }
  }
  // lanes 4 apart hold the same columns
#pragma unroll
  for (int off = 4; off <= 16; off <<= 1)
#pragma unroll
    for (int k = 0; k < 8; ++k) s1[k] += __shfl_xor_sync(0xffffffffu, s1[k], off);
  const int lane = wt & 31;
  if (lane < 4) {
    float* row = s_stat + (4 * t + (wt >> 5)) * 32;
#pragma unroll
    for (int k = 0; k < 8; ++k) row[8 * (k >> 1) + 2 * lane + (k & 1)] = s1[k];
  }
}

struct L2FwdSmem {
  static constexpr int kB = 25 * 32 * 128;       // weights: [tap][32 co][128 B] (ci 0..15 used)            102,400
  static constexpr int kYs = 196 * 32 * 4;       // conv output of the image, [pixel][32]                     25,088
  static constexpr int kMisc = 1024 * 4;         // statistics and classifier scratch                          4,096
  static constexpr int kTotal = 1024 + kPatchAlloc + kB + kYs + kMisc;
};

// The forward's CTA: every compute thread owns the same pixel d of two pooling windows, win and win + 98 (392 threads, the
// 4-lanes-per-window order of L1Map kept), in 13 warps.  The register budget of 416 threads holds both pixels' accumulators and
// the 32-value statistics reduction without local memory, and every conv1 weight read from shared memory serves two pixels.
constexpr int kFwdPix = 392;
constexpr int kFwdThreads = 416;
constexpr int kFwdWarps = kFwdThreads / 32;

// conv1 output of one pixel → y1 (for direct callers of convnet_fwd).
__device__ __forceinline__ void l1_store_y(float* __restrict__ y1, int n, const L1Map& m, const float (&acc)[16]) {
  float4* yp = reinterpret_cast<float4*>(y1 + ((static_cast<size_t>(n) * 28 + m.r) * 28 + m.c) * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q) yp[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
}

// BN + ReLU + 2×2 max-pool of one pixel's window (two shuffles; called by every lane) → conv2's patch and the global frame p1n.
__device__ __forceinline__ void l1_pool_store(const float (&acc)[16], const L1Map& m, const float* s_scale, const float* s_shift, uint8_t* sa,
                                              float* __restrict__ p1n) {
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
    *reinterpret_cast<float4*>(sa + sw128_off(P, m.d)) = o;   // conv2 reads this one
    reinterpret_cast<float4*>(p1n + P * 16)[m.d] = o;          // backward (conv2 wgrad) reads this one
  }
}

// =====================================================================================================================
// Whole forward pass in ONE kernel: layer 1 and layer 2 (+ classifier) of an image run in the same CTA, so the pooled
// layer-1 activations never leave the SM on their way into conv2 — they are written straight into the swizzled,
// zero-haloed shared-memory patch the wgmma descriptors read (the global copy is still written: backward needs it) —
// and the conv2 weights are staged while conv1 computes.  Two grid barriers (BN1 and BN2 batch statistics), one launch.
// Ce = ScaledCe: the cross-entropy rider computes scale · (mean cross-entropy) and its gradient (gradient accumulation: 1/k).
// Ce = SmoothCe: the same with class weights, label smoothing, any ignore_index and the sum (fused_convnet.h).
// Ce = SoftCe: the SmoothCe options with class-probability targets.
// =====================================================================================================================
__device__ __forceinline__ float ce_scale(const FusedCe&) { return 1.f; }
__device__ __forceinline__ float ce_scale(const ScaledCe& ce) { return ce.scale; }
// whether the cross-entropy rider is on
__device__ __forceinline__ bool ce_on(const FusedCe& ce) { return ce.target != nullptr; }
__device__ __forceinline__ bool ce_on(const SoftCe& ce) { return ce.target_probs != nullptr; }

template <class Ce = FusedCe>
__global__ void __launch_bounds__(kFwdThreads, 1)
convnet_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ g1,
                   const float* __restrict__ be1, float* __restrict__ y1, float* __restrict__ p1, float* saved1, float* rm1, float* rv1,
                   long long* nbt1, float mom1, float eps1, const float* __restrict__ w2, const float* __restrict__ b2,
                   const float* __restrict__ g2, const float* __restrict__ be2, float* __restrict__ y2, float* __restrict__ out, float* saved2,
                   float* rm2, float* rv2, long long* nbt2, float mom2, float eps2, const float* __restrict__ fcw,
                   const float* __restrict__ fcb, float* __restrict__ logits, int ncls, float* partials, GridSync gs, Ce ce) {
  constexpr bool kScaled = std::is_same_v<Ce, ScaledCe>;
  constexpr bool kSmooth = std::is_same_v<Ce, SmoothCe>;
  constexpr bool kSoft = std::is_same_v<Ce, SoftCe>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                  // conv2 input patch, written by this CTA's layer-1 epilogue
  uint8_t* sb = sa + kPatchAlloc;                      // conv2 weights
  float* ys = reinterpret_cast<float*>(sb + L2FwdSmem::kB);
  float* misc = ys + 196 * 32;                         // 1024 floats
  float* s_part = misc;                                // [8 warps][32] conv2 sums / [13 warps][16] classifier partials
  float* s_scale2 = misc + 576;                        // [32]
  float* s_shift2 = misc + 608;                        // [32]
  __shared__ float xs[32 * 32];
  __shared__ __align__(16) float ws[25 * 16];
  __shared__ float red[kFwdWarps * 32];
  __shared__ float s_tmp[kFwdWarps * 32];
  __shared__ float s_stat[64];   // an image's means, then the batch's (mean, var): layer 1 in [0, 32), layer 2 in [0, 64)
  __shared__ float s_scale[16], s_shift[16];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;
  // pixel d of windows win and win + 98; the threads past kFwdPix own none (L1Map(784) is not valid)
  const L1Map m0(tid < kFwdPix ? tid : 784), m1(tid < kFwdPix ? tid + kFwdPix : 784);
  GridBar bar(gs);
  TRACE_INIT();
  trace(0, 0);

  // conv2 weights [co][ci][tap] → the swizzled K-major tiles [tap][co][ci], one float per cp.async: nothing is held in registers
  // while they fly, behind conv1.  One (co, ci) pair per thread and its 25 taps, so that the 32 lanes of a copy write 32 different
  // banks (consecutive taps are 4 KiB apart in shared memory: one bank).
  for (int pair = tid; pair < 32 * 16; pair += kFwdThreads) {
    const int co = pair >> 4, ci = pair & 15;
    const uint32_t dst = smem_u32(sb + sw128_off(co, ci >> 2) + (ci & 3) * 4);
#pragma unroll
    for (int tap = 0; tap < 25; ++tap) cp_async_4(dst + tap * 4096, w2 + pair * 25 + tap);
  }
  cp_async_commit();
  // the patch's zero halo: the 64 bytes (channels 0..15) the descriptors read of each halo row.  The slack rows past 324 are left
  // as they are: only the padding rows of tile 1 read them, and those outputs are dropped.
  for (int i = tid; i < 128 * 4; i += kFwdThreads)
    *reinterpret_cast<float4*>(sa + sw128_off(patch_halo_row(i >> 2), i & 3)) = make_float4(0.f, 0.f, 0.f, 0.f);
  {   // the image and conv1's weights are requested together: one round trip, not two in a row
    L1Image<kFwdThreads> img;
    img.load(x + static_cast<size_t>(n) * 784, tid);
    const float w1v = tid < 400 ? w1[(tid & 15) * 25 + (tid >> 4)] : 0.f;
    img.store(xs, tid);
    if (tid < 400) ws[tid] = w1v;   // [tap][co]
  }
  __syncthreads();
  trace(0, 11);

  // ---- layer 1: both pixels in the FMA order of one pixel per thread, so y1 does not depend on the CTA shape ---------------
  float acc[2][16];
  float(&acc0)[16] = acc[0];
  float(&acc1)[16] = acc[1];
  {
    const int xoff[2] = {m0.r * 32 + m0.c, m1.r * 32 + m1.c};
    conv1_pixels<2, 16>(xs, ws, b1, xoff, acc);
  }
  trace(0, 1);
  // this image's [Σy (16) | M2 (16)] (fold_centred_stats): Σy first, then the squared deviations about the image's mean
  {
    float v[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = m0.valid ? acc0[j] + acc1[j] : 0.f;
    warp_transpose_reduce16(v, lane);
    if (lane < 16) red[warp * 16 + lane] = v[0];
  }
  __syncthreads();
  if (tid < 16) {
    float s = 0.f;
#pragma unroll
    for (int wi = 0; wi < kFwdWarps; ++wi) s += red[wi * 16 + tid];
    partials[static_cast<size_t>(n) * 32 + tid] = s;
    s_stat[tid] = s / 784.f;
  }
  __syncthreads();
  {
    float v[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float d0 = acc0[j] - s_stat[j], d1 = acc1[j] - s_stat[j];
      v[j] = m0.valid ? fmaf(d1, d1, d0 * d0) : 0.f;
    }
    warp_transpose_reduce16(v, lane);
    if (lane < 16) red[kFwdWarps * 16 + warp * 16 + lane] = v[0];
  }
  __syncthreads();
  if (tid < 16) {
    float s = 0.f;
#pragma unroll
    for (int wi = 0; wi < kFwdWarps; ++wi) s += red[kFwdWarps * 16 + wi * 16 + tid];
    partials[static_cast<size_t>(n) * 32 + 16 + tid] = s;
  }
  trace(0, 2);
  bar.arrive(gs);
  // in the barrier's shadow: the pooled frame's zero halo (backward reads it; nothing in this kernel does)
  float* p1n = p1 + static_cast<size_t>(n) * 324 * 16;
  for (int i = tid; i < 128 * 4; i += kFwdThreads)
    reinterpret_cast<float4*>(p1n + patch_halo_row(i >> 2) * 16)[i & 3] = make_float4(0.f, 0.f, 0.f, 0.f);
  bar.wait(gs);
  trace(0, 3);
  fold_centred_stats<16, kFwdThreads, 6>(partials, B, 784.f, s_tmp, red, s_stat);
  if (tid < 16) {
    const float cnt = static_cast<float>(B) * 784.f;
    const float mean = s_stat[tid], var = s_stat[16 + tid];
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
  l1_pool_store(acc0, m0, s_scale, s_shift, sa, p1n);
  l1_pool_store(acc1, m1, s_scale, s_shift, sa, p1n);
  if (y1 && m0.valid) {   // y1 for direct callers (nothing in this kernel reads it; backward B recomputes it): drains behind conv2
    l1_store_y(y1, n, m0, acc0);
    l1_store_y(y1, n, m1, acc1);
  }
  cp_async_wait<0>();         // this thread's weight copies have landed
  fence_proxy_async_smem();   // generic-proxy writes of the patch and of the weights → visible to the tensor core
  __syncthreads();
  trace(0, 4);
  // ---- layer 2: 2 × 100 wgmma (K = 8, M = 64 each), output tile t by warpgroup t -------------------------------------------
  const int wg = warpgroup_index();
  if (wg < 2) l2_conv_wgmma(sa, sb, b2, ys, s_part, wg, tid & 127);
  __syncthreads();
  trace(0, 5);
  // this image's [Σy (32) | M2 (32)] (fold_centred_stats): Σy from the epilogue, the squared deviations about the image's mean
  // from ys, 15 or 16 pixels of one channel per thread
  float* partials2 = partials + static_cast<size_t>(B) * 32;
  if (tid < 32) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += s_part[w * 32 + tid];
    partials2[static_cast<size_t>(n) * 64 + tid] = s;
    s_stat[tid] = s / 196.f;
  }
  __syncthreads();
  {
    const int c = lane;
    const float mu = s_stat[c];
    float q = 0.f;
    for (int pix = warp; pix < 196; pix += kFwdWarps) {
      const float d = ys[pix * 32 + ((((c >> 2) + pix) & 7) << 2) + (c & 3)] - mu;
      q = fmaf(d, d, q);
    }
    red[warp * 32 + lane] = q;
  }
  __syncthreads();
  if (tid < 32) {
    float s = 0.f;
#pragma unroll
    for (int wi = 0; wi < kFwdWarps; ++wi) s += red[wi * 32 + tid];
    partials2[static_cast<size_t>(n) * 64 + 32 + tid] = s;
  }
  trace(0, 6);
  bar.arrive(gs);
  float* fcs = reinterpret_cast<float*>(sb + 8192);   // classifier weights, staged behind the pooled activations (conv2's weights are dead)
  // only where they fit before ys, which is still being read: up to 15 classes; 16 are read from global memory
  const bool fc_staged = logits != nullptr && (reinterpret_cast<uintptr_t>(fcw) & 15) == 0 && ncls * 1568 * 4 <= L2FwdSmem::kB - 8192;
  if (fc_staged) {
    for (int i = tid; i < ncls * 392; i += kFwdThreads) cp_async_16(smem_u32(fcs + 4 * i), fcw + 4 * i, 16);
    cp_async_commit();
  }
  __shared__ std::conditional_t<kSmooth || kSoft, float, int> s_counted;   // SmoothCe, SoftCe: the divisor D
  if constexpr (kSoft) {
    if (tid == 0) s_counted = ce.sum ? 1.f : static_cast<float>(B);   // every image counts
  } else if constexpr (kSmooth) {
    if (ce.target != nullptr && warp == 0) {
      // in the barrier's shadow: D = Σ w_t over the counted images (their number without weights) for the mean, 1 for the sum;
      // every CTA sums the same B ≤ #SM terms in the same order, so all agree bit for bit
      float d = 0.f;
      if (!ce.sum) {
        for (int r = lane; r < B; r += 32) {
          const long long tr = ce.target[r];
          if (tr >= 0 && tr < ncls && tr != ce.ignore_index) d += ce.weight ? ce.weight[tr] : 1.f;
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) d += __shfl_xor_sync(0xffffffffu, d, off);
      }
      if (lane == 0) s_counted = ce.sum ? 1.f : d;
    }
  } else if (ce.target != nullptr && warp == 0) {
    // in the barrier's shadow: the cross-entropy's mean is over the images whose target lies in [0, ncls) (torch's ignore_index);
    // every CTA counts them, B ≤ one per SM
    int counted = 0;
#pragma unroll 4
    for (int r = lane; r < B; r += 32) {
      const long long tr = ce.target[r];
      counted += (tr >= 0 && tr < ncls) ? 1 : 0;
    }
    counted = __reduce_add_sync(0xffffffffu, counted);
    if (lane == 0) s_counted = counted;
  }
  for (int i = tid; i < 196 * 8; i += kFwdThreads) {   // in the barrier's shadow: conv2's output for the backward pass
    const int pix = i >> 3, q = i & 7;
    reinterpret_cast<float4*>(y2 + (static_cast<size_t>(n) * 196 + pix) * 32)[q] = reinterpret_cast<const float4*>(ys + pix * 32)[(q + pix) & 7];
  }
  bar.wait(gs);
  griddep_launch_dependents();   // no CTA waits for another from here on: the layer-2 backward's grid may be set up
  trace(0, 7);
  fold_centred_stats<32, kFwdThreads, 11>(partials2, B, 196.f, s_tmp, red, s_stat);
  if (tid < 32) {
    const float cnt = static_cast<float>(B) * 196.f;
    const float mean = s_stat[tid], var = s_stat[32 + tid];
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
  for (int i = tid; i < 1568; i += kFwdThreads) {
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
  for (int i = tid; i < 1568; i += kFwdThreads) out[static_cast<size_t>(n) * 1568 + i] = pool[i];
  if (logits != nullptr) {
    // classifier: thread t owns features t, t + 416, t + 832 and t + 1248 (< 1568) for every class (≤ 16): all weight loads
    // independent
    float accv[16], pv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) pv[u] = (tid + u * kFwdThreads < 1568) ? pool[tid + u * kFwdThreads] : 0.f;
#pragma unroll
    for (int c16 = 0; c16 < 16; ++c16) {
      float sacc = 0.f;
      if (c16 < ncls) {
        const float* wr = (fc_staged ? fcs : fcw) + static_cast<size_t>(c16) * 1568 + tid;
        sacc = pv[0] * wr[0];
#pragma unroll
        for (int u = 1; u < 4; ++u)
          if (tid + u * kFwdThreads < 1568) sacc = fmaf(pv[u], wr[u * kFwdThreads], sacc);
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
#pragma unroll
        for (int wi = 0; wi < kFwdWarps; ++wi) lg += s_part[wi * 16 + lane];
        logits[static_cast<size_t>(n) * ncls + lane] = lg;
      }
      trace(0, 9);
      if (ce_on(ce)) {
        // cross-entropy of this image and its gradient for a unit incoming gradient, divided by the number of counted images; an
        // ignored image adds no term and gets a zero gradient
        const auto counted = s_counted;   // SmoothCe, SoftCe: the divisor D
        float mx = lg;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        const float e = lane < ncls ? __expf(lg - mx) : 0.f;
        float ssum = e;
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, off);
        if constexpr (kSoft) {
          // term = Σ_c a_c·(lse − l_c), gradient (p_c·S − a_c) / D, with a_c = w_c·q'_c, q' = q·(1−ε) + ε/C and S = Σ_c a_c; lane c
          // reads q_c and w_c, the sums over classes are shuffle reductions
          float a = 0.f;
          if (lane < ncls)
            a = (ce.weight ? ce.weight[lane] : 1.f) *
                (ce.target_probs[static_cast<size_t>(n) * ncls + lane] * (1.f - ce.smoothing) + ce.smoothing / static_cast<float>(ncls));
          const float lse = mx + __logf(ssum);
          float S = a, term = lane < ncls ? a * (lse - lg) : 0.f;
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) {
            S += __shfl_xor_sync(0xffffffffu, S, off);
            term += __shfl_xor_sync(0xffffffffu, term, off);
          }
          if (lane < ncls) ce.dlogits[static_cast<size_t>(n) * ncls + lane] = (e / ssum * S - a) / counted * ce.scale;
          if (lane == 0) ce.loss_parts[n] = term;
        } else {
          const long long t = ce.target[n];
          bool t_ok = t >= 0 && t < ncls;
          if constexpr (kSmooth) t_ok = t_ok && t != ce.ignore_index;
          const float lt = __shfl_sync(0xffffffffu, lg, t_ok ? static_cast<int>(t) : 0);
          if constexpr (kSmooth) {
            // term = (1-ε)·w_t·(lse − l_t) + (ε/C)·Σ_c w_c·(lse − l_c), gradient [(1-ε)·w_t·(p_c − [c=t]) + (ε/C)·(W·p_c − w_c)] / D;
            // lane c holds w_c, the sums over classes are shuffle reductions
            const float wc = lane < ncls ? (ce.weight ? ce.weight[lane] : 1.f) : 0.f;
            const float wt = __shfl_sync(0xffffffffu, wc, t_ok ? static_cast<int>(t) : 0);
            const float lse = mx + __logf(ssum);
            float wsum = wc, smooth = lane < ncls ? wc * (lse - lg) : 0.f;
#pragma unroll
            for (int off = 16; off >= 1; off >>= 1) {
              wsum += __shfl_xor_sync(0xffffffffu, wsum, off);
              smooth += __shfl_xor_sync(0xffffffffu, smooth, off);
            }
            const float keep = 1.f - ce.smoothing, eps_c = ce.smoothing / static_cast<float>(ncls);
            if (lane < ncls) {
              const float p = e / ssum;
              ce.dlogits[static_cast<size_t>(n) * ncls + lane] =
                  (t_ok ? (keep * wt * (p - (t == lane ? 1.f : 0.f)) + eps_c * (wsum * p - wc)) / counted : 0.f) * ce.scale;
            }
            // D = 0 (a mean over zero total weight): no term, so that either fold gives torch's 0 / 0 = NaN
            if (lane == 0) ce.loss_parts[n] = t_ok && counted != 0.f ? keep * wt * (lse - lt) + eps_c * smooth : 0.f;
          } else {
            if (lane < ncls) {
              // ScaledCe: the rounding of autograd's grad · scale behind the unscaled loss
              if constexpr (kScaled)
                ce.dlogits[static_cast<size_t>(n) * ncls + lane] = (t_ok ? (e / ssum - (t == lane ? 1.f : 0.f)) / static_cast<float>(counted) : 0.f) * ce.scale;
              else
                ce.dlogits[static_cast<size_t>(n) * ncls + lane] = t_ok ? (e / ssum - (t == lane ? 1.f : 0.f)) / static_cast<float>(counted) : 0.f;
            }
            if (lane == 0) ce.loss_parts[n] = t_ok ? mx + __logf(ssum) - lt : 0.f;
          }
        }
        // for a mean folded later (ScaledCe: the divisor is the count over the scale; SmoothCe, SoftCe: D over the scale)
        if (lane == 0 && n == 0)
          ce.loss_parts[B] = (kScaled || kSmooth || kSoft) ? static_cast<float>(counted) / ce_scale(ce) : static_cast<float>(counted);
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
              *ce.loss = sl / ((kScaled || kSmooth || kSoft) ? static_cast<float>(counted) / ce_scale(ce) : static_cast<float>(counted));
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
  // the classifier's backward: fc weights [16][1568] | dlogits [B ≤ 160][16] | pooled slice [B ≤ 160][16]
  static constexpr int kFcW = 16 * 1568 * 4, kFcDl = 160 * 16 * 4, kFcP = 160 * 16 * 4;
  static constexpr int kTotalFc = kTotal + kFcW + kFcDl + kFcP;
  // WG: conv2's weight-gradient operands (Conv2Wg).  The x copies are written in the grid barrier's shadow over the fc weights, dead
  // by then, and dyᵀ after the barrier over the end of the fc weights and the dlogits / pooled slices, which the classifier's
  // weight gradient in the shadow was the last to read.
  static constexpr int kXT = kPatchAlloc + kB + 4096;
  static constexpr int kDyT = kXT + Conv2Wg::kXBytes;
  // the data gradient's edge rows (l2_dgrad_edge_slot), behind dyᵀ in both forms (past the end of the FC layout)
  static constexpr int kDxEdge = kDyT + Conv2Wg::kDyT;
  static constexpr int kDxEdgeBytes = 9 * 10 * 16 * 4;
  static constexpr int kTotalWg = 1024 + kDxEdge + kDxEdgeBytes;
  static_assert(Conv2Wg::kXBytes <= kFcW && kDxEdge >= kTotalFc - 1024 && kTotalWg == 230016 && kTotalWg <= 227 * 1024,
                "conv2 weight-gradient operand and data-gradient edge placement");
};

// conv2's data gradient with the filter columns in N.  D'[q][16·kw + ci] = Σ_{kh, co} dy[q + 18·kh][co] · Bd[5·kh + kw][ci][co] over
// patch rows q = 0..255 (four M = 64 tiles; q + 18·kh ≤ 327 stays inside the zeroed patch), then dx[p][ci] = Σ_kw D'[p + kw][16·kw + ci]
// with kw = 0, 1, 2, 3, 4 added in that order.  Warp w of the warpgroup holds 16-row range r = 4·tile + w of a tile's accumulators;
// row p + kw of its own rows comes from a lane of the same warp (shuffles), and the first four rows of range r + 1 (columns kw > row)
// from the edge buffer: slot l2_dgrad_edge_slot(r) holds range r's rows s = 0..3 at entry kw·(kw − 1)/2 + s, [10][16] floats.
// Tiles 2 and 3 run first, so range 8 is in the buffer when range 7 needs it.  Range r takes slot (r + 1) mod 9: the first pass
// (ranges 8..15) fills slots 0..7 and the second (ranges 0..7) slots 1..8, so it keeps range 8's slot 0 and overwrites only slots
// the first pass has finished reading.
__device__ __forceinline__ int l2_dgrad_edge_slot(int r) { return (r + 1) % 9; }

// Range r's edge rows from its accumulators a (row s = 16r + s is element half 0 of lanes 4s .. 4s + 3).
__device__ __forceinline__ void l2_dgrad_edge_store(const float (&a)[40], float* edge, int r, int lane) {
  const int s = lane >> 2, t4 = lane & 3;
  if (s >= 4) return;
  float* slot = edge + l2_dgrad_edge_slot(r) * 160;
#pragma unroll
  for (int kw = 1; kw < 5; ++kw)
    if (kw > s)
#pragma unroll
      for (int cg = 0; cg < 2; ++cg) {
        const int e = 4 * (2 * kw + cg);
        *reinterpret_cast<float2*>(slot + (kw * (kw - 1) / 2 + s) * 16 + 8 * cg + 2 * t4) = make_float2(a[e], a[e + 1]);
      }
}

// dx of range r (dxn = the image's [324][16] frame): the thread's output rows are p = 16r + g + 8·hh (g = lane / 4), its columns
// ci = 8·cg + 2·(lane mod 4) + b, as in the accumulator fragment.  Row p + kw sits in lane 4·((g + kw) mod 8) + lane mod 4, in the
// other accumulator half when g + kw wraps past 7 and in range r + 1 when it also wraps past the range (only the dropped rows
// p ≥ 248 of range 15 reach past row 255).
__device__ __forceinline__ void l2_dgrad_epilogue(const float (&a)[40], const float* edge, float* __restrict__ dxn, int r, int lane) {
  const int g = lane >> 2, t4 = lane & 3;
  float o[2][2][2];   // [hh][cg][b]
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int cg = 0; cg < 2; ++cg)
#pragma unroll
      for (int b = 0; b < 2; ++b) o[hh][cg][b] = a[4 * cg + 2 * hh + b];
  const float* next = edge + l2_dgrad_edge_slot(r + 1) * 160;
#pragma unroll
  for (int kw = 1; kw < 5; ++kw) {
    const int src = 4 * ((g + kw) & 7) + t4;
    const bool send_upper = g < kw;       // the row this lane sends to lane g − kw is in its upper half
    const bool take_next = g + kw >= 8;   // row p + kw of the upper half lies in range r + 1
#pragma unroll
    for (int cg = 0; cg < 2; ++cg)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int e = 4 * (2 * kw + cg) + b;
        const float lo = __shfl_sync(0xffffffffu, send_upper ? a[e + 2] : a[e], src);
        const float hi = __shfl_sync(0xffffffffu, a[e + 2], src);
        o[0][cg][b] += lo;
        o[1][cg][b] += !take_next ? hi : r < 15 ? next[(kw * (kw - 1) / 2 + g + kw - 8) * 16 + 8 * cg + 2 * t4 + b] : 0.f;
      }
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int p = 16 * r + g + 8 * hh, oh = p / kPW, ow = p - oh * kPW;
    if (oh < 14 && ow < 14)
#pragma unroll
      for (int cg = 0; cg < 2; ++cg)
        *reinterpret_cast<float2*>(dxn + ((oh + 2) * kPW + ow + 2) * 16 + 8 * cg + 2 * t4) = make_float2(o[hh][cg][0], o[hh][cg][1]);
  }
}

// The classifier's backward rides along: the gradient of the pooled activations is computed on the fly,
// d(out)[n][k] = Σ_j dlogits[n][j] · Wfc[j][k] (fc weights staged in smem once per CTA); the classifier's weight
// gradient dWfc[j][k] = Σ_n dlogits[n][j] · out[n][k] is produced in 16-column slices, one slice per CTA (all images, fixed
// order: deterministic, no partials), the bias gradient by the CTA that owns "slice 98".
// WG: conv2's weight-gradient partial of the image (Conv2Wg) is computed here on wgmma, issued by warpgroup 0 while warpgroup 1 issues
// the data gradient's: the x copies are written from conv2's input frame x2 in the shadow of the grid barrier, dyᵀ from the
// registers that write the dy patch.  The global dy frame is then not written: nothing reads it.
// WG = false writes the dy frame instead and no partials.  No training step runs it: it is the reference the tests feed to
// conv2_wgrad_partials_kernel, and the two together are the only bit-exact check of the K-major operand copies the WG form writes.
// ACC (accumulate mode, gradient accumulation over micro-batches, needs WG): every gradient this kernel writes — dfcw, dfcb, dgamma,
// dbeta — and the folded loss become g = g_old + v, one fp32 add, the rounding of autograd's accumulation of a temporary.
template <bool WG, bool ACC = false>
__global__ void __launch_bounds__(kL2Threads, 1)
convnet_l2_bwd_kernel(const float* __restrict__ y /*[B,14,14,32]*/,
                      const float* __restrict__ saved, const float* __restrict__ gamma, const float* __restrict__ beta,
                      const float* __restrict__ w, float* dgamma, float* dbeta, float* __restrict__ dy /*[B,18,18,32] zero-haloed frame*/,
                      float* __restrict__ dx /*[B,18,18,16] frame, interior written*/, float* __restrict__ dysum /*[B,32]*/,
                      float* partials, GridSync gs,
                      const float* __restrict__ dlogits /*[B,ncls]*/, const float* __restrict__ fcw /*[ncls,1568]*/,
                      const float* __restrict__ pooled /*[B,1568] = forward's out*/, float* dfcw /*[ncls,1568]*/, float* dfcb /*[ncls]*/,
                      int ncls, const float* __restrict__ loss_parts /*[B] or null*/, float* loss_out,
                      // WG only
                      const float* __restrict__ x2 /*[B,18,18,16] = conv2's input frame*/, float* __restrict__ wpart /*[B][400][32]*/) {
  static_assert(WG || !ACC, "accumulate mode is a variant of the kernel with conv2's weight gradient");
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
  float* s_fcw = misc + 1024;                                   // [ncls][1568]
  float* s_dl = s_fcw + L2BwdSmem::kFcW / 4;                    // [B][16] (columns >= ncls zero)
  float* s_pool = s_dl + L2BwdSmem::kFcDl / 4;                  // [B][16] slice of the pooled activations
  uint8_t* s_xt = smem + L2BwdSmem::kXT;                        // WG: conv2's x copies
  uint8_t* s_dyt = smem + L2BwdSmem::kDyT;                      // WG: conv2's dyᵀ
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = blockIdx.x, B = gridDim.x;

  griddep_wait();   // programmatic launch behind the forward: everything below reads its outputs or the grid-barrier words
  GridBar bar(gs);
  TRACE_INIT();
  const bool trace_wg1_ = (threadIdx.x == 128) && (*reinterpret_cast<volatile int*>(&g_trace_on) != 0);   // the data gradient's end
  trace(3, 0);
  // WG: the loads of conv2's x copies, written in the grid barrier's shadow (the forward kernel wrote x2)
  Conv2WgX<kL2Threads> xr;
  if constexpr (WG) xr.load(x2 + static_cast<size_t>(n) * Conv2Wg::kFrame * 16, tid);
  {
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
  cp_async_wait<0>();
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
      float best = -INFINITY, ya = 0.f;   // ya = y at the arg-max, so that no index into yv depends on data (no local memory)
#pragma unroll
      for (int d = 0; d < 4; ++d) {
        const int p = (2 * ph + (d >> 1)) * 14 + 2 * pw + (d & 1);
        yv[k][d] = y[(static_cast<size_t>(n) * 196 + p) * 32 + c];
        const float z = fmaf(yv[k][d], sc, sh);
        if (d == 0) ya = yv[k][0];
        if (z > best) { best = z; arg[k] = d; ya = yv[k][d]; }
      }
      // d(out) of this window from the classifier: Σ_j dlogits[n][j] · Wfc[j][c·49 + pp]
      const float* wk = s_fcw + c * 49 + pp;       // bank = (17·c + pp) mod 32: conflict-free across the warp's 32 channels
      const float* dl = s_dl + n * 16;
      float g0 = 0.f, g1 = 0.f;
#pragma unroll
      for (int j = 0; j < 16; j += 2) {            // independent smem loads (classes >= ncls: dlogits column is zero, weight not read)
        g0 = fmaf(dl[j], j < ncls ? wk[j * 1568] : 0.f, g0);
        g1 = fmaf(dl[j + 1], j + 1 < ncls ? wk[(j + 1) * 1568] : 0.f, g1);
      }
      const float go = g0 + g1;
      dzv[k] = best > 0.f ? go : 0.f;
      const float xh = (ya - mu) * is;
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
  // conv2's x copies, over the classifier weights (dead since the __syncthreads above)
  if constexpr (WG) xr.store(s_xt, tid);
  // zero halo of the global dy frame (the weight gradient sums over all 324 positions)
  if constexpr (!WG) {
    for (int i = tid; i < 324 * 8; i += kL2Threads) {
      const int P = i >> 3, pr = P / 18, pc = P - pr * 18;
      if (pr < 2 || pr >= 16 || pc < 2 || pc >= 16) reinterpret_cast<float4*>(dy + (static_cast<size_t>(n) * 324 + P) * 32)[i & 7] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  {
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
          float* dst = dfcw + static_cast<size_t>(j) * 1568 + slice * 16 + kl;
          if constexpr (ACC) *dst = *dst + ((a[0] + a[1]) + (a[2] + a[3]));
          else *dst = (a[0] + a[1]) + (a[2] + a[3]);
        }
      } else {
        if (dfcb != nullptr && tid < ncls) {
          float a = 0.f;
          for (int r = 0; r < B; ++r) a += s_dl[r * 16 + tid];
          if constexpr (ACC) dfcb[tid] = dfcb[tid] + a;
          else dfcb[tid] = a;
        }
        if (loss_parts != nullptr && warp == 7) {   // the forward kernel left one cross-entropy term per image and the number of
          const float counted = __ldg(loss_parts + B);   // counted images after them: batch mean, fixed order
          float sl = 0.f;
          for (int r = lane; r < B; r += 32) sl += __ldg(loss_parts + r);
#pragma unroll
          for (int off = 16; off >= 1; off >>= 1) sl += __shfl_xor_sync(0xffffffffu, sl, off);
          if constexpr (ACC) { if (lane == 0) *loss_out = *loss_out + sl / counted; }
          else if (lane == 0) *loss_out = sl / counted;
        }
      }
    }
  }
  bar.wait(gs);
  griddep_launch_dependents();   // the kernel's only grid barrier is behind it: the layer-1 backward's grid may be set up
  trace(3, 3);
  fold_rows<64>(partials, B, s_tmp, s_tot);
  trace(3, 4);
  if (n == 0 && tid < 32) {
    if constexpr (ACC) {
      if (dbeta) dbeta[tid] = dbeta[tid] + s_tot[tid];
      if (dgamma) dgamma[tid] = dgamma[tid] + s_tot[32 + tid];
    } else {
      if (dbeta) dbeta[tid] = s_tot[tid];
      if (dgamma) dgamma[tid] = s_tot[32 + tid];
    }
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
          if constexpr (!WG) dy[(static_cast<size_t>(n) * 324 + P) * 32 + c] = v;  // frame for the weight-gradient kernel (TMA)
          else *reinterpret_cast<float*>(s_dyt + conv2_dyt_off(c, P - Conv2Wg::kFirst)) = tf32_round(v);   // conv2's dyᵀ
          *reinterpret_cast<float*>(sa + sw128_off(P, c >> 2) + (c & 3) * 4) = v;   // same frame in smem for the data-gradient MMAs
          dsum += v;
        }
      }
    }
    s_part[g * 64 + c] = dsum;
    if constexpr (WG) {
      // the 60 halo positions of dyᵀ's window: P = 18·pr + 16 .. 18·pr + 19 for pr = 2..14, then 286..293
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int h = g + 8 * k;
        if (h < 60) *reinterpret_cast<float*>(s_dyt + conv2_dyt_off(c, (h < 52 ? 18 * (2 + (h >> 2)) + 16 + (h & 3) : 286 + h - 52) - Conv2Wg::kFirst)) = 0.f;
      }
    }
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
  // ---- conv2 data gradient: 80 wgmma m64n80k8 by the warpgroup of warps 4..7, two M tiles at a time (l2_dgrad_epilogue); next to
  // it (WG) conv2's weight-gradient partial, 320 wgmma m64n32k8 by warps 0..3 -------------------------------------------------------
  const int wg = warpgroup_index();
  if constexpr (WG) {
    if (wg == 0) {
      conv2_wgrad_wgmma(smem_u32(s_xt), smem_u32(s_dyt), wpart + static_cast<size_t>(n) * 400 * 32, tid);
      trace(3, 7);
    }
  }
  if (wg == 1) {
    const int wq = warp - 4;
    float* edge = reinterpret_cast<float*>(smem + L2BwdSmem::kDxEdge);
    float* dxn = dx + static_cast<size_t>(n) * 324 * 16;
    const uint64_t ad0 = gmma_desc_kmajor<128>(smem_u32(sa)), bd0 = gmma_desc_kmajor<128>(smem_u32(sb));
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
      const int t0 = 2 - 2 * pass;   // tiles 2, 3, then 0, 1
      float acc[2][40];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 40; ++e) acc[h][e] = 0.f;
      wgmma_fence();
#pragma unroll 1
      for (int kh = 0; kh < 5; ++kh) {
        // A: the patch from row 64·t0 + 18·kh; B: the 80 rows (kw, ci) of taps 5·kh .. 5·kh + 4, one 1024-byte-aligned block
        const uint64_t ad = ad0 + static_cast<uint64_t>(((64 * t0 + kh * kPW) * 128) >> 4);
        const uint64_t bd = bd0 + static_cast<uint64_t>((kh * 5 * 2048) >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k)   // K = 32 output channels = four K=8 steps
#pragma unroll
          for (int h = 0; h < 2; ++h) wgmma_m64n80k8_tf32(acc[h], ad + ((h * 64 * 128 + k * 32) >> 4), bd + ((k * 32) >> 4), (kh | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (pass == 1) asm volatile("bar.sync 1, 128;" ::: "memory");   // the first pass has read its edge slots
#pragma unroll
      for (int h = 0; h < 2; ++h) l2_dgrad_edge_store(acc[h], edge, 4 * (t0 + h) + wq, lane);
      asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
      for (int h = 0; h < 2; ++h) l2_dgrad_epilogue(acc[h], edge, dxn, 4 * (t0 + h) + wq, lane);
    }
    trace_stamp(trace_wg1_, 3, 8);
  }
  __syncthreads();
  bar.finish(gs);
  trace(3, 6);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------

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

void launch_conv2_wgrad_partials(const float* dy2_pad, const float* x2_pad, int B, float* wpart, cudaStream_t st) {
  opt_in_smem(conv2_wgrad_partials_kernel, kConv2WgSmem);
  conv2_wgrad_partials_kernel<<<B, 128, kConv2WgSmem, st>>>(dy2_pad, x2_pad, wpart);
  check_launch("conv2_wgrad_partials");
}

template <class Rider>
void launch_convnet_l1_bwd_wgrad(const float* dp, const float* y, const float* w1, const float* b1, const float* x, const float* saved,
                                 const float* gamma, const float* beta, float* dgamma, float* dbeta, float* dw, float* db, const float* wpart,
                                 const float* dysum2, float* dw2, float* db2, int B, float* partials, float* partials_w, GridSync gs, cudaStream_t st,
                                 Rider rider, bool accumulate) {
  auto kernel = accumulate ? convnet_l1_bwd_kernel<Rider, true> : convnet_l1_bwd_kernel<Rider>;
  launch_cooperative(kernel, B, kL1Threads, static_cast<size_t>(kL1BwdSmem), st, "convnet_l1_bwd_wgrad", true, dp, y, w1, b1, x, saved,
                     gamma, beta, dgamma, dbeta, dw, db, partials, partials_w, gs, wpart, dysum2, dw2, db2, rider);
}
#define PDT_L1_BWD_WGRAD(R)                                                                                                            \
  template void launch_convnet_l1_bwd_wgrad<R>(const float*, const float*, const float*, const float*, const float*, const float*,       \
                                               const float*, const float*, float*, float*, float*, float*, const float*, const float*, float*, \
                                               float*, int, float*, float*, GridSync, cudaStream_t, R, bool);
PDT_L1_BWD_WGRAD(SgdRider)
PDT_L1_BWD_WGRAD(AdamRider)
PDT_L1_BWD_WGRAD(ClipRider<SgdRider>)
PDT_L1_BWD_WGRAD(ClipRider<AdamRider>)
PDT_L1_BWD_WGRAD(AmsgradRider)
PDT_L1_BWD_WGRAD(ClipRider<AmsgradRider>)
PDT_L1_BWD_WGRAD(RmspropRider)
PDT_L1_BWD_WGRAD(ClipRider<RmspropRider>)
PDT_L1_BWD_WGRAD(AdagradRider)
PDT_L1_BWD_WGRAD(ClipRider<AdagradRider>)
#undef PDT_L1_BWD_WGRAD

void launch_convnet_fwd(const float* x, const float* w1, const float* b1, const float* g1, const float* be1, float* y1, float* p1, float* saved1,
                        float* rm1, float* rv1, long long* nbt1, float mom1, float eps1, const float* w2, const float* b2, const float* g2,
                        const float* be2, float* y2, float* out, float* saved2, float* rm2, float* rv2, long long* nbt2, float mom2, float eps2,
                        const float* fcw, const float* fcb, float* logits, int ncls, int B, float* partials, GridSync gs, cudaStream_t st,
                        SoftCe ce) {
  if (logits != nullptr && ncls > 16) throw std::invalid_argument("convnet_fwd: the fused classifier handles at most 16 classes");
  if ((ce.target != nullptr || ce.target_probs != nullptr) && logits == nullptr)
    throw std::invalid_argument("convnet_fwd: the fused cross-entropy needs the fused classifier");
  if (ce.target != nullptr && ce.target_probs != nullptr)
    throw std::invalid_argument("convnet_fwd: class-index and class-probability targets are exclusive");
  if (!(ce.scale > 0.f)) throw std::invalid_argument("convnet_fwd: the cross-entropy scale must be positive");
  if (!(ce.smoothing >= 0.f && ce.smoothing <= 1.f)) throw std::invalid_argument("convnet_fwd: label smoothing must lie in [0, 1]");
  if (ce.target_probs != nullptr) {
    launch_cooperative(convnet_fwd_kernel<SoftCe>, B, kFwdThreads, static_cast<size_t>(L2FwdSmem::kTotal), st, "convnet_fwd", false, x, w1, b1, g1, be1, y1, p1,
                       saved1, rm1, rv1, nbt1, mom1, eps1, w2, b2, g2, be2, y2, out, saved2, rm2, rv2, nbt2, mom2, eps2, fcw, fcb, logits, ncls, partials,
                       gs, ce);
    return;
  }
  if (ce.target != nullptr && !ce.is_default(ncls)) {
    launch_cooperative(convnet_fwd_kernel<SmoothCe>, B, kFwdThreads, static_cast<size_t>(L2FwdSmem::kTotal), st, "convnet_fwd", false, x, w1, b1, g1, be1, y1, p1,
                       saved1, rm1, rv1, nbt1, mom1, eps1, w2, b2, g2, be2, y2, out, saved2, rm2, rv2, nbt2, mom2, eps2, fcw, fcb, logits, ncls, partials,
                       gs, static_cast<const SmoothCe&>(ce));
    return;
  }
  if (ce.target != nullptr && ce.scale != 1.f) {
    launch_cooperative(convnet_fwd_kernel<ScaledCe>, B, kFwdThreads, static_cast<size_t>(L2FwdSmem::kTotal), st, "convnet_fwd", false, x, w1, b1, g1, be1, y1, p1,
                       saved1, rm1, rv1, nbt1, mom1, eps1, w2, b2, g2, be2, y2, out, saved2, rm2, rv2, nbt2, mom2, eps2, fcw, fcb, logits, ncls, partials,
                       gs, static_cast<const ScaledCe&>(ce));
    return;
  }
  launch_cooperative(convnet_fwd_kernel<FusedCe>, B, kFwdThreads, static_cast<size_t>(L2FwdSmem::kTotal), st, "convnet_fwd", false, x, w1, b1, g1, be1, y1, p1, saved1,
                     rm1, rv1, nbt1, mom1, eps1, w2, b2, g2, be2, y2, out, saved2, rm2, rv2, nbt2, mom2, eps2, fcw, fcb, logits, ncls, partials, gs,
                     static_cast<const FusedCe&>(ce));
}

void launch_convnet_l2_bwd_fc(const float* dlogits, const float* fcw, const float* pooled, float* dfcw, float* dfcb, int ncls, const float* y,
                              const float* saved, const float* gamma, const float* beta, const float* w, float* dgamma, float* dbeta, float* dy,
                              float* dx, float* dysum, int B, float* partials, GridSync gs, cudaStream_t st, const float* loss_parts, float* loss_out,
                              const float* x2, float* wpart, bool accumulate) {
  if (ncls < 1 || ncls > 16) throw std::invalid_argument("convnet_l2_bwd_fc: 1..16 classes");
  if (B > 160) throw std::invalid_argument("convnet_l2_bwd_fc: batch too large for the staged dlogits");
  if (accumulate && x2 == nullptr) throw std::invalid_argument("convnet_l2_bwd_fc: accumulate mode needs conv2's input frame (x2)");
  auto kernel = accumulate ? convnet_l2_bwd_kernel<true, true> : x2 != nullptr ? convnet_l2_bwd_kernel<true> : convnet_l2_bwd_kernel<false>;
  const int smem = std::max(L2BwdSmem::kTotalFc, L2BwdSmem::kTotalWg);   // every form has the data gradient's edge buffer
  launch_cooperative(kernel, B, kL2Threads, static_cast<size_t>(smem), st, "convnet_l2_bwd_fc", true, y, saved, gamma, beta, w, dgamma, dbeta, dy,
                     dx, dysum, partials, gs, dlogits, fcw, pooled, dfcw, dfcb, ncls, loss_parts, loss_out, x2, wpart);
}

}  // namespace pdt
