// wgmma / TMA kernels for sm_90a (hand-written PTX; no CUTLASS): the per-op 5x5 convolution of the ConvNet's conv2
// (16→32 channels, 88% of the model's FLOPs; ref: ddp_example.py:30).
//
//  * conv5x5_wgmma_im2col_kernel — forward and data gradient as an implicit GEMM: M = output pixels (128 per tile),
//    N = output channels, K = 25 taps × input channels.  The im2col A-tile of every filter tap is one
//    cp.async.bulk.tensor im2col load (the TMA unit zero-fills the padding halo), the repacked weights (B) are TMA-loaded
//    once per CTA and stay resident in smem, and one warpgroup issues wgmma.mma_async ... .tf32 with the fp32 accumulator
//    in its registers.  The forward epilogue adds the bias, folds the per-channel statistics BatchNorm needs (saving a
//    full re-read of y) and writes the tile with a TMA store.
//  * conv5x5_wgrad_mma_kernel — weight and bias gradient: persistent split-K over pixel tiles on warp-level mma.sync (both
//    operands are MN-major, which TF32 wgmma does not accept); wgrad_fold_kernel then sums the per-CTA partials in a fixed
//    order.
// TF32 inputs / fp32 accumulate is the same numerics contract the reference gets from cuDNN (torch allows TF32 in
// convolutions by default).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>

#include "conv_wgmma.h"
#include "hopper_ptx.cuh"
#include "wgrad_win.cuh"
#include "cuda_utils.h"
#include "grid_fold.cuh"

namespace pdt {

namespace {

using namespace ptx;

constexpr int kTileM = 128;

// =====================================================================================================
// Implicit-GEMM 5x5 convolution, fully TMA-fed: the im2col A-tile of every filter tap is ONE
// cp.async.bulk.tensor.4d...im2col instruction (hardware walks 128 consecutive output pixels through
// W→H→N, applies the (kw,kh) tap offset and zero-fills the padding halo), so there are no producer
// warps at all: warp 4 = TMA, warps 0-3 = the warpgroup that issues the wgmma (two M = 64 halves of the
// 128-pixel tile) and runs the epilogue from its register accumulators.
//   CK = 16 (fwd):  rows of 64 B  → SWIZZLE_64B smem/wgmma layout, 2 K=8 steps per tap
//   CK = 32 (dgrad): rows of 128 B → SWIZZLE_128B,                4 K=8 steps per tap
// Weights: Bm[NOUT][25·CK] (K index = tap·CK + c), one TMA box per tap, resident in smem.
// =====================================================================================================
__device__ __forceinline__ void tma_load_im2col_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c, int w, int h, int n,
                                                   uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

template <int CK, int NOUT>
struct ConvTmaCfg {
  static constexpr int kRowB = CK * 4;                       // bytes per pixel per tap
  static constexpr int kATapBytes = kTileM * kRowB;          // 8 KB / 16 KB
  // One pipeline stage = one filter ROW (5 taps, 5 TMA loads on one mbarrier): the per-stage
  // handshake (TMA issue → full → MMA → empty) costs the same whatever the payload, so a stage
  // carries five taps rather than one.
  static constexpr int kTapsPerStage = 5;
  static constexpr int kAStageBytes = kTapsPerStage * kATapBytes;   // 40 KB / 80 KB
  static constexpr int kStages = CK == 16 ? 3 : 2;
  static constexpr int kBTapBytes = NOUT * kRowB;            // 2 KB
  static constexpr int kSyBytes = CK == 16 ? kTileM * 128 : 0;  // output staging only for the TMA-stored forward
  static constexpr int kAccBytes = kTileM * (NOUT + 1) * 4;  // accumulator rows, one per epilogue thread
  static constexpr int kThreads = 160;
  static constexpr size_t kSmem = 2048 + kStages * kAStageBytes + 25 * kBTapBytes + kSyBytes + kAccBytes + 2048;
};

template <int CK, int NOUT, bool FWD>
__global__ void __launch_bounds__(160, 1) conv5x5_wgmma_im2col_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_b,
                                                                  const __grid_constant__ CUtensorMap tm_y, const float* __restrict__ bias,
                                                                  float* __restrict__ y, float* stats, int centred, ReduceScratch scr, int B,
                                                                  int H, int W, int num_tiles) {
  using Cfg = ConvTmaCfg<CK, NOUT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;
  uint8_t* sb = sa + Cfg::kStages * Cfg::kAStageBytes;
  uint8_t* sy = sb + 25 * Cfg::kBTapBytes;
  sy = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sy) + 1023) & ~uintptr_t(1023));
  float* sacc = reinterpret_cast<float*>(sy + Cfg::kSyBytes);   // [128][NOUT + 1]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sacc + kTileM * (NOUT + 1));
  uint64_t* full = bars;
  uint64_t* empty = full + Cfg::kStages;
  uint64_t* b_full = empty + Cfg::kStages;
  float* s_part = reinterpret_cast<float*>(b_full + 2);   // [4][2*NOUT] + [2*NOUT]
  __shared__ int s_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int M = B * H * W;
  if (tid == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_b);
    if (FWD) tma_prefetch_desc(&tm_y);
    for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 128); }
    mbar_init(b_full, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      mbar_arrive_expect_tx(b_full, 25 * Cfg::kBTapBytes);
      for (int t = 0; t < 25; ++t) tma_load_2d(sb + t * Cfg::kBTapBytes, &tm_b, b_full, t * CK, 0);
      int g = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int p0 = tile * kTileM;
        const int ow0 = p0 % W, oh0 = (p0 / W) % H, n0 = p0 / (W * H);
        for (int kh = 0; kh < 5; ++kh, ++g) {
          const int s = g % Cfg::kStages;
          mbar_wait(&empty[s], ((g / Cfg::kStages) & 1) ^ 1);
          mbar_arrive_expect_tx(&full[s], Cfg::kAStageBytes);
          // base pixel = output pixel shifted by the lower corner (-pad); the tap goes in the offsets
#pragma unroll
          for (int kw = 0; kw < 5; ++kw)
            tma_load_im2col_4d(sa + s * Cfg::kAStageBytes + kw * Cfg::kATapBytes, &tm_x, &full[s], 0, ow0 - 2, oh0 - 2, n0,
                               static_cast<uint16_t>(kw), static_cast<uint16_t>(kh));
        }
      }
    }
  } else {
    // ---- warps 0..3: wgmma issue + epilogue, thread = tile row -----------------------------------------------
    const int et = tid, r = tid;
    mbar_wait(b_full, 0);
    int g = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      float acc[2][NOUT / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < NOUT / 2; ++e) acc[h][e] = 0.f;
      for (int kh = 0; kh < 5; ++kh, ++g) {
        const int s = g % Cfg::kStages;
        mbar_wait(&full[s], (g / Cfg::kStages) & 1);
        const uint32_t a0 = smem_u32(sa + s * Cfg::kAStageBytes), b0 = smem_u32(sb + kh * 5 * Cfg::kBTapBytes);
        wgmma_fence();
#pragma unroll
        for (int kw = 0; kw < 5; ++kw)
#pragma unroll
          for (int k = 0; k < CK / 8; ++k)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              wgmma_tf32<NOUT>(acc[h], gmma_desc_kmajor<Cfg::kRowB>(a0 + kw * Cfg::kATapBytes + h * 64 * Cfg::kRowB + k * 32),
                               gmma_desc_kmajor<Cfg::kRowB>(b0 + kw * Cfg::kBTapBytes + k * 32), (kh | kw | k) != 0);
        wgmma_commit();
        wgmma_wait<0>();
        mbar_arrive(&empty[s]);                 // this thread's share of the stage has been read
      }
      asm volatile("bar.sync 1, 128;" ::: "memory");   // the previous tile's rows have been read out of sacc
#pragma unroll
      for (int h = 0; h < 2; ++h) wgmma_frag_store<NOUT>(acc[h], sacc, NOUT + 1, 64 * h, tid);
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float v[NOUT];
#pragma unroll
      for (int j = 0; j < NOUT; ++j) v[j] = sacc[r * (NOUT + 1) + j];
      const int p = tile * kTileM + r;
      const bool valid = p < M;
      if (bias) {
#pragma unroll
        for (int j = 0; j < NOUT; ++j) v[j] += bias[j];
      }
      if constexpr (FWD) {
        asm volatile("bar.sync 1, 128;" ::: "memory");  // previous tile's TMA store has finished reading sy
#pragma unroll
        for (int q = 0; q < NOUT / 4; ++q) {
          float4 o = valid ? make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<float4*>(sy + r * 128 + ((q ^ (r & 7)) << 4)) = o;
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (et == 0) {
          tma_store_2d(&tm_y, sy, 0, tile * kTileM);
          tma_store_commit();
        }
        if (stats) {
          // the tile's per-channel sums of d = y − K and d² over its valid rows (rows past M are zeros in sy); lane = channel.
          // K = 0 gives Σy and Σy².  Centred, K is the tile's first row, and the tile's M2 = Σd² − (Σd)²/n then cancels only in
          // proportion to ((mean − K)/std)², a property of the data's spread rather than of the size of its mean
          const int q = lane >> 2, e = lane & 3;
          const int w4 = et >> 5;  // 0..3: rows 32*w4 .. 32*w4+31
          const int nvalid = min(kTileM, M - tile * kTileM);
          const float K = centred ? reinterpret_cast<const float*>(sy + (q << 4))[e] : 0.f;
          float s1 = 0.f, s2 = 0.f;
          for (int rr = w4 * 32; rr < w4 * 32 + 32; ++rr) {
            const float val = reinterpret_cast<const float*>(sy + rr * 128 + ((q ^ (rr & 7)) << 4))[e];
            const float d = rr < nvalid ? val - K : 0.f;
            s1 += d;
            s2 += d * d;
          }
          s_part[w4 * 2 * NOUT + lane] = s1;
          s_part[w4 * 2 * NOUT + NOUT + lane] = s2;
          asm volatile("bar.sync 1, 128;" ::: "memory");
          float* tile_sums = s_part + 8 * NOUT;
          if (et < 2 * NOUT) tile_sums[et] = s_part[et] + s_part[2 * NOUT + et] + s_part[4 * NOUT + et] + s_part[6 * NOUT + et];
          asm volatile("bar.sync 1, 128;" ::: "memory");
          if (centred) {
            if (et < NOUT) {   // [Σd, Σd²] → [Σy, M2] (thread et < 32 holds channel et's K)
              const float sd = tile_sums[et], n = static_cast<float>(nvalid);
              tile_sums[NOUT + et] = fmaxf(tile_sums[NOUT + et] - sd * sd / n, 0.f);
              tile_sums[et] = fmaf(n, K, sd);
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");
            grid_fold_centred(tile_sums, NOUT, kTileM, M, tile, num_tiles, scr, s_part, &s_last, et, 128, NamedSync<1, 128>{},
                              [&](int i, float mean, float m2) {
                                stats[i] = mean;
                                stats[NOUT + i] = m2;
                                if (i == 0) stats[2 * NOUT] = static_cast<float>(M);
                              });
          } else {
            grid_fold(tile_sums, 2 * NOUT, tile, num_tiles, scr, s_part, &s_last, et, 128, NamedSync<1, 128>{}, [&](int i, float tot) {
              stats[i] = tot;
              if (i == 0) stats[2 * NOUT] = static_cast<float>(M);
            });
          }
        }
        if (et == 0) tma_store_wait_read();
      } else {
        if (valid) {
          float* o = y + static_cast<size_t>(p) * NOUT;
#pragma unroll
          for (int q = 0; q < NOUT / 4; ++q) *reinterpret_cast<float4*>(o + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
        }
      }
    }
  }
}

// Weight repack for the implicit GEMM: Bm[NOUT][25*CK], K index = tap*CK + c (the kernel loads one [NOUT][CK] box per tap)
//   FWD  : Bm[co][tap*16+ci] = w[co][ci][tap]
//   DGRAD: Bm[ci][tap*32+co] = w[co][ci][24-tap]
template <bool FWD>
__global__ void repack_weights_dense_kernel(const float* __restrict__ w, float* __restrict__ bm, int Cout, int Cin) {
  const int CK = FWD ? Cin : Cout, NOUT = FWD ? Cout : Cin;
  const int kk = 25 * CK;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NOUT * kk) return;
  const int n = i / kk, k = i % kk, tap = k / CK, c = k % CK;
  bm[i] = FWD ? w[(n * Cin + c) * 25 + tap] : w[(c * Cin + n) * 25 + (24 - tap)];
}

// =====================================================================================================
// conv2 weight gradient on the tensor cores:   dWᵀ[m = tap·16+ci][co] = Σ_pixels xcol[p][m] · dy[p][co]
//
// The reduction runs over output pixels, i.e. over the *slow* dimension of both operands (MN-major):
//   A = im2col(x)   [64 pixels][128 of the 416 im2col columns]   gathered by cp.async (zero fill), 16-byte units XOR-swizzled
//   B = dy tile     [128 pixels][32 channels]                    one TMA box per tile, SWIZZLE_128B
// M = 416 is covered by four 128-row accumulators living in registers for the CTA's whole lifetime
// (persistent split-K over pixel tiles); column 400 of the im2col is a column of ones, so the
// bias gradient Σ_p dy[p][co] falls out of the same MMAs.  Each CTA deposits one partial
// [416][32]; wgrad_fold_kernel sums the ≤ #SM partials in CTA order (deterministic) and scatters
// into torch's [co][ci][5][5] layout.
// =====================================================================================================
struct WgradCfg {
  static constexpr int kMUsed = 416;                  // 25 taps × 16 ch, + ones column (400), + pad
  static constexpr int kMTiles = 4;
  static constexpr int kHalfPix = 64;                 // pixels per A stage
  static constexpr int kStages = 4, kLag = 1;
  static constexpr int kAStageBytes = kHalfPix * 512; // [64 pixels][128 im2col columns], 16-byte units XOR-swizzled
  static constexpr int kBStages = 2, kBStageBytes = kTileM * 128;
  static constexpr int kThreads = 160;
  static constexpr size_t kSmem = 1024 + kStages * kAStageBytes + kBStages * kBStageBytes + 1024;
};

// Both GEMM operands have the pixels (the reduction dimension) outermost — MN-major — which TF32 wgmma does not
// accept, so the four producer warps also run the MMAs, warp-level mma.sync m16n8k8 (wgrad_win.cuh): warp w owns
// rows 32w .. 32w+31 of every 128-row M tile, and all four M tiles stay in registers across the CTA's pixel tiles.
__global__ void __launch_bounds__(160, 1) conv5x5_wgrad_mma_kernel(const float* __restrict__ x, const __grid_constant__ CUtensorMap tm_dy,
                                                                    const float* __restrict__ ones, float* __restrict__ partials, int B,
                                                                    int H, int W, int num_tiles) {
  using Cfg = WgradCfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;
  uint8_t* sb = sa + Cfg::kStages * Cfg::kAStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sb + Cfg::kBStages * Cfg::kBStageBytes);
  uint64_t* bfull = bars;
  uint64_t* bempty = bfull + Cfg::kBStages;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int M = B * H * W;
  if (tid == 0) {
    tma_prefetch_desc(&tm_dy);
    for (int s = 0; s < Cfg::kBStages; ++s) { mbar_init(&bfull[s], 1); mbar_init(&bempty[s], 128); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const int s = it % Cfg::kBStages;
        mbar_wait(&bempty[s], ((it / Cfg::kBStages) & 1) ^ 1);
        mbar_arrive_expect_tx(&bfull[s], Cfg::kBStageBytes);
        tma_load_2d(sb + s * Cfg::kBStageBytes, &tm_dy, &bfull[s], 0, tile * kTileM);   // rows ≥ M arrive as zeros
      }
    }
    return;
  }
  // ---- warps 0-3: im2col gather (64 pixels × 128 columns per stage), then the MMAs of the stage kLag behind --------
  float acc[Cfg::kMTiles][2][4][4];
#pragma unroll
  for (int mt = 0; mt < Cfg::kMTiles; ++mt)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[mt][j][nt][e] = 0.f;
  // stage q (the q-th of the CTA) holds M tile (q / 2) % 4, pixel half q % 2 of the CTA's tile q / 8
  auto mma_stage = [&](int q) {
    const int mt = (q >> 1) & 3, h = q & 1, it = q >> 3, bs = it % Cfg::kBStages;
    mbar_wait(&bfull[bs], (it / Cfg::kBStages) & 1);
    const float* xs = reinterpret_cast<const float*>(sa + (q % Cfg::kStages) * Cfg::kAStageBytes);
    const float* dys = reinterpret_cast<const float*>(sb + bs * Cfg::kBStageBytes);
#pragma unroll
    for (int m = 0; m < Cfg::kMTiles; ++m)
      if (m == mt) wgrad_win_atom<Cfg::kHalfPix, 128>(acc[m], xs, 0, warp * 32, dys, h * Cfg::kHalfPix, lane);
    if (mt == Cfg::kMTiles - 1 && h == 1) mbar_arrive(&bempty[bs]);   // the last stage of this pixel tile has read dy
  };
  const int u = tid & 31;                 // 16-byte unit inside the 128-column row: tap_local = u/4, channels 4(u%4)..
  const int tap_local = u >> 2, c4 = (u & 3) * 4;
  const int t4 = tid >> 5;                // this thread fills pixel rows t4 + 4j of a stage
  int g = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    for (int mt = 0; mt < Cfg::kMTiles; ++mt) {
      const int tap = mt * 8 + tap_local;
      const int kh = tap / 5 - 2, kw = tap % 5 - 2;
      for (int h = 0; h < 2; ++h, ++g) {
        const int s = g % Cfg::kStages;
        const uint32_t dst0 = smem_u32(sa + s * Cfg::kAStageBytes) + t4 * 512;   // row t4 + 4j, unit u stored at u ^ (row % 8)
        int p = tile * kTileM + h * Cfg::kHalfPix + t4;
        int ow = p % W, oh = (p / W) % H;               // NHWC: pixel p lives at x + 16 p, so only bounds need (oh, ow)
        const int tap_delta = (kh * W + kw) * 16 + c4;
#pragma unroll 4
        for (int j = 0; j < 16; ++j) {
          const float* src = x;
          uint32_t bytes = 0;
          if (p < M) {
            if (tap < 25) {
              const int ih = oh + kh, iw = ow + kw;
              if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
                src = x + static_cast<size_t>(p) * 16 + tap_delta;
                bytes = 16;
              }
            } else if (tap == 25 && c4 == 0) {
              src = ones;  // {1,0,0,0}: im2col column 400 ≡ 1 → row 400 of dWᵀ is the bias gradient
              bytes = 16;
            }
          }
          cp_async_16(dst0 + j * 2048 + ((u ^ (t4 | ((j & 1) << 2))) << 4), src, bytes);
          p += 4;
          ow += 4;
          if (ow >= W) { ow -= W; oh = (oh + 1 == H) ? 0 : oh + 1; }
        }
        cp_async_commit();
        if (g >= Cfg::kLag) {
          cp_async_wait<Cfg::kLag>();
          asm volatile("bar.sync 1, 128;" ::: "memory");   // stage g - kLag has landed for every producer thread
          mma_stage(g - Cfg::kLag);
        }
      }
    }
  }
  cp_async_wait<0>();
  asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
  for (int q = Cfg::kLag; q >= 1; --q)
    if (g - q >= 0) mma_stage(g - q);
  // ---- this CTA's partial [416][32] ------------------------------------------------------------------------------
#pragma unroll
  for (int mt = 0; mt < Cfg::kMTiles; ++mt) {
    const int m0 = mt * kTileM + warp * 32;
    if (m0 < Cfg::kMUsed) wgrad_win_atom_store(acc[mt], partials + (static_cast<size_t>(blockIdx.x) * Cfg::kMUsed + m0) * 32, lane, Cfg::kMUsed - m0);
  }
}

// dw[co][ci][tap] = Σ_cta partial[cta][tap*16+ci][co];  db[co] = Σ_cta partial[cta][400][co]
__global__ void __launch_bounds__(256) wgrad_fold_kernel(const float* __restrict__ partials, int nparts, float* __restrict__ dw,
                                                         float* __restrict__ db) {
  // one CTA per im2col row m (401 of them): lane = output channel, the 8 warps stride over the
  // per-CTA partials (≤ 132/8 = 17 loads each on an H100, two in flight), sub-sums folded in warp order
  __shared__ float s_sub[8][32];
  const int m = blockIdx.x, co = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* p = partials + static_cast<size_t>(m) * 32 + co;
  const size_t stride = static_cast<size_t>(WgradCfg::kMUsed) * 32;
  float s0 = 0.f, s1 = 0.f;
  int c = warp;
  for (; c + 8 < nparts; c += 16) {
    s0 += p[c * stride];
    s1 += p[(c + 8) * stride];
  }
  if (c < nparts) s0 += p[c * stride];
  s_sub[warp][co] = s0 + s1;
  __syncthreads();
  if (warp == 0) {
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) s += s_sub[w8][co];
    if (m < 400) dw[(co * 16 + (m & 15)) * 25 + (m >> 4)] = s;
    else if (db) db[co] = s;
  }
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
CUtensorMap make_tmap_2d(const float* base, uint64_t inner, uint64_t outer, uint32_t box_inner, uint32_t box_outer,
                         CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  CUtensorMap m;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {inner * sizeof(float)};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = driver().cuTensorMapEncodeTiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed: " + cu_error(r));
  return m;
}

// NHWC activation [N,H,W,C] as a rank-4 im2col tensor map for a 5x5 / pad 2 / stride 1 window:
// bounding box lower corner = -pad, upper corner = pad - (filter - 1); 128 pixels × C channels per load.
CUtensorMap make_tmap_im2col(const float* base, int C, int W, int H, int N, CUtensorMapSwizzle swizzle) {
  const DriverApi& d = driver();
  if (!d.cuTensorMapEncodeIm2col) throw std::runtime_error("cuTensorMapEncodeIm2col is not available in this driver");
  CUtensorMap m;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * 4, static_cast<cuuint64_t>(W) * C * 4, static_cast<cuuint64_t>(H) * W * C * 4};
  int lower[2] = {-2, -2}, upper[2] = {-2, -2};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = d.cuTensorMapEncodeIm2col(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, lower, upper,
                                         static_cast<cuuint32_t>(C), static_cast<cuuint32_t>(kTileM), estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeIm2col failed: " + cu_error(r));
  return m;
}

// device buffers, one per (device, slot): 0 = forward weights, 1 = data-gradient weights, 2 = the weight gradient's ones
// column; allocated on first use (outside graph capture)
float* repack_buffer(int slot_id, size_t floats) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, std::pair<float*, size_t>> bufs;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> g(mu);
  auto& slot = bufs[{dev, slot_id}];
  if (slot.second < floats) {
    if (slot.first) cudaFree(slot.first);
    cudaError_t e = cudaMalloc(&slot.first, floats * sizeof(float));
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaMalloc(repack buffer): ") + cudaGetErrorString(e));
    slot.second = floats;
  }
  return slot.first;
}

}  // namespace

bool conv_wgmma_supported(const ConvShape& s) { return s.Cin == 16 && s.Cout == 32; }

void launch_conv5x5_fwd_im2col(const float* x, const float* w, const float* bias, float* y, float* stats, bool centred, ConvShape s,
                               ReduceScratch scr, cudaStream_t st) {
  if (!conv_wgmma_supported(s)) throw std::invalid_argument("conv5x5 im2col: only 16→32 channels are implemented");
  using Cfg = ConvTmaCfg<16, 32>;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  if (stats && (static_cast<long long>(tiles + tiles / kFoldGroup + 1) * 64 > scr.capacity_floats || tiles / kFoldGroup + 2 > scr.fold_counters))
    throw std::invalid_argument("conv5x5 im2col: scratch too small");
  float* bm = repack_buffer(0, static_cast<size_t>(32) * 400);
  repack_weights_dense_kernel<true><<<(32 * 400 + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights_dense(fwd)");
  CUtensorMap tm_x = make_tmap_im2col(x, 16, s.W, s.H, s.B, CU_TENSOR_MAP_SWIZZLE_64B);
  CUtensorMap tm_b = make_tmap_2d(bm, 400, 32, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B);
  CUtensorMap tm_y = make_tmap_2d(y, 32, static_cast<uint64_t>(M), 32, kTileM);
  auto kern = conv5x5_wgmma_im2col_kernel<16, 32, true>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_b, tm_y, bias, y, stats, centred ? 1 : 0, scr, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_wgmma_im2col(fwd)");
}

void launch_conv5x5_dgrad_im2col(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st) {
  if (!conv_wgmma_supported(s)) throw std::invalid_argument("conv5x5 im2col dgrad: only 16→32 channels are implemented");
  using Cfg = ConvTmaCfg<32, 16>;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  float* bm = repack_buffer(1, static_cast<size_t>(16) * 800);
  repack_weights_dense_kernel<false><<<(16 * 800 + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights_dense(dgrad)");
  CUtensorMap tm_x = make_tmap_im2col(dy, 32, s.W, s.H, s.B, CU_TENSOR_MAP_SWIZZLE_128B);
  CUtensorMap tm_b = make_tmap_2d(bm, 800, 16, 32, 16, CU_TENSOR_MAP_SWIZZLE_128B);
  auto kern = conv5x5_wgmma_im2col_kernel<32, 16, false>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_b, tm_b, nullptr, dx, nullptr, 0, ReduceScratch{}, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_wgmma_im2col(dgrad)");
}

void launch_conv5x5_wgrad_mma(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st) {
  if (!conv_wgmma_supported(s)) throw std::invalid_argument("conv5x5 wgrad (mma): only 16→32 channels are implemented");
  using Cfg = WgradCfg;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  const int grid = std::min(tiles, sm_count());
  if (static_cast<long long>(grid) * Cfg::kMUsed * 32 > scr.capacity_floats) throw std::invalid_argument("conv5x5 wgrad (mma): scratch too small");
  // {1,0,0,0}: source of the im2col "ones" column; written once per device, outside any graph capture
  static std::mutex mu;
  static std::map<int, bool> ones_ready;
  float* ones = repack_buffer(2, 4);
  {
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    if (!ones_ready[dev]) {
      const float h[4] = {1.f, 0.f, 0.f, 0.f};
      cudaError_t e = cudaMemcpy(ones, h, sizeof(h), cudaMemcpyHostToDevice);
      if (e != cudaSuccess) throw std::runtime_error(std::string("cudaMemcpy(ones): ") + cudaGetErrorString(e));
      ones_ready[dev] = true;
    }
  }
  CUtensorMap tm_dy = make_tmap_2d(dy, 32, static_cast<uint64_t>(M), 32, kTileM, CU_TENSOR_MAP_SWIZZLE_128B);
  opt_in_smem(conv5x5_wgrad_mma_kernel, Cfg::kSmem);
  conv5x5_wgrad_mma_kernel<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(x, tm_dy, ones, scr.partials, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_wgrad_mma");
  wgrad_fold_kernel<<<401, 256, 0, st>>>(scr.partials, grid, dw, db);
  check_launch("wgrad_fold");
}

}  // namespace pdt
