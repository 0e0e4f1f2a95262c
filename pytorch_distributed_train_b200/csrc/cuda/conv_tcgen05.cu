// wgmma / TMA kernels for sm_90a (hand-written PTX; no CUTLASS).  The file and the "umma" kernel names date from the
// first (Blackwell) version of the project; the kernels are Hopper's.
//
//  * gemm_tf32_umma_kernel — D[M,N] = A[M,K]·B[N,K]^T: both operands arrive by TMA
//    (cp.async.bulk.tensor, SWIZZLE_128B), one warpgroup issues wgmma.mma_async ... .tf32,
//    the fp32 accumulator lives in its registers.  It is the self-test
//    for every descriptor/barrier convention used below (tests/test_gpu_ops.py).
//  * conv5x5_umma_kernel — the ConvNet's conv2 (88% of the model's FLOPs; ref:
//    ddp_example.py:30) and its data gradient as an implicit GEMM: M = output pixels (128 per
//    tile), N = output channels, K = 25 taps × input channels.  The im2col A-tile is never
//    materialised in global memory: four producer warps gather it straight from the NHWC
//    activation with 16-byte cp.async (zero-fill for the padding halo) into the 128B-swizzled
//    K-major layout the wgmma descriptor expects; the repacked weights (B) are TMA-loaded once
//    per CTA and stay resident in smem; the epilogue adds the bias, folds the per-channel
//    Σy/Σy² that BatchNorm needs (saving a full re-read of y) and writes the tile with a TMA
//    store.  TF32 inputs / fp32 accumulate is the same numerics contract the reference gets from
//    cuDNN (torch allows TF32 in convolutions by default).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <map>
#include <mutex>
#include <stdexcept>
#include <string>

#include "conv_tcgen05.h"
#include "umma_ptx.cuh"
#include "wgrad_win.cuh"
#include "cuda_utils.h"
#include "grid_fold.cuh"
#include "grid_sync.cuh"

namespace pdt {

namespace {

using namespace ptx;

constexpr int kTileM = 128;
constexpr int kChunkK = 32;            // fp32 elements per 128-byte swizzle row
constexpr int kStageBytes = kTileM * 128;

// =====================================================================================================
// TF32 GEMM self-test:  one CTA per 128-row × NB-column tile of D; 4-stage TMA ring; 160 threads
// (warps 0-3 = the wgmma warpgroup, warp 4 = TMA producer)
// =====================================================================================================
template <int NB>  // N block = 16, 32 or 64 columns
struct GemmCfg {
  static constexpr int kStages = 4;
  static constexpr int kBBytes = NB * 128;
  static constexpr size_t kSmem = 1024 + kStages * (kStageBytes + kBBytes) + 256;
};

template <int NB>
__global__ void __launch_bounds__(160, 1) gemm_tf32_umma_kernel(const __grid_constant__ CUtensorMap tm_a,
                                                                const __grid_constant__ CUtensorMap tm_b, float* __restrict__ d, int M,
                                                                int N, int K) {
  using Cfg = GemmCfg<NB>;
  constexpr int kN = NB < 32 ? NB : 32;   // wgmma N per instruction
  constexpr int kNI = NB / kN;            // instructions per 64-row half
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;
  uint8_t* sb = smem + Cfg::kStages * kStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sb + Cfg::kStages * Cfg::kBBytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::kStages;

  const int tid = threadIdx.x, warp = tid >> 5;
  const int m0 = blockIdx.x * kTileM, n0 = blockIdx.y * NB;
  const int nk = (K + kChunkK - 1) / kChunkK;

  if (tid == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 128); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    if (elect_one()) {
      for (int kc = 0; kc < nk; ++kc) {
        const int s = kc % Cfg::kStages;
        mbar_wait(&empty[s], ((kc / Cfg::kStages) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], kStageBytes + Cfg::kBBytes);
        tma_load_2d(sa + s * kStageBytes, &tm_a, &full[s], kc * kChunkK, m0);
        tma_load_2d(sb + s * Cfg::kBBytes, &tm_b, &full[s], kc * kChunkK, n0);
      }
    }
    return;
  }
  float acc[2][kNI][kN / 2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < kNI; ++i)
#pragma unroll
      for (int e = 0; e < kN / 2; ++e) acc[h][i][e] = 0.f;
  for (int kc = 0; kc < nk; ++kc) {
    const int s = kc % Cfg::kStages;
    mbar_wait(&full[s], (kc / Cfg::kStages) & 1);
    const uint32_t a0 = smem_u32(sa + s * kStageBytes), b0 = smem_u32(sb + s * Cfg::kBBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kChunkK / 8; ++k)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < kNI; ++i)
          wgmma_tf32<kN>(acc[h][i], gmma_desc_kmajor<128>(a0 + h * 64 * 128 + k * 32), gmma_desc_kmajor<128>(b0 + i * kN * 128 + k * 32),
                         (kc | k) != 0);
    wgmma_commit();
    wgmma_wait<0>();
    mbar_arrive(&empty[s]);
  }
  // epilogue straight from the register fragments
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < kNI; ++i)
#pragma unroll
      for (int e = 0; e < kN / 2; ++e) {
        const int row = m0 + 64 * h + wgmma_frag_row(tid, e), col = n0 + i * kN + wgmma_frag_col(tid, e);
        if (row < M && col < N) d[static_cast<size_t>(row) * N + col] = acc[h][i][e];
      }
}

// =====================================================================================================
// Weight repack for the implicit GEMM:  Bm[NOUT][NCHUNK*32], K index = tap*CK + c  (zero padded)
//   FWD : Bm[co][tap*16+ci] = w[co][ci][tap]
//   DGRAD: Bm[ci][tap*32+co] = w[co][ci][24-tap]
// =====================================================================================================
template <bool FWD>
__global__ void repack_weights_kernel(const float* __restrict__ w, float* __restrict__ bm, int Cout, int Cin) {
  const int CK = FWD ? Cin : Cout, NOUT = FWD ? Cout : Cin;
  const int tpc = kChunkK / CK, nchunk = (25 + tpc - 1) / tpc, kpad = nchunk * kChunkK;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NOUT * kpad) return;
  const int n = i / kpad, k = i % kpad, tap = k / CK, c = k % CK;
  float v = 0.f;
  if (tap < 25) v = FWD ? w[(n * Cin + c) * 25 + tap] : w[(c * Cin + n) * 25 + (24 - tap)];
  bm[i] = v;
}

// =====================================================================================================
// Implicit-GEMM 5x5 convolution on wgmma
// =====================================================================================================
template <int CK, int NOUT>
struct ConvCfg {
  static constexpr int kTapsPerChunk = kChunkK / CK;                           // 2 (fwd) / 1 (dgrad)
  static constexpr int kChunks = (25 + kTapsPerChunk - 1) / kTapsPerChunk;     // 13 / 25
  // 8 smem stages but only 3 cp.async groups in flight per thread: a chunk is multiplied kLag
  // iterations after it was issued, so the copies of the next chunks overlap the MMAs.
  static constexpr int kStages = 8;
  static constexpr int kLag = 3;
  static constexpr int kBChunkBytes = NOUT * 128;
  static constexpr int kAccBytes = kTileM * (NOUT + 1) * 4;
  static constexpr int kThreads = 160;                                         // 4 producer/MMA/epilogue warps + TMA warp
  // alignment slack + A ring + resident B + output staging + accumulator rows + (barriers, stat partials)
  static constexpr size_t kSmem = 1024 + kStages * kStageBytes + kChunks * kBChunkBytes + kTileM * 128 + kAccBytes + 2048;
};

template <int CK, int NOUT, bool FWD>
__global__ void __launch_bounds__(160, 1) conv5x5_umma_kernel(const float* __restrict__ x, const __grid_constant__ CUtensorMap tm_b,
                                                              const __grid_constant__ CUtensorMap tm_y, const float* __restrict__ bias,
                                                              float* __restrict__ y, float* stats, ReduceScratch scr, int B, int H, int W,
                                                              int num_tiles) {
  using Cfg = ConvCfg<CK, NOUT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                                  // [stages][128 rows][128 B] swizzled
  uint8_t* sb = sa + Cfg::kStages * kStageBytes;                       // [chunks][NOUT rows][128 B] swizzled (TMA)
  uint8_t* sy = sb + Cfg::kChunks * Cfg::kBChunkBytes;                 // [128 rows][128 B] swizzled output staging
  float* sacc = reinterpret_cast<float*>(sy + kTileM * 128);          // [128][NOUT + 1] accumulator rows
  uint64_t* b_full = reinterpret_cast<uint64_t*>(sacc + kTileM * (NOUT + 1));
  float* s_part = reinterpret_cast<float*>(b_full + 2);               // [4 warps][2*NOUT] + [2*NOUT]
  __shared__ int s_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int M = B * H * W;

  if (tid == 0) {
    tma_prefetch_desc(&tm_b);
    if (FWD) tma_prefetch_desc(&tm_y);
    mbar_init(b_full, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    // ---- weights: one TMA box per K-chunk, resident for the CTA's lifetime -------------------------
    if (elect_one()) {
      mbar_arrive_expect_tx(b_full, Cfg::kChunks * Cfg::kBChunkBytes);
      for (int c = 0; c < Cfg::kChunks; ++c) tma_load_2d(sb + c * Cfg::kBChunkBytes, &tm_b, b_full, c * kChunkK, 0);
    }
  } else {
    // ---- warps 0-3: im2col producers, wgmma issue (the chunk issued kLag iterations earlier), epilogue --------
    // A stage is refilled kStages chunks after it was filled; its MMAs completed kStages − kLag iterations before.
    static_assert(Cfg::kLag < Cfg::kStages, "conv5x5_umma: the lag must be shorter than the ring");
    const uint64_t bdesc0 = gmma_desc_kmajor<128>(smem_u32(sb));
    auto mma_chunk = [&](float (&acc)[2][NOUT / 2], int c, int s) {
      const uint32_t a0 = smem_u32(sa + s * kStageBytes);
      const uint64_t bd = bdesc0 + static_cast<uint64_t>((c * Cfg::kBChunkBytes) >> 4);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kChunkK / 8; ++k)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          wgmma_tf32<NOUT>(acc[h], gmma_desc_kmajor<128>(a0 + h * 64 * 128 + k * 32), bd + ((k * 32) >> 4), (c | k) != 0);
      wgmma_commit();
      wgmma_wait<0>();
    };
    mbar_wait(b_full, 0);
    const int u = tid & 7;                       // 16-byte column inside the 128-byte K row
    const int tap_in_chunk = (u * 4) / CK;       // which tap of the chunk this column belongs to
    const int c4 = (u * 4) % CK;                 // channel offset inside the tap
    int g = 0, it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      // the 8 rows this thread fills: r = tid/8 + 16 j
      int row_off[8], row_h[8], row_w[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int r = (tid >> 3) + 16 * j;
        const int p = tile * kTileM + r;
        if (p < M) {
          const int ow = p % W, oh = (p / W) % H, n = p / (W * H);
          row_off[j] = ((n * H + oh) * W + ow) * CK;
          row_h[j] = oh;
          row_w[j] = ow;
        } else {
          row_off[j] = 0;
          row_h[j] = -100000;  // every tap falls outside → zero fill
          row_w[j] = 0;
        }
      }
      float acc[2][NOUT / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < NOUT / 2; ++e) acc[h][e] = 0.f;
      for (int c = 0; c < Cfg::kChunks; ++c, ++g) {
        const int s = g % Cfg::kStages;
        const int tap = c * Cfg::kTapsPerChunk + tap_in_chunk;
        const int kh = tap / 5 - 2, kw = tap % 5 - 2;
        const int delta = (kh * W + kw) * CK + c4;
        const uint32_t stage = smem_u32(sa + s * kStageBytes);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int r = (tid >> 3) + 16 * j;
          const int ih = row_h[j] + kh, iw = row_w[j] + kw;
          const bool ok = tap < 25 && ih >= 0 && ih < H && iw >= 0 && iw < W;
          const float* src = ok ? x + row_off[j] + delta : x;
          cp_async_16(stage + r * 128 + ((u ^ (r & 7)) << 4), src, ok ? 16u : 0u);
        }
        cp_async_commit();
        if (c >= Cfg::kLag) {
          cp_async_wait<Cfg::kLag>();            // chunk c-kLag of this thread has landed
          fence_proxy_async_smem();              // generic-proxy writes → visible to the tensor core (async proxy)
          asm volatile("bar.sync 1, 128;" ::: "memory");   // ... and that of every producer thread
          mma_chunk(acc, c - Cfg::kLag, (g - Cfg::kLag) % Cfg::kStages);
        }
      }
      // drain this tile (its accumulator is needed now): the kLag chunks still in flight; the lag bookkeeping restarts
      // with the next tile
      cp_async_wait<0>();
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
      for (int q = Cfg::kLag; q >= 1; --q) mma_chunk(acc, Cfg::kChunks - q, (g - q) % Cfg::kStages);
      // ---- epilogue ----------------------------------------------------------------------------------
#pragma unroll
      for (int h = 0; h < 2; ++h) wgmma_frag_store<NOUT>(acc[h], sacc, NOUT + 1, 64 * h, tid);
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float v[NOUT];
#pragma unroll
      for (int j = 0; j < NOUT; ++j) v[j] = sacc[tid * (NOUT + 1) + j];
      const int r = tid;  // 0..127 = tile row
      const int p = tile * kTileM + r;
      const bool valid = p < M;
      if (bias) {
#pragma unroll
        for (int j = 0; j < NOUT; ++j) v[j] += bias[j];
      }
      if constexpr (FWD) {
        // stage the tile (swizzled like the tensor map) for the TMA store and the column sums
        asm volatile("bar.sync 1, 128;" ::: "memory");  // previous tile's TMA store has finished reading sy
#pragma unroll
        for (int q = 0; q < NOUT / 4; ++q) {
          float4 o = valid ? make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
          *reinterpret_cast<float4*>(sy + r * 128 + ((q ^ (r & 7)) << 4)) = o;
        }
        fence_proxy_async_smem();
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (tid == 0) {
          tma_store_2d(&tm_y, sy, 0, tile * kTileM);
          tma_store_commit();
        }
        if (stats) {
          // column sums over this warp's 32 rows: lane = channel
          float s1 = 0.f, s2 = 0.f;
          const int q = lane >> 2, e = lane & 3;
          for (int rr = warp * 32; rr < warp * 32 + 32; ++rr) {
            const float val = reinterpret_cast<const float*>(sy + rr * 128 + ((q ^ (rr & 7)) << 4))[e];
            s1 += val;
            s2 += val * val;
          }
          s_part[warp * 2 * NOUT + lane] = s1;
          s_part[warp * 2 * NOUT + NOUT + lane] = s2;
          asm volatile("bar.sync 1, 128;" ::: "memory");
          float* tile_sums = s_part + 8 * NOUT;  // [2*NOUT]
          if (tid < 2 * NOUT) tile_sums[tid] = s_part[tid] + s_part[2 * NOUT + tid] + s_part[4 * NOUT + tid] + s_part[6 * NOUT + tid];
          asm volatile("bar.sync 1, 128;" ::: "memory");
          // tiles are the contributors of the two-level deterministic fold (grid_fold.cuh)
          grid_fold(tile_sums, 2 * NOUT, tile, num_tiles, scr, s_part, &s_last, tid, 128, NamedSync<1, 128>{}, [&](int i, float tot) {
            stats[i] = tot;
            if (i == 0) stats[2 * NOUT] = static_cast<float>(M);
          });
        }
        if (tid == 0) tma_store_wait_read();
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
__global__ void __launch_bounds__(160, 1) conv5x5_umma_tma_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_b,
                                                                  const __grid_constant__ CUtensorMap tm_y, const float* __restrict__ bias,
                                                                  float* __restrict__ y, float* stats, ReduceScratch scr, int B, int H, int W,
                                                                  int num_tiles) {
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
          float s1 = 0.f, s2 = 0.f;
          const int q = lane >> 2, e = lane & 3;
          const int w4 = et >> 5;  // 0..3: rows 32*w4 .. 32*w4+31
          for (int rr = w4 * 32; rr < w4 * 32 + 32; ++rr) {
            const float val = reinterpret_cast<const float*>(sy + rr * 128 + ((q ^ (rr & 7)) << 4))[e];
            s1 += val;
            s2 += val * val;
          }
          s_part[w4 * 2 * NOUT + lane] = s1;
          s_part[w4 * 2 * NOUT + NOUT + lane] = s2;
          asm volatile("bar.sync 1, 128;" ::: "memory");
          float* tile_sums = s_part + 8 * NOUT;
          if (et < 2 * NOUT) tile_sums[et] = s_part[et] + s_part[2 * NOUT + et] + s_part[4 * NOUT + et] + s_part[6 * NOUT + et];
          asm volatile("bar.sync 1, 128;" ::: "memory");
          grid_fold(tile_sums, 2 * NOUT, tile, num_tiles, scr, s_part, &s_last, et, 128, NamedSync<1, 128>{}, [&](int i, float tot) {
            stats[i] = tot;
            if (i == 0) stats[2 * NOUT] = static_cast<float>(M);
          });
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

// =====================================================================================================
// EXPERIMENTAL (not covered by the test suite, not reachable unless impl == "win" is requested):
// "window" implicit-GEMM 5x5 convolution — every input pixel is loaded ONCE.
//
// The im2col kernels above gather 128 pixels × 25 taps = 3,200 rows per tile through TMA.  Here a tile is R output rows of one image
// in *padded-width* coordinates (PW = W + 4 positions per row, M = R·PW ≤ 128 MMA rows of which R·W are real
// outputs): ONE tiled TMA box {32 ch, PW, R + 4 rows} brings the zero-haloed patch (hardware OOB fill
// provides the halo and, for C = 16, the upper half of the 128-byte row), and tap (kh, kw) is the same
// buffer read through a K-major SWIZZLE_128B descriptor that starts (kh·PW + kw) rows in (base offset 0: the swizzle
// phase follows the absolute address, tools/exp_rowshift.py).  Index math checked on the CPU by
// tools/emulate_window_conv.py.
// Weights: Bm[NOUT][25·32] (K index = tap·32 + c, zero padded for C = 16), resident in smem.
// =====================================================================================================

template <int NOUT>
struct ConvWinCfg {
  static constexpr int kRowB = 128;                          // bytes per padded position (32 floats, upper half zero for C=16)
  static constexpr int kPatchRowsMax = 256;                  // PW·(R+4) positions per tile, box limit
  static constexpr int kAStageBytes = kPatchRowsMax * kRowB + 1024;   // + slack: the last taps of padding rows read past the box
  static constexpr int kStages = 2;
  static constexpr int kBTapBytes = NOUT * kRowB;            // 4 KB / 2 KB
  static constexpr int kSyBytes = kTileM * 128;              // row staging for the BN statistics
  static constexpr int kAccBytes = kTileM * (NOUT + 1) * 4;  // accumulator rows, one per epilogue thread
  static constexpr int kThreads = 160;
  static constexpr size_t kSmem = 2048 + kStages * kAStageBytes + 25 * kBTapBytes + kSyBytes + kAccBytes + 2048;
};

template <int CK, int NOUT, bool FWD>
__global__ void __launch_bounds__(160, 1) conv5x5_umma_win_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_b,
                                                                  const float* __restrict__ bias, float* __restrict__ y, float* stats,
                                                                  ReduceScratch scr, int B, int H, int W, int R, int num_tiles, int bo_mode) {
  using Cfg = ConvWinCfg<NOUT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                                        // stages start 1024-aligned (kAStageBytes % 1024 == 0)
  uint8_t* sb = sa + Cfg::kStages * Cfg::kAStageBytes;
  uint8_t* sy = sb + 25 * Cfg::kBTapBytes;
  float* sacc = reinterpret_cast<float*>(sy + Cfg::kSyBytes);   // [128][NOUT + 1]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sacc + kTileM * (NOUT + 1));
  uint64_t* full = bars;
  uint64_t* empty = full + Cfg::kStages;
  uint64_t* b_full = empty + Cfg::kStages;
  float* s_part = reinterpret_cast<float*>(b_full + 2);   // [4][2*NOUT] + [2*NOUT]
  __shared__ int s_last;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int PW = W + 4, tiles_per_img = H / R, Mrows = R * PW;
  const int M = B * H * W;
  if (tid == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_b);
    for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 128); }
    mbar_init(b_full, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warpgroup_index() == 1) {
    if (elect_one()) {
      mbar_arrive_expect_tx(b_full, 25 * Cfg::kBTapBytes);
      for (int t = 0; t < 25; ++t) tma_load_2d(sb + t * Cfg::kBTapBytes, &tm_b, b_full, t * 32, 0);
      const uint32_t patch_bytes = static_cast<uint32_t>(Cfg::kRowB) * PW * (R + 4);
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const int n = tile / tiles_per_img, oh0 = (tile % tiles_per_img) * R;
        const int s = it % Cfg::kStages;
        mbar_wait(&empty[s], ((it / Cfg::kStages) & 1) ^ 1);
        mbar_arrive_expect_tx(&full[s], patch_bytes);
        tma_load_4d(sa + s * Cfg::kAStageBytes, &tm_x, &full[s], 0, -2, oh0 - 2, n);   // halo and channel pad: OOB zero fill
      }
    }
  } else {
    // ---- warps 0..3: wgmma issue + epilogue; thread = padded position of the tile --------------------------------
    const int et = tid, r = tid;
    const int rr = r / PW, owp = r - rr * PW;
    const bool real = r < Mrows && owp < W;   // 4 of every PW positions (and rows ≥ R·PW) are padding
    mbar_wait(b_full, 0);
    int it = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
      const int s = it % Cfg::kStages;
      const int n = tile / tiles_per_img, oh0 = (tile % tiles_per_img) * R;
      mbar_wait(&full[s], (it / Cfg::kStages) & 1);
      float acc[2][NOUT / 2];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < NOUT / 2; ++e) acc[h][e] = 0.f;
      const uint32_t a0 = smem_u32(sa + s * Cfg::kAStageBytes), b0 = smem_u32(sb);
      wgmma_fence();
      for (int kh = 0; kh < 5; ++kh) {
#pragma unroll
        for (int kw = 0; kw < 5; ++kw) {
          const uint32_t arow = a0 + static_cast<uint32_t>(kh * PW + kw) * Cfg::kRowB;
#pragma unroll
          for (int k = 0; k < CK / 8; ++k) {   // C = 16: the zero upper half of the row is simply not multiplied
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t astart = arow + h * 64 * Cfg::kRowB + k * 32;
              uint64_t ad = gmma_desc_kmajor<128>(astart);
              if (bo_mode) ad |= static_cast<uint64_t>((astart >> 7) & 7) << 49;
              wgmma_tf32<NOUT>(acc[h], ad, gmma_desc_kmajor<128>(b0 + (kh * 5 + kw) * Cfg::kBTapBytes + k * 32), (kh | kw | k) != 0);
            }
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      mbar_arrive(&empty[s]);
      asm volatile("bar.sync 1, 128;" ::: "memory");   // the previous tile's rows have been read out of sacc
#pragma unroll
      for (int h = 0; h < 2; ++h) wgmma_frag_store<NOUT>(acc[h], sacc, NOUT + 1, 64 * h, tid);
      asm volatile("bar.sync 1, 128;" ::: "memory");
      float v[NOUT];
#pragma unroll
      for (int j = 0; j < NOUT; ++j) v[j] = sacc[r * (NOUT + 1) + j];
      if (bias) {
#pragma unroll
        for (int j = 0; j < NOUT; ++j) v[j] += bias[j];
      }
      if (real) {
        float* o = y + (static_cast<size_t>(n * H + oh0 + rr) * W + owp) * NOUT;
#pragma unroll
        for (int q = 0; q < NOUT / 4; ++q) *reinterpret_cast<float4*>(o + 4 * q) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
      }
      if constexpr (FWD) {
        if (stats) {
          asm volatile("bar.sync 1, 128;" ::: "memory");  // the previous tile's statistics pass has finished reading sy
#pragma unroll
          for (int q = 0; q < NOUT / 4; ++q) {
            float4 o4 = real ? make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]) : make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4*>(sy + r * 128 + ((q ^ (r & 7)) << 4)) = o4;
          }
          asm volatile("bar.sync 1, 128;" ::: "memory");
          float s1 = 0.f, s2 = 0.f;
          const int q = lane >> 2, e = lane & 3;
          const int w4 = et >> 5;
          for (int r2 = w4 * 32; r2 < w4 * 32 + 32; ++r2) {
            const float val = reinterpret_cast<const float*>(sy + r2 * 128 + ((q ^ (r2 & 7)) << 4))[e];
            s1 += val;
            s2 += val * val;
          }
          s_part[w4 * 2 * NOUT + lane] = s1;
          s_part[w4 * 2 * NOUT + NOUT + lane] = s2;
          asm volatile("bar.sync 1, 128;" ::: "memory");
          float* tile_sums = s_part + 8 * NOUT;
          if (et < 2 * NOUT) tile_sums[et] = s_part[et] + s_part[2 * NOUT + et] + s_part[4 * NOUT + et] + s_part[6 * NOUT + et];
          asm volatile("bar.sync 1, 128;" ::: "memory");
          grid_fold(tile_sums, 2 * NOUT, tile, num_tiles, scr, s_part, &s_last, et, 128, NamedSync<1, 128>{}, [&](int i, float tot) {
            stats[i] = tot;
            if (i == 0) stats[2 * NOUT] = static_cast<float>(M);
          });
        }
      }
    }
  }
}

// Bm[NOUT][25·32]: K index = tap·32 + c, channels ≥ CK zero (window kernel: 128-byte rows for every C)
template <bool FWD>
__global__ void repack_weights_pad32_kernel(const float* __restrict__ w, float* __restrict__ bm, int Cout, int Cin) {
  const int CK = FWD ? Cin : Cout, NOUT = FWD ? Cout : Cin;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NOUT * 800) return;
  const int n = i / 800, k = i % 800, tap = k / 32, c = k % 32;
  float v = 0.f;
  if (c < CK) v = FWD ? w[(n * Cin + c) * 25 + tap] : w[(c * Cin + n) * 25 + (24 - tap)];
  bm[i] = v;
}

// Bm[NOUT][25*CK] without K padding (the TMA-fed kernel loads one [NOUT][CK] box per tap)
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
__global__ void __launch_bounds__(160, 1) conv5x5_wgrad_umma_kernel(const float* __restrict__ x, const __grid_constant__ CUtensorMap tm_dy,
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

// =====================================================================================================
// conv2 weight gradient, fully TMA-fed ("window" formulation; used by the cooperative fused layers, whose activations
// live in zero-haloed 18×18 frames):   dWᵀ[(kh, kw, ci)][co] = Σ_P  xpad[P + (kh−2)·18 + (kw−2)][ci] · dypad[P][co]
// over the padded positions P of every image (dypad is zero outside the 14×14 interior, so the halo and the frame
// padding contribute nothing).  Two horizontally adjacent taps of one pixel are 32 *contiguous* floats of the NHWC
// frame, so the 32-row M atom of tap pair (kh, kw/2) is a row of an overlapping-row view of xpad (row pitch 64 B, row
// length 128 B) read (kh−2)·18 + (kw−2) rows from the position: each image's view (384 rows) and its 256 dy positions
// from the first interior one arrive as eight TMA boxes, and the 15 tap pairs (q = 3·kh + kw/2; pair (kh, 4-5) carries
// a dummy sixth column) are computed by four warps with mma.sync (wgrad_win.cuh), accumulated over the CTA's images in
// registers.  One CTA per image at most; per-CTA partial [512][32] (rows q·32 + (kw&1)·16 + ci); the bias gradient
// comes from per-image Σdy rows (layer-2 backward).
// =====================================================================================================
struct WgradWinCfg {
  static constexpr int kFrame = 18 * 18;              // padded positions per image
  static constexpr int kFirst = 2 * 18 + 2;           // first interior position
  static constexpr int kMRows = 512;
  static constexpr int kABoxes = 6, kABytes = kABoxes * 64 * 128;   // overlapping-row view of one image, 64-row boxes
  static constexpr int kBBytes = 2 * kTileM * 128;                   // dy at 256 positions
  static constexpr int kThreads = 128;
  static constexpr size_t kSmem = 1024 + kABytes + kBBytes + 1024;
};

__global__ void __launch_bounds__(128, 1) conv5x5_wgrad_win_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_dy,
                                                                   float* __restrict__ partials, int B, const float* __restrict__ dysum,
                                                                   float* __restrict__ dw, float* __restrict__ db, GridSync gs) {
  using Cfg = WgradWinCfg;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;
  uint8_t* sb = sa + Cfg::kABytes;
  uint64_t* ld_full = reinterpret_cast<uint64_t*>(sb + Cfg::kBBytes);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  GridBar bar(gs);
  if (tid == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_dy);
    mbar_init(ld_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  float acc[4][2][4][4];   // warp w: tap pairs q = 4w .. 4w+3
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[a][j][nt][e] = 0.f;
  int it = 0;
  for (int n = blockIdx.x; n < B; n += gridDim.x, ++it) {
    if (tid == 0) {
      const int frame0 = n * Cfg::kFrame;
      mbar_arrive_expect_tx(ld_full, Cfg::kABytes + Cfg::kBBytes);
      for (int bx = 0; bx < Cfg::kABoxes; ++bx) tma_load_2d(sa + bx * 8192, &tm_x, ld_full, 0, frame0 + 64 * bx);   // rows past the tensor are zero-filled
      tma_load_2d(sb, &tm_dy, ld_full, 0, frame0 + Cfg::kFirst);
      tma_load_2d(sb + kTileM * 128, &tm_dy, ld_full, 0, frame0 + Cfg::kFirst + kTileM);
    }
    mbar_wait(ld_full, it & 1);
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int q = warp * 4 + a, kh = q / 3, kw = 2 * (q - kh * 3);
      if (q < 15) wgrad_win_atom(acc[a], reinterpret_cast<const float*>(sa), Cfg::kFirst + (kh - 2) * 18 + (kw - 2), 0,
                                 reinterpret_cast<const float*>(sb), 0, lane);
    }
    __syncthreads();   // every warp is done with this image's tiles before the next loads overwrite them
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int q = warp * 4 + a;
    if (q < 15) wgrad_win_atom_store(acc[a], partials + (static_cast<size_t>(blockIdx.x) * Cfg::kMRows + q * 32) * 32, lane);
  }
  if (dw == nullptr) return;   // two-launch variant: wgrad_win_fold_kernel folds
  // ---- in-kernel fold (cooperative launch): after a grid barrier every CTA folds a share of the 400 × 32 outputs over the
  //      per-CTA partials in a fixed order — thread = (co, one of six partial classes), classes combined through smem ----------
  bar.sync(gs);
  float* s_f = reinterpret_cast<float*>(smem);   // [4][32]
  const int co = tid & 31, part = tid >> 5, nparts = gridDim.x;
  for (int i = blockIdx.x; i < 401; i += gridDim.x) {
    float acc = 0.f;
    if (i < 400) {
      const int tap = i >> 4, ci = i & 15, kh = tap / 5, kw = tap - kh * 5;
      const int m = (3 * kh + (kw >> 1)) * 32 + (kw & 1) * 16 + ci;
      const float* p = partials + static_cast<size_t>(m) * 32 + co;
      const size_t stride = static_cast<size_t>(Cfg::kMRows) * 32;
      for (int c = part; c < nparts; c += 32) {   // eight independent L2 loads in flight
        float t[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) t[j] = (c + 4 * j < nparts) ? __ldcg(p + static_cast<size_t>(c + 4 * j) * stride) : 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += t[j];
      }
    } else {
      for (int n = part; n < B; n += 4) acc += __ldcg(dysum + static_cast<size_t>(n) * 32 + co);
    }
    __syncthreads();
    s_f[part * 32 + co] = acc;
    __syncthreads();
    if (part == 0) {
      const float tot = (s_f[co] + s_f[32 + co]) + (s_f[64 + co] + s_f[96 + co]);
      if (i < 400) dw[(co * 16 + (i & 15)) * 25 + (i >> 4)] = tot;
      else if (db) db[co] = tot;
    }
  }
}

// dw[co][ci][kh][kw] = Σ_cta partial[cta][q·32 + (kw&1)·16 + ci][co] with q = 3·kh + kw/2;  db[co] = Σ_n dysum[n][co]
__global__ void __launch_bounds__(256) wgrad_win_fold_kernel(const float* __restrict__ partials, int nparts, const float* __restrict__ dysum, int B,
                                                             float* __restrict__ dw, float* __restrict__ db) {
  __shared__ float s_sub[8][32];
  const int i = blockIdx.x, co = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float s0 = 0.f, s1 = 0.f;
  if (i < 400) {
    const int tap = i >> 4, ci = i & 15, kh = tap / 5, kw = tap - kh * 5;
    const int m = (3 * kh + (kw >> 1)) * 32 + (kw & 1) * 16 + ci;
    const float* p = partials + static_cast<size_t>(m) * 32 + co;
    const size_t stride = static_cast<size_t>(WgradWinCfg::kMRows) * 32;
    int c = warp;
    for (; c + 8 < nparts; c += 16) {
      s0 += p[c * stride];
      s1 += p[(c + 8) * stride];
    }
    if (c < nparts) s0 += p[c * stride];
  } else {
    for (int n = warp; n < B; n += 8) s0 += dysum[static_cast<size_t>(n) * 32 + co];
  }
  s_sub[warp][co] = s0 + s1;
  __syncthreads();
  if (warp == 0) {
    float s = 0.f;
#pragma unroll
    for (int w8 = 0; w8 < 8; ++w8) s += s_sub[w8][co];
    if (i < 400) dw[(co * 16 + (i & 15)) * 25 + (i >> 4)] = s;
    else if (db) db[co] = s;
  }
}

// =====================================================================================================
// Hardware probe of the descriptor convention the window convolutions rely on: can a K-major swizzled A
// operand start at an arbitrary ROW of a larger smem buffer?  A [256][ROWB/4] tile is loaded once by TMA;
// the wgmma reads rows [shift, shift+128) through descriptors whose start address is base + shift·ROWB,
// with the base-offset field either 0 (mode 0) or (start >> 7) & 7 (mode 1).  D[128][32] = A[shift:shift+128] · Bᵀ.
// Not used by any product path; run by tools/exp_rowshift.py.
// =====================================================================================================
template <int ROWB>
__global__ void __launch_bounds__(128, 1) umma_rowshift_probe_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                                                                     float* __restrict__ d, int shift, int mode) {
  constexpr int kRows = 256, kN = 32, kK = ROWB / 4;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sa = smem;                         // [256][ROWB]
  uint8_t* sb = smem + kRows * ROWB;          // [32][ROWB]   (1024-aligned: 256·ROWB is a multiple of 1024)
  uint64_t* bar = reinterpret_cast<uint64_t*>(sb + 4096);
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, kRows * ROWB + kN * ROWB);
    tma_load_2d(sa, &tm_a, bar, 0, 0);
    tma_load_2d(sb, &tm_b, bar, 0, 0);
  }
  mbar_wait(bar, 0);
  float acc[2][16];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[h][e] = 0.f;
  const uint32_t a0 = smem_u32(sa) + static_cast<uint32_t>(shift) * ROWB, b0 = smem_u32(sb);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kK / 8; ++k)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const uint32_t astart = a0 + h * 64 * ROWB + k * 32;
      uint64_t ad = gmma_desc_kmajor<ROWB>(astart);
      if (mode == 1) ad |= static_cast<uint64_t>((astart >> 7) & 7) << 49;
      wgmma_m64n32k8_tf32(acc[h], ad, gmma_desc_kmajor<ROWB>(b0 + k * 32), k != 0);
    }
  wgmma_commit();
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 16; ++e) d[(64 * h + wgmma_frag_row(tid, e)) * kN + wgmma_frag_col(tid, e)] = acc[h][e];
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
// NHWC activation as a 4-D tiled map {C, W, H, N} with a box of {32 channels, box_w, box_h, 1}: coordinates may start
// outside the tensor (negative w/h, channels ≥ C) — the hardware zero-fills, which is the conv halo and the channel pad.
CUtensorMap make_tmap_nhwc_patch(const float* base, int C, int W, int H, int N, int box_w, int box_h) {
  CUtensorMap m;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * 4, static_cast<cuuint64_t>(W) * C * 4, static_cast<cuuint64_t>(H) * W * C * 4};
  cuuint32_t box[4] = {32, static_cast<cuuint32_t>(box_w), static_cast<cuuint32_t>(box_h), 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = driver().cuTensorMapEncodeTiled(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, estr,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(nhwc patch) failed: " + cu_error(r));
  return m;
}

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

void check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("launch of ") + what + " failed: " + cudaGetErrorString(e));
  count_kernel_launch();
}

template <typename K>
void opt_in_smem(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  if (e != cudaSuccess) throw std::runtime_error(std::string("cudaFuncSetAttribute(smem): ") + cudaGetErrorString(e));
}

// repacked-weight buffers, one per (device, direction); allocated on first use (outside graph capture)
float* repack_buffer(int dir, size_t floats) {
  static std::mutex mu;
  static std::map<std::pair<int, int>, std::pair<float*, size_t>> bufs;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> g(mu);
  auto& slot = bufs[{dev, dir}];
  if (slot.second < floats) {
    if (slot.first) cudaFree(slot.first);
    cudaError_t e = cudaMalloc(&slot.first, floats * sizeof(float));
    if (e != cudaSuccess) throw std::runtime_error(std::string("cudaMalloc(repack buffer): ") + cudaGetErrorString(e));
    slot.second = floats;
  }
  return slot.first;
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

}  // namespace

bool conv_tcgen05_supported(const ConvShape& s) { return s.Cin == 16 && s.Cout == 32; }

void launch_conv5x5_fwd_tcgen05(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s, ReduceScratch scr,
                                cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 tcgen05: only 16→32 channels are implemented");
  using Cfg = ConvCfg<16, 32>;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  if (stats && (static_cast<long long>(tiles + tiles / kFoldGroup + 1) * 64 > scr.capacity_floats || tiles / kFoldGroup + 2 > scr.counters))
    throw std::invalid_argument("conv5x5 tcgen05: scratch too small");
  const int kpad = Cfg::kChunks * kChunkK;
  float* bm = repack_buffer(0, static_cast<size_t>(32) * kpad);
  repack_weights_kernel<true><<<(32 * kpad + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights(fwd)");
  CUtensorMap tm_b = make_tmap_2d(bm, kpad, 32, kChunkK, 32);
  CUtensorMap tm_y = make_tmap_2d(y, 32, static_cast<uint64_t>(M), 32, kTileM);
  auto kern = conv5x5_umma_kernel<16, 32, true>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(x, tm_b, tm_y, bias, y, stats, scr, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_umma(fwd)");
}

void launch_conv5x5_dgrad_tcgen05(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 tcgen05 dgrad: only 16→32 channels are implemented");
  using Cfg = ConvCfg<32, 16>;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  const int kpad = Cfg::kChunks * kChunkK;
  float* bm = repack_buffer(1, static_cast<size_t>(16) * kpad);
  repack_weights_kernel<false><<<(16 * kpad + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights(dgrad)");
  CUtensorMap tm_b = make_tmap_2d(bm, kpad, 16, kChunkK, 16);
  auto kern = conv5x5_umma_kernel<32, 16, false>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(dy, tm_b, tm_b, nullptr, dx, nullptr, ReduceScratch{}, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_umma(dgrad)");
}

void launch_conv5x5_fwd_tma(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s, ReduceScratch scr,
                            cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 tma: only 16→32 channels are implemented");
  using Cfg = ConvTmaCfg<16, 32>;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  if (stats && (static_cast<long long>(tiles + tiles / kFoldGroup + 1) * 64 > scr.capacity_floats || tiles / kFoldGroup + 2 > scr.counters))
    throw std::invalid_argument("conv5x5 tma: scratch too small");
  float* bm = repack_buffer(3, static_cast<size_t>(32) * 400);
  repack_weights_dense_kernel<true><<<(32 * 400 + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights_dense(fwd)");
  CUtensorMap tm_x = make_tmap_im2col(x, 16, s.W, s.H, s.B, CU_TENSOR_MAP_SWIZZLE_64B);
  CUtensorMap tm_b = make_tmap_2d(bm, 400, 32, 16, 32, CU_TENSOR_MAP_SWIZZLE_64B);
  CUtensorMap tm_y = make_tmap_2d(y, 32, static_cast<uint64_t>(M), 32, kTileM);
  auto kern = conv5x5_umma_tma_kernel<16, 32, true>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_b, tm_y, bias, y, stats, scr, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_umma_tma(fwd)");
}

void launch_conv5x5_dgrad_tma(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 tma dgrad: only 16→32 channels are implemented");
  using Cfg = ConvTmaCfg<32, 16>;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  float* bm = repack_buffer(4, static_cast<size_t>(16) * 800);
  repack_weights_dense_kernel<false><<<(16 * 800 + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights_dense(dgrad)");
  CUtensorMap tm_x = make_tmap_im2col(dy, 32, s.W, s.H, s.B, CU_TENSOR_MAP_SWIZZLE_128B);
  CUtensorMap tm_b = make_tmap_2d(bm, 800, 16, 32, 16, CU_TENSOR_MAP_SWIZZLE_128B);
  auto kern = conv5x5_umma_tma_kernel<32, 16, false>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_b, tm_b, nullptr, dx, nullptr, ReduceScratch{}, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_umma_tma(dgrad)");
}

// ---- experimental window kernels (see conv5x5_umma_win_kernel) -----------------------------------------------
static int win_rows_per_tile(const ConvShape& s) {
  const int PW = s.W + 4;
  int R = 0;
  for (int r = 1; r <= s.H; ++r)
    if (s.H % r == 0 && r * PW <= kTileM && (r + 4) * PW <= 256 && r + 4 <= 256) R = r;
  return R;
}
static int win_base_offset_mode() {
  static const int m = [] { const char* e = getenv("PDT_WIN_BASE_OFFSET"); return e ? atoi(e) : 0; }();
  return m;
}

void launch_conv5x5_fwd_win(const float* x, const float* w, const float* bias, float* y, float* stats, ConvShape s, ReduceScratch scr,
                            cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 win: only 16→32 channels are implemented");
  using Cfg = ConvWinCfg<32>;
  const int R = win_rows_per_tile(s);
  if (R == 0) throw std::invalid_argument("conv5x5 win: no row tiling fits 128 MMA rows for this image size");
  const int tiles = s.B * (s.H / R);
  if (stats && (static_cast<long long>(tiles + tiles / kFoldGroup + 1) * 64 > scr.capacity_floats || tiles / kFoldGroup + 2 > scr.counters))
    throw std::invalid_argument("conv5x5 win: scratch too small");
  float* bm = repack_buffer(5, static_cast<size_t>(32) * 800);
  repack_weights_pad32_kernel<true><<<(32 * 800 + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights_pad32(fwd)");
  CUtensorMap tm_x = make_tmap_nhwc_patch(x, 16, s.W, s.H, s.B, s.W + 4, R + 4);
  CUtensorMap tm_b = make_tmap_2d(bm, 800, 32, 32, 32, CU_TENSOR_MAP_SWIZZLE_128B);
  auto kern = conv5x5_umma_win_kernel<16, 32, true>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_b, bias, y, stats, scr, s.B, s.H, s.W, R, tiles, win_base_offset_mode());
  check_launch("conv5x5_umma_win(fwd)");
}

void launch_conv5x5_dgrad_win(const float* dy, const float* w, float* dx, ConvShape s, cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 win dgrad: only 16→32 channels are implemented");
  using Cfg = ConvWinCfg<16>;
  const int R = win_rows_per_tile(s);
  if (R == 0) throw std::invalid_argument("conv5x5 win dgrad: no row tiling fits 128 MMA rows for this image size");
  const int tiles = s.B * (s.H / R);
  float* bm = repack_buffer(6, static_cast<size_t>(16) * 800);
  repack_weights_pad32_kernel<false><<<(16 * 800 + 255) / 256, 256, 0, st>>>(w, bm, 32, 16);
  check_launch("repack_weights_pad32(dgrad)");
  CUtensorMap tm_x = make_tmap_nhwc_patch(dy, 32, s.W, s.H, s.B, s.W + 4, R + 4);
  CUtensorMap tm_b = make_tmap_2d(bm, 800, 16, 32, 16, CU_TENSOR_MAP_SWIZZLE_128B);
  auto kern = conv5x5_umma_win_kernel<32, 16, false>;
  opt_in_smem(kern, Cfg::kSmem);
  const int grid = std::min(tiles, sm_count());
  kern<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_b, nullptr, dx, nullptr, ReduceScratch{}, s.B, s.H, s.W, R, tiles, win_base_offset_mode());
  check_launch("conv5x5_umma_win(dgrad)");
}

void launch_conv5x5_wgrad_tcgen05(const float* dy, const float* x, float* dw, float* db, ConvShape s, ReduceScratch scr, cudaStream_t st) {
  if (!conv_tcgen05_supported(s)) throw std::invalid_argument("conv5x5 tcgen05 wgrad: only 16→32 channels are implemented");
  using Cfg = WgradCfg;
  const int M = s.B * s.H * s.W;
  const int tiles = (M + kTileM - 1) / kTileM;
  const int grid = std::min(tiles, sm_count());
  if (static_cast<long long>(grid) * Cfg::kMUsed * 32 > scr.capacity_floats) throw std::invalid_argument("conv5x5 tcgen05 wgrad: scratch too small");
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
  opt_in_smem(conv5x5_wgrad_umma_kernel, Cfg::kSmem);
  conv5x5_wgrad_umma_kernel<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(x, tm_dy, ones, scr.partials, s.B, s.H, s.W, tiles);
  check_launch("conv5x5_wgrad_umma");
  wgrad_fold_kernel<<<401, 256, 0, st>>>(scr.partials, grid, dw, db);
  check_launch("wgrad_fold");
}

void make_wgrad_win_tmaps(const float* x_pad, const float* dy_pad, int B, CUtensorMap* tm_x, CUtensorMap* tm_dy) {
  const uint64_t rows = static_cast<uint64_t>(B) * WgradWinCfg::kFrame;
  // overlapping-row view of the haloed NHWC frames: row r = the 32 floats starting at position r (two adjacent pixels × 16 ch)
  cuuint64_t dims[2] = {32, rows - 1};
  cuuint64_t strides[1] = {64};
  cuuint32_t box[2] = {32, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = driver().cuTensorMapEncodeTiled(tm_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(x_pad), dims, strides, box, estr,
                                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled(overlapping rows) failed: " + cu_error(r));
  *tm_dy = make_tmap_2d(dy_pad, 32, rows, 32, kTileM, CU_TENSOR_MAP_SWIZZLE_128B);
}

void launch_conv5x5_wgrad_win(const float* dy_pad, const float* x_pad, const float* dysum, float* dw, float* db, int B, ReduceScratch scr,
                              cudaStream_t st, GridSync gs) {
  using Cfg = WgradWinCfg;
  const int grid = std::min(B, sm_count());
  if (static_cast<long long>(grid) * Cfg::kMRows * 32 > scr.capacity_floats) throw std::invalid_argument("conv5x5 wgrad (window): scratch too small");
  CUtensorMap tm_x, tm_dy;
  make_wgrad_win_tmaps(x_pad, dy_pad, B, &tm_x, &tm_dy);
  opt_in_smem(conv5x5_wgrad_win_kernel, Cfg::kSmem);
  static const bool one_launch = [] { const char* e = getenv("PDT_WGRAD_WIN_FOLD"); return !(e && e[0] == '0'); }();
  if (one_launch && gs.epoch != nullptr) {
    // cooperative launch (one CTA per SM at most): the fold happens after a grid barrier inside the kernel
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(Cfg::kThreads);
    cfg.dynamicSmemBytes = Cfg::kSmem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, conv5x5_wgrad_win_kernel, tm_x, tm_dy, scr.partials, B, dysum, dw, db, gs);
    if (e != cudaSuccess) throw std::runtime_error(std::string("launch of conv5x5_wgrad_win failed: ") + cudaGetErrorString(e));
    count_kernel_launch();
    return;
  }
  conv5x5_wgrad_win_kernel<<<grid, Cfg::kThreads, Cfg::kSmem, st>>>(tm_x, tm_dy, scr.partials, B, nullptr, nullptr, nullptr, GridSync{nullptr, nullptr});
  check_launch("conv5x5_wgrad_win");
  wgrad_win_fold_kernel<<<401, 256, 0, st>>>(scr.partials, grid, dysum, B, dw, db);
  check_launch("wgrad_win_fold");
}

void launch_gemm_tf32_tcgen05(const float* a, const float* b, float* d, int M, int N, int K, cudaStream_t st) {
  if (N % 16 != 0 || N < 16 || N > 256) throw std::invalid_argument("gemm_tf32_tcgen05: N must be a multiple of 16 in [16, 256]");
  if (K % 4 != 0 || K < 4) throw std::invalid_argument("gemm_tf32_tcgen05: K must be a positive multiple of 4 (16-byte rows for TMA)");
  CUtensorMap tm_a = make_tmap_2d(a, static_cast<uint64_t>(K), static_cast<uint64_t>(M), kChunkK, kTileM);
  const int mtiles = (M + kTileM - 1) / kTileM;
#define PDT_GEMM_CASE(NB)                                                                    \
  if (N <= NB || NB == 64) {                                                                 \
    CUtensorMap tm_b = make_tmap_2d(b, static_cast<uint64_t>(K), static_cast<uint64_t>(N), kChunkK, NB); \
    auto kern = gemm_tf32_umma_kernel<NB>;                                                   \
    opt_in_smem(kern, GemmCfg<NB>::kSmem);                                                   \
    kern<<<dim3(mtiles, (N + NB - 1) / NB), 160, GemmCfg<NB>::kSmem, st>>>(tm_a, tm_b, d, M, N, K); \
    check_launch("gemm_tf32_umma");                                                          \
    return;                                                                                  \
  }
  PDT_GEMM_CASE(16)
  PDT_GEMM_CASE(32)
  PDT_GEMM_CASE(64)
#undef PDT_GEMM_CASE
}

void launch_umma_rowshift_probe(const float* a, const float* b, float* d, int rowb, int shift, int mode, cudaStream_t st) {
  if (rowb != 64 && rowb != 128) throw std::invalid_argument("umma_rowshift_probe: row bytes must be 64 or 128");
  if (shift < 0 || shift > 128) throw std::invalid_argument("umma_rowshift_probe: shift must be in [0, 128]");
  const int kf = rowb / 4;
  const CUtensorMapSwizzle sw = rowb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUtensorMap tm_a = make_tmap_2d(a, kf, 256, kf, 256, sw);
  CUtensorMap tm_b = make_tmap_2d(b, kf, 32, kf, 32, sw);
  const size_t smem = 1024 + 256 * static_cast<size_t>(rowb) + 4096 + 256;
  if (rowb == 128) {
    opt_in_smem(umma_rowshift_probe_kernel<128>, smem);
    umma_rowshift_probe_kernel<128><<<1, 128, smem, st>>>(tm_a, tm_b, d, shift, mode);
  } else {
    opt_in_smem(umma_rowshift_probe_kernel<64>, smem);
    umma_rowshift_probe_kernel<64><<<1, 128, smem, st>>>(tm_a, tm_b, d, shift, mode);
  }
  check_launch("umma_rowshift_probe");
}

}  // namespace pdt
