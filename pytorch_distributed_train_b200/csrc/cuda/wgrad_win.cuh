// conv2 (16→32, 5×5) weight gradient of one image in the "window" formulation, shared by the stand-alone kernel
// (conv_tcgen05.cu) and the layer-1 backward kernel that carries it along (fused_convnet.cu):
//   dWᵀ[(kh, kw, ci)][co] = Σ_P xpad[P + (kh−2)·18 + (kw−2)][ci] · dypad[P][co]
// over the 256 padded positions P from the first interior one.  Two horizontally adjacent taps of one position are 32
// contiguous floats of the NHWC frame, so a 32-row "atom" of the M dimension (tap pair × 16 channels) is one row of the
// overlapping-row view of the frame (row r = positions r, r+1).  Both operands have the reduction dimension (positions)
// outermost — MN-major — which TF32 wgmma does not accept, so this is warp-level mma.sync m16n8k8 reading the swizzled
// tiles directly.  The im2col weight gradient (conv_tcgen05.cu) uses the same per-warp step.
// Trade-off: on the previous (Blackwell) generation these MMAs ran asynchronously from one extra warp while the layer-1
// SIMT warps worked; here they are synchronous warp-level MMAs.  In the layer-1 backward kernel they run on 15 of its warps
// just before the second grid barrier, i.e. on the critical path of the step: about 13 µs of the ~40 µs layer-1 backward
// kernel and of the ~99 µs replayed step at batch 100 (H100 SXM, 700 W limit; tools/fused_trace.py).  Feeding wgmma instead
// would need a K-major (transposed) copy of both operands in shared memory.
#pragma once
#include <cstdint>

namespace pdt {
namespace ptx {

__device__ __forceinline__ uint32_t f32_to_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}
// D(16×8) += A(16×8, row) · B(8×8, col); fragments per the PTX ISA m16n8k8 .tf32 layout
__device__ __forceinline__ void mma_m16n8k8_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Operand tiles are swizzled: element (row r, column c) of a tile with PITCH floats per row sits at r·PITCH + (c ^ 4·(r mod 8)),
// i.e. the 16-byte chunk index is XORed with r mod 8 — for 128-byte rows this is TMA's SWIZZLE_128B (tile 1024-byte aligned).
// The four rows a fragment load touches differ in r mod 8, so the loads below are free of bank conflicts.

// One warp: acc (32 rows of an atom × 32 output channels) += Σ_{P < KPOS} x[P][i] · dy[P][co], where x[P][i] is element
// (xrow0 + P, xcol0 + i) of the swizzled tile xs (the window kernels: row xrow0 + P of the overlapping-row view) and dy[P][co]
// element (dyrow0 + P, co) of the swizzled tile dys ([rows][32]).  acc[j][nt][e] holds D[16j + g + 8·(e >> 1)][8nt + 2·t4 + (e & 1)]
// with g = lane / 4, t4 = lane % 4.  UNROLL: K steps per loop iteration (1 where registers are scarce).
template <int KPOS = 256, int XPITCH = 32, int UNROLL = 2>
__device__ __forceinline__ void wgrad_win_atom(float (&acc)[2][4][4], const float* xs, int xrow0, int xcol0, const float* dys, int dyrow0,
                                               int lane) {
  const int g = lane >> 2, t4 = lane & 3;
  // p0 advances by 8 rows, so the swizzle of this lane's rows is loop-invariant; row + 4 flips bit 2 of r mod 8 (XOR 16 floats)
  const int kx = ((xrow0 + t4) & 7) << 2, kd = ((dyrow0 + t4) & 7) << 2;
  const int c0 = (xcol0 + g) ^ kx, c1 = (xcol0 + g + 8) ^ kx, c2 = (xcol0 + g + 16) ^ kx, c3 = (xcol0 + g + 24) ^ kx;
  const float* xa = xs + (xrow0 + t4) * XPITCH;
  const float* da = dys + (dyrow0 + t4) * 32;
#pragma unroll UNROLL
  for (int p0 = 0; p0 < KPOS; p0 += 8, xa += 8 * XPITCH, da += 8 * 32) {
    const float* xb = xa + 4 * XPITCH;
    const float* db = da + 4 * 32;
    uint32_t b[4][2];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      b[nt][0] = f32_to_tf32(da[(8 * nt + g) ^ kd]);
      b[nt][1] = f32_to_tf32(db[(8 * nt + g) ^ kd ^ 16]);
    }
    const uint32_t a0[4] = {f32_to_tf32(xa[c0]), f32_to_tf32(xa[c1]), f32_to_tf32(xb[c0 ^ 16]), f32_to_tf32(xb[c1 ^ 16])};
    const uint32_t a1[4] = {f32_to_tf32(xa[c2]), f32_to_tf32(xa[c3]), f32_to_tf32(xb[c2 ^ 16]), f32_to_tf32(xb[c3 ^ 16])};
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      mma_m16n8k8_tf32(acc[0][nt], a0, b[nt][0], b[nt][1]);
      mma_m16n8k8_tf32(acc[1][nt], a1, b[nt][0], b[nt][1]);
    }
  }
}

// Write the 32 × 32 atom accumulator to out[row][co] (row pitch 32 floats, out = the atom's first row); rows ≥ rows_valid
// are skipped.
__device__ __forceinline__ void wgrad_win_atom_store(const float (&acc)[2][4][4], float* out, int lane, int rows_valid = 32) {
  const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      if (16 * j + g < rows_valid)
        *reinterpret_cast<float2*>(out + (16 * j + g) * 32 + 8 * nt + 2 * t4) = make_float2(acc[j][nt][0], acc[j][nt][1]);
      if (16 * j + g + 8 < rows_valid)
        *reinterpret_cast<float2*>(out + (16 * j + g + 8) * 32 + 8 * nt + 2 * t4) = make_float2(acc[j][nt][2], acc[j][nt][3]);
    }
}

}  // namespace ptx
}  // namespace pdt
