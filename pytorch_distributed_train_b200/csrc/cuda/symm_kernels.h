// Host-callable launchers for the NVLink collective kernels (implemented in symm_kernels.cu).
// No torch types here: raw pointers, byte offsets into the symmetric heap, a CUDA stream.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>

#include "symm_device.h"

namespace pdt {

// Must match pdt::DType / pdt::ReduceOp (csrc/cpu/cpu_backend.h).  The reducing launchers take AVG as SUM (the caller passes
// 1/world in `scale`), reject a scale != 1 on integer and bool types, run SUM / MAX on bool as logical OR and PRODUCT / MIN as
// logical AND, and reject AVG on bool.  MIN / MAX propagate NaN from any rank.
enum SymmDType : int { SD_F32 = 0, SD_F64 = 1, SD_F16 = 2, SD_BF16 = 3, SD_I8 = 4, SD_U8 = 5, SD_I32 = 6, SD_I64 = 7, SD_BOOL = 8, SD_I16 = 9 };
enum SymmOp : int { SO_SUM = 0, SO_AVG = 1, SO_PROD = 2, SO_MIN = 3, SO_MAX = 4, SO_BAND = 5, SO_BOR = 6, SO_BXOR = 7 };

struct SymmLaunchCfg {
  int blocks = 0;    // 0 = auto
  int threads = 0;   // 0 = auto
};

// out[i] = scale * reduce_r(in_r[i]).  `in`/`out` are ordinary local device pointers (may alias,
// need not live in the heap).  Every rank pushes its vector into slot[rank] of every peer's staging
// area at `stage_off` (P2P stores, or one multimem.st when use_mc), one cross-GPU barrier, then a
// local rank-ordered reduction ⇒ bitwise identical results on all ranks.  Staging must hold
// world × round_up(nbytes,16) bytes and alternate between two halves call to call.
void launch_allreduce_oneshot_push(const SymmDev& d, const void* in, void* out, size_t stage_off, size_t count,
                                   int dtype, int op, double scale, bool use_mc, SymmLaunchCfg cfg, cudaStream_t s);

// In-place on a symmetric buffer at heap offset `buf_off` (same offset on every rank):
// reduce-scatter (rank r owns slice r) + all-gather.  nvls=true: multimem.ld_reduce +
// multimem.st through the switch (f32/f16/bf16 SUM only, 2 barriers); otherwise P2P loads
// (3 barriers).
void launch_allreduce_twoshot(const SymmDev& d, size_t buf_off, size_t count, int dtype, int op, double scale, bool nvls,
                              SymmLaunchCfg cfg, cudaStream_t s);

// dst (local pointer) <- nbytes at heap offset src_off of rank `root`.  exit_barrier: the source
// may be overwritten right after the kernel (false when the source is double-buffered staging).
void launch_broadcast_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, int root, bool exit_barrier,
                           SymmLaunchCfg cfg, cudaStream_t s);
// dst[r*dst_stride ...] <- rank r's nbytes at heap offset src_off, for all r.
void launch_allgather_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, size_t dst_stride, bool exit_barrier,
                           SymmLaunchCfg cfg, cudaStream_t s);
// dst[r*stride ...] <- nbytes of rank r's block [my_rank] (sources hold world blocks, `stride` apart).
void launch_alltoall_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, size_t stride, bool exit_barrier,
                          SymmLaunchCfg cfg, cudaStream_t s);
// Every rank has parked total_vec 16-byte vectors at heap offset `stage_off`; after one barrier this rank reduces
// vectors [begin_vec, begin_vec + count_vec) over all ranks (rank order) into `out` (local pointer; count_vec may be 0).
void launch_reduce_pull(const SymmDev& d, size_t stage_off, size_t begin_vec, size_t count_vec, size_t total_vec, void* out, int dtype, int op,
                        double scale, SymmLaunchCfg cfg, cudaStream_t s);
// Device-signalled point-to-point chunk (see p2p_send_kernel): `slot_off` is the heap offset of the (sender → receiver)
// slot inside the RECEIVER's heap, `seq` the pair's chunk sequence number (1, 2, …; same on both ends).
constexpr int kSymmP2PBlocks = 16;
void launch_p2p_send(const SymmDev& d, const void* src, size_t nbytes, int dst_rank, size_t slot_off, unsigned int seq, cudaStream_t s);
void launch_p2p_recv(const SymmDev& d, void* dst, size_t nbytes, int src_rank, size_t slot_off, unsigned int seq, cudaStream_t s);
void launch_barrier(const SymmDev& d, cudaStream_t s);

// Fused: mean-allreduce of a flat fp32 gradient vector (one-shot push) + SGD update of the flat
// fp32 parameter vector with the same layout:  g <- mean_r(g_r);  p <- p - lr * (g [+ wd*p]).
// The grad allreduce and the optimizer step of a small model in ONE launch.  Optional rider: `bcast_bytes` of
// `bcast_buf` (a local pointer, same meaning on every rank) are replaced by `bcast_root`'s contents, staged behind
// the world gradient slots (staging must hold world × count × 4 + bcast_bytes).
void launch_allreduce_sgd_oneshot(const SymmDev& d, float* grad, float* param, float* momentum_buf, size_t stage_off,
                                  size_t count, float scale, const float* lr_dev, float lr, float momentum, float dampening,
                                  float weight_decay, bool nesterov, bool first_step, bool use_mc, SymmLaunchCfg cfg,
                                  cudaStream_t s, void* bcast_buf = nullptr, size_t bcast_bytes = 0, int bcast_root = 0);

}  // namespace pdt
