// sm_90a collective kernels over NVLink peer / multicast memory.
//
// These are the product's communication path (BASELINE.json north star): the DDP
// bucket allreduce, the per-step BatchNorm-buffer broadcast and SyncBatchNorm's statistic
// exchange all run here, as plain kernel launches with device-side cross-GPU barriers, so they
// can be issued from an autograd hook on a side stream *and* captured in a CUDA graph.  What the
// reference stack does with NCCL (ref: ddp_example.py:64 → c10d reducer → ncclAllReduce) plus
// 10 per-parameter scale kernels is one launch here: flatten is free (gradients live in the
// bucket), the 1/world scale — and optionally the SGD update — are fused into the reduce.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>
#include <stdexcept>
#include <string>

#include "cuda_utils.h"
#include "symm_kernels.h"

namespace pdt {

namespace {

// ---- element traits -----------------------------------------------------------------------------
template <typename T> struct Acc { using type = T; };
template <> struct Acc<__half> { using type = float; };
template <> struct Acc<__nv_bfloat16> { using type = float; };

template <typename T> __device__ __forceinline__ typename Acc<T>::type to_acc(T v) { return v; }
template <> __device__ __forceinline__ float to_acc<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_acc<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_acc(typename Acc<T>::type v) { return v; }
template <> __device__ __forceinline__ __half from_acc<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_acc<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// MIN / MAX propagate a NaN whichever rank holds it (torch.minimum / torch.maximum): `b != b` is false for integers.
template <typename A, int OP> __device__ __forceinline__ A combine(A a, A b) {
  if constexpr (OP == SO_SUM || OP == SO_AVG) return a + b;
  else if constexpr (OP == SO_PROD) return a * b;
  else if constexpr (OP == SO_MIN) return (b < a || b != b) ? b : a;
  else if constexpr (OP == SO_MAX) return (b > a || b != b) ? b : a;
  else if constexpr (OP == SO_BAND) { if constexpr (std::is_integral<A>::value) return a & b; else return a; }
  else if constexpr (OP == SO_BOR) { if constexpr (std::is_integral<A>::value) return a | b; else return a; }
  else { if constexpr (std::is_integral<A>::value) return a ^ b; else return a; }
}

// The launchers take the scale as a double and reject a scale != 1 on integer types; the kernels convert it once to the
// accumulator type, so an fp64 reduction is scaled by the fp64 value.
template <typename A> __device__ __forceinline__ A apply_scale(A v, A scale) {
  if constexpr (std::is_floating_point<A>::value) return v * scale;
  else return v;
}

__device__ __forceinline__ uint4 ld_vec(const void* p) { return *reinterpret_cast<const uint4*>(p); }
// peer / staging reads: bypass L1 (another GPU's writes must not be served from a stale line)
__device__ __forceinline__ uint4 ld_vec_nc(const void* p) {
  uint4 v;
  asm volatile("ld.global.relaxed.sys.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_vec(void* p, uint4 v) { *reinterpret_cast<uint4*>(p) = v; }
__device__ __forceinline__ void st_vec_sys(void* p, uint4 v) {
  asm volatile("st.global.relaxed.sys.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void mc_st_vec(void* p, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(__uint_as_float(v.x)),
               "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)), "f"(__uint_as_float(v.w))
               : "memory");
}

template <typename T> struct VecOf { static constexpr int N = 16 / sizeof(T); };

template <typename T, int OP>
__device__ __forceinline__ void acc_init(typename Acc<T>::type (&a)[VecOf<T>::N], uint4 v) {
  const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
  for (int k = 0; k < VecOf<T>::N; ++k) a[k] = to_acc<T>(e[k]);
}
template <typename T, int OP>
__device__ __forceinline__ void acc_add(typename Acc<T>::type (&a)[VecOf<T>::N], uint4 v) {
  const T* e = reinterpret_cast<const T*>(&v);
#pragma unroll
  for (int k = 0; k < VecOf<T>::N; ++k) a[k] = combine<typename Acc<T>::type, OP>(a[k], to_acc<T>(e[k]));
}
template <typename T>
__device__ __forceinline__ uint4 acc_pack(typename Acc<T>::type (&a)[VecOf<T>::N], typename Acc<T>::type scale) {
  uint4 v;
  T* e = reinterpret_cast<T*>(&v);
#pragma unroll
  for (int k = 0; k < VecOf<T>::N; ++k) e[k] = from_acc<T>(apply_scale(a[k], scale));
  return v;
}

// ---- one-shot push allreduce -----------------------------------------------------------------------
// nvec: number of 16-byte vectors (host pads the tail into a scratch vector); slot stride = nvec*16.
template <typename T, int OP, bool MC>
__global__ void __launch_bounds__(512) allreduce_oneshot_push_kernel(const __grid_constant__ SymmDev d, const uint4* __restrict__ in, uint4* out,
                                                                      size_t stage_off, size_t nvec, double scale) {
  SymmEpoch ep(d, blockIdx.x);
  const auto sc = static_cast<typename Acc<T>::type>(scale);
  const size_t slot_bytes = nvec * 16;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  // phase 1: publish my vector into slot[rank] on every GPU
  for (size_t i = first; i < nvec; i += stride) {
    uint4 v = ld_vec(in + i);
    const size_t off = stage_off + static_cast<size_t>(d.rank) * slot_bytes + i * 16;
    if constexpr (MC) {
      mc_st_vec(d.mc + off, v);
    } else {
#pragma unroll
      for (int r = 0; r < kSymmMaxWorld; ++r)
        if (r < d.world) st_vec_sys(d.peer[r] + off, v);
    }
  }
  symm_barrier_block(d, blockIdx.x, ep.next());
  // phase 2: every slot is now complete locally; reduce in rank order
  const char* base = d.peer[d.rank] + stage_off;
  for (size_t i = first; i < nvec; i += stride) {
    typename Acc<T>::type a[VecOf<T>::N];
    acc_init<T, OP>(a, ld_vec_nc(base + i * 16));
    for (int r = 1; r < d.world; ++r) acc_add<T, OP>(a, ld_vec_nc(base + static_cast<size_t>(r) * slot_bytes + i * 16));
    st_vec(out + i, acc_pack<T>(a, sc));
  }
  ep.commit(d, blockIdx.x);
}

// ---- fused one-shot allreduce + SGD (+ optional broadcast) ---------------------------------------------------
// The DDP reducer's per-chunk launch when the optimizer is fused into the reduction.  One cross-GPU barrier:
//   push my gradient chunk into slot[rank] of every peer's staging half  (P2P stores, or one multimem.st)
//   [root only] push `bc_nvec` vectors of the module-buffer arena into every peer's staging, behind the slots
//   barrier
//   rank-ordered sum × scale → averaged gradient (kept in `grad`, like the reference's allreduce) → SGD update
//   copy the broadcast payload from my staging into my buffer arena
// The broadcast goes through staging, not straight into the peers' arenas: a slower peer may still be running the
// forward pass that read-modify-writes its own running statistics.
template <bool MC>
__global__ void __launch_bounds__(512) allreduce_sgd_oneshot_kernel(const __grid_constant__ SymmDev d, float4* grad, float4* param, float4* mom,
                                                                    size_t stage_off, size_t nvec, float scale,
                                                                    const float* lr_dev, float lr_host, float momentum,
                                                                    float dampening, float wd, int nesterov, int first_step,
                                                                    uint4* bc_buf, size_t bc_nvec, int bc_root) {
  SymmEpoch ep(d, blockIdx.x);
  const size_t slot_bytes = nvec * 16;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (size_t i = first; i < nvec; i += stride) {
    uint4 v = ld_vec(grad + i);
    const size_t off = stage_off + static_cast<size_t>(d.rank) * slot_bytes + i * 16;
    if constexpr (MC) {
      mc_st_vec(d.mc + off, v);
    } else {
#pragma unroll
      for (int r = 0; r < kSymmMaxWorld; ++r)
        if (r < d.world) st_vec_sys(d.peer[r] + off, v);
    }
  }
  const size_t bc_off = stage_off + static_cast<size_t>(d.world) * slot_bytes;
  if (bc_nvec && d.rank == bc_root) {
    for (size_t i = first; i < bc_nvec; i += stride) {
      uint4 v = ld_vec(bc_buf + i);
      if constexpr (MC) {
        mc_st_vec(d.mc + bc_off + i * 16, v);
      } else {
#pragma unroll
        for (int r = 0; r < kSymmMaxWorld; ++r)
          if (r < d.world) st_vec_sys(d.peer[r] + bc_off + i * 16, v);
      }
    }
  }
  const float lr = lr_dev ? *lr_dev : lr_host;
  symm_barrier_block(d, blockIdx.x, ep.next());
  const char* base = d.peer[d.rank] + stage_off;
  for (size_t i = first; i < nvec; i += stride) {
    float a[4];
    acc_init<float, SO_SUM>(a, ld_vec_nc(base + i * 16));
    for (int r = 1; r < d.world; ++r) acc_add<float, SO_SUM>(a, ld_vec_nc(base + static_cast<size_t>(r) * slot_bytes + i * 16));
    float4 g = make_float4(a[0] * scale, a[1] * scale, a[2] * scale, a[3] * scale);
    grad[i] = g;  // .grad holds the averaged gradient, as after the reference's allreduce
    float4 p = param[i];
    if (wd != 0.f) { g.x += wd * p.x; g.y += wd * p.y; g.z += wd * p.z; g.w += wd * p.w; }
    if (momentum != 0.f) {
      float4 b;
      if (first_step) b = g;
      else {
        b = mom[i];
        const float k = 1.f - dampening;
        b.x = momentum * b.x + k * g.x; b.y = momentum * b.y + k * g.y; b.z = momentum * b.z + k * g.z; b.w = momentum * b.w + k * g.w;
      }
      mom[i] = b;
      if (nesterov) { g.x += momentum * b.x; g.y += momentum * b.y; g.z += momentum * b.z; g.w += momentum * b.w; }
      else g = b;
    }
    p.x -= lr * g.x; p.y -= lr * g.y; p.z -= lr * g.z; p.w -= lr * g.w;
    param[i] = p;
  }
  if (bc_nvec && d.rank != bc_root) {
    const char* src = d.peer[d.rank] + bc_off;
    for (size_t i = first; i < bc_nvec; i += stride) st_vec(bc_buf + i, ld_vec_nc(src + i * 16));
  }
  ep.commit(d, blockIdx.x);
}

// ---- two-shot allreduce, in place on a symmetric buffer ---------------------------------------------
template <typename T> __device__ __forceinline__ uint4 nvls_ld_reduce(const void* p);
template <> __device__ __forceinline__ uint4 nvls_ld_reduce<float>(const void* p) {
  float4 f = multimem_ld_reduce_f32x4(p);
  return make_uint4(__float_as_uint(f.x), __float_as_uint(f.y), __float_as_uint(f.z), __float_as_uint(f.w));
}
template <> __device__ __forceinline__ uint4 nvls_ld_reduce<__half>(const void* p) { return multimem_ld_reduce_f16x8(p); }
template <> __device__ __forceinline__ uint4 nvls_ld_reduce<__nv_bfloat16>(const void* p) { return multimem_ld_reduce_bf16x8(p); }

template <typename T, int OP, bool NVLS>
__global__ void __launch_bounds__(512) allreduce_twoshot_kernel(const __grid_constant__ SymmDev d, size_t buf_off, size_t nvec, double scale) {
  SymmEpoch ep(d, blockIdx.x);
  const auto sc = static_cast<typename Acc<T>::type>(scale);
  const size_t per = (nvec + d.world - 1) / d.world;  // vectors per slice
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  symm_barrier_block(d, blockIdx.x, ep.next());  // every rank's input is in place
  {
    const size_t lo = per * d.rank, hi = min(nvec, lo + per);
    for (size_t j = first; lo + j < hi; j += stride) {
      const size_t off = buf_off + (lo + j) * 16;
      if constexpr (NVLS) {
        uint4 v = nvls_ld_reduce<T>(d.mc + off);
        if (scale != 1.0) {
          typename Acc<T>::type a[VecOf<T>::N];
          acc_init<T, OP>(a, v);
          v = acc_pack<T>(a, sc);
        }
        mc_st_vec(d.mc + off, v);  // lands in every rank's buffer
      } else {
        typename Acc<T>::type a[VecOf<T>::N];
        acc_init<T, OP>(a, ld_vec_nc(d.peer[0] + off));
        for (int r = 1; r < d.world; ++r) acc_add<T, OP>(a, ld_vec_nc(d.peer[r] + off));
        st_vec(d.peer[d.rank] + off, acc_pack<T>(a, sc));
      }
    }
  }
  symm_barrier_block(d, blockIdx.x, ep.next());  // all slices reduced (NVLS: and delivered)
  if constexpr (!NVLS) {
    for (int k = 1; k < d.world; ++k) {
      const int q = (d.rank + k) % d.world;  // stagger peers so links are used evenly
      const size_t lo = per * q, hi = min(nvec, lo + per);
      for (size_t j = first; lo + j < hi; j += stride) {
        const size_t off = buf_off + (lo + j) * 16;
        st_vec(d.peer[d.rank] + off, ld_vec_nc(d.peer[q] + off));
      }
    }
    symm_barrier_block(d, blockIdx.x, ep.next());  // nobody overwrites a slice a peer still reads
  }
  ep.commit(d, blockIdx.x);
}

// ---- reduce-scatter / rooted reduce: the first half of a two-shot ------------------------------------------------
// Every rank has parked its whole contribution (nvec 16-byte vectors) at `stage_off` of its own heap.  After one
// barrier a rank reduces vectors [begin, begin + count) over all ranks, in rank order, straight out of the peers'
// memory, into `out` — reduce_scatter: everybody takes its slice (inbound (N−1)/N·S per GPU, the minimum);
// reduce(root): the root takes everything, the others only attend the barrier.
template <typename T, int OP>
__global__ void __launch_bounds__(512) reduce_pull_kernel(const __grid_constant__ SymmDev d, size_t stage_off, size_t begin, size_t count, uint4* out,
                                                          double scale) {
  SymmEpoch ep(d, blockIdx.x);
  const auto sc = static_cast<typename Acc<T>::type>(scale);
  symm_barrier_block(d, blockIdx.x, ep.next());
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < count; i += stride) {
    const size_t off = stage_off + (begin + i) * 16;
    typename Acc<T>::type a[VecOf<T>::N];
    acc_init<T, OP>(a, ld_vec_nc(d.peer[0] + off));
    for (int r = 1; r < d.world; ++r) acc_add<T, OP>(a, ld_vec_nc(d.peer[r] + off));
    st_vec(out + i, acc_pack<T>(a, sc));
  }
  ep.commit(d, blockIdx.x);
}

// ---- pull-style data movement -------------------------------------------------------------------------
// mode 0: broadcast (root → dst), 1: allgather, 2: alltoall
__global__ void __launch_bounds__(512) pull_kernel(const __grid_constant__ SymmDev d, size_t src_off, char* dst, size_t nbytes, size_t dst_stride,
                                                   int root, int mode, int exit_barrier) {
  SymmEpoch ep(d, blockIdx.x);
  symm_barrier_block(d, blockIdx.x, ep.next());
  if (dst == nullptr) {   // a rank that only attends (gather on a non-root rank): barriers, no copies
    if (exit_barrier) symm_barrier_block(d, blockIdx.x, ep.next());
    ep.commit(d, blockIdx.x);
    return;
  }
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nvec = nbytes / 16, tail = nbytes % 16;
  const int n_src = mode == 0 ? 1 : d.world;
  for (int k = 0; k < n_src; ++k) {
    const int q = mode == 0 ? root : (d.rank + k) % d.world;
    if (mode == 0 && d.rank == root && dst == d.peer[root] + src_off) break;  // in place at the root
    const char* src = d.peer[q] + src_off + (mode == 2 ? static_cast<size_t>(d.rank) * dst_stride : 0);
    char* out = dst + (mode == 0 ? 0 : static_cast<size_t>(q) * dst_stride);
    const uintptr_t mis = reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(out);
    if ((mis & 15) == 0) {
      for (size_t i = first; i < nvec; i += stride) st_vec(out + i * 16, ld_vec_nc(src + i * 16));
      if (tail && blockIdx.x == 0 && threadIdx.x < tail)
        out[nvec * 16 + threadIdx.x] = *reinterpret_cast<const volatile char*>(src + nvec * 16 + threadIdx.x);
    } else if (((mis | nbytes) & 3) == 0) {  // small / oddly-strided slices (e.g. 5 floats per rank): word copies
      for (size_t i = first; i < nbytes / 4; i += stride)
        reinterpret_cast<uint32_t*>(out)[i] = *reinterpret_cast<const volatile uint32_t*>(src + i * 4);
    } else {
      for (size_t i = first; i < nbytes; i += stride) out[i] = *reinterpret_cast<const volatile char*>(src + i);
    }
  }
  if (exit_barrier) symm_barrier_block(d, blockIdx.x, ep.next());
  ep.commit(d, blockIdx.x);
}

// ---- point-to-point: device-signalled, no host round trip ---------------------------------------------------------------
// A message travels in chunks through a slot of the RECEIVER's heap reserved for this sender.  Per (pair, block) there
// are two monotonically increasing flags: `ready` in the receiver's signal pad (written by the sender after its
// stores, release.sys) and `ack` in the sender's pad (written by the receiver once the chunk has been copied out).
// Chunk k of the pair carries sequence number k (host-side counters on both ends, identical chunking), so nothing is
// ever reset: send(k) waits for ack ≥ k−1, writes, publishes ready = k; recv(k) waits for ready ≥ k, copies, acks k.
// Both are ordinary kernels on the caller's stream.  Rows [0, kP2PBlocks) of the channel hold `ready`, rows
// [kP2PAckRow, …) hold `ack`.
constexpr int kP2PAckRow = 80;

__device__ __forceinline__ void p2p_wait(const SymmDev& d, const uint32_t* flag, uint32_t want, int peer) {
  uint32_t v = ld_acquire_sys(flag);
  if (static_cast<int32_t>(v - want) < 0) {
    const unsigned long long t0 = globaltimer_ns();
    int spins = 0;
    while (static_cast<int32_t>((v = ld_acquire_sys(flag)) - want) < 0) {
      if (++spins > 64) {
        __nanosleep(40);
        if ((spins & 1023) == 0 && globaltimer_ns() - t0 > d.timeout_ns) symm_trap_timeout(d, peer, want, v);
      }
    }
  }
}

__global__ void __launch_bounds__(512) p2p_send_kernel(const __grid_constant__ SymmDev d, const char* __restrict__ src, size_t nbytes, int dst_rank,
                                                       size_t slot_off, uint32_t seq) {
  if (threadIdx.x == 0) p2p_wait(d, symm_flag_row(d, d.rank, kP2PAckRow + blockIdx.x) + dst_rank, seq - 1, dst_rank);   // previous chunk consumed
  __syncthreads();
  char* out = d.peer[dst_rank] + slot_off;
  const size_t nvec = nbytes / 16, tail = nbytes % 16;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x, first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
    for (size_t i = first; i < nvec; i += stride) st_vec_sys(out + i * 16, ld_vec(src + i * 16));
    if (blockIdx.x == 0 && threadIdx.x < tail) out[nvec * 16 + threadIdx.x] = src[nvec * 16 + threadIdx.x];
  } else {
    for (size_t i = first; i < nbytes; i += stride) out[i] = src[i];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(symm_flag_row(d, dst_rank, blockIdx.x) + d.rank, seq);
  }
}

__global__ void __launch_bounds__(512) p2p_recv_kernel(const __grid_constant__ SymmDev d, char* __restrict__ dst, size_t nbytes, int src_rank,
                                                       size_t slot_off, uint32_t seq) {
  if (threadIdx.x == 0) p2p_wait(d, symm_flag_row(d, d.rank, blockIdx.x) + src_rank, seq, src_rank);
  __syncthreads();
  const char* in = d.peer[d.rank] + slot_off;
  const size_t nvec = nbytes / 16, tail = nbytes % 16;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x, first = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    for (size_t i = first; i < nvec; i += stride) st_vec(dst + i * 16, ld_vec_nc(in + i * 16));
    if (blockIdx.x == 0 && threadIdx.x < tail) dst[nvec * 16 + threadIdx.x] = *reinterpret_cast<const volatile char*>(in + nvec * 16 + threadIdx.x);
  } else {
    for (size_t i = first; i < nbytes; i += stride) dst[i] = *reinterpret_cast<const volatile char*>(in + i);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();
    st_release_sys(symm_flag_row(d, src_rank, kP2PAckRow + blockIdx.x) + d.rank, seq);
  }
}

__global__ void barrier_kernel(const __grid_constant__ SymmDev d) {
  SymmEpoch ep(d, 0);
  symm_barrier_block(d, 0, ep.next());
  ep.commit(d, 0);
}

// ---- launch helpers -------------------------------------------------------------------------------------
int auto_blocks(size_t nvec, int threads, int cap) {
  size_t b = (nvec + static_cast<size_t>(threads) * 2 - 1) / (static_cast<size_t>(threads) * 2);
  return static_cast<int>(std::max<size_t>(1, std::min<size_t>(b, static_cast<size_t>(cap))));
}

// Which (dtype, op) pairs get a kernel.  SUM exists for every dtype (it is what DDP, SyncBatchNorm and the object
// collectives use); MIN / MAX / PROD for the 32/64-bit types; the bitwise ops for the integer types they are defined on.
// Everything else is rejected at dispatch instead of being instantiated (the full cross product was 210 kernels and a
// 9.7 MB object for combinations nothing ever calls).
template <typename T, int OP> constexpr bool op_supported() {
  if (OP == SO_SUM) return true;
  if (OP == SO_PROD || OP == SO_MIN || OP == SO_MAX)
    return std::is_same<T, float>::value || std::is_same<T, double>::value || std::is_same<T, int>::value || std::is_same<T, long long>::value;
  return std::is_same<T, int>::value || std::is_same<T, long long>::value || std::is_same<T, unsigned char>::value;
}

#define PDT_OP_CASE(T, OPC, ...)                                                                                      \
  {                                                                                                                   \
    constexpr int OP = OPC;                                                                                           \
    if constexpr (op_supported<T, OPC>()) { __VA_ARGS__; }                                                           \
    else throw std::invalid_argument("this reduce op is not implemented for this dtype on the NVLink backend");     \
    break;                                                                                                            \
  }
#define PDT_DISPATCH_OP(T, OPV, ...)                                  \
  switch (OPV) {                                                      \
    case SO_SUM: case SO_AVG: PDT_OP_CASE(T, SO_SUM, __VA_ARGS__)     \
    case SO_PROD: PDT_OP_CASE(T, SO_PROD, __VA_ARGS__)                \
    case SO_MIN: PDT_OP_CASE(T, SO_MIN, __VA_ARGS__)                  \
    case SO_MAX: PDT_OP_CASE(T, SO_MAX, __VA_ARGS__)                  \
    case SO_BAND: PDT_OP_CASE(T, SO_BAND, __VA_ARGS__)                \
    case SO_BOR: PDT_OP_CASE(T, SO_BOR, __VA_ARGS__)                  \
    case SO_BXOR: PDT_OP_CASE(T, SO_BXOR, __VA_ARGS__)                \
    default: throw std::invalid_argument("unsupported reduce op");    \
  }

#define PDT_DISPATCH_TYPE(DT, ...)                                             \
  switch (DT) {                                                                \
    case SD_F32: { using T = float; __VA_ARGS__; break; }                      \
    case SD_F64: { using T = double; __VA_ARGS__; break; }                     \
    case SD_F16: { using T = __half; __VA_ARGS__; break; }                     \
    case SD_BF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }             \
    case SD_I8: { using T = signed char; __VA_ARGS__; break; }                 \
    case SD_U8: case SD_BOOL: { using T = unsigned char; __VA_ARGS__; break; } \
    case SD_I16: { using T = short; __VA_ARGS__; break; }                      \
    case SD_I32: { using T = int; __VA_ARGS__; break; }                        \
    case SD_I64: { using T = long long; __VA_ARGS__; break; }                  \
    default: throw std::invalid_argument("unsupported dtype for NVLink collectives"); \
  }

// The op a launcher runs for (dtype, op), after rejecting what has no defined result.  A scale ≠ 1 on an integer type would be
// dropped (apply_scale), so it is an error.  On bool, SUM is logical OR and PRODUCT logical AND, as torch's NCCL backend maps them
// (to MAX / MIN); on 0/1 bytes MIN and MAX are AND and OR as well, and AVG has no bool result.
int checked_op(int dtype, int op, double scale) {
  const bool floating = dtype == SD_F32 || dtype == SD_F64 || dtype == SD_F16 || dtype == SD_BF16;
  if (scale != 1.0 && !floating) throw std::invalid_argument("a reduction scale is only defined for floating-point tensors");
  if (dtype != SD_BOOL) return op;
  switch (op) {
    case SO_SUM: case SO_MAX: case SO_BOR: return SO_BOR;
    case SO_PROD: case SO_MIN: case SO_BAND: return SO_BAND;
    case SO_BXOR: return SO_BXOR;
    default: throw std::invalid_argument("AVG is not defined for bool tensors");
  }
}

size_t elem_size(int dtype) {
  switch (dtype) {
    case SD_F32: case SD_I32: return 4;
    case SD_F64: case SD_I64: return 8;
    case SD_F16: case SD_BF16: case SD_I16: return 2;
    default: return 1;
  }
}

}  // namespace

void launch_allreduce_oneshot_push(const SymmDev& d, const void* in, void* out, size_t stage_off, size_t count, int dtype,
                                   int op, double scale, bool use_mc, SymmLaunchCfg cfg, cudaStream_t s) {
  const size_t nbytes = count * elem_size(dtype);
  if (nbytes % 16 != 0) throw std::invalid_argument("oneshot push: byte count must be a multiple of 16 (caller pads)");
  op = checked_op(dtype, op, scale);
  const size_t nvec = nbytes / 16;
  if (nvec == 0) return;
  const int threads = cfg.threads ? cfg.threads : 256;
  const int blocks = std::min(cfg.blocks ? cfg.blocks : auto_blocks(nvec, threads, 64), kSymmMaxBlocks);
  PDT_DISPATCH_TYPE(dtype, PDT_DISPATCH_OP(T, op, {
    if (use_mc) allreduce_oneshot_push_kernel<T, OP, true><<<blocks, threads, 0, s>>>(d, static_cast<const uint4*>(in), static_cast<uint4*>(out), stage_off, nvec, scale);
    else allreduce_oneshot_push_kernel<T, OP, false><<<blocks, threads, 0, s>>>(d, static_cast<const uint4*>(in), static_cast<uint4*>(out), stage_off, nvec, scale);
  }));
  check_launch("allreduce_oneshot_push");
}

void launch_allreduce_sgd_oneshot(const SymmDev& d, float* grad, float* param, float* momentum_buf, size_t stage_off,
                                  size_t count, float scale, const float* lr_dev, float lr, float momentum, float dampening,
                                  float weight_decay, bool nesterov, bool first_step, bool use_mc, SymmLaunchCfg cfg,
                                  cudaStream_t s, void* bcast_buf, size_t bcast_bytes, int bcast_root) {
  if (count % 4 != 0) throw std::invalid_argument("allreduce_sgd: element count must be a multiple of 4");
  if (bcast_bytes % 16 != 0) throw std::invalid_argument("allreduce_sgd: broadcast payload must be a multiple of 16 bytes");
  const size_t nvec = count / 4;
  if (nvec == 0) return;
  const int threads = cfg.threads ? cfg.threads : 256;
  const int blocks = std::min(cfg.blocks ? cfg.blocks : auto_blocks(nvec, threads, 64), kSymmMaxBlocks);
  const size_t bc_nvec = bcast_buf ? bcast_bytes / 16 : 0;
  if (use_mc)
    allreduce_sgd_oneshot_kernel<true><<<blocks, threads, 0, s>>>(d, reinterpret_cast<float4*>(grad), reinterpret_cast<float4*>(param),
                                                                  reinterpret_cast<float4*>(momentum_buf), stage_off, nvec, scale, lr_dev, lr,
                                                                  momentum, dampening, weight_decay, nesterov, first_step,
                                                                  static_cast<uint4*>(bcast_buf), bc_nvec, bcast_root);
  else
    allreduce_sgd_oneshot_kernel<false><<<blocks, threads, 0, s>>>(d, reinterpret_cast<float4*>(grad), reinterpret_cast<float4*>(param),
                                                                   reinterpret_cast<float4*>(momentum_buf), stage_off, nvec, scale, lr_dev, lr,
                                                                   momentum, dampening, weight_decay, nesterov, first_step,
                                                                   static_cast<uint4*>(bcast_buf), bc_nvec, bcast_root);
  check_launch("allreduce_sgd_oneshot");
}

void launch_allreduce_twoshot(const SymmDev& d, size_t buf_off, size_t count, int dtype, int op, double scale, bool nvls,
                              SymmLaunchCfg cfg, cudaStream_t s) {
  const size_t nbytes = count * elem_size(dtype);
  if (nbytes % 16 != 0 || buf_off % 16 != 0) throw std::invalid_argument("twoshot: buffer must be 16-byte aligned and sized");
  op = checked_op(dtype, op, scale);
  const size_t nvec = nbytes / 16;
  if (nvec == 0) return;
  const int threads = cfg.threads ? cfg.threads : 512;
  const size_t per = (nvec + d.world - 1) / d.world;
  // the two-shot kernels use at most one CTA per SM
  const int blocks = std::min(cfg.blocks ? cfg.blocks : auto_blocks(per, threads, sm_count()), kSymmMaxBlocks);
  if (nvls) {
    if (!d.mc) throw std::runtime_error("twoshot nvls requested but the heap has no multicast mapping");
    if (!(op == SO_SUM || op == SO_AVG)) throw std::invalid_argument("NVLS reduction supports SUM only");
    switch (dtype) {
      case SD_F32: allreduce_twoshot_kernel<float, SO_SUM, true><<<blocks, threads, 0, s>>>(d, buf_off, nvec, scale); break;
      case SD_F16: allreduce_twoshot_kernel<__half, SO_SUM, true><<<blocks, threads, 0, s>>>(d, buf_off, nvec, scale); break;
      case SD_BF16: allreduce_twoshot_kernel<__nv_bfloat16, SO_SUM, true><<<blocks, threads, 0, s>>>(d, buf_off, nvec, scale); break;
      default: throw std::invalid_argument("NVLS reduction supports f32/f16/bf16 only");
    }
  } else {
    PDT_DISPATCH_TYPE(dtype, PDT_DISPATCH_OP(T, op, { allreduce_twoshot_kernel<T, OP, false><<<blocks, threads, 0, s>>>(d, buf_off, nvec, scale); }));
  }
  check_launch("allreduce_twoshot");
}

static void launch_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, size_t dst_stride, int root, int mode,
                        bool exit_barrier, SymmLaunchCfg cfg, cudaStream_t s) {
  const int threads = cfg.threads ? cfg.threads : 512;
  const int blocks = std::min(cfg.blocks ? cfg.blocks : auto_blocks(nbytes / 16 + 1, threads, 64), kSymmMaxBlocks);
  pull_kernel<<<blocks, threads, 0, s>>>(d, src_off, static_cast<char*>(dst), nbytes, dst_stride, root, mode, exit_barrier ? 1 : 0);
  check_launch("pull_kernel");
}
void launch_broadcast_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, int root, bool exit_barrier,
                           SymmLaunchCfg cfg, cudaStream_t s) {
  launch_pull(d, src_off, dst, nbytes, 0, root, 0, exit_barrier, cfg, s);
}
void launch_allgather_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, size_t dst_stride, bool exit_barrier,
                           SymmLaunchCfg cfg, cudaStream_t s) {
  launch_pull(d, src_off, dst, nbytes, dst_stride, 0, 1, exit_barrier, cfg, s);
}
void launch_alltoall_pull(const SymmDev& d, size_t src_off, void* dst, size_t nbytes, size_t stride, bool exit_barrier,
                          SymmLaunchCfg cfg, cudaStream_t s) {
  launch_pull(d, src_off, dst, nbytes, stride, 0, 2, exit_barrier, cfg, s);
}
void launch_reduce_pull(const SymmDev& d, size_t stage_off, size_t begin_vec, size_t count_vec, size_t total_vec, void* out, int dtype, int op,
                        double scale, SymmLaunchCfg cfg, cudaStream_t s) {
  if (stage_off % 16 != 0) throw std::invalid_argument("reduce_pull: staging offset must be 16-byte aligned");
  op = checked_op(dtype, op, scale);
  const int threads = cfg.threads ? cfg.threads : 512;
  // every rank must launch the same grid (the barrier is per block): size it by the whole vector, not by this rank's share
  const int blocks = std::min(cfg.blocks ? cfg.blocks : auto_blocks(total_vec / std::max(1, d.world) + 1, threads, 64), kSymmMaxBlocks);
  PDT_DISPATCH_TYPE(dtype, PDT_DISPATCH_OP(T, op, { reduce_pull_kernel<T, OP><<<blocks, threads, 0, s>>>(d, stage_off, begin_vec, count_vec, static_cast<uint4*>(out), scale); }));
  check_launch("reduce_pull");
}

void launch_p2p_send(const SymmDev& d, const void* src, size_t nbytes, int dst_rank, size_t slot_off, unsigned int seq, cudaStream_t s) {
  p2p_send_kernel<<<kSymmP2PBlocks, 512, 0, s>>>(d, static_cast<const char*>(src), nbytes, dst_rank, slot_off, seq);
  check_launch("p2p_send");
}
void launch_p2p_recv(const SymmDev& d, void* dst, size_t nbytes, int src_rank, size_t slot_off, unsigned int seq, cudaStream_t s) {
  p2p_recv_kernel<<<kSymmP2PBlocks, 512, 0, s>>>(d, static_cast<char*>(dst), nbytes, src_rank, slot_off, seq);
  check_launch("p2p_recv");
}

void launch_barrier(const SymmDev& d, cudaStream_t s) {
  barrier_kernel<<<1, 32, 0, s>>>(d);
  check_launch("barrier_kernel");
}

}  // namespace pdt
