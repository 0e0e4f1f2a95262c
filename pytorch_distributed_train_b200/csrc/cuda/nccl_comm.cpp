// Thin libnccl binding — the *measured baseline and correctness oracle* for the NVLink kernels (`--comm nccl`).  The
// library is resolved with dlopen at first use so the extension imports on machines without it.
#include <c10/cuda/CUDAGuard.h>
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>
#include <mutex>

#include "cuda_comm.h"
#include "cuda_utils.h"

namespace pdt {

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*CommAbort)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Reduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*ReduceScatter)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  std::string error;
};

NcclApi& api() {
  static NcclApi a;
  static std::once_flag once;
  std::call_once(once, [] {
    // torch has normally mapped its bundled libnccl.so.2 already; RTLD_NOLOAD finds that copy first
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
      a.lib = dlopen(name, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
      if (a.lib) break;
    }
    if (!a.lib)
      for (const char* name : {"libnccl.so.2", "libnccl.so"}) {
        a.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
        if (a.lib) break;
      }
    if (!a.lib) {
      a.error = std::string("cannot load libnccl: ") + dlerror();
      return;
    }
    auto sym = [&](const char* n) {
      void* p = dlsym(a.lib, n);
      if (!p && a.error.empty()) a.error = std::string("libnccl lacks symbol ") + n;
      return p;
    };
#define PDT_NCCL_SYM(field, name) a.field = reinterpret_cast<decltype(a.field)>(sym(name))
    PDT_NCCL_SYM(GetVersion, "ncclGetVersion");
    PDT_NCCL_SYM(GetUniqueId, "ncclGetUniqueId");
    PDT_NCCL_SYM(CommInitRank, "ncclCommInitRank");
    PDT_NCCL_SYM(CommDestroy, "ncclCommDestroy");
    PDT_NCCL_SYM(CommAbort, "ncclCommAbort");
    PDT_NCCL_SYM(GetErrorString, "ncclGetErrorString");
    PDT_NCCL_SYM(AllReduce, "ncclAllReduce");
    PDT_NCCL_SYM(Broadcast, "ncclBroadcast");
    PDT_NCCL_SYM(Reduce, "ncclReduce");
    PDT_NCCL_SYM(AllGather, "ncclAllGather");
    PDT_NCCL_SYM(ReduceScatter, "ncclReduceScatter");
    PDT_NCCL_SYM(Send, "ncclSend");
    PDT_NCCL_SYM(Recv, "ncclRecv");
    PDT_NCCL_SYM(GroupStart, "ncclGroupStart");
    PDT_NCCL_SYM(GroupEnd, "ncclGroupEnd");
#undef PDT_NCCL_SYM
  });
  return a;
}

void nccl_check(ncclResult_t r, const char* what) {
  if (r != ncclSuccess) throw std::runtime_error(std::string("NCCL error in ") + what + ": " + api().GetErrorString(r));
}

ncclDataType_t nccl_dtype(at::ScalarType t) {
  switch (t) {
    case at::kFloat: return ncclFloat32;
    case at::kDouble: return ncclFloat64;
    case at::kHalf: return ncclFloat16;
    case at::kBFloat16: return ncclBfloat16;
    case at::kChar: return ncclInt8;
    case at::kByte: case at::kBool: return ncclUint8;
    case at::kInt: return ncclInt32;
    case at::kLong: return ncclInt64;
    default: TORCH_CHECK(false, "NCCL: unsupported dtype ", c10::toString(t));
  }
}

// On bool, SUM is logical OR and PRODUCT logical AND (as torch's NCCL backend maps them): MAX and MIN of 0/1 bytes.  AVG has no
// bool result.
ncclRedOp_t nccl_op(ReduceOp op, at::ScalarType t) {
  if (t == at::kBool) {
    TORCH_CHECK(op != ReduceOp::AVG, "NCCL: AVG is not defined for bool tensors");
    if (op == ReduceOp::SUM) return ncclMax;
    if (op == ReduceOp::PRODUCT) return ncclMin;
  }
  switch (op) {
    case ReduceOp::SUM: return ncclSum;
    case ReduceOp::AVG: return ncclAvg;
    case ReduceOp::PRODUCT: return ncclProd;
    case ReduceOp::MIN: return ncclMin;
    case ReduceOp::MAX: return ncclMax;
    default: TORCH_CHECK(false, "NCCL: bitwise reductions are not supported");
  }
}

}  // namespace

bool NcclComm::available() { return api().lib != nullptr && api().error.empty(); }

std::string NcclComm::version() {
  if (!available()) return "unavailable: " + api().error;
  int v = 0;
  api().GetVersion(&v);
  return std::to_string(v / 10000) + "." + std::to_string((v / 100) % 100) + "." + std::to_string(v % 100);
}

NcclComm::NcclComm(std::shared_ptr<Store> store, int rank, int size, int device, Millis timeout) : CudaCommBase(rank, size, device) {
  (void)timeout;
  TORCH_CHECK(available(), "NCCL backend requested but ", api().error);
  c10::cuda::CUDAGuard guard(device);
  ncclUniqueId id;
  if (rank == 0) {
    nccl_check(api().GetUniqueId(&id), "ncclGetUniqueId");
    store->set("nccl/uid", std::string(reinterpret_cast<const char*>(&id), sizeof(id)));
  } else {
    std::string blob = store->get("nccl/uid");
    TORCH_CHECK(blob.size() == sizeof(id), "NCCL: bad unique id in store");
    std::memcpy(&id, blob.data(), sizeof(id));
  }
  ncclComm_t c;
  nccl_check(api().CommInitRank(&c, size, id, rank), "ncclCommInitRank");
  comm_ = c;
  barrier_buf_ = at::zeros({1}, at::TensorOptions().dtype(at::kFloat).device(at::Device(at::kCUDA, static_cast<c10::DeviceIndex>(device))));
}

NcclComm::~NcclComm() { shutdown(); }

void NcclComm::shutdown() {
  if (!comm_) return;
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
  api().CommDestroy(static_cast<ncclComm_t>(comm_));
  comm_ = nullptr;
}

std::shared_ptr<CommWork> NcclComm::allreduce(at::Tensor t, ReduceOp op, double postscale) {
  check(t, "allreduce");
  record("allreduce", &t);
  return enqueue({t}, [&](cudaStream_t s) {
    nccl_check(api().AllReduce(t.data_ptr(), t.data_ptr(), static_cast<size_t>(t.numel()), nccl_dtype(t.scalar_type()), nccl_op(op, t.scalar_type()),
                               static_cast<ncclComm_t>(comm_), s),
               "ncclAllReduce");
    if (postscale != 1.0) {
      // the baseline pays a separate scale kernel, like the reference's per-parameter divide
      c10::cuda::CUDAStreamGuard sg(comm_stream_);
      t.mul_(postscale);
    }
  });
}
std::shared_ptr<CommWork> NcclComm::broadcast(at::Tensor t, int root) {
  check(t, "broadcast");
  record("broadcast", &t);
  return enqueue({t}, [&](cudaStream_t s) {
    nccl_check(api().Broadcast(t.data_ptr(), t.data_ptr(), t.nbytes(), ncclUint8, root, static_cast<ncclComm_t>(comm_), s), "ncclBroadcast");
  });
}
std::shared_ptr<CommWork> NcclComm::allgather(at::Tensor out, at::Tensor in) {
  check(out, "allgather output");
  check(in, "allgather input");
  TORCH_CHECK(out.numel() == in.numel() * size_, "allgather: output must hold world_size × input elements");
  record("allgather", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    nccl_check(api().AllGather(in.data_ptr(), out.data_ptr(), in.nbytes(), ncclUint8, static_cast<ncclComm_t>(comm_), s), "ncclAllGather");
  });
}
std::shared_ptr<CommWork> NcclComm::reduce(at::Tensor t, ReduceOp op, int root) {
  check(t, "reduce");
  record("reduce", &t);
  return enqueue({t}, [&](cudaStream_t s) {
    nccl_check(api().Reduce(t.data_ptr(), t.data_ptr(), static_cast<size_t>(t.numel()), nccl_dtype(t.scalar_type()), nccl_op(op, t.scalar_type()), root,
                            static_cast<ncclComm_t>(comm_), s),
               "ncclReduce");
  });
}
std::shared_ptr<CommWork> NcclComm::reduce_scatter(at::Tensor out, at::Tensor in, ReduceOp op) {
  check(out, "reduce_scatter output");
  check(in, "reduce_scatter input");
  record("reduce_scatter", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    nccl_check(api().ReduceScatter(in.data_ptr(), out.data_ptr(), static_cast<size_t>(out.numel()), nccl_dtype(in.scalar_type()), nccl_op(op, in.scalar_type()),
                                   static_cast<ncclComm_t>(comm_), s),
               "ncclReduceScatter");
  });
}
std::shared_ptr<CommWork> NcclComm::alltoall(at::Tensor out, at::Tensor in) {
  check(out, "alltoall output");
  check(in, "alltoall input");
  TORCH_CHECK(in.numel() == out.numel() && in.numel() % size_ == 0, "alltoall: equal splits required");
  record("alltoall", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    const size_t blk = in.nbytes() / size_;
    nccl_check(api().GroupStart(), "ncclGroupStart");
    for (int r = 0; r < size_; ++r) {
      nccl_check(api().Send(static_cast<const char*>(in.data_ptr()) + r * blk, blk, ncclUint8, r, static_cast<ncclComm_t>(comm_), s), "ncclSend");
      nccl_check(api().Recv(static_cast<char*>(out.data_ptr()) + r * blk, blk, ncclUint8, r, static_cast<ncclComm_t>(comm_), s), "ncclRecv");
    }
    nccl_check(api().GroupEnd(), "ncclGroupEnd");
  });
}
std::shared_ptr<CommWork> NcclComm::send(at::Tensor t, int dst) {
  check(t, "send");
  record("send", &t);
  return enqueue({t}, [&](cudaStream_t s) { nccl_check(api().Send(t.data_ptr(), t.nbytes(), ncclUint8, dst, static_cast<ncclComm_t>(comm_), s), "ncclSend"); });
}
std::shared_ptr<CommWork> NcclComm::recv(at::Tensor t, int src) {
  check(t, "recv");
  record("recv", &t);
  return enqueue({t}, [&](cudaStream_t s) { nccl_check(api().Recv(t.data_ptr(), t.nbytes(), ncclUint8, src, static_cast<ncclComm_t>(comm_), s), "ncclRecv"); });
}
std::shared_ptr<CommWork> NcclComm::barrier() {
  record("barrier", nullptr);
  return enqueue({barrier_buf_}, [&](cudaStream_t s) {
    nccl_check(api().AllReduce(barrier_buf_.data_ptr(), barrier_buf_.data_ptr(), 1, ncclFloat32, ncclSum, static_cast<ncclComm_t>(comm_), s),
               "ncclAllReduce(barrier)");
  });
}

}  // namespace pdt
