// Tensor-level collective interface implemented by every backend:
//   CpuComm     – TCP mesh on host tensors (csrc/cpu)                        ["gloo" slot]
//   SymmComm    – sm_90a kernels over NVLink peer / multicast memory (csrc/cuda) [product path]
//   NcclComm    – thin libnccl binding, measured baseline + oracle only       ["--comm nccl"]
// Semantics follow the ProcessGroup contract the reference relies on
// (ref: ddp_example.py:50,64; torch c10d ProcessGroup.hpp / Work.hpp): collectives are
// enqueued in program order, CUDA collectives are stream-ordered after the caller's current
// stream and `wait()` is a stream wait, never a host block.
#pragma once
#include <ATen/ATen.h>

#include <algorithm>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../cpu/cpu_backend.h"

namespace pdt {

class CommWork {
 public:
  virtual ~CommWork() = default;
  // CPU: block the host. CUDA: make the current stream wait for the collective.
  virtual void wait() = 0;
  // Block the host until the result is visible (CPU: same as wait()).
  virtual void synchronize() = 0;
  virtual bool is_completed() = 0;
};

// A point in device time: an event on the compute (or comm) stream for CUDA backends, the host clock otherwise.
// The reducer's logger is built on these so that its numbers are *device* times, not host enqueue times.
class DeviceStamp {
 public:
  virtual ~DeviceStamp() = default;
  virtual bool ready() = 0;                                   // has the device passed this point?
  virtual double us_since(DeviceStamp& earlier) = 0;          // both must be ready()
};

// Hyper-parameters of the SGD update fused into a gradient reduction (Comm::allreduce_sgd).
struct FusedSgd {
  double lr = 0, momentum = 0, dampening = 0, weight_decay = 0;
  bool nesterov = false, first_step = false;
  at::Tensor lr_tensor;      // optional device scalar (CUDA-graph friendly schedules); overrides lr
};

class Comm {
 public:
  virtual ~Comm() = default;
  virtual int rank() const = 0;
  virtual int size() const = 0;
  virtual std::string backend_name() const = 0;
  virtual bool is_cuda() const = 0;

  // Flat storage for gradient buckets / parameter arenas. SymmComm returns a view into the
  // peer-mapped symmetric heap so reduce kernels can read every rank's copy directly.
  virtual at::Tensor alloc_flat(int64_t numel, at::ScalarType dtype, const at::Device& device) {
    return at::zeros({numel}, at::TensorOptions().dtype(dtype).device(device));
  }
  // t <- reduce(t over ranks) * postscale   (postscale folded into the kernel / last pass)
  virtual std::shared_ptr<CommWork> allreduce(at::Tensor t, ReduceOp op, double postscale) = 0;
  virtual std::shared_ptr<CommWork> broadcast(at::Tensor t, int root) = 0;
  // out has size() * in.numel() elements, rank-major.
  virtual std::shared_ptr<CommWork> allgather(at::Tensor out, at::Tensor in) = 0;
  virtual std::shared_ptr<CommWork> reduce(at::Tensor t, ReduceOp op, int root);
  virtual std::shared_ptr<CommWork> reduce_scatter(at::Tensor out, at::Tensor in, ReduceOp op);
  virtual std::shared_ptr<CommWork> gather(at::Tensor out, at::Tensor in, int root);
  virtual std::shared_ptr<CommWork> scatter(at::Tensor out, at::Tensor in, int root);
  virtual std::shared_ptr<CommWork> alltoall(at::Tensor out, at::Tensor in);
  virtual std::shared_ptr<CommWork> send(at::Tensor t, int dst);
  virtual std::shared_ptr<CommWork> recv(at::Tensor t, int src);
  virtual std::shared_ptr<CommWork> barrier() = 0;
  virtual void shutdown() {}

  // grad <- mean_r(grad_r);  param <- SGD(param, grad)  on flat fp32 vectors of equal layout — the DDP reducer's
  // per-chunk launch when the optimizer is fused into the reduction.  `bcast` (optional): afterwards every rank's
  // `bcast` tensor holds `bcast_root`'s contents (DDP's BatchNorm-buffer sync riding on the last chunk).
  // Default: allreduce + ATen ops + broadcast; SymmComm runs ONE kernel with one cross-GPU barrier.
  virtual std::shared_ptr<CommWork> allreduce_sgd(at::Tensor grad, at::Tensor param, at::Tensor momentum_buf, const FusedSgd& h,
                                                  at::Tensor bcast, int bcast_root);
  // Device-time marks for the reducer's logger.  on_comm_stream: mark the backend's collective stream instead of
  // the caller's.  capturing(): a CUDA graph is being recorded (no timing marks, no host-visible state).
  virtual std::shared_ptr<DeviceStamp> stamp(bool on_comm_stream = false);
  virtual bool capturing() const { return false; }

  // Flight recorder: ring of the last K collectives issued on this rank.
  struct Record { uint64_t seq; std::string op; int64_t numel; std::string dtype; double t_enqueue; };
  std::vector<Record> flight_records() const;

 protected:
  void record(const char* op, const at::Tensor* t);
  mutable std::mutex rec_mu_;
  std::vector<Record> ring_;
  uint64_t seq_ = 0;
  static constexpr size_t kRing = 64;
};

DType to_dtype(at::ScalarType t);

// ---- CPU ------------------------------------------------------------------------------
class CpuComm : public Comm {
 public:
  CpuComm(std::shared_ptr<Store> store, int rank, int size, Millis timeout, const std::string& bind_host)
      : be_(std::make_shared<CpuBackend>(std::move(store), rank, size, timeout, bind_host)) {}
  int rank() const override { return be_->rank(); }
  int size() const override { return be_->size(); }
  std::string backend_name() const override { return "cpu"; }
  bool is_cuda() const override { return false; }
  std::shared_ptr<CommWork> allreduce(at::Tensor t, ReduceOp op, double postscale) override;
  std::shared_ptr<CommWork> broadcast(at::Tensor t, int root) override;
  std::shared_ptr<CommWork> allgather(at::Tensor out, at::Tensor in) override;
  std::shared_ptr<CommWork> reduce(at::Tensor t, ReduceOp op, int root) override;
  std::shared_ptr<CommWork> reduce_scatter(at::Tensor out, at::Tensor in, ReduceOp op) override;
  std::shared_ptr<CommWork> gather(at::Tensor out, at::Tensor in, int root) override;
  std::shared_ptr<CommWork> scatter(at::Tensor out, at::Tensor in, int root) override;
  std::shared_ptr<CommWork> alltoall(at::Tensor out, at::Tensor in) override;
  std::shared_ptr<CommWork> send(at::Tensor t, int dst) override;
  std::shared_ptr<CommWork> recv(at::Tensor t, int src) override;
  std::shared_ptr<CommWork> barrier() override;
  void shutdown() override { be_->shutdown(); }
  CpuBackend& backend() { return *be_; }

 private:
  std::shared_ptr<CpuBackend> be_;
};

}  // namespace pdt
