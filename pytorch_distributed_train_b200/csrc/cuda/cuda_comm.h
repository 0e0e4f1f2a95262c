// GPU communicators: SymmComm (product: NVLink peer/multicast kernels) and NcclComm (baseline).
#pragma once
#include <ATen/cuda/CUDAEvent.h>
#include <c10/cuda/CUDAStream.h>

#include <memory>

#include "../comm/comm.h"
#include "symm_kernels.h"
#include "symm_mem.h"

namespace pdt {

// Stream-ordered completion handle: wait() makes the *current* stream wait for the collective
// (ProcessGroupNCCL semantics the reference relies on); never blocks the host.
class CudaWork : public CommWork {
 public:
  CudaWork(int device, std::vector<at::Tensor> keep) : device_(device), keep_(std::move(keep)) {}
  at::cuda::CUDAEvent& done() { return done_; }
  void wait() override;
  void synchronize() override;
  bool is_completed() override;

 private:
  int device_;
  at::cuda::CUDAEvent done_{cudaEventDisableTiming};
  std::vector<at::Tensor> keep_;
};

class CudaCommBase : public Comm {
 public:
  CudaCommBase(int rank, int size, int device);
  int rank() const override { return rank_; }
  int size() const override { return size_; }
  bool is_cuda() const override { return true; }
  int device() const { return device_; }
  c10::cuda::CUDAStream comm_stream() const { return comm_stream_; }
  std::shared_ptr<DeviceStamp> stamp(bool on_comm_stream = false) override;   // timing event on the compute / comm stream
  bool capturing() const override;

 protected:
  // Runs fn(stream) on the comm stream, ordered after the caller's current stream; the tensors
  // are kept alive (and their blocks marked in use on the comm stream) until completion.
  std::shared_ptr<CommWork> enqueue(const std::vector<at::Tensor>& tensors, const std::function<void(cudaStream_t)>& fn);
  void check(const at::Tensor& t, const char* what) const;
  int rank_, size_, device_;
  c10::cuda::CUDAStream comm_stream_;
};

class SymmComm : public CudaCommBase {
 public:
  SymmComm(std::shared_ptr<Store> store, int rank, int size, int device, Millis timeout, size_t heap_bytes);
  ~SymmComm() override;
  std::string backend_name() const override { return "nvlink"; }
  at::Tensor alloc_flat(int64_t numel, at::ScalarType dtype, const at::Device& device) override;
  std::shared_ptr<CommWork> allreduce(at::Tensor t, ReduceOp op, double postscale) override;
  std::shared_ptr<CommWork> broadcast(at::Tensor t, int root) override;
  std::shared_ptr<CommWork> allgather(at::Tensor out, at::Tensor in) override;
  std::shared_ptr<CommWork> reduce(at::Tensor t, ReduceOp op, int root) override;
  std::shared_ptr<CommWork> reduce_scatter(at::Tensor out, at::Tensor in, ReduceOp op) override;
  std::shared_ptr<CommWork> gather(at::Tensor out, at::Tensor in, int root) override;
  std::shared_ptr<CommWork> scatter(at::Tensor out, at::Tensor in, int root) override;
  std::shared_ptr<CommWork> alltoall(at::Tensor out, at::Tensor in) override;
  // Point-to-point over the symmetric heap, device-signalled: the sender stores chunks into its slot of the receiver's
  // heap and raises a flag there, the receiver copies out and acknowledges — two plain kernels, no host synchronisation.
  // Eager up to one slot (32 MiB / world); longer messages need the matching recv posted.
  std::shared_ptr<CommWork> send(at::Tensor t, int dst) override;
  std::shared_ptr<CommWork> recv(at::Tensor t, int src) override;
  std::shared_ptr<CommWork> barrier() override;
  void shutdown() override;
  // ONE kernel on the comm stream: one-shot mean-allreduce of the gradient chunk + SGD update (+ buffer broadcast).
  std::shared_ptr<CommWork> allreduce_sgd(at::Tensor grad, at::Tensor param, at::Tensor momentum_buf, const FusedSgd& h, at::Tensor bcast,
                                          int bcast_root) override;

  // Same collective launched directly on the caller's current stream (channel kChanInline):
  // no stream hop — used where the result is needed by the very next kernel (SyncBatchNorm).
  void allreduce_inline(at::Tensor t, ReduceOp op, double postscale);
  void broadcast_inline(at::Tensor t, int root);
  // Fused mean-allreduce(grad) + SGD(param) in one launch on the caller's stream.
  void allreduce_sgd_inline(at::Tensor grad, at::Tensor param, c10::optional<at::Tensor> momentum_buf, double lr,
                            c10::optional<at::Tensor> lr_tensor, double momentum, double dampening, double weight_decay,
                            bool nesterov, bool first_step);

  SymmetricHeap& heap() { return *heap_; }
  bool has_multicast() const { return heap_->has_multicast(); }
  // tuning knobs (also read from PDT_AR_* environment variables)
  void set_algo(const std::string& algo) { algo_ = algo; }
  std::string algo() const { return algo_; }
  void set_oneshot_max_bytes(int64_t n) { oneshot_max_ = static_cast<size_t>(n); }
  void set_launch(int blocks, int threads) { cfg_.blocks = blocks; cfg_.threads = threads; }
  std::string describe() const;
  int status() const { return heap_->status(); }
  // Human-readable form of the device-written status word (see symm_trap_timeout in symm_device.h).
  std::string status_string() const {
    const int s = heap_->status();
    if (s == 0) return "ok";
    if ((static_cast<unsigned>(s) & 0xFF000000u) == 0x7D000000u)
      return "device-side barrier timeout on rank " + std::to_string(rank_) + ": channel " + std::to_string((s >> 20) & 0xF) +
             " never heard from rank " + std::to_string((s >> 16) & 0xF) + " (waiting for epoch …" + std::to_string(s & 0xFFFF) + ")";
    return "unknown status " + std::to_string(s);
  }

 private:
  void do_allreduce(at::Tensor& t, ReduceOp op, double scale, int channel, cudaStream_t s);
  void do_broadcast(at::Tensor& t, int root, int channel, cudaStream_t s);
  std::shared_ptr<SymmetricHeap> heap_;  // shared with every tensor carved out of it (see alloc_flat)
  std::shared_ptr<Store> store_;         // control plane of send/recv
  uint64_t send_seq_[kSymmMaxWorld] = {}, recv_seq_[kSymmMaxWorld] = {};
  uint64_t alloc_seq_ = 0;               // alloc_flat is collective: sequence number of the store exchange
  std::string algo_ = "auto";   // auto | oneshot | oneshot_mc | twoshot | nvls
  size_t oneshot_max_ = 512 * 1024;
  SymmLaunchCfg cfg_;
  bool down_ = false;
};

class NcclComm : public CudaCommBase {
 public:
  NcclComm(std::shared_ptr<Store> store, int rank, int size, int device, Millis timeout);
  ~NcclComm() override;
  std::string backend_name() const override { return "nccl-lib"; }
  std::shared_ptr<CommWork> allreduce(at::Tensor t, ReduceOp op, double postscale) override;
  std::shared_ptr<CommWork> broadcast(at::Tensor t, int root) override;
  std::shared_ptr<CommWork> allgather(at::Tensor out, at::Tensor in) override;
  std::shared_ptr<CommWork> reduce(at::Tensor t, ReduceOp op, int root) override;
  std::shared_ptr<CommWork> reduce_scatter(at::Tensor out, at::Tensor in, ReduceOp op) override;
  std::shared_ptr<CommWork> alltoall(at::Tensor out, at::Tensor in) override;
  std::shared_ptr<CommWork> send(at::Tensor t, int dst) override;
  std::shared_ptr<CommWork> recv(at::Tensor t, int src) override;
  std::shared_ptr<CommWork> barrier() override;
  void shutdown() override;
  static bool available();
  static std::string version();

 private:
  void* comm_ = nullptr;
  at::Tensor barrier_buf_;
};

}  // namespace pdt
