// Gradient reducer: the native half of our DistributedDataParallel.
//
// What it has to do is fixed by how the reference uses DDP (ref: ddp_example.py:64,91 →
// c10d reducer.hpp:45-584): fire as each parameter's gradient is accumulated, pack gradients
// into flat buckets, launch one collective per bucket as soon as the bucket is complete (in
// bucket order, overlapped with the rest of backward), and finish at the end of backward.
// How it does it is ours:
//   * gradients live *in* the bucket (param.grad is a view) so "flatten" is free; on the
//     SymmComm backend the bucket is peer-mapped NVLink memory that remote GPUs read directly;
//   * the 1/world_size scale is folded into the collective (`postscale`) instead of a
//     per-parameter multiply kernel (the reference path spends 10 tiny kernels on it);
//   * bucket layout is rebuilt once from the observed grad-ready order, planner in C++.
#pragma once
#include <ATen/ATen.h>
#include <pybind11/pybind11.h>
#include <torch/csrc/autograd/function.h>

#include <chrono>
#include <deque>
#include <memory>
#include <mutex>
#include <optional>
#include <unordered_map>
#include <vector>

#include "../comm/comm.h"
#include "bucket_plan.h"

namespace pdt {

namespace py = pybind11;

struct GradBucket {
  int64_t index;
  bool is_last;
  at::Tensor buffer;                    // flat, undivided local gradients
  std::vector<at::Tensor> gradients;    // views into buffer, one per parameter
  std::vector<at::Tensor> parameters;
  std::vector<int64_t> offsets, lengths;
};

struct ReducerStats {
  int64_t num_iterations = 0;
  int64_t num_buckets_reduced = 0;       // lifetime
  int64_t num_rebuilds = 0;
  std::vector<int64_t> bucket_sizes_bytes;
  std::vector<int64_t> grad_ready_order;  // previous iteration
  std::vector<std::vector<int64_t>> bucket_indices;
  // DEVICE times of the last resolved iteration, microseconds: event marks on the compute / comm streams for CUDA
  // backends (host clock for the CPU backend).  Iterations recorded into a CUDA graph are not timed.
  double forward_us = 0, backward_compute_us = 0, backward_comm_us = 0, backward_total_us = 0;
  double backward_comm_exposed_us = 0;    // how long the compute stream stalled at the end of backward waiting for the reduction
  int64_t reduce_chunks = 0;              // collectives launched per synchronised backward (sub-bucket chunks)
  // running means over the synchronised iterations after the first kStatsWarmup (the reference's logger samples
  // the same quantities every 100 iterations after the first 10, hdr:reducer.hpp:33,166-170)
  int64_t timed_iterations = 0;
  double avg_forward_us = 0, avg_backward_compute_us = 0, avg_backward_comm_us = 0, avg_backward_comm_exposed_us = 0;
  bool has_rebuilt = false;
  bool gradient_as_bucket_view = true;
  bool find_unused_parameters = false;
  int64_t total_param_bytes = 0;
  int64_t copies_into_bucket = 0;         // grads that were not already bucket views (lifetime)
};

class Reducer {
 public:
  Reducer(std::vector<at::Tensor> params, std::vector<std::vector<int64_t>> bucket_indices,
          std::shared_ptr<Comm> comm, int64_t bucket_bytes_cap, int64_t first_bucket_bytes_cap,
          bool find_unused_parameters, bool gradient_as_bucket_view, bool static_graph);
  ~Reducer();

  void prepare_for_forward();
  // Arms the hooks for the coming backward. `outputs` is only inspected when
  // find_unused_parameters is on.
  void prepare_for_backward(const std::vector<at::Tensor>& outputs);
  // no_sync(): when false the hooks are inert and gradients just accumulate locally.
  void set_require_sync(bool v) { require_sync_ = v; }
  // Rebuild-once protocol: rank 0 proposes, everybody applies (layout agreed via the store).
  bool should_rebuild() const;
  std::vector<std::vector<int64_t>> propose_rebuild() const;
  void apply_rebuild(const std::vector<std::vector<int64_t>>& bucket_indices);
  // Python comm hook: hook(bucket: GradBucket) -> Tensor | object-with-wait()->Tensor
  void register_comm_hook(py::object hook);
  ReducerStats stats() const;
  std::vector<at::Tensor> bucket_buffers() const;
  // Per-parameter bucket slot (param order): kernels may write gradients straight into these.
  std::vector<at::Tensor> grad_views() const;
  // True when every parameter's .grad currently aliases its bucket slot.
  bool grads_are_views() const;
  // Re-point every param.grad at its bucket view (zeroing the bucket): used by the graph
  // engine so backward writes land directly in comm-visible memory.
  void install_grad_views(bool zero);
  void set_postscale(double s) { postscale_ = s; }
  // The optimizer reduces: buckets are filled and gradients re-pointed exactly as in a synchronised
  // backward, but no collective is launched (a fused allreduce+update kernel consumes the flat buckets).
  void set_defer_comm(bool on) { defer_comm_ = on; }
  bool defer_comm() const { return defer_comm_; }
  // Sub-bucket overlap: a bucket is reduced in up to `max_chunks` contiguous pieces of at least
  // `min_chunk_bytes`, each launched from the autograd hook as soon as its last gradient is ready, so the transfer
  // of early layers' gradients overlaps the rest of backward even when the whole model fits one bucket.
  void set_chunking(int64_t min_chunk_bytes, int64_t max_chunks);
  // Optimizer fused into the reduction: every chunk is reduced AND applied (Comm::allreduce_sgd) from the hook; the
  // last chunk also carries the module-buffer broadcast.  `param_flat` / `momentum_flat` mirror bucket 0 element
  // for element.  Requires a single bucket and no comm hook.  Pass an undefined param_flat to switch it off.
  void set_fused_sgd(at::Tensor param_flat, at::Tensor momentum_flat, FusedSgd hyper, at::Tensor bcast, int64_t bcast_root);
  bool fused_sgd() const { return fused_param_.defined(); }

 private:
  struct Chunk {
    size_t first_slot = 0, end_slot = 0;  // slots [first, end) of the bucket
    int64_t off = 0, len = 0;             // element range of bucket.flat (16-byte aligned on both ends)
    size_t pending = 0;
    std::shared_ptr<CommWork> work;
  };
  struct Bucket {
    at::Tensor flat;
    std::vector<Chunk> chunks;
    std::vector<size_t> slot_chunk;        // slot -> chunk index
    size_t next_chunk = 0;
    std::vector<int64_t> params;          // global param indices
    std::vector<at::Tensor> views;        // same order as params
    std::vector<int64_t> offsets, lengths;
    size_t pending = 0;
    bool launched = false;
    std::shared_ptr<CommWork> work;
    py::object py_future;                  // when a comm hook is installed
    at::Tensor hook_result;
  };
  struct Loc { size_t bucket, slot; };

  void build_buckets(const std::vector<std::vector<int64_t>>& bucket_indices);
  void autograd_hook(size_t index);
  void mark_variable_ready(size_t index);
  void launch_ready_buckets();
  void launch_bucket(size_t b);
  void launch_chunk(size_t b, size_t c);
  void plan_chunks(Bucket& bk) const;
  void resolve_timings();
  void finalize_backward();
  void search_unused(const std::vector<at::Tensor>& outputs);

  std::vector<at::Tensor> params_;
  std::shared_ptr<Comm> comm_;
  int64_t bucket_bytes_cap_, first_bucket_bytes_cap_;
  bool find_unused_, grad_as_view_, static_graph_;
  bool require_sync_ = true;
  bool expect_hooks_ = false;
  bool callback_queued_ = false;
  bool has_rebuilt_ = false;
  double postscale_;
  bool defer_comm_ = false;

  std::vector<Bucket> buckets_;
  std::vector<Loc> locs_;
  size_t next_bucket_ = 0;
  std::vector<char> ready_;               // per param, this iteration
  std::vector<char> locally_unused_;      // per param, this iteration
  std::vector<int64_t> ready_order_, prev_ready_order_;
  std::vector<std::pair<std::shared_ptr<torch::autograd::Node>, uintptr_t>> hooks_;
  std::unordered_map<torch::autograd::Node*, size_t> acc_to_index_;
  py::object comm_hook_;
  bool has_comm_hook_ = false;
  mutable std::mutex mu_;

  int64_t min_chunk_bytes_ = 32 * 1024, max_chunks_ = 4;
  at::Tensor fused_param_, fused_momentum_, fused_bcast_;
  FusedSgd fused_hyper_;
  int fused_bcast_root_ = 0;

  // device-time marks of one iteration (see ReducerStats); resolved lazily once the device has passed them
  struct Marks {
    std::shared_ptr<DeviceStamp> fwd_start, bwd_start, first_ready, comm_end, before_wait, after_wait;
    int64_t iteration = 0;
  };
  Marks cur_;
  std::deque<Marks> unresolved_;
  bool timing_this_iter_ = false;
  bool saw_first_hook_ = false;
  ReducerStats stats_;
};

}  // namespace pdt
