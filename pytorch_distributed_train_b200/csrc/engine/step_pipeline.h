// Host side of a graph-replayed training step (engine.GraphedTrainStep): everything the training thread does around
// `cudaGraphLaunch` — staging the next batch into the step's input buffers on a copy stream, ordering it against the
// replays that read / wrote those buffers, shipping every loss to pinned host memory on a side stream — as three native
// calls instead of ~25 Python-level stream / event / copy operations, whose host time was comparable to the device time
// of a replayed step (the input loop was host-bound).
//
// Ordering per input buffer set i (two sets, one captured graph each):
//   copy stream : wait done[i] (the replay that last read set i) → copy batch → record ready[i]
//   step stream : wait ready[i] → wait loss_read[i] (the previous loss of graph i has left the device) → replay → record done[i]
//   d2h stream  : wait (event recorded on the step stream after the replay) → copy loss → record slot event
// Copies go through at::Tensor::copy_, so pinned sources stay registered with the caching host allocator.
#pragma once
#include <ATen/ATen.h>
#include <ATen/cuda/CUDAEvent.h>
#include <c10/cuda/CUDAStream.h>

#include <memory>
#include <vector>

namespace pdt {

class StepPipeline {
 public:
  static constexpr int kRing = 16;   // loss slots: a handle stays readable for kRing - 1 further steps
  StepPipeline(int device, int num_sets, at::ScalarType loss_dtype);
  // Queue the copy of `src` into `dst` (input set i) and make the current stream wait for it.  inputs_ready: device-resident
  // sources are complete already (otherwise the copy is ordered behind the current stream).
  void stage_inputs(int i, const std::vector<at::Tensor>& dst, const std::vector<at::Tensor>& src, bool inputs_ready, bool overlap);
  // After the replay of graph i was queued on the current stream.
  void replayed(int i);
  // Queue the device→host copy of `loss` (the static loss tensor of graph i); returns the generation number of the handle.
  int64_t loss_to_host(int i, const at::Tensor& loss);
  // Blocks until the copy of generation `gen` has landed; throws if the slot has been reused.
  double loss_value(int64_t gen);

 private:
  int device_;
  c10::cuda::CUDAStream copy_, d2h_;
  std::vector<std::unique_ptr<at::cuda::CUDAEvent>> ready_, done_;
  std::vector<at::cuda::CUDAEvent*> loss_read_;   // per set: slot event of the last loss copy (nullptr: none pending)
  std::vector<std::unique_ptr<at::cuda::CUDAEvent>> slot_ev_;
  at::cuda::CUDAEvent after_, src_ready_;   // after_: behind the replay (loss hand-off); src_ready_: device-resident sources
  at::Tensor host_;   // pinned [kRing]
  int64_t gen_ = 0;
};

}  // namespace pdt
