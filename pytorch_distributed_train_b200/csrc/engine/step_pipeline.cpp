#include "step_pipeline.h"

#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/util/Exception.h>

namespace pdt {

namespace {
// dst.copy_(src, non_blocking) on `stream`.  A device-resident source of the same dtype and layout is one cudaMemcpyAsync: the
// dispatcher's copy_ costs microseconds of host time per tensor, and a replayed step's device time is not much larger than the
// host time of the loop that feeds it — every microsecond the host saves is lead it keeps over the device through a host stall.
// Anything else (pinned host sources above all, which must stay registered with the caching host allocator) goes through copy_.
void stage_copy(const at::Tensor& dst, const at::Tensor& src, c10::cuda::CUDAStream stream) {
  if (src.is_cuda() && dst.is_cuda() && src.get_device() == dst.get_device() && src.scalar_type() == dst.scalar_type() &&
      src.numel() == dst.numel() && src.is_contiguous() && dst.is_contiguous()) {
    C10_CUDA_CHECK(cudaMemcpyAsync(dst.data_ptr(), src.data_ptr(), src.nbytes(), cudaMemcpyDeviceToDevice, stream.stream()));
    return;
  }
  c10::cuda::CUDAStreamGuard sg(stream);
  dst.copy_(src, /*non_blocking=*/true);
}
}  // namespace

StepPipeline::StepPipeline(int device, int num_sets, at::ScalarType loss_dtype)
    : device_(device),
      copy_(c10::cuda::getStreamFromPool(/*isHighPriority=*/false, device)),
      d2h_(c10::cuda::getStreamFromPool(/*isHighPriority=*/false, device)),
      after_(cudaEventDisableTiming),
      src_ready_(cudaEventDisableTiming) {
  TORCH_CHECK(num_sets >= 1, "StepPipeline: at least one input set");
  c10::cuda::CUDAGuard g(device_);
  auto cur = c10::cuda::getCurrentCUDAStream(device_);
  for (int i = 0; i < num_sets; ++i) {
    ready_.emplace_back(new at::cuda::CUDAEvent(cudaEventDisableTiming));
    done_.emplace_back(new at::cuda::CUDAEvent(cudaEventDisableTiming));
    done_.back()->record(cur);   // "nobody is reading this set"
    loss_read_.push_back(nullptr);
  }
  for (int s = 0; s < kRing; ++s) slot_ev_.emplace_back(new at::cuda::CUDAEvent(cudaEventDisableTiming));
  host_ = at::zeros({kRing}, at::TensorOptions().dtype(loss_dtype).pinned_memory(true));
}

void StepPipeline::stage_inputs(int i, const std::vector<at::Tensor>& dst, const std::vector<at::Tensor>& src, bool inputs_ready, bool overlap) {
  TORCH_CHECK(i >= 0 && i < static_cast<int>(ready_.size()) && dst.size() == src.size(), "StepPipeline::stage_inputs: bad arguments");
  c10::cuda::CUDAGuard g(device_);
  auto cur = c10::cuda::getCurrentCUDAStream(device_);
  if (overlap) {
    done_[i]->block(copy_);   // the replay that last read this set has finished
    if (!inputs_ready) {
      bool any_dev = false;
      for (const auto& t : src) any_dev = any_dev || t.is_cuda();
      if (any_dev) {   // device-resident sources may still be in flight on the caller's stream
        src_ready_.record(cur);
        src_ready_.block(copy_);
      }
    }
    for (size_t k = 0; k < dst.size(); ++k) stage_copy(dst[k], src[k], copy_);
    ready_[i]->record(copy_);
    ready_[i]->block(cur);
  } else {
    for (size_t k = 0; k < dst.size(); ++k) stage_copy(dst[k], src[k], cur);
  }
  if (loss_read_[i] != nullptr) {   // loss_to_host() of this graph's previous replay has read the loss buffer
    loss_read_[i]->block(cur);
    loss_read_[i] = nullptr;
  }
}

void StepPipeline::replayed(int i) {
  c10::cuda::CUDAGuard g(device_);
  done_[i]->record(c10::cuda::getCurrentCUDAStream(device_));
}

int64_t StepPipeline::loss_to_host(int i, const at::Tensor& loss) {
  TORCH_CHECK(loss.numel() == 1 && loss.scalar_type() == host_.scalar_type(), "StepPipeline::loss_to_host: scalar loss of the captured dtype expected");
  c10::cuda::CUDAGuard g(device_);
  const int slot = static_cast<int>(gen_ % kRing);
  if (gen_ >= kRing) slot_ev_[slot]->synchronize();   // the slot's previous value has been delivered (and may be overwritten)
  auto cur = c10::cuda::getCurrentCUDAStream(device_);
  after_.record(cur);        // the replay (and anything the caller queued behind it)
  after_.block(d2h_);
  {
    c10::cuda::CUDAStreamGuard sg(d2h_);
    host_.select(0, slot).copy_(loss.detach().reshape({}), /*non_blocking=*/true);
  }
  slot_ev_[slot]->record(d2h_);
  loss_read_[i] = slot_ev_[slot].get();
  return ++gen_;
}

double StepPipeline::loss_value(int64_t gen) {
  TORCH_CHECK(gen >= 1 && gen <= gen_, "StepPipeline::loss_value: unknown handle");
  TORCH_CHECK(gen_ - gen < kRing, "HostLoss: read too late — the pinned slot has been reused (handles stay valid for ", kRing - 1, " further steps)");
  const int slot = static_cast<int>((gen - 1) % kRing);
  slot_ev_[slot]->synchronize();
  return host_.select(0, slot).item<double>();
}

}  // namespace pdt
