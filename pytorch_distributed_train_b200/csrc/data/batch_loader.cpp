#include "batch_loader.h"

#include <c10/util/Exception.h>

#include <chrono>
#include <cstdlib>
#include <cstring>

#if PDT_WITH_CUDA
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAEvent.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#endif

namespace pdt {

namespace {
// uint8 → float32 × scale (ToTensor).  78,400 elements per MNIST batch: the AVX2 loop is an order of magnitude faster than the scalar one —
// the difference between a loader that keeps up with a 0.1 ms training step and one that does not.
#if defined(__x86_64__)
__attribute__((target("avx2"), optimize("O3"))) void u8_to_f32_avx2(const uint8_t* __restrict p, float* __restrict o, int64_t n, float sc) {
  for (int64_t k = 0; k < n; ++k) o[k] = static_cast<float>(p[k]) * sc;
}
#endif
__attribute__((optimize("O3"))) void u8_to_f32_generic(const uint8_t* __restrict p, float* __restrict o, int64_t n, float sc) {
  for (int64_t k = 0; k < n; ++k) o[k] = static_cast<float>(p[k]) * sc;
}
void u8_to_f32(const uint8_t* p, float* o, int64_t n, float sc) {
#if defined(__x86_64__)
  static const bool avx2 = __builtin_cpu_supports("avx2");
  if (avx2) return u8_to_f32_avx2(p, o, n, sc);
#endif
  u8_to_f32_generic(p, o, n, sc);
}
}  // namespace

BatchStager::BatchStager(at::Tensor data, at::Tensor targets, std::vector<int64_t> sample_shape, int64_t batch_size, bool drop_last,
                         double scale, int64_t depth, bool pin_memory, int device)
    : data_(std::move(data)), targets_(std::move(targets)), sample_shape_(std::move(sample_shape)), batch_(batch_size),
      depth_(std::max<int64_t>(depth, 2)), drop_last_(drop_last), pin_(pin_memory), scale_(scale), device_(device) {
  TORCH_CHECK(data_.device().is_cpu() && targets_.device().is_cpu() && data_.is_contiguous() && targets_.is_contiguous(),
              "BatchStager: dataset tensors must be contiguous CPU tensors");
  TORCH_CHECK(data_.scalar_type() == at::kByte || data_.scalar_type() == at::kFloat, "BatchStager: data must be uint8 or float32");
  TORCH_CHECK(data_.dim() >= 1 && targets_.dim() == 1 && data_.size(0) == targets_.size(0), "BatchStager: data/targets disagree");
  TORCH_CHECK(batch_ > 0, "BatchStager: batch size must be positive");
  row_elems_ = data_.numel() / std::max<int64_t>(data_.size(0), 1);
  int64_t want = 1;
  for (auto d : sample_shape_) want *= d;
  TORCH_CHECK(want == row_elems_, "BatchStager: sample_shape does not match the dataset rows");
  ring_.resize(static_cast<size_t>(depth_));
  int64_t slot_index = 0;
  for (auto& s : ring_) {
    alloc_slot(s);
    s.seq = slot_index++;   // slot i takes batches i, i + depth, i + 2·depth, … (numbered across epochs)
  }
}

BatchStager::~BatchStager() { stop_worker(); }

void BatchStager::alloc_slot(Slot& s) {
  std::vector<int64_t> shp{batch_};
  shp.insert(shp.end(), sample_shape_.begin(), sample_shape_.end());
  auto io = at::TensorOptions().dtype(at::kFloat).device(at::kCPU).pinned_memory(pin_);
  auto to = at::TensorOptions().dtype(targets_.scalar_type()).device(at::kCPU).pinned_memory(pin_);
  s.images = at::empty(shp, io);
  s.targets = at::empty({batch_}, to);
  s.out = std::make_shared<std::atomic<int>>(0);
}

void BatchStager::stop_worker() {
  {
    std::lock_guard<std::mutex> g(mu_);
    stop_ = true;
  }
  cv_.notify_all();
  for (auto& t : workers_) if (t.joinable()) t.join();
  workers_.clear();
  stop_ = false;
  running_ = false;
}

void BatchStager::start(at::Tensor indices) {
  TORCH_CHECK(indices.device().is_cpu() && indices.scalar_type() == at::kLong && indices.dim() == 1, "BatchStager.start: int64 CPU index vector expected");
  stop_worker();
  indices_ = indices.contiguous();
  const int64_t n = indices_.numel();
  nbatches_ = drop_last_ ? n / batch_ : (n + batch_ - 1) / batch_;
  // Batches are numbered across epochs (consume_ never resets): the slots handed back in the previous epoch whose CUDA events are
  // still pending stay in the ring's normal reaping order instead of being waited for here — with a 75-step epoch (8 ranks) that
  // wait (the device is ~15 steps behind the host) stalled the training thread for milliseconds per epoch.
  base_ = consume_;
  produce_ = 0;
  error_ = nullptr;
  st_fill_us_ = st_wait_free_us_ = st_next_wait_us_ = st_ready_sum_ = st_alloc_us_ = 0;
  st_allocs_ = 0;
  st_next_calls_ = 0;
  ++epoch_;
  for (auto& s : ring_) {
    if (s.state == 1) s.state = 0;   // staged for the abandoned epoch: its number (seq) now belongs to a batch of this epoch
  }
  running_ = true;
  if (const char* e = std::getenv("PDT_LOADER_WORKERS")) nworkers_ = std::max(1, std::atoi(e));
  nworkers_ = static_cast<int>(std::min<int64_t>(nworkers_, std::max<int64_t>(1, depth_ / 2)));
  for (int w = 0; w < nworkers_; ++w) workers_.emplace_back([this, w] { this->worker(w); });
}

void BatchStager::worker(int w) {
  // an exception in a std::thread would terminate the process: park it and let the consumer's next() rethrow it
  try {
    worker_loop(w);
  } catch (...) {
    {
      std::lock_guard<std::mutex> g(mu_);
      if (!error_) error_ = std::current_exception();
    }
    cv_.notify_all();
  }
}

void BatchStager::worker_loop(int w) {
#if PDT_WITH_CUDA
  if (pin_ && device_ >= 0) cudaSetDevice(device_);
#endif
  const int64_t n = indices_.numel();
  const int64_t* idx = indices_.data_ptr<int64_t>();
  const int64_t N = data_.size(0);
  const size_t tsize = targets_.element_size();
  for (int64_t b = base_ + w; b < base_ + nbatches_; b += nworkers_) {   // b: global batch number, b - base_: index in this epoch
    Slot& s = ring_[static_cast<size_t>(b % depth_)];
    const auto tw0 = std::chrono::steady_clock::now();
    {
      std::unique_lock<std::mutex> lk(mu_);
      cv_.wait(lk, [&] { return stop_ || (s.state == 0 && s.seq == b); });   // free (handed back, consumer's event completed) and it is batch b's turn
      if (stop_) return;
    }
    const auto tw1 = std::chrono::steady_clock::now();
    // a batch somebody still holds (list(loader), a stashed view) is never overwritten: the slot gets fresh buffers, the old ones
    // live on until the last tensor handed out over them dies (see next(): outstanding-tensor counter)
    bool fresh = false;
    if (s.out->load(std::memory_order_acquire) != 0) {
      alloc_slot(s);
      fresh = true;
    }
    const auto tw1b = std::chrono::steady_clock::now();
    const int64_t lo = (b - base_) * batch_, hi = std::min(n, lo + batch_);
    float* out = s.images.data_ptr<float>();
    char* tout = static_cast<char*>(s.targets.data_ptr());
    const char* tin = static_cast<const char*>(targets_.data_ptr());
    if (data_.scalar_type() == at::kByte) {
      const uint8_t* src = data_.data_ptr<uint8_t>();
      const float sc = static_cast<float>(scale_);
      for (int64_t i = lo; i < hi; ++i) {
        const int64_t r = idx[i];
        TORCH_CHECK(r >= 0 && r < N, "BatchStager: index ", r, " out of range");
        if (i + 3 < hi) {   // the sampler's order is random: pull the row three samples ahead towards the cache while this one converts
          const int64_t rn = idx[i + 3];
          if (rn >= 0 && rn < N) {
            const char* pn = reinterpret_cast<const char*>(src + rn * row_elems_);
            for (int64_t off = 0; off < row_elems_; off += 64) __builtin_prefetch(pn + off, 0, 1);
          }
        }
        const uint8_t* p = src + r * row_elems_;
        float* o = out + (i - lo) * row_elems_;
        u8_to_f32(p, o, row_elems_, sc);
        std::memcpy(tout + (i - lo) * tsize, tin + r * tsize, tsize);
      }
    } else {
      const float* src = data_.data_ptr<float>();
      const float sc = static_cast<float>(scale_);
      for (int64_t i = lo; i < hi; ++i) {
        const int64_t r = idx[i];
        TORCH_CHECK(r >= 0 && r < N, "BatchStager: index ", r, " out of range");
        if (i + 3 < hi) {
          const int64_t rn = idx[i + 3];
          if (rn >= 0 && rn < N) {
            const char* pn = reinterpret_cast<const char*>(src + rn * row_elems_);
            for (int64_t off = 0; off < row_elems_ * 4; off += 64) __builtin_prefetch(pn + off, 0, 1);
          }
        }
        const float* p = src + r * row_elems_;
        float* o = out + (i - lo) * row_elems_;
        if (sc == 1.f) std::memcpy(o, p, static_cast<size_t>(row_elems_) * sizeof(float));
        else for (int64_t k = 0; k < row_elems_; ++k) o[k] = p[k] * sc;
        std::memcpy(tout + (i - lo) * tsize, tin + r * tsize, tsize);
      }
    }
    const auto tw2 = std::chrono::steady_clock::now();
    {
      std::lock_guard<std::mutex> g(mu_);
      s.rows = hi - lo;
      s.state = 1;
      ++produce_;
      st_wait_free_us_ += std::chrono::duration<double, std::micro>(tw1 - tw0).count();
      st_fill_us_ += std::chrono::duration<double, std::micro>(tw2 - tw1b).count();
      st_alloc_us_ += std::chrono::duration<double, std::micro>(tw1b - tw1).count();
      st_allocs_ += fresh ? 1 : 0;
    }
    cv_.notify_all();
  }
}

std::vector<double> BatchStager::stats() const {
  std::lock_guard<std::mutex> g(const_cast<std::mutex&>(mu_));
  return {static_cast<double>(produce_), st_fill_us_, st_wait_free_us_, static_cast<double>(st_next_calls_), st_ready_sum_, st_next_wait_us_,
          static_cast<double>(st_allocs_), st_alloc_us_};
}

void BatchStager::reap_events_locked() {
  // events complete in the order they were recorded: stop at the first one that has not
  for (int64_t b = reap_; b < consume_; ++b) {
    Slot& p = ring_[static_cast<size_t>(b % depth_)];
    if (p.state != 3) break;
#if PDT_WITH_CUDA
    if (p.event && !static_cast<at::cuda::CUDAEvent*>(p.event.get())->query()) break;
#endif
    p.event.reset();
    p.state = 0;
    p.seq = b + depth_;
    reap_ = b + 1;
  }
}

bool BatchStager::next(at::Tensor* images, at::Tensor* targets) {
  // The consumer moves on.  The batch handed out TWO calls ago goes back to the ring: its tensors are no longer referenced by an
  // ordinary `for batch in loader` loop (the loop variables and the iterator's own frame still hold the *previous* batch while this
  // call runs — releasing that one here made the retention check below re-allocate its pinned buffers on every step whenever the
  // device was idle).  Everything the consumer enqueued on its current stream for that batch precedes the event.
  if (prev_handed_ >= 0) {
    Slot& p = ring_[static_cast<size_t>(prev_handed_ % depth_)];
    std::shared_ptr<void> ev;
#if PDT_WITH_CUDA
    if (pin_ && device_ >= 0) {
      c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device_));
      auto* e = new at::cuda::CUDAEvent(cudaEventDisableTiming);
      e->record(c10::cuda::getCurrentCUDAStream(static_cast<c10::DeviceIndex>(device_)));
      ev = std::shared_ptr<void>(e, [](void* q) { delete static_cast<at::cuda::CUDAEvent*>(q); });
    }
#endif
    {
      std::lock_guard<std::mutex> g(mu_);
      p.event = std::move(ev);
      p.state = 3;
      reap_events_locked();
    }
    cv_.notify_all();
  }
  prev_handed_ = last_handed_;
  last_handed_ = -1;
  if (consume_ >= base_ + nbatches_) return false;
  Slot& s = ring_[static_cast<size_t>(consume_ % depth_)];
  {
    std::unique_lock<std::mutex> lk(mu_);
    const auto tn0 = std::chrono::steady_clock::now();
    ++st_next_calls_;
    for (const auto& q : ring_) st_ready_sum_ += q.state == 1 ? 1.0 : 0.0;
    struct Acc {
      double& dst;
      std::chrono::steady_clock::time_point t0;
      ~Acc() { dst += std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t0).count(); }
    } acc{st_next_wait_us_, tn0};
    while (s.state != 1) {
      if (error_) {   // a worker failed (bad index, allocation failure): surface it on the training thread
        std::exception_ptr e = error_;
        lk.unlock();
        std::rethrow_exception(e);
      }
      // the batch is not staged yet: maybe every slot is waiting for the device — keep reaping while we wait
      const int64_t before = reap_;
      reap_events_locked();
      if (reap_ != before) {
        lk.unlock();
        cv_.notify_all();
        lk.lock();
        continue;
      }
      cv_.wait_for(lk, std::chrono::microseconds(20));
    }
    s.state = 2;
  }
  // Hand out FRESH tensor objects over the slot's buffers.  Their storage deleter keeps the buffers alive and counts the tensors
  // still in user hands — the retention check of the worker.  (Handing out the ring's own tensors and looking at use_count() does
  // not work: once a tensor has had a Python wrapper, the wrapper and the TensorImpl keep each other alive, so the count never
  // returns to one and every refill re-allocated its pinned buffers.)
  {
    std::vector<int64_t> shp{s.rows};
    shp.insert(shp.end(), sample_shape_.begin(), sample_shape_.end());
    auto out = s.out;
    at::Tensor keep_i = s.images, keep_t = s.targets;
    out->fetch_add(2, std::memory_order_acq_rel);
    *images = at::from_blob(s.images.data_ptr(), shp, [out, keep_i](void*) { out->fetch_sub(1, std::memory_order_acq_rel); },
                            at::TensorOptions().dtype(at::kFloat).device(at::kCPU));
    *targets = at::from_blob(s.targets.data_ptr(), {s.rows}, [out, keep_t](void*) { out->fetch_sub(1, std::memory_order_acq_rel); },
                             at::TensorOptions().dtype(targets_.scalar_type()).device(at::kCPU));
  }
  last_handed_ = consume_;
  ++consume_;
  return true;
}

}  // namespace pdt
