// Native batch stager behind data.DataLoader (ref: ddp_example.py:73-78 — DataLoader(batch_size=100, num_workers=0,
// pin_memory=True, sampler=...); torch/utils/data/dataloader.py:773-805 for the contract).
//
// The reference pays 100 PIL decodes + default_collate + pin_memory() on the training thread per step.  Here a C++
// worker thread (no GIL, no intra-op thread pool) gathers the sampler's indices out of the dataset tensor, converts
// uint8 → float32 on the way (ToTensor's 1/255), and writes straight into a ring of pinned buffers that is allocated
// once — a graph-replayed step is ~0.1 ms, and a pool miss in the pinned allocator (cudaHostAlloc) or a descheduled
// OpenMP worker was measured stalling the Python loader for tens of milliseconds.
//
// Ring safety: a slot is refilled only after (1) the consumer has asked for a later batch, (2) the CUDA event recorded
// on the consumer's stream at that moment has completed (so `.to(device, non_blocking=True)` copies out of the slot
// are done), and (3) nobody else holds a reference to the slot's tensors — if the user kept a batch (list(loader)),
// the slot gets fresh buffers instead of being overwritten.  The events are *queried by the consumer thread* (inside
// next(), oldest first): a worker parked in cudaEventSynchronize spins inside the driver and slowed every CUDA call of
// the training thread by several times; the worker itself never touches CUDA.
#pragma once
#include <ATen/ATen.h>

#include <atomic>
#include <condition_variable>
#include <exception>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

namespace pdt {

class BatchStager {
 public:
  BatchStager(at::Tensor data, at::Tensor targets, std::vector<int64_t> sample_shape, int64_t batch_size, bool drop_last, double scale,
              int64_t depth, bool pin_memory, int device);
  ~BatchStager();
  // Begin an epoch over `indices` (int64, CPU).  Any unfinished epoch is abandoned.
  void start(at::Tensor indices);
  // Next batch as (images float32 [b, *sample_shape], targets [b]); returns false at the end of the epoch.
  // Blocks (release the GIL around it) until the worker has staged the batch.
  bool next(at::Tensor* images, at::Tensor* targets);
  int64_t num_batches() const { return nbatches_; }
  // Diagnostics since start(): {batches produced, µs the worker spent filling, µs it waited for a free slot,
  // next() calls, Σ ready slots seen at next(), µs next() waited, slots re-allocated because a batch was still referenced, µs spent on that}
  std::vector<double> stats() const;

 private:
  struct Slot {
    at::Tensor images, targets;   // the slot's (pinned) buffers; handed out as from_blob views that count themselves
    std::shared_ptr<std::atomic<int>> out;   // tensors over these buffers still alive outside the ring
    int state = 0;          // 0 free, 1 ready, 2 handed out, 3 returned (waiting for the consumer's CUDA event)
    int64_t rows = 0;
    int64_t seq = 0;        // the batch index this slot takes next (several workers fill slots concurrently)
    std::shared_ptr<void> event;   // at::cuda::CUDAEvent recorded when the consumer moved on (opaque here)
  };
  void worker(int w);
  void worker_loop(int w);
  void alloc_slot(Slot& s);
  void reap_events_locked();   // returned slots whose event has completed become free (consumer thread, mu_ held)
  void stop_worker();

  at::Tensor data_, targets_, indices_;
  std::vector<int64_t> sample_shape_;
  int64_t batch_, row_elems_, nbatches_ = 0, depth_;
  bool drop_last_, pin_;
  double scale_;
  int device_;
  std::vector<Slot> ring_;
  std::vector<std::thread> workers_;   // worker w stages batches w, w + W, ... (PDT_LOADER_WORKERS, default 1)
  int nworkers_ = 1;
  std::mutex mu_;
  std::condition_variable cv_;
  int64_t produce_ = 0, consume_ = 0, reap_ = 0, epoch_ = 0, base_ = 0;   // consume_/reap_/base_: global batch numbers
  double st_fill_us_ = 0, st_wait_free_us_ = 0, st_next_wait_us_ = 0, st_ready_sum_ = 0;
  int64_t st_next_calls_ = 0, st_allocs_ = 0;
  double st_alloc_us_ = 0;
  int64_t last_handed_ = -1, prev_handed_ = -1;
  bool stop_ = false, running_ = false;
  std::exception_ptr error_;   // first exception of a worker thread, rethrown by next()
};

}  // namespace pdt
