// CPU collective backend ("gloo"-equivalent plumbing path; ref: ddp_example.py:105 --backend,
// BASELINE.json config 1). Own design: full TCP mesh bootstrapped through the Store, one FIFO
// worker thread per process group (identical op order on every rank), deterministic reduction
// order (results are bitwise identical across ranks).
#pragma once
#include <condition_variable>
#include <deque>
#include <exception>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "../common/net.h"
#include "../store/store.h"

namespace pdt {

enum class DType : int { F32 = 0, F64 = 1, F16 = 2, BF16 = 3, I8 = 4, U8 = 5, I32 = 6, I64 = 7, BOOL = 8, I16 = 9 };
enum class ReduceOp : int { SUM = 0, AVG = 1, PRODUCT = 2, MIN = 3, MAX = 4, BAND = 5, BOR = 6, BXOR = 7 };

size_t dtype_size(DType t);
// dst = dst (op) src, elementwise, `count` elements.
void reduce_inplace(void* dst, const void* src, size_t count, DType t, ReduceOp op);
void scale_inplace(void* dst, size_t count, DType t, double factor);

// Completion handle. wait() rethrows the worker's exception on the caller's thread.
class Work {
 public:
  void wait(Millis timeout);
  bool is_completed();
  bool is_success();
  std::string error();
  // internal
  void finish(std::exception_ptr e);

 private:
  std::mutex mu_;
  std::condition_variable cv_;
  bool done_ = false;
  std::exception_ptr err_;
};

class CpuBackend {
 public:
  CpuBackend(std::shared_ptr<Store> store, int rank, int size, Millis timeout, const std::string& bind_host);
  ~CpuBackend();
  int rank() const { return rank_; }
  int size() const { return size_; }
  Millis timeout() const { return timeout_; }

  // Asynchronous API: the op is queued to the worker; buffers must stay alive until wait().
  std::shared_ptr<Work> allreduce(void* buf, size_t count, DType t, ReduceOp op);
  std::shared_ptr<Work> broadcast(void* buf, size_t nbytes, int root);
  std::shared_ptr<Work> allgather(const void* in, void* out, size_t nbytes_per_rank);
  std::shared_ptr<Work> reduce(void* buf, size_t count, DType t, ReduceOp op, int root);
  std::shared_ptr<Work> reduce_scatter(const void* in, void* out, size_t count_per_rank, DType t, ReduceOp op);
  std::shared_ptr<Work> gather(const void* in, void* out, size_t nbytes_per_rank, int root);
  std::shared_ptr<Work> scatter(const void* in, void* out, size_t nbytes_per_rank, int root);
  std::shared_ptr<Work> alltoall(const void* in, void* out, size_t nbytes_per_rank);
  std::shared_ptr<Work> send(const void* buf, size_t nbytes, int dst);
  std::shared_ptr<Work> recv(void* buf, size_t nbytes, int src);
  std::shared_ptr<Work> barrier();

  // Fault injection for the failure tests: the next `n` ops on this rank
  // sleep `ms` before running / are silently skipped.
  void inject_delay(int n_ops, int ms) { delay_ops_ = n_ops; delay_ms_ = ms; }
  void inject_skip(int n_ops) { skip_ops_ = n_ops; }
  uint64_t ops_completed() const { return seq_done_; }
  void shutdown();

 private:
  std::shared_ptr<Work> submit(std::function<void()> fn);
  void worker_loop();
  int peer(int r) const { return socks_[r].get(); }
  // blocking bodies (worker thread only)
  void do_allreduce(void* buf, size_t count, DType t, ReduceOp op);
  void do_broadcast(void* buf, size_t nbytes, int root);
  void do_allgather(const void* in, void* out, size_t nb);
  void do_reduce(void* buf, size_t count, DType t, ReduceOp op, int root);
  void do_reduce_scatter(const void* in, void* out, size_t cpr, DType t, ReduceOp op);

  std::shared_ptr<Store> store_;
  int rank_, size_;
  Millis timeout_;
  std::vector<Fd> socks_;  // socks_[r] = connection to rank r (invalid for r == rank_)
  std::thread worker_;
  std::mutex mu_;
  std::condition_variable cv_;
  std::deque<std::pair<std::function<void()>, std::shared_ptr<Work>>> queue_;
  bool stop_ = false;
  std::atomic<int> delay_ops_{0}, delay_ms_{0}, skip_ops_{0};
  std::atomic<uint64_t> seq_done_{0};
  std::vector<char> scratch_;
};

}  // namespace pdt
