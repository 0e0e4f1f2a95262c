#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDACachingAllocator.h>
#include <c10/cuda/CUDAGuard.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <sstream>

#include "cuda_comm.h"
#include "cuda_utils.h"

namespace pdt {

// ---- CudaWork / CudaCommBase ----------------------------------------------------------------------
void CudaWork::wait() {
  done_.block(c10::cuda::getCurrentCUDAStream(device_));
  // tensors stay referenced by `keep_` until this handle dies; the caching allocator has also
  // been told about the comm stream (recordStream), so dropping them early is safe too.
}
void CudaWork::synchronize() {
  done_.synchronize();
  keep_.clear();
}
bool CudaWork::is_completed() { return done_.query(); }

CudaCommBase::CudaCommBase(int rank, int size, int device)
    : rank_(rank), size_(size), device_(device), comm_stream_(c10::cuda::getStreamFromPool(/*isHighPriority=*/true, device)) {}

void CudaCommBase::check(const at::Tensor& t, const char* what) const {
  TORCH_CHECK(t.is_cuda(), "pdt ", backend_name(), " backend: ", what, " tensor must be a CUDA tensor (got ", t.device(), ")");
  TORCH_CHECK(t.device().index() == device_, "pdt ", backend_name(), " backend: ", what, " tensor lives on cuda:", t.device().index(),
              " but this process group drives cuda:", device_);
  TORCH_CHECK(t.is_contiguous(), "pdt ", backend_name(), " backend: ", what, " tensor must be contiguous");
}

std::shared_ptr<CommWork> CudaCommBase::enqueue(const std::vector<at::Tensor>& tensors,
                                               const std::function<void(cudaStream_t)>& fn) {
  c10::cuda::CUDAGuard guard(device_);
  auto cur = c10::cuda::getCurrentCUDAStream(device_);
  auto work = std::make_shared<CudaWork>(device_, tensors);
  at::cuda::CUDAEvent ready(cudaEventDisableTiming);
  ready.record(cur);
  ready.block(comm_stream_);
  for (auto& t : tensors)
    if (t.defined() && t.is_cuda() && t.storage().data_ptr().get_deleter() == c10::cuda::CUDACachingAllocator::get()->raw_deleter())
      c10::cuda::CUDACachingAllocator::recordStream(t.storage().data_ptr(), comm_stream_);
  fn(comm_stream_.stream());
  work->done().record(comm_stream_);
  return work;
}

namespace {
class CudaStamp : public DeviceStamp {
 public:
  explicit CudaStamp(c10::cuda::CUDAStream s) : ev_(cudaEventDefault) { ev_.record(s); }
  bool ready() override { return ev_.query(); }
  double us_since(DeviceStamp& earlier) override { return static_cast<double>(static_cast<CudaStamp&>(earlier).ev_.elapsed_time(ev_)) * 1e3; }

 private:
  at::cuda::CUDAEvent ev_;
};
}  // namespace

std::shared_ptr<DeviceStamp> CudaCommBase::stamp(bool on_comm_stream) {
  c10::cuda::CUDAGuard guard(device_);
  return std::make_shared<CudaStamp>(on_comm_stream ? comm_stream_ : c10::cuda::getCurrentCUDAStream(device_));
}

bool CudaCommBase::capturing() const {
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(c10::cuda::getCurrentCUDAStream(device_).stream(), &st);
  return st != cudaStreamCaptureStatusNone;
}

// ---- SymmComm ---------------------------------------------------------------------------------------
SymmComm::SymmComm(std::shared_ptr<Store> store, int rank, int size, int device, Millis timeout, size_t heap_bytes)
    : CudaCommBase(rank, size, device) {
  c10::cuda::CUDAGuard guard(device);
  store_ = store;
  heap_ = std::make_shared<SymmetricHeap>(std::move(store), rank, size, device, heap_bytes, timeout);
  if (const char* a = getenv("PDT_AR_ALGO")) algo_ = a;
  // One-shot / two-shot crossover: at N = 2 a one-shot push moves the same bytes as a two-shot, so it stays ahead up to
  // large messages; at N = 8 it sends 7× the data and falls behind much earlier.  These switch points were chosen on the
  // previous NVLink generation and have not been re-measured on H100 (NVLink 4); tools/allreduce_sweep.py measures them,
  // PDT_AR_ONESHOT_MAX overrides them.
  oneshot_max_ = size <= 2 ? (size_t(4) << 20) : size <= 4 ? (size_t(1) << 20) : (size_t(512) << 10);
  if (const char* m = getenv("PDT_AR_ONESHOT_MAX")) oneshot_max_ = static_cast<size_t>(atoll(m));
  if (const char* b = getenv("PDT_AR_BLOCKS")) cfg_.blocks = atoi(b);
  if (const char* t = getenv("PDT_AR_THREADS")) cfg_.threads = atoi(t);
}

SymmComm::~SymmComm() { shutdown(); }

void SymmComm::shutdown() {
  if (down_) return;
  down_ = true;
  cudaSetDevice(device_);
  cudaDeviceSynchronize();
}

std::string SymmComm::describe() const {
  std::ostringstream os;
  os << "SymmComm(rank=" << rank_ << "/" << size_ << ", device=" << device_ << ", transport=" << heap_->transport()
     << ", multicast=" << (heap_->has_multicast() ? "yes" : "no") << ", heap=" << (heap_->heap_bytes() >> 20) << "MiB, algo=" << algo_
     << ", oneshot_max=" << oneshot_max_ << ")";
  return os.str();
}

at::Tensor SymmComm::alloc_flat(int64_t numel, at::ScalarType dtype, const at::Device& device) {
  TORCH_CHECK(device.is_cuda() && device.index() == device_, "alloc_flat: device mismatch");
  const size_t nbytes = static_cast<size_t>(std::max<int64_t>(numel, 1)) * c10::elementSize(dtype);
  // alloc_flat is a *collective* (every rank calls it in the same order — DDP construction, bucket rebuild, optimizer
  // fusion).  Kernels address peers as peer[r] + local_offset, so the allocator state must be identical everywhere:
  //  (1) blocks parked by tensor deleters are released only if *every* rank has parked them (set intersection
  //      exchanged through the store), after the device has drained (no in-flight kernel can still touch them);
  //  (2) the offset handed out is cross-checked against rank 0's and a mismatch raises instead of corrupting memory.
  const uint64_t seq = alloc_seq_++;
  const std::string base = "symm/alloc/" + std::to_string(seq) + "/";
  if (size_ > 1) {
    std::vector<size_t> mine = heap_->pending_frees();
    std::string blob(reinterpret_cast<const char*>(mine.data()), mine.size() * sizeof(size_t));
    store_->set(base + "f/" + std::to_string(rank_), blob);
    std::vector<size_t> common = mine;
    for (int r = 0; r < size_ && !common.empty(); ++r) {
      if (r == rank_) continue;
      const std::string theirs = store_->get(base + "f/" + std::to_string(r));
      std::vector<size_t> v(theirs.size() / sizeof(size_t));
      std::memcpy(v.data(), theirs.data(), v.size() * sizeof(size_t));
      std::vector<size_t> both;
      std::set_intersection(common.begin(), common.end(), v.begin(), v.end(), std::back_inserter(both));
      common.swap(both);
    }
    if (!common.empty()) {
      c10::cuda::CUDAGuard guard(device_);
      PDT_CUDA_CHECK(cudaDeviceSynchronize());
      heap_->apply_frees(common);
    }
  }
  void* p = heap_->alloc(nbytes, 256);
  if (size_ > 1) {
    const std::string off = std::to_string(heap_->offset_of(p));
    store_->set(base + "o/" + std::to_string(rank_), off);
    const std::string off0 = rank_ == 0 ? off : store_->get(base + "o/0");
    if (off0 != off) {
      heap_->free(p);
      TORCH_CHECK(false, "symmetric heap diverged: allocation #", seq, " (", nbytes, " B) landed at offset ", off, " on rank ", rank_,
                  " but at ", off0, " on rank 0 — ranks must issue the same sequence of alloc_flat calls");
    }
  }
  // the tensor co-owns the heap: parameters/buckets may outlive the communicator object
  std::shared_ptr<SymmetricHeap> heap = heap_;
  at::Tensor t = at::from_blob(p, {numel}, [heap, p](void*) { heap->free(p); }, at::TensorOptions().dtype(dtype).device(device));
  t.zero_();
  return t;
}

static int to_symm_dtype(at::ScalarType t) { return static_cast<int>(to_dtype(t)); }

void SymmComm::do_allreduce(at::Tensor& t, ReduceOp op, double scale, int channel, cudaStream_t s) {
  const size_t nbytes = t.nbytes();
  if (nbytes == 0) return;
  if (op == ReduceOp::AVG) { scale *= 1.0 / size_; op = ReduceOp::SUM; }
  const int dt = to_symm_dtype(t.scalar_type());
  const bool floating = at::isFloatingType(t.scalar_type());
  TORCH_CHECK(scale == 1.0 || floating, "postscale is only defined for floating-point tensors");
  const bool aligned = (reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0) && (nbytes % 16 == 0);
  const bool in_heap = aligned && heap_->contains(t.data_ptr(), nbytes);
  const bool nvls_ok = heap_->has_multicast() && op == ReduceOp::SUM &&
                       (t.scalar_type() == at::kFloat || t.scalar_type() == at::kHalf || t.scalar_type() == at::kBFloat16);
  const size_t half = heap_->staging_half_bytes(channel);
  const size_t slot_bytes = (nbytes + 15) / 16 * 16;
  std::string algo = algo_;
  if (algo == "auto") {
    if (slot_bytes * size_ <= half && nbytes <= oneshot_max_) algo = heap_->has_multicast() ? "oneshot_mc" : "oneshot";
    // with two ranks the switch adds a hop and reduces nothing: peer loads are preferred to NVLS
    else algo = (nvls_ok && size_ > 2) ? "nvls" : "twoshot";
  }
  if ((algo == "oneshot" || algo == "oneshot_mc") && slot_bytes * size_ > half) algo = nvls_ok ? "nvls" : "twoshot";
  if (algo == "oneshot_mc" && !heap_->has_multicast()) algo = "oneshot";
  if (algo == "nvls" && !nvls_ok) algo = "twoshot";
  SymmDev d = heap_->dev(channel);
  if (size_ == 1) {
    if (scale != 1.0) t.mul_(scale);
    return;
  }
  if (algo == "oneshot" || algo == "oneshot_mc") {
    const int parity = heap_->next_parity(channel);
    const size_t stage = heap_->staging_off(channel, parity);
    if (aligned) {
      launch_allreduce_oneshot_push(d, t.data_ptr(), t.data_ptr(), stage, static_cast<size_t>(t.numel()), dt, static_cast<int>(op), scale,
                                    algo == "oneshot_mc", cfg_, s);
    } else {
      // odd size / alignment: bounce through a padded scratch vector
      const int64_t es = static_cast<int64_t>(t.element_size());
      const int64_t padded = static_cast<int64_t>(slot_bytes) / es;
      at::Tensor tmp = at::zeros({padded}, t.options());
      tmp.narrow(0, 0, t.numel()).copy_(t.view(-1));
      launch_allreduce_oneshot_push(d, tmp.data_ptr(), tmp.data_ptr(), stage, static_cast<size_t>(padded), dt, static_cast<int>(op), scale,
                                    algo == "oneshot_mc", cfg_, s);
      t.view(-1).copy_(tmp.narrow(0, 0, t.numel()));
    }
    return;
  }
  // two-shot family works in place on symmetric memory
  if (in_heap) {
    launch_allreduce_twoshot(d, heap_->offset_of(t.data_ptr()), static_cast<size_t>(t.numel()), dt, static_cast<int>(op), scale,
                             algo == "nvls", cfg_, s);
    return;
  }
  // ordinary tensor: stream it through the staging area in chunks (copy-in, reduce in place, copy-out)
  const size_t es = t.element_size();
  const size_t chunk_elems = (half / 16 * 16) / es;
  char* p = static_cast<char*>(t.data_ptr());
  size_t done = 0;
  const size_t total = static_cast<size_t>(t.numel());
  while (done < total) {
    const size_t n = std::min(chunk_elems, total - done);
    const size_t n_pad = ((n * es + 15) / 16 * 16) / es;
    const int parity = heap_->next_parity(channel);
    const size_t stage = heap_->staging_off(channel, parity);
    char* stg = heap_->local_base() + stage;
    if (n_pad != n) PDT_CUDA_CHECK(cudaMemsetAsync(stg + n * es, 0, (n_pad - n) * es, s));
    PDT_CUDA_CHECK(cudaMemcpyAsync(stg, p + done * es, n * es, cudaMemcpyDeviceToDevice, s));
    launch_allreduce_twoshot(d, stage, n_pad, dt, static_cast<int>(op), scale, algo == "nvls", cfg_, s);
    PDT_CUDA_CHECK(cudaMemcpyAsync(p + done * es, stg, n * es, cudaMemcpyDeviceToDevice, s));
    done += n;
  }
}

std::shared_ptr<CommWork> SymmComm::allreduce(at::Tensor t, ReduceOp op, double postscale) {
  check(t, "allreduce");
  record("allreduce", &t);
  return enqueue({t}, [&](cudaStream_t s) {
    c10::cuda::CUDAStreamGuard sg(comm_stream_);  // the odd-size bounce path issues ATen ops
    do_allreduce(t, op, postscale, kChanComm, s);
  });
}

void SymmComm::allreduce_inline(at::Tensor t, ReduceOp op, double postscale) {
  check(t, "allreduce");
  record("allreduce_inline", &t);
  c10::cuda::CUDAGuard guard(device_);
  do_allreduce(t, op, postscale, kChanInline, c10::cuda::getCurrentCUDAStream(device_).stream());
}

void SymmComm::allreduce_sgd_inline(at::Tensor grad, at::Tensor param, c10::optional<at::Tensor> momentum_buf, double lr,
                                    c10::optional<at::Tensor> lr_tensor, double momentum, double dampening, double weight_decay,
                                    bool nesterov, bool first_step) {
  check(grad, "allreduce_sgd grad");
  check(param, "allreduce_sgd param");
  TORCH_CHECK(grad.scalar_type() == at::kFloat && param.scalar_type() == at::kFloat && grad.numel() == param.numel(),
              "allreduce_sgd: flat fp32 grad/param vectors of equal length required");
  TORCH_CHECK(grad.numel() % 4 == 0 && reinterpret_cast<uintptr_t>(grad.data_ptr()) % 16 == 0 &&
                  reinterpret_cast<uintptr_t>(param.data_ptr()) % 16 == 0,
              "allreduce_sgd: vectors must be 16-byte aligned with length % 4 == 0");
  float* mom = nullptr;
  if (momentum != 0.0) {
    TORCH_CHECK(momentum_buf.has_value() && momentum_buf->numel() == grad.numel(), "allreduce_sgd: momentum buffer required");
    mom = momentum_buf->data_ptr<float>();
  }
  record("allreduce_sgd", &grad);
  c10::cuda::CUDAGuard guard(device_);
  cudaStream_t s = c10::cuda::getCurrentCUDAStream(device_).stream();
  const size_t nbytes = grad.nbytes();
  const int channel = kChanInline;
  TORCH_CHECK(nbytes * size_ <= heap_->staging_half_bytes(channel),
              "allreduce_sgd: flat gradient too large for the one-shot staging area (", nbytes, " B × ", size_, ")");
  const int parity = heap_->next_parity(channel);
  launch_allreduce_sgd_oneshot(heap_->dev(channel), grad.data_ptr<float>(), param.data_ptr<float>(), mom,
                               heap_->staging_off(channel, parity), static_cast<size_t>(grad.numel()), 1.0f / size_,
                               lr_tensor.has_value() ? lr_tensor->data_ptr<float>() : nullptr, static_cast<float>(lr),
                               static_cast<float>(momentum), static_cast<float>(dampening), static_cast<float>(weight_decay), nesterov,
                               first_step, heap_->has_multicast() && algo_ != "oneshot", cfg_, s);
}

std::shared_ptr<CommWork> SymmComm::allreduce_sgd(at::Tensor grad, at::Tensor param, at::Tensor momentum_buf, const FusedSgd& h, at::Tensor bcast,
                                                  int bcast_root) {
  check(grad, "allreduce_sgd grad");
  check(param, "allreduce_sgd param");
  const bool fits = grad.scalar_type() == at::kFloat && param.scalar_type() == at::kFloat && grad.numel() == param.numel() &&
                    grad.numel() % 4 == 0 && reinterpret_cast<uintptr_t>(grad.data_ptr()) % 16 == 0 &&
                    reinterpret_cast<uintptr_t>(param.data_ptr()) % 16 == 0 &&
                    (!momentum_buf.defined() || reinterpret_cast<uintptr_t>(momentum_buf.data_ptr()) % 16 == 0);
  const size_t bc_bytes = (bcast.defined() && size_ > 1) ? bcast.nbytes() : 0;
  const bool bc_ok = bc_bytes == 0 || (bcast.is_cuda() && bcast.is_contiguous() && bc_bytes % 16 == 0 &&
                                       reinterpret_cast<uintptr_t>(bcast.data_ptr()) % 16 == 0);
  const size_t need = grad.nbytes() * static_cast<size_t>(size_) + bc_bytes;
  if (size_ == 1 || !fits || !bc_ok || need > heap_->staging_half_bytes(kChanComm))
    return Comm::allreduce_sgd(grad, param, momentum_buf, h, bcast, bcast_root);  // composition: allreduce + ATen + broadcast
  TORCH_CHECK(h.momentum == 0 || (momentum_buf.defined() && momentum_buf.numel() == grad.numel()), "allreduce_sgd: momentum buffer required");
  record("allreduce_sgd", &grad);
  std::vector<at::Tensor> keep{grad, param};
  if (momentum_buf.defined()) keep.push_back(momentum_buf);
  if (bc_bytes) keep.push_back(bcast);
  if (h.lr_tensor.defined()) keep.push_back(h.lr_tensor);
  return enqueue(keep, [&](cudaStream_t s) {
    const int parity = heap_->next_parity(kChanComm);
    launch_allreduce_sgd_oneshot(heap_->dev(kChanComm), grad.data_ptr<float>(), param.data_ptr<float>(),
                                 (h.momentum != 0 && momentum_buf.defined()) ? momentum_buf.data_ptr<float>() : nullptr,
                                 heap_->staging_off(kChanComm, parity), static_cast<size_t>(grad.numel()), 1.0f / size_,
                                 h.lr_tensor.defined() ? h.lr_tensor.data_ptr<float>() : nullptr, static_cast<float>(h.lr),
                                 static_cast<float>(h.momentum), static_cast<float>(h.dampening), static_cast<float>(h.weight_decay),
                                 h.nesterov, h.first_step, heap_->has_multicast() && algo_ != "oneshot", cfg_, s,
                                 bc_bytes ? bcast.data_ptr() : nullptr, bc_bytes, bcast_root);
  });
}

void SymmComm::do_broadcast(at::Tensor& t, int root, int channel, cudaStream_t s) {
  const size_t nbytes = t.nbytes();
  if (nbytes == 0 || size_ == 1) return;
  SymmDev d = heap_->dev(channel);
  if (heap_->contains(t.data_ptr(), nbytes)) {
    launch_broadcast_pull(d, heap_->offset_of(t.data_ptr()), t.data_ptr(), nbytes, root, /*exit_barrier=*/true, cfg_, s);
    return;
  }
  const size_t half = heap_->staging_half_bytes(channel);
  char* p = static_cast<char*>(t.data_ptr());
  for (size_t done = 0; done < nbytes; done += half) {
    const size_t n = std::min(half, nbytes - done);
    const size_t stage = heap_->staging_off(channel, heap_->next_parity(channel));
    if (rank_ == root) PDT_CUDA_CHECK(cudaMemcpyAsync(heap_->local_base() + stage, p + done, n, cudaMemcpyDeviceToDevice, s));
    // the root's destination is its own (already correct) tensor: pull into it anyway would be a
    // self-copy from staging — harmless and keeps every rank on the same barrier sequence
    launch_broadcast_pull(d, stage, p + done, n, root, /*exit_barrier=*/false, cfg_, s);
  }
}

std::shared_ptr<CommWork> SymmComm::broadcast(at::Tensor t, int root) {
  check(t, "broadcast");
  TORCH_CHECK(root >= 0 && root < size_, "broadcast: invalid root");
  record("broadcast", &t);
  return enqueue({t}, [&](cudaStream_t s) { do_broadcast(t, root, kChanComm, s); });
}

void SymmComm::broadcast_inline(at::Tensor t, int root) {
  check(t, "broadcast");
  TORCH_CHECK(root >= 0 && root < size_, "broadcast: invalid root");
  record("broadcast_inline", &t);
  c10::cuda::CUDAGuard guard(device_);
  do_broadcast(t, root, kChanInline, c10::cuda::getCurrentCUDAStream(device_).stream());
}

// ---- point-to-point ------------------------------------------------------------------------------------
// Device-signalled (p2p_send_kernel / p2p_recv_kernel): the sender stores the chunk into the slot the receiver's heap
// reserves for it and raises a flag in the receiver's signal pad; the receiver copies the chunk out and raises the
// acknowledgement in the sender's pad.  No store traffic, no stream synchronisation, plain kernels on the caller's stream.
// Messages up to one slot (32 MiB / world) are eager; longer ones advance chunk by chunk as the receiver acknowledges.
namespace {
constexpr int kChanP2P = 3;
}  // namespace

std::shared_ptr<CommWork> SymmComm::send(at::Tensor t, int dst) {
  check(t, "send");
  TORCH_CHECK(dst >= 0 && dst < size_ && dst != rank_, "send: invalid destination rank ", dst);
  record("send", &t);
  c10::cuda::CUDAGuard guard(device_);
  auto cur = c10::cuda::getCurrentCUDAStream(device_);
  const size_t slot = (2 * heap_->staging_half_bytes(kChanP2P) / static_cast<size_t>(size_)) / 256 * 256;
  const size_t slot_off = heap_->staging_off(kChanP2P, 0) + static_cast<size_t>(rank_) * slot;   // my slot in the receiver's heap
  const size_t nbytes = t.nbytes();
  const char* p = static_cast<const char*>(t.data_ptr());
  size_t done = 0;
  do {
    const size_t n = std::min(slot, nbytes - done);
    launch_p2p_send(heap_->dev(kChanP2P), p + done, n, dst, slot_off, static_cast<unsigned int>(++send_seq_[dst]), cur.stream());
    done += n;
  } while (done < nbytes);
  auto work = std::make_shared<CudaWork>(device_, std::vector<at::Tensor>{t});
  work->done().record(cur);
  return work;
}

std::shared_ptr<CommWork> SymmComm::recv(at::Tensor t, int src) {
  check(t, "recv");
  TORCH_CHECK(src >= 0 && src < size_ && src != rank_, "recv: invalid source rank ", src);
  record("recv", &t);
  c10::cuda::CUDAGuard guard(device_);
  auto cur = c10::cuda::getCurrentCUDAStream(device_);
  const size_t slot = (2 * heap_->staging_half_bytes(kChanP2P) / static_cast<size_t>(size_)) / 256 * 256;
  const size_t slot_off = heap_->staging_off(kChanP2P, 0) + static_cast<size_t>(src) * slot;     // the sender's slot in my heap
  const size_t nbytes = t.nbytes();
  char* p = static_cast<char*>(t.data_ptr());
  size_t done = 0;
  do {
    const size_t n = std::min(slot, nbytes - done);
    launch_p2p_recv(heap_->dev(kChanP2P), p + done, n, src, slot_off, static_cast<unsigned int>(++recv_seq_[src]), cur.stream());
    done += n;
  } while (done < nbytes);
  auto work = std::make_shared<CudaWork>(device_, std::vector<at::Tensor>{t});
  work->done().record(cur);
  return work;
}

std::shared_ptr<CommWork> SymmComm::allgather(at::Tensor out, at::Tensor in) {
  check(out, "allgather output");
  check(in, "allgather input");
  TORCH_CHECK(out.numel() == in.numel() * size_ && out.scalar_type() == in.scalar_type(),
              "allgather: output must hold world_size × input elements of the same dtype");
  record("allgather", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    const size_t nbytes = in.nbytes();
    if (nbytes == 0) return;
    if (size_ == 1) {
      PDT_CUDA_CHECK(cudaMemcpyAsync(out.data_ptr(), in.data_ptr(), nbytes, cudaMemcpyDeviceToDevice, s));
      return;
    }
    SymmDev d = heap_->dev(kChanComm);
    const size_t half = heap_->staging_half_bytes(kChanComm);
    const char* src = static_cast<const char*>(in.data_ptr());
    char* dst = static_cast<char*>(out.data_ptr());
    for (size_t done = 0; done < nbytes; done += half) {
      const size_t n = std::min(half, nbytes - done);
      const size_t stage = heap_->staging_off(kChanComm, heap_->next_parity(kChanComm));
      PDT_CUDA_CHECK(cudaMemcpyAsync(heap_->local_base() + stage, src + done, n, cudaMemcpyDeviceToDevice, s));
      launch_allgather_pull(d, stage, dst + done, n, nbytes, /*exit_barrier=*/false, cfg_, s);
    }
  });
}

std::shared_ptr<CommWork> SymmComm::alltoall(at::Tensor out, at::Tensor in) {
  check(out, "alltoall output");
  check(in, "alltoall input");
  TORCH_CHECK(in.numel() == out.numel() && in.numel() % size_ == 0 && in.scalar_type() == out.scalar_type(), "alltoall: equal splits required");
  record("alltoall", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    const size_t total = in.nbytes(), blk = total / size_;
    if (total == 0) return;
    TORCH_CHECK(total <= heap_->staging_half_bytes(kChanComm), "alltoall: message larger than the staging area (", total, " B)");
    const size_t stage = heap_->staging_off(kChanComm, heap_->next_parity(kChanComm));
    PDT_CUDA_CHECK(cudaMemcpyAsync(heap_->local_base() + stage, in.data_ptr(), total, cudaMemcpyDeviceToDevice, s));
    if (size_ == 1) {
      PDT_CUDA_CHECK(cudaMemcpyAsync(out.data_ptr(), in.data_ptr(), total, cudaMemcpyDeviceToDevice, s));
      return;
    }
    launch_alltoall_pull(heap_->dev(kChanComm), stage, out.data_ptr(), blk, blk, /*exit_barrier=*/false, cfg_, s);
  });
}

// ---- rooted / scattered collectives: one barrier-synchronised kernel over the staging area each, no clone + allreduce ------
std::shared_ptr<CommWork> SymmComm::reduce(at::Tensor t, ReduceOp op, int root) {
  check(t, "reduce");
  TORCH_CHECK(root >= 0 && root < size_, "reduce: invalid root");
  TORCH_CHECK(op != ReduceOp::AVG || at::isFloatingType(t.scalar_type()), "reduce: AVG is only defined for floating-point tensors");
  record("reduce", &t);
  return enqueue({t}, [&](cudaStream_t s) {
    const size_t nbytes = t.nbytes();
    if (nbytes == 0 || size_ == 1) return;
    double scale = 1.0;
    ReduceOp rop = op;
    if (op == ReduceOp::AVG) { scale = 1.0 / size_; rop = ReduceOp::SUM; }
    const size_t half = heap_->staging_half_bytes(kChanComm) / 16 * 16;
    char* p = static_cast<char*>(t.data_ptr());
    for (size_t done = 0; done < nbytes; done += half) {
      const size_t n = std::min(half, nbytes - done), n_pad = (n + 15) / 16 * 16;
      const size_t stage = heap_->staging_off(kChanComm, heap_->next_parity(kChanComm));
      char* stg = heap_->local_base() + stage;
      if (n_pad != n) PDT_CUDA_CHECK(cudaMemsetAsync(stg + n, 0, n_pad - n, s));
      PDT_CUDA_CHECK(cudaMemcpyAsync(stg, p + done, n, cudaMemcpyDeviceToDevice, s));
      // the root reduces every rank's parked chunk back into its own staging copy (an exact 16-byte multiple), then takes it
      launch_reduce_pull(heap_->dev(kChanComm), stage, 0, rank_ == root ? n_pad / 16 : 0, n_pad / 16, stg, to_symm_dtype(t.scalar_type()),
                         static_cast<int>(rop), scale, cfg_, s);
      if (rank_ == root) PDT_CUDA_CHECK(cudaMemcpyAsync(p + done, stg, n, cudaMemcpyDeviceToDevice, s));
    }
  });
}

std::shared_ptr<CommWork> SymmComm::reduce_scatter(at::Tensor out, at::Tensor in, ReduceOp op) {
  check(out, "reduce_scatter output");
  check(in, "reduce_scatter input");
  TORCH_CHECK(in.numel() == out.numel() * size_ && in.scalar_type() == out.scalar_type(), "reduce_scatter: input must hold world_size × output elements");
  TORCH_CHECK(op != ReduceOp::AVG || at::isFloatingType(out.scalar_type()), "reduce_scatter: AVG is only defined for floating-point tensors");
  record("reduce_scatter", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    const size_t slice = out.nbytes();
    if (slice == 0) return;
    if (size_ == 1) {
      PDT_CUDA_CHECK(cudaMemcpyAsync(out.data_ptr(), in.data_ptr(), slice, cudaMemcpyDeviceToDevice, s));
      return;
    }
    double scale = 1.0;
    ReduceOp rop = op;
    if (op == ReduceOp::AVG) { scale = 1.0 / size_; rop = ReduceOp::SUM; }
    // a chunk = the same piece of every rank's slice, parked slice-major with 16-byte padded pieces
    const size_t half = heap_->staging_half_bytes(kChanComm);
    const size_t piece_max = (half / size_) / 16 * 16;
    const char* src = static_cast<const char*>(in.data_ptr());
    char* dst = static_cast<char*>(out.data_ptr());
    for (size_t done = 0; done < slice; done += piece_max) {
      const size_t n = std::min(piece_max, slice - done), n_pad = (n + 15) / 16 * 16;
      const size_t stage = heap_->staging_off(kChanComm, heap_->next_parity(kChanComm));
      char* stg = heap_->local_base() + stage;
      for (int r = 0; r < size_; ++r) {
        if (n_pad != n) PDT_CUDA_CHECK(cudaMemsetAsync(stg + r * n_pad + n, 0, n_pad - n, s));
        PDT_CUDA_CHECK(cudaMemcpyAsync(stg + r * n_pad, src + r * slice + done, n, cudaMemcpyDeviceToDevice, s));
      }
      if (n_pad == n) {
        launch_reduce_pull(heap_->dev(kChanComm), stage, static_cast<size_t>(rank_) * (n_pad / 16), n_pad / 16, size_ * (n_pad / 16), dst + done,
                           to_symm_dtype(out.scalar_type()), static_cast<int>(rop), scale, cfg_, s);
      } else {  // ragged tail: reduce into the (now free) own piece of the staging copy, then copy the exact bytes out
        char* tmp = stg + static_cast<size_t>(rank_) * n_pad;
        launch_reduce_pull(heap_->dev(kChanComm), stage, static_cast<size_t>(rank_) * (n_pad / 16), n_pad / 16, size_ * (n_pad / 16), tmp,
                           to_symm_dtype(out.scalar_type()), static_cast<int>(rop), scale, cfg_, s);
        PDT_CUDA_CHECK(cudaMemcpyAsync(dst + done, tmp, n, cudaMemcpyDeviceToDevice, s));
      }
    }
  });
}

std::shared_ptr<CommWork> SymmComm::gather(at::Tensor out, at::Tensor in, int root) {
  check(in, "gather input");
  TORCH_CHECK(root >= 0 && root < size_, "gather: invalid root");
  if (rank_ == root) {
    check(out, "gather output");
    TORCH_CHECK(out.numel() == in.numel() * size_ && out.scalar_type() == in.scalar_type(), "gather: output must hold world_size × input elements");
  }
  record("gather", &in);
  return enqueue({out, in}, [&](cudaStream_t s) {
    const size_t nbytes = in.nbytes();
    if (nbytes == 0) return;
    if (size_ == 1) {
      PDT_CUDA_CHECK(cudaMemcpyAsync(out.data_ptr(), in.data_ptr(), nbytes, cudaMemcpyDeviceToDevice, s));
      return;
    }
    const size_t half = heap_->staging_half_bytes(kChanComm);
    const char* src = static_cast<const char*>(in.data_ptr());
    char* dst = rank_ == root ? static_cast<char*>(out.data_ptr()) : nullptr;
    for (size_t done = 0; done < nbytes; done += half) {
      const size_t n = std::min(half, nbytes - done);
      const size_t stage = heap_->staging_off(kChanComm, heap_->next_parity(kChanComm));
      PDT_CUDA_CHECK(cudaMemcpyAsync(heap_->local_base() + stage, src + done, n, cudaMemcpyDeviceToDevice, s));
      // only the root pulls; everybody else just attends the barrier (dst == nullptr)
      launch_allgather_pull(heap_->dev(kChanComm), stage, dst ? dst + done : nullptr, n, nbytes, /*exit_barrier=*/false, cfg_, s);
    }
  });
}

std::shared_ptr<CommWork> SymmComm::scatter(at::Tensor out, at::Tensor in, int root) {
  check(out, "scatter output");
  TORCH_CHECK(root >= 0 && root < size_, "scatter: invalid root");
  if (rank_ == root) {
    check(in, "scatter input");
    TORCH_CHECK(in.numel() == out.numel() * size_ && in.scalar_type() == out.scalar_type(), "scatter: input must hold world_size × output elements");
  }
  record("scatter", &out);
  return enqueue({out, in}, [&](cudaStream_t s) {
    const size_t blk = out.nbytes();
    if (blk == 0) return;
    if (size_ == 1) {
      PDT_CUDA_CHECK(cudaMemcpyAsync(out.data_ptr(), in.data_ptr(), blk, cudaMemcpyDeviceToDevice, s));
      return;
    }
    const size_t half = heap_->staging_half_bytes(kChanComm);
    const size_t piece_max = (half / size_) / 16 * 16;
    char* dst = static_cast<char*>(out.data_ptr());
    for (size_t done = 0; done < blk; done += piece_max) {
      const size_t n = std::min(piece_max, blk - done), n_pad = (n + 15) / 16 * 16;
      const size_t stage = heap_->staging_off(kChanComm, heap_->next_parity(kChanComm));
      if (rank_ == root) {
        const char* src = static_cast<const char*>(in.data_ptr());
        for (int r = 0; r < size_; ++r)
          PDT_CUDA_CHECK(cudaMemcpyAsync(heap_->local_base() + stage + r * n_pad, src + r * blk + done, n, cudaMemcpyDeviceToDevice, s));
      }
      // every rank pulls its own piece out of the root's staging area
      launch_broadcast_pull(heap_->dev(kChanComm), stage + static_cast<size_t>(rank_) * n_pad, dst + done, n, root, /*exit_barrier=*/false, cfg_, s);
    }
  });
}

std::shared_ptr<CommWork> SymmComm::barrier() {
  record("barrier", nullptr);
  return enqueue({}, [&](cudaStream_t s) {
    if (size_ > 1) launch_barrier(heap_->dev(kChanComm), s);
  });
}

}  // namespace pdt
