#include "cpu_backend.h"

#include <unistd.h>

#include <algorithm>
#include <cmath>
#include <cstring>

namespace pdt {

// ---------------------------------------------------------------------------------------
// dtype helpers
size_t dtype_size(DType t) {
  switch (t) {
    case DType::F32: case DType::I32: return 4;
    case DType::F64: case DType::I64: return 8;
    case DType::F16: case DType::BF16: case DType::I16: return 2;
    default: return 1;
  }
}

namespace {

inline float bf16_to_f32(uint16_t h) {
  uint32_t u = static_cast<uint32_t>(h) << 16;
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f32_to_bf16(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x40);  // NaN
  uint32_t lsb = (u >> 16) & 1u;
  u += 0x7fffu + lsb;  // round to nearest even
  return static_cast<uint16_t>(u >> 16);
}
inline float f16_to_f32(uint16_t h) {
  uint32_t sign = (h & 0x8000u) << 16;
  uint32_t exp = (h >> 10) & 0x1f;
  uint32_t man = h & 0x3ffu;
  uint32_t u;
  if (exp == 0) {
    if (man == 0) u = sign;
    else {
      int e = -1;
      do { ++e; man <<= 1; } while (!(man & 0x400u));
      man &= 0x3ffu;
      u = sign | ((127 - 15 - e) << 23) | (man << 13);
    }
  } else if (exp == 31) u = sign | 0x7f800000u | (man << 13);
  else u = sign | ((exp + 112) << 23) | (man << 13);
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}
inline uint16_t f32_to_f16(float f) {
  uint32_t x;
  std::memcpy(&x, &f, 4);
  uint32_t sign = (x >> 16) & 0x8000u;
  int32_t exp = static_cast<int32_t>((x >> 23) & 0xff) - 127 + 15;
  uint32_t man = x & 0x7fffffu;
  if (((x >> 23) & 0xff) == 0xff) return static_cast<uint16_t>(sign | 0x7c00u | (man ? 0x200u : 0));
  if (exp >= 31) return static_cast<uint16_t>(sign | 0x7c00u);
  if (exp <= 0) {
    if (exp < -10) return static_cast<uint16_t>(sign);
    man |= 0x800000u;
    uint32_t shift = static_cast<uint32_t>(14 - exp);
    uint32_t half = man >> shift;
    uint32_t rem = man & ((1u << shift) - 1);
    uint32_t mid = 1u << (shift - 1);
    if (rem > mid || (rem == mid && (half & 1))) ++half;
    return static_cast<uint16_t>(sign | half);
  }
  uint32_t half = (static_cast<uint32_t>(exp) << 10) | (man >> 13);
  uint32_t rem = man & 0x1fffu;
  if (rem > 0x1000u || (rem == 0x1000u && (half & 1))) ++half;
  return static_cast<uint16_t>(sign | half);
}

template <typename T>
void reduce_t(T* d, const T* s, size_t n, ReduceOp op) {
  switch (op) {
    case ReduceOp::SUM: case ReduceOp::AVG: for (size_t i = 0; i < n; ++i) d[i] = d[i] + s[i]; break;
    case ReduceOp::PRODUCT: for (size_t i = 0; i < n; ++i) d[i] = d[i] * s[i]; break;
    case ReduceOp::MIN: for (size_t i = 0; i < n; ++i) d[i] = std::min(d[i], s[i]); break;
    case ReduceOp::MAX: for (size_t i = 0; i < n; ++i) d[i] = std::max(d[i], s[i]); break;
    default: throw std::invalid_argument("bitwise reduce op on a non-integer dtype");
  }
}
template <typename T>
void reduce_int(T* d, const T* s, size_t n, ReduceOp op) {
  switch (op) {
    case ReduceOp::BAND: for (size_t i = 0; i < n; ++i) d[i] = d[i] & s[i]; break;
    case ReduceOp::BOR: for (size_t i = 0; i < n; ++i) d[i] = d[i] | s[i]; break;
    case ReduceOp::BXOR: for (size_t i = 0; i < n; ++i) d[i] = d[i] ^ s[i]; break;
    default: reduce_t(d, s, n, op);
  }
}
template <float (*Load)(uint16_t), uint16_t (*Store)(float)>
void reduce_half(uint16_t* d, const uint16_t* s, size_t n, ReduceOp op) {
  for (size_t i = 0; i < n; ++i) {
    float a = Load(d[i]), b = Load(s[i]), r;
    switch (op) {
      case ReduceOp::SUM: case ReduceOp::AVG: r = a + b; break;
      case ReduceOp::PRODUCT: r = a * b; break;
      case ReduceOp::MIN: r = std::min(a, b); break;
      case ReduceOp::MAX: r = std::max(a, b); break;
      default: throw std::invalid_argument("bitwise reduce op on a floating dtype");
    }
    d[i] = Store(r);
  }
}

}  // namespace

void reduce_inplace(void* dst, const void* src, size_t n, DType t, ReduceOp op) {
  switch (t) {
    case DType::F32: reduce_t(static_cast<float*>(dst), static_cast<const float*>(src), n, op); break;
    case DType::F64: reduce_t(static_cast<double*>(dst), static_cast<const double*>(src), n, op); break;
    case DType::F16: reduce_half<f16_to_f32, f32_to_f16>(static_cast<uint16_t*>(dst), static_cast<const uint16_t*>(src), n, op); break;
    case DType::BF16: reduce_half<bf16_to_f32, f32_to_bf16>(static_cast<uint16_t*>(dst), static_cast<const uint16_t*>(src), n, op); break;
    case DType::I8: reduce_int(static_cast<int8_t*>(dst), static_cast<const int8_t*>(src), n, op); break;
    case DType::U8: case DType::BOOL: reduce_int(static_cast<uint8_t*>(dst), static_cast<const uint8_t*>(src), n, op); break;
    case DType::I16: reduce_int(static_cast<int16_t*>(dst), static_cast<const int16_t*>(src), n, op); break;
    case DType::I32: reduce_int(static_cast<int32_t*>(dst), static_cast<const int32_t*>(src), n, op); break;
    case DType::I64: reduce_int(static_cast<int64_t*>(dst), static_cast<const int64_t*>(src), n, op); break;
  }
}

void scale_inplace(void* dst, size_t n, DType t, double f) {
  switch (t) {
    case DType::F32: { auto* p = static_cast<float*>(dst); float ff = static_cast<float>(f); for (size_t i = 0; i < n; ++i) p[i] *= ff; break; }
    case DType::F64: { auto* p = static_cast<double*>(dst); for (size_t i = 0; i < n; ++i) p[i] *= f; break; }
    case DType::F16: { auto* p = static_cast<uint16_t*>(dst); for (size_t i = 0; i < n; ++i) p[i] = f32_to_f16(f16_to_f32(p[i]) * static_cast<float>(f)); break; }
    case DType::BF16: { auto* p = static_cast<uint16_t*>(dst); for (size_t i = 0; i < n; ++i) p[i] = f32_to_bf16(bf16_to_f32(p[i]) * static_cast<float>(f)); break; }
    case DType::I32: { auto* p = static_cast<int32_t*>(dst); for (size_t i = 0; i < n; ++i) p[i] = static_cast<int32_t>(p[i] * f); break; }
    case DType::I64: { auto* p = static_cast<int64_t*>(dst); for (size_t i = 0; i < n; ++i) p[i] = static_cast<int64_t>(p[i] * f); break; }
    default: throw std::invalid_argument("AVG is not defined for this dtype");
  }
}

// ---------------------------------------------------------------------------------------
// Work
void Work::wait(Millis timeout) {
  std::unique_lock<std::mutex> g(mu_);
  if (!cv_.wait_for(g, timeout, [&] { return done_; }))
    throw TimeoutError("collective did not complete within " + std::to_string(timeout.count()) +
                       " ms (a peer rank is likely dead or diverged)");
  if (err_) std::rethrow_exception(err_);
}
bool Work::is_completed() { std::lock_guard<std::mutex> g(mu_); return done_; }
bool Work::is_success() { std::lock_guard<std::mutex> g(mu_); return done_ && !err_; }
std::string Work::error() {
  std::lock_guard<std::mutex> g(mu_);
  if (!err_) return "";
  try { std::rethrow_exception(err_); } catch (const std::exception& e) { return e.what(); } catch (...) { return "unknown"; }
}
void Work::finish(std::exception_ptr e) {
  { std::lock_guard<std::mutex> g(mu_); done_ = true; err_ = e; }
  cv_.notify_all();
}

// ---------------------------------------------------------------------------------------
// CpuBackend
CpuBackend::CpuBackend(std::shared_ptr<Store> store, int rank, int size, Millis timeout, const std::string& bind_host)
    : store_(std::move(store)), rank_(rank), size_(size), timeout_(timeout) {
  socks_.resize(size_);
  if (size_ > 1) {
    int port = 0;
    Fd lfd = tcp_listen(bind_host, 0, &port);
    std::string host = bind_host.empty() ? "127.0.0.1" : bind_host;
    store_->set("cpu/addr/" + std::to_string(rank_), host + ":" + std::to_string(port));
    // higher rank dials lower rank; the dialer announces its rank in a 4-byte hello
    for (int r = 0; r < rank_; ++r) {
      std::string addr = store_->get("cpu/addr/" + std::to_string(r));
      auto colon = addr.rfind(':');
      Fd s = tcp_connect(addr.substr(0, colon), std::stoi(addr.substr(colon + 1)), timeout_);
      int32_t me = rank_;
      send_all(s.get(), &me, 4, timeout_);
      socks_[r] = std::move(s);
    }
    for (int k = rank_ + 1; k < size_; ++k) {
      Fd s = tcp_accept(lfd.get(), timeout_);
      int32_t who = -1;
      recv_all(s.get(), &who, 4, timeout_);
      if (who <= rank_ || who >= size_ || socks_[who].valid())
        throw std::runtime_error("cpu backend: unexpected hello from rank " + std::to_string(who));
      socks_[who] = std::move(s);
    }
    for (int r = 0; r < size_; ++r)
      if (r != rank_) set_nonblocking(socks_[r].get(), true);
  }
  worker_ = std::thread([this] { worker_loop(); });
}

CpuBackend::~CpuBackend() { shutdown(); }

void CpuBackend::shutdown() {
  {
    std::lock_guard<std::mutex> g(mu_);
    if (stop_) return;
    stop_ = true;
  }
  cv_.notify_all();
  if (worker_.joinable()) worker_.join();
  for (auto& s : socks_) s.reset();
}

void CpuBackend::worker_loop() {
  while (true) {
    std::pair<std::function<void()>, std::shared_ptr<Work>> item;
    {
      std::unique_lock<std::mutex> g(mu_);
      cv_.wait(g, [&] { return stop_ || !queue_.empty(); });
      if (queue_.empty()) return;  // stop requested and drained
      item = std::move(queue_.front());
      queue_.pop_front();
    }
    std::exception_ptr err;
    try {
      if (delay_ops_.load() > 0) {
        --delay_ops_;
        ::usleep(static_cast<useconds_t>(delay_ms_.load()) * 1000);
      }
      if (skip_ops_.load() > 0) --skip_ops_;
      else item.first();
    } catch (...) {
      err = std::current_exception();
    }
    ++seq_done_;
    item.second->finish(err);
  }
}

std::shared_ptr<Work> CpuBackend::submit(std::function<void()> fn) {
  auto w = std::make_shared<Work>();
  {
    std::lock_guard<std::mutex> g(mu_);
    if (stop_) throw std::runtime_error("process group has been shut down");
    queue_.emplace_back(std::move(fn), w);
  }
  cv_.notify_one();
  return w;
}

// ---- blocking bodies -------------------------------------------------------------------
void CpuBackend::do_broadcast(void* buf, size_t nbytes, int root) {
  if (size_ == 1 || nbytes == 0) return;
  // binomial tree rooted at `root` (log2(N) rounds)
  int vrank = (rank_ - root + size_) % size_;
  int mask = 1;
  while (mask < size_) {
    if (vrank & mask) {
      int src = (vrank - mask + root) % size_;
      recv_all(peer(src), buf, nbytes, timeout_);
      break;
    }
    mask <<= 1;
  }
  mask >>= 1;
  while (mask > 0) {
    if (vrank + mask < size_ && !(vrank & (mask - 1)) && !(vrank & mask)) {
      int dst = (vrank + mask + root) % size_;
      send_all(peer(dst), buf, nbytes, timeout_);
    }
    mask >>= 1;
  }
}

void CpuBackend::do_allgather(const void* in, void* out, size_t nb) {
  char* o = static_cast<char*>(out);
  if (in != o + static_cast<size_t>(rank_) * nb) std::memcpy(o + static_cast<size_t>(rank_) * nb, in, nb);
  if (size_ == 1 || nb == 0) return;
  // ring: in step s forward the block received in step s-1
  int right = (rank_ + 1) % size_, left = (rank_ - 1 + size_) % size_;
  for (int s = 0; s < size_ - 1; ++s) {
    int send_blk = (rank_ - s + size_) % size_;
    int recv_blk = (rank_ - s - 1 + size_) % size_;
    send_recv(peer(right), o + static_cast<size_t>(send_blk) * nb, nb, peer(left), o + static_cast<size_t>(recv_blk) * nb, nb, timeout_);
  }
}

void CpuBackend::do_allreduce(void* buf, size_t count, DType t, ReduceOp op) {
  size_t es = dtype_size(t);
  size_t nbytes = count * es;
  if (size_ > 1 && count > 0) {
    if (nbytes <= 64 * 1024 || count < static_cast<size_t>(size_) * 8) {
      // Latency path: everybody gets everybody's vector, reduces locally in rank order
      // → bitwise identical on every rank.
      scratch_.resize(nbytes * static_cast<size_t>(size_));
      do_allgather(buf, scratch_.data(), nbytes);
      std::memcpy(buf, scratch_.data(), nbytes);
      for (int r = 1; r < size_; ++r) reduce_inplace(buf, scratch_.data() + static_cast<size_t>(r) * nbytes, count, t, op);
    } else {
      // Bandwidth path: ring reduce-scatter then ring all-gather over N nearly equal chunks.
      std::vector<size_t> off(size_ + 1);
      for (int i = 0; i <= size_; ++i) off[i] = count * static_cast<size_t>(i) / static_cast<size_t>(size_);
      size_t max_chunk = 0;
      for (int i = 0; i < size_; ++i) max_chunk = std::max(max_chunk, off[i + 1] - off[i]);
      scratch_.resize(max_chunk * es);
      char* b = static_cast<char*>(buf);
      int right = (rank_ + 1) % size_, left = (rank_ - 1 + size_) % size_;
      for (int s = 0; s < size_ - 1; ++s) {
        int sc = (rank_ - s + size_) % size_;
        int rc = (rank_ - s - 1 + size_) % size_;
        size_t sn = off[sc + 1] - off[sc], rn = off[rc + 1] - off[rc];
        send_recv(peer(right), b + off[sc] * es, sn * es, peer(left), scratch_.data(), rn * es, timeout_);
        reduce_inplace(b + off[rc] * es, scratch_.data(), rn, t, op);
      }
      // rank r now owns fully reduced chunk (r+1)%N
      for (int s = 0; s < size_ - 1; ++s) {
        int sc = (rank_ + 1 - s + size_) % size_;
        int rc = (rank_ - s + size_) % size_;
        size_t sn = off[sc + 1] - off[sc], rn = off[rc + 1] - off[rc];
        send_recv(peer(right), b + off[sc] * es, sn * es, peer(left), b + off[rc] * es, rn * es, timeout_);
      }
    }
  }
  if (op == ReduceOp::AVG) scale_inplace(buf, count, t, 1.0 / static_cast<double>(size_));
}

void CpuBackend::do_reduce(void* buf, size_t count, DType t, ReduceOp op, int root) {
  size_t nbytes = count * dtype_size(t);
  if (size_ > 1 && count > 0) {
    if (rank_ == root) {
      scratch_.resize(nbytes);
      std::vector<char> acc(nbytes);
      // rank order 0..N-1 regardless of root, for determinism
      bool first = true;
      for (int r = 0; r < size_; ++r) {
        const char* src;
        if (r == rank_) src = static_cast<const char*>(buf);
        else { recv_all(peer(r), scratch_.data(), nbytes, timeout_); src = scratch_.data(); }
        if (first) { std::memcpy(acc.data(), src, nbytes); first = false; }
        else reduce_inplace(acc.data(), src, count, t, op);
      }
      std::memcpy(buf, acc.data(), nbytes);
    } else {
      send_all(peer(root), buf, nbytes, timeout_);
    }
  }
  if (op == ReduceOp::AVG && rank_ == root) scale_inplace(buf, count, t, 1.0 / static_cast<double>(size_));
}

void CpuBackend::do_reduce_scatter(const void* in, void* out, size_t cpr, DType t, ReduceOp op) {
  size_t es = dtype_size(t);
  std::vector<char> tmp(static_cast<const char*>(in), static_cast<const char*>(in) + cpr * es * static_cast<size_t>(size_));
  do_allreduce(tmp.data(), cpr * static_cast<size_t>(size_), t, op);
  std::memcpy(out, tmp.data() + static_cast<size_t>(rank_) * cpr * es, cpr * es);
}

// ---- async wrappers --------------------------------------------------------------------
// On bool, SUM is logical OR and PRODUCT logical AND (torch's NCCL backend maps them to MAX / MIN, and so do the GPU backends);
// on 0/1 bytes MIN and MAX are AND and OR as well.  AVG has no bool result.  Checked before any byte moves, on every rank alike.
static ReduceOp checked_op(DType t, ReduceOp op) {
  if (t != DType::BOOL) return op;
  switch (op) {
    case ReduceOp::SUM: case ReduceOp::MAX: case ReduceOp::BOR: return ReduceOp::BOR;
    case ReduceOp::PRODUCT: case ReduceOp::MIN: case ReduceOp::BAND: return ReduceOp::BAND;
    case ReduceOp::BXOR: return ReduceOp::BXOR;
    default: throw std::invalid_argument("AVG is not defined for bool tensors");
  }
}

std::shared_ptr<Work> CpuBackend::allreduce(void* buf, size_t count, DType t, ReduceOp op) {
  op = checked_op(t, op);
  return submit([=] { do_allreduce(buf, count, t, op); });
}
std::shared_ptr<Work> CpuBackend::broadcast(void* buf, size_t nbytes, int root) {
  if (root < 0 || root >= size_) throw std::invalid_argument("broadcast: invalid root rank");
  return submit([=] { do_broadcast(buf, nbytes, root); });
}
std::shared_ptr<Work> CpuBackend::allgather(const void* in, void* out, size_t nb) {
  return submit([=] { do_allgather(in, out, nb); });
}
std::shared_ptr<Work> CpuBackend::reduce(void* buf, size_t count, DType t, ReduceOp op, int root) {
  if (root < 0 || root >= size_) throw std::invalid_argument("reduce: invalid root rank");
  op = checked_op(t, op);
  return submit([=] { do_reduce(buf, count, t, op, root); });
}
std::shared_ptr<Work> CpuBackend::reduce_scatter(const void* in, void* out, size_t cpr, DType t, ReduceOp op) {
  op = checked_op(t, op);
  return submit([=] { do_reduce_scatter(in, out, cpr, t, op); });
}
std::shared_ptr<Work> CpuBackend::gather(const void* in, void* out, size_t nb, int root) {
  return submit([=] {
    if (rank_ == root) {
      char* o = static_cast<char*>(out);
      std::memcpy(o + static_cast<size_t>(rank_) * nb, in, nb);
      for (int r = 0; r < size_; ++r)
        if (r != rank_) recv_all(peer(r), o + static_cast<size_t>(r) * nb, nb, timeout_);
    } else {
      send_all(peer(root), in, nb, timeout_);
    }
  });
}
std::shared_ptr<Work> CpuBackend::scatter(const void* in, void* out, size_t nb, int root) {
  return submit([=] {
    if (rank_ == root) {
      const char* i = static_cast<const char*>(in);
      for (int r = 0; r < size_; ++r)
        if (r != rank_) send_all(peer(r), i + static_cast<size_t>(r) * nb, nb, timeout_);
      std::memcpy(out, i + static_cast<size_t>(rank_) * nb, nb);
    } else {
      recv_all(peer(root), out, nb, timeout_);
    }
  });
}
std::shared_ptr<Work> CpuBackend::alltoall(const void* in, void* out, size_t nb) {
  return submit([=] {
    const char* i = static_cast<const char*>(in);
    char* o = static_cast<char*>(out);
    std::memcpy(o + static_cast<size_t>(rank_) * nb, i + static_cast<size_t>(rank_) * nb, nb);
    for (int s = 1; s < size_; ++s) {
      int to = (rank_ + s) % size_, from = (rank_ - s + size_) % size_;
      send_recv(peer(to), i + static_cast<size_t>(to) * nb, nb, peer(from), o + static_cast<size_t>(from) * nb, nb, timeout_);
    }
  });
}
std::shared_ptr<Work> CpuBackend::send(const void* buf, size_t nbytes, int dst) {
  if (dst < 0 || dst >= size_ || dst == rank_) throw std::invalid_argument("send: invalid destination rank");
  return submit([=] { send_all(peer(dst), buf, nbytes, timeout_); });
}
std::shared_ptr<Work> CpuBackend::recv(void* buf, size_t nbytes, int src) {
  if (src < 0 || src >= size_ || src == rank_) throw std::invalid_argument("recv: invalid source rank");
  return submit([=] { recv_all(peer(src), buf, nbytes, timeout_); });
}
std::shared_ptr<Work> CpuBackend::barrier() {
  return submit([=] {
    int32_t token = 1;
    do_allreduce(&token, 1, DType::I32, ReduceOp::SUM);
  });
}

}  // namespace pdt
