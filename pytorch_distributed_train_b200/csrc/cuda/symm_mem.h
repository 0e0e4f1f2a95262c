// Symmetric memory heap across the per-GPU processes of one node.
//
// This is the substrate of the NVLink-native backend: every rank owns one
// physically contiguous heap (cuMemCreate), exports it as a POSIX fd, ships the fd to its peers
// over an AF_UNIX socket (SCM_RIGHTS; names published through the Store) and maps every peer's
// heap into its own address space, so a kernel can load/store any rank's memory directly over
// NVLink 5 / NVSwitch.  When the driver supports it the heaps are additionally bound to one
// multicast object so `multimem.ld_reduce` / `multimem.st` reach all replicas through the
// switch (NVLS).  If fd export is not permitted (containers), the legacy cudaIpc path provides
// plain P2P without multicast.
//
// Heap layout (identical on every rank, so "same offset" == "same tensor"):
//   [ signal pads | staging (per channel, double-buffered) | user area (first-fit allocator) ]
#pragma once
#include <cstddef>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "../store/store.h"
#include "symm_device.h"

namespace pdt {

class SymmetricHeap {
 public:
  // Collective over (store, rank, world): every rank must construct with the same sizes.
  SymmetricHeap(std::shared_ptr<Store> store, int rank, int world, int device, size_t heap_bytes, Millis timeout);
  ~SymmetricHeap();
  SymmetricHeap(const SymmetricHeap&) = delete;

  int rank() const { return rank_; }
  int world() const { return world_; }
  int device() const { return device_; }
  bool has_multicast() const { return mc_base_ != nullptr; }
  const char* transport() const { return vmm_ ? "vmm" : "cudaIpc"; }
  size_t heap_bytes() const { return heap_bytes_; }
  char* base(int r) const { return peer_base_[r]; }
  char* local_base() const { return peer_base_[rank_]; }
  char* mc_base() const { return mc_base_; }

  // Device-visible descriptor for a channel (passed by value to kernels).
  SymmDev dev(int channel) const;
  // Staging area of a channel: two halves of staging_half_bytes(channel) each.
  size_t staging_off(int channel, int half) const;
  size_t staging_half_bytes(int channel) const;
  // Host-side parity flip, one per collective issued on the channel (all ranks issue the same
  // sequence, so parities agree).
  int next_parity(int channel) { return parity_[channel]++ & 1; }
  int peek_parity(int channel) const { return parity_[channel] & 1; }

  // User area.  Offsets are identical across ranks because every rank performs the same sequence of alloc calls and
  // frees are applied only at collective points: free() parks the block; SymmComm::alloc_flat exchanges the parked
  // sets and releases exactly the blocks every rank has dropped (pending_frees / apply_frees).
  void* alloc(size_t nbytes, size_t align = 256);
  void free(void* p);
  std::vector<size_t> pending_frees() const;
  void apply_frees(const std::vector<size_t>& offsets);
  bool contains(const void* p, size_t nbytes) const;
  size_t offset_of(const void* p) const { return static_cast<const char*>(p) - peer_base_[rank_]; }
  size_t user_bytes_in_use() const;

  // Host-mapped status word the kernels write on timeout: 0 = ok.
  int status() const { return *status_host_; }
  void clear_status() { *status_host_ = 0; }
  void set_timeout_ns(unsigned long long ns) { timeout_ns_ = ns; }

 private:
  void setup_vmm(std::shared_ptr<Store> store, Millis timeout);
  void setup_ipc(std::shared_ptr<Store> store, Millis timeout);
  void setup_multicast(std::shared_ptr<Store> store, Millis timeout);
  void exchange_fds(std::shared_ptr<Store> store, const std::string& tag, int my_fd, std::vector<int>* peer_fds, Millis timeout);

  int rank_, world_, device_;
  size_t heap_bytes_ = 0;
  bool vmm_ = false;
  std::vector<char*> peer_base_;
  char* mc_base_ = nullptr;
  uint32_t* epochs_ = nullptr;       // device, local: [kSymmChannels][kSymmMaxBlocks]
  int* status_host_ = nullptr;       // pinned + mapped
  int* status_dev_ = nullptr;
  unsigned long long timeout_ns_ = 20ull * 1000 * 1000 * 1000;
  int parity_[kSymmChannels] = {0};

  // layout
  size_t signal_bytes_ = 0;
  size_t staging_off_[kSymmChannels] = {0};
  size_t staging_half_[kSymmChannels] = {0};
  size_t user_off_ = 0;

  // allocator
  mutable std::mutex mu_;
  std::map<size_t, size_t> free_;    // offset -> size
  std::map<size_t, size_t> used_;    // offset -> size
  std::set<size_t> pending_;         // parked frees (offsets), released at the next collective alloc
  void release_locked(size_t off);

  // driver handles (VMM path)
  std::vector<unsigned long long> handles_;
  unsigned long long mc_handle_ = 0;
  size_t mc_size_ = 0;
};

}  // namespace pdt
