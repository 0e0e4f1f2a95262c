#include "cuda_utils.h"

#include <atomic>
#include <mutex>

namespace pdt {

namespace {
template <typename F>
bool load(const char* name, F* out, bool required) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint(name, &fn, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || fn == nullptr) {
    (void)cudaGetLastError();
    if (required) throw std::runtime_error(std::string("CUDA driver entry point unavailable: ") + name);
    return false;
  }
  *out = reinterpret_cast<F>(fn);
  return true;
}
}  // namespace

const DriverApi& driver() {
  static DriverApi api;
  static std::once_flag once;
  static std::string err;
  std::call_once(once, [] {
    try {
      int n = 0;
      if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        (void)cudaGetLastError();
        throw std::runtime_error("no CUDA device / driver available");
      }
      load("cuGetErrorString", &api.cuGetErrorString, true);
      load("cuDeviceGetAttribute", &api.cuDeviceGetAttribute, true);
      load("cuMemGetAllocationGranularity", &api.cuMemGetAllocationGranularity, true);
      load("cuMemCreate", &api.cuMemCreate, true);
      load("cuMemRelease", &api.cuMemRelease, true);
      load("cuMemExportToShareableHandle", &api.cuMemExportToShareableHandle, true);
      load("cuMemImportFromShareableHandle", &api.cuMemImportFromShareableHandle, true);
      load("cuMemAddressReserve", &api.cuMemAddressReserve, true);
      load("cuMemAddressFree", &api.cuMemAddressFree, true);
      load("cuMemMap", &api.cuMemMap, true);
      load("cuMemUnmap", &api.cuMemUnmap, true);
      load("cuMemSetAccess", &api.cuMemSetAccess, true);
      load("cuCtxGetDevice", &api.cuCtxGetDevice, true);
      load("cuTensorMapEncodeTiled", &api.cuTensorMapEncodeTiled, true);
      load("cuTensorMapEncodeIm2col", &api.cuTensorMapEncodeIm2col, false);
      api.multicast_api = load("cuMulticastCreate", &api.cuMulticastCreate, false) &&
                          load("cuMulticastAddDevice", &api.cuMulticastAddDevice, false) &&
                          load("cuMulticastBindMem", &api.cuMulticastBindMem, false) &&
                          load("cuMulticastGetGranularity", &api.cuMulticastGetGranularity, false) &&
                          load("cuMulticastUnbind", &api.cuMulticastUnbind, false);
    } catch (const std::exception& e) {
      err = e.what();
    }
  });
  if (!err.empty()) throw std::runtime_error("CUDA driver API not usable: " + err);
  return api;
}

static std::atomic<long long> g_launches{0};
static std::atomic<bool> g_exiting{false};
void mark_process_exiting() { g_exiting.store(true); }
bool process_exiting() { return g_exiting.load(); }
void count_kernel_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long kernel_launch_count() { return g_launches.load(std::memory_order_relaxed); }

void check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) throw std::runtime_error(std::string("launch of ") + what + " failed: " + cudaGetErrorString(e));
  count_kernel_launch();
}

constexpr int kMaxDevices = 64;

// attribute `attr` of the current device, queried once per device into cached[device] (0 = not queried yet)
static int cached_attribute(cudaDeviceAttr attr, std::atomic<int>* cached) {
  int dev = 0;
  PDT_CUDA_CHECK(cudaGetDevice(&dev));
  int n = dev < kMaxDevices ? cached[dev].load(std::memory_order_relaxed) : 0;
  if (n == 0) {
    PDT_CUDA_CHECK(cudaDeviceGetAttribute(&n, attr, dev));
    if (dev < kMaxDevices) cached[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

int sm_count() {
  static std::atomic<int> cached[kMaxDevices];
  return cached_attribute(cudaDevAttrMultiProcessorCount, cached);
}

size_t smem_optin_limit() {
  static std::atomic<int> cached[kMaxDevices];
  return static_cast<size_t>(cached_attribute(cudaDevAttrMaxSharedMemoryPerBlockOptin, cached));
}

std::string cu_error(CUresult r) {
  const char* s = nullptr;
  try {
    if (driver().cuGetErrorString(r, &s) == CUDA_SUCCESS && s) return std::string(s) + " (" + std::to_string(static_cast<int>(r)) + ")";
  } catch (...) {
  }
  return "CUresult " + std::to_string(static_cast<int>(r));
}

}  // namespace pdt
