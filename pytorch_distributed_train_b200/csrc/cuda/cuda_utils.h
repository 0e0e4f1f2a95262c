// CUDA runtime/driver helpers shared by the host-side glue (no torch headers here).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstddef>
#include <stdexcept>
#include <string>
#include <utility>

namespace pdt {

#define PDT_CUDA_CHECK(expr)                                                                        \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      throw std::runtime_error(std::string("CUDA error at ") + __FILE__ + ":" + std::to_string(__LINE__) + \
                               " (" #expr "): " + cudaGetErrorString(_e));                          \
  } while (0)

// Driver entry points are resolved through the runtime (cudaGetDriverEntryPoint) so that the
// library links without libcuda.so and imports on GPU-less build boxes.
struct DriverApi {
  CUresult (*cuGetErrorString)(CUresult, const char**) = nullptr;
  CUresult (*cuDeviceGetAttribute)(int*, CUdevice_attribute, CUdevice) = nullptr;
  CUresult (*cuMemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags) = nullptr;
  CUresult (*cuMemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long) = nullptr;
  CUresult (*cuMemRelease)(CUmemGenericAllocationHandle) = nullptr;
  CUresult (*cuMemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long) = nullptr;
  CUresult (*cuMemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType) = nullptr;
  CUresult (*cuMemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long) = nullptr;
  CUresult (*cuMemAddressFree)(CUdeviceptr, size_t) = nullptr;
  CUresult (*cuMemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long) = nullptr;
  CUresult (*cuMemUnmap)(CUdeviceptr, size_t) = nullptr;
  CUresult (*cuMemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t) = nullptr;
  CUresult (*cuMulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*) = nullptr;
  CUresult (*cuMulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice) = nullptr;
  CUresult (*cuMulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long) = nullptr;
  CUresult (*cuMulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags) = nullptr;
  CUresult (*cuMulticastUnbind)(CUmemGenericAllocationHandle, CUdevice, size_t, size_t) = nullptr;
  CUresult (*cuTensorMapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                     const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill) = nullptr;
  CUresult (*cuTensorMapEncodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill) = nullptr;
  CUresult (*cuCtxGetDevice)(CUdevice*) = nullptr;
  bool multicast_api = false;
};

const DriverApi& driver();  // throws if the driver cannot be reached (no GPU)
std::string cu_error(CUresult r);

#define PDT_CU_CHECK(expr)                                                                           \
  do {                                                                                               \
    CUresult _r = (expr);                                                                            \
    if (_r != CUDA_SUCCESS)                                                                          \
      throw std::runtime_error(std::string("CUDA driver error at ") + __FILE__ + ":" + std::to_string(__LINE__) + \
                               " (" #expr "): " + ::pdt::cu_error(_r));                              \
  } while (0)

// Every launcher of this library reports here, so benchmarks can state how many of *our* kernels
// ran in a timed region (during CUDA-graph capture: how many were recorded into the graph).
void count_kernel_launch(int n = 1);
long long kernel_launch_count();
// Set from a Python atexit hook: destructors that would call into a dying CUDA driver skip their work.
void mark_process_exiting();
bool process_exiting();

// Call right after a <<<...>>> launch: throws if the launch failed, counts it otherwise.
void check_launch(const char* what);

// Multiprocessor count of the current device (queried once per device).
int sm_count();
// Dynamic shared memory one block of the current device may opt in to (queried once per device): the bound of opt_in_smem.
size_t smem_optin_limit();

// Kernels that use more than the default 48 KB of dynamic shared memory must opt in first.
template <typename K>
void opt_in_smem(K kernel, size_t bytes) {
  if (bytes > 48 * 1024) PDT_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
}

// Cooperative launch: all CTAs are co-resident, so they may wait for each other at a grid barrier (grid_sync.cuh).
// programmatic: a programmatic dependent launch — the grid may start before the kernel ahead of it in the stream has finished, once
// that kernel calls griddep_launch_dependents(); the kernel must call griddep_wait() before it reads anything that kernel wrote
// (hopper_ptx.cuh), and before it touches a grid-barrier word.
template <typename... KArgs, typename... Args>
void launch_cooperative(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, const char* what, bool programmatic,
                        Args&&... args) {
  opt_in_smem(kernel, smem);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = programmatic ? 2 : 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
  if (e != cudaSuccess) throw std::runtime_error(std::string("launch of ") + what + " failed: " + cudaGetErrorString(e));
  count_kernel_launch();
}

}  // namespace pdt
