// Host-side device bookkeeping of the C-ABI entry points: every entry runs on the device that owns
// its first device pointer (not on whatever device happens to be current), and every per-process
// cache (SM count, granted dynamic shared memory, scratch) is kept per device.
#pragma once
#include <cuda_runtime.h>

#include "../../include/sbi_b200.h"

namespace sbi {

constexpr int kMaxDev = 32;

inline int cur_dev() {
  int d = 0;
  if (cudaGetDevice(&d) != cudaSuccess) { cudaGetLastError(); d = 0; }
  return (d >= 0 && d < kMaxDev) ? d : 0;
}

// Makes the device owning `p` current for the lifetime of the guard (no-op for null / host / already
// current).  cudaPointerGetAttributes and cudaSetDevice are legal during stream capture.
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(const void* p) {
    if (p == nullptr) return;
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return; }
    if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) return;
    int cur = 0;
    if (cudaGetDevice(&cur) != cudaSuccess) { cudaGetLastError(); return; }
    if (a.device != cur && cudaSetDevice(a.device) == cudaSuccess) prev = cur;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

inline int dev_num_sms() {
  static int n[kMaxDev] = {0};
  const int d = cur_dev();
  if (n[d] == 0) {
    cudaDeviceProp p;
    n[d] = (cudaGetDeviceProperties(&p, d) == cudaSuccess) ? p.multiProcessorCount : 132;
  }
  return n[d];
}

// Raise the dynamic shared-memory limit of a kernel once per (kernel, size): steady-state
// launches -- and launches recorded during CUDA-graph capture -- make no attribute calls.  Kernels of
// the same signature share a type, so each kernel of a translation unit takes its own ID.
template <int ID, class K>
static int set_smem(K kernel, int bytes) {
  static int granted_[kMaxDev] = {0};
  int& granted = granted_[cur_dev()];
  if (bytes > 227 * 1024) return SBI_ESMEM;
  if (bytes <= granted) return 0;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return (int)e;
  granted = bytes;
  return 0;
}

}  // namespace sbi
