// Host side of the C-ABI entry points: every entry runs on the device that owns its first device pointer (not on
// whatever device happens to be current), every per-process cache (SM count, granted dynamic shared memory)
// is kept per device, and every row-tile kernel is sized and launched through the helpers below.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <initializer_list>
#include <mutex>
#include <unordered_map>
#include <utility>

#include "../../include/sbi_b200.h"

namespace sbi {

constexpr int kMaxDev = 32;
constexpr int kMaxSmemBytes = 227 * 1024;   // dynamic shared memory one CTA may opt into on sm_90

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

// Raise the dynamic shared-memory limit of `kernel` on the current device when `bytes` exceeds what it was
// granted before: steady-state launches -- and launches recorded during CUDA-graph capture -- make no
// attribute call.
inline int set_smem(const void* kernel, int bytes) {
  static std::mutex mu;
  static std::unordered_map<const void*, int> granted_[kMaxDev];
  if (bytes > kMaxSmemBytes) return SBI_ESMEM;
  const int d = cur_dev();
  std::lock_guard<std::mutex> lock(mu);
  int& granted = granted_[d][kernel];
  if (bytes <= granted) return 0;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return (int)e;
  granted = bytes;
  return 0;
}

// Grid of a launch: `ctas` CTAs along x.  `early`: programmatic stream serialization -- the grid may start once
// every CTA of the kernel before it in the stream has run griddepcontrol.launch_dependents, so it must itself
// wait for whatever of that kernel's output it reads.
struct Grid {
  int ctas;
  bool early;
  Grid(int n, bool e = false) : ctas(n), early(e) {}
};

// Opt `kernel` into `smem_bytes` of dynamic shared memory, launch it and return the launch status.
template <class... P, class... A>
int launch(void (*kernel)(P...), Grid grid, int threads, int smem_bytes, cudaStream_t s, A&&... args) {
  if (int e = set_smem(reinterpret_cast<const void*>(kernel), smem_bytes)) return e;
  if (grid.early) {
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid.ctas);
    cfg.blockDim = dim3((unsigned)threads);
    cfg.dynamicSmemBytes = (size_t)smem_bytes;
    cfg.stream = s;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
  } else {
    kernel<<<grid.ctas, threads, smem_bytes, s>>>(std::forward<A>(args)...);
  }
  return (int)cudaGetLastError();
}

// Grid of a persistent kernel over TM-row tiles: `per_sm` CTAs per SM, never more CTAs than tiles.
inline int tile_grid(int64_t R, int TM, int per_sm) {
  return (int)std::min<int64_t>((R + TM - 1) / TM, (int64_t)dev_num_sms() * per_sm);
}

// CTAs per SM of the SIMT forward kernels: two when the layout takes at most 110 KB, else one.
inline int per_sm_110k(int bytes) { return bytes <= 110 * 1024 ? 2 : 1; }

// Partial-gradient slabs of a VJP over TM-row tiles: one per CTA, at most one CTA per SM.
inline int vjp_parts(int64_t R, int TM) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((R + TM - 1) / TM, dev_num_sms()));
}

// Large batches (two 64-row tiles per SM or more) take 64-row tiles when the model's 64-row layout
// (`bytes64`) fits; a model that only fits a 32-row tile evaluates every batch on 32-row tiles.
inline bool use_64_rows(int64_t R, int bytes64) {
  return R >= (int64_t)64 * dev_num_sms() * 2 && bytes64 <= kMaxSmemBytes;
}

// The weight ring of the SIMT kernels: 2 to 8 slots of `wcap` floats, and every chunk -- a multiple of 4
// weight rows of `row_len` floats -- fits one slot.
struct RingChunk {
  int rows, row_len;
};
inline bool ring_ok(std::initializer_list<RingChunk> chunks, int nbuf, int wcap) {
  if (nbuf < 2 || nbuf > 8) return false;
  for (const RingChunk& c : chunks)
    if ((c.rows & 3) || c.rows < 4 || c.rows * c.row_len > wcap) return false;
  return true;
}

}  // namespace sbi
