// Gradient reduction + clip_grad_norm_ + Adam, restating the reference training step
// (/root/reference/sbi/inference/trainers/base.py:1181-1187: clip_grad_norm_(max_norm) then
// torch.optim.Adam.step with torch defaults) on one flat parameter buffer.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/sbi_b200.h"
#include "common.cuh"
#include "device.cuh"

namespace sbi {

// grad[p] = sum_i gpart[i][p] ; fixed summation order -> bitwise reproducible
__device__ __forceinline__ float block_sum(float v, float* red);

// 64 float4 columns per block, the partials split over 4 thread groups (more loads in flight),
// combined in shared memory in a fixed order
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ gpart, int n_part, int64_t n4,
                       float* __restrict__ grad, const uint8_t* __restrict__ mask,
                       float* __restrict__ sumsq_part) {
  __shared__ float red[32];
  __shared__ float4 part[3][64];
  const int col = threadIdx.x & 63, grp = threadIdx.x >> 6;
  const int64_t i = (int64_t)blockIdx.x * 64 + col;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n4) {
    const float4* src = reinterpret_cast<const float4*>(gpart) + i;
#pragma unroll 8
    for (int p = grp; p < n_part; p += 4) {
      const float4 v = __ldg(src + (int64_t)p * n4);
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
  }
  if (grp > 0) part[grp - 1][col] = a;
  __syncthreads();
  float ss = 0.f;
  if (grp == 0 && i < n4) {
#pragma unroll
    for (int g = 0; g < 3; ++g) {
      const float4 v = part[g][col];
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    reinterpret_cast<float4*>(grad)[i] = a;
    if (sumsq_part != nullptr) {
      if (mask != nullptr) {
        const uchar4 mk = reinterpret_cast<const uchar4*>(mask)[i];
        if (!mk.x) a.x = 0.f;
        if (!mk.y) a.y = 0.f;
        if (!mk.z) a.z = 0.f;
        if (!mk.w) a.w = 0.f;
      }
      ss = fmaf(a.x, a.x, fmaf(a.y, a.y, fmaf(a.z, a.z, a.w * a.w)));
    }
  }
  if (sumsq_part != nullptr) {   // one deterministic partial per block (fixed reduction tree)
    const float tot = block_sum(ss, red);
    if (threadIdx.x == 0) sumsq_part[blockIdx.x] = tot;
  }
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    float t = (l < (blockDim.x >> 5)) ? red[l] : 0.f;
    t = warp_sum(t);
    if (l == 0) red[0] = t;
  }
  __syncthreads();
  const float out = red[0];
  __syncthreads();
  return out;
}

// Every CTA first recomputes the full gradient norm (n is ~1e5: 0.4 MB from L2), identically
// and deterministically, then updates its own slice.  No cross-CTA dependency, no atomics.
// d_step[0] = optimizer step count, d_step[1] = CTA completion counter (last CTA bumps step).
__global__ void __launch_bounds__(256)
adam_clip_kernel(float* __restrict__ params, const float* __restrict__ grad,
                 float* __restrict__ state, int32_t* __restrict__ d_step,
                 const uint8_t* __restrict__ mask, int64_t n, float lr, float beta1, float beta2,
                 float eps, float max_norm, float gscale, const float* __restrict__ sumsq_part,
                 int n_sumsq) {
  __shared__ float red[32];
  __shared__ float s_bc1, s_bc2s;
  float clip = 1.f;
  if (max_norm > 0.f) {
    float tot;
    if (sumsq_part != nullptr) {
      // per-block partials of sum g^2 from reduce_partials: fixed-order sum, identical in every CTA
      float ss = 0.f;
      for (int i = threadIdx.x; i < n_sumsq; i += blockDim.x) ss += __ldg(sumsq_part + i);
      tot = block_sum(ss, red) * gscale * gscale;
    } else {
      // every CTA recomputes the full norm (e.g. after an all-reduce): float4 loads, 4 chains
      float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
      const int64_t n4 = n >> 2;
      const float4* g4 = reinterpret_cast<const float4*>(grad);
      const uchar4* m4 = reinterpret_cast<const uchar4*>(mask);
      for (int64_t i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 g = __ldg(g4 + i);
        if (mask != nullptr) {
          const uchar4 mk = m4[i];
          if (!mk.x) g.x = 0.f;
          if (!mk.y) g.y = 0.f;
          if (!mk.z) g.z = 0.f;
          if (!mk.w) g.w = 0.f;
        }
        s0 = fmaf(g.x, g.x, s0); s1 = fmaf(g.y, g.y, s1); s2 = fmaf(g.z, g.z, s2); s3 = fmaf(g.w, g.w, s3);
      }
      for (int64_t i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) {
        float g = __ldg(grad + i);
        if (mask != nullptr && mask[i] == 0) g = 0.f;
        s0 = fmaf(g, g, s0);
      }
      tot = block_sum((s0 + s1) + (s2 + s3), red) * gscale * gscale;
    }
    const float c = max_norm / (sqrtf(tot) + 1e-6f);
    clip = c >= 1.f ? 1.f : c;   // a NaN norm gives a NaN clip for every entry, as torch.clamp(max=1) does
  }
  if (threadIdx.x == 0) {
    // bias corrections 1 - beta^t in double like torch (python floats), by repeated squaring: ~2 log2(t)
    // FP64 multiplies instead of a software pow()
    const int t = d_step[0] + 1;
    double p1 = 1.0, p2 = 1.0, b1 = (double)beta1, b2 = (double)beta2;
    for (int e = t; e > 0; e >>= 1) {
      if (e & 1) { p1 *= b1; p2 *= b2; }
      b1 *= b1;
      b2 *= b2;
    }
    s_bc1 = (float)(1.0 - p1);
    s_bc2s = (float)sqrt(1.0 - p2);
  }
  __syncthreads();
  const float step_size = lr / s_bc1;
  const float bc2s = s_bc2s;
  float* m = state;
  float* v = state + n;
  const int64_t per = (n + gridDim.x - 1) / gridDim.x;
  const int64_t lo = (int64_t)blockIdx.x * per;
  const int64_t hi = lo + per < n ? lo + per : n;
  for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    if (mask != nullptr && mask[i] == 0) continue;
    const float g = grad[i] * gscale * clip;
    const float mi = m[i] + (g - m[i]) * (1.f - beta1);          // exp_avg.lerp_(grad, 1-beta1)
    const float vi = fmaf(g * g, 1.f - beta2, v[i] * beta2);     // mul_(beta2).addcmul_(g,g,1-beta2)
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2s + eps;
    params[i] = params[i] - step_size * (mi / denom);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int done = atomicAdd(d_step + 1, 1);
    if (done == (int)gridDim.x - 1) {
      d_step[1] = 0;
      d_step[0] = d_step[0] + 1;
    }
  }
}

// -sum of the finite entries of a log-prob vector and the count of non-finite ones (the epoch
// statistics of the validation pass, trainers/base.py:1195-1225 + assert_all_finite): one block,
// fixed summation order (deterministic).
__global__ void __launch_bounds__(1024)
nll_stats_kernel(const float* __restrict__ lp, int64_t n, float* __restrict__ out) {
  __shared__ float s_sum[32], s_bad[32];
  float a = 0.f, b = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = lp[i];
    if (isfinite(v)) a -= v; else b += 1.f;
  }
  a = warp_sum(a);
  b = warp_sum(b);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_sum[w] = a; s_bad[w] = b; }
  __syncthreads();
  if (w == 0) {
    a = s_sum[l];
    b = s_bad[l];
    a = warp_sum(a);
    b = warp_sum(b);
    if (l == 0) { out[0] = a; out[1] = b; }
  }
}

}  // namespace sbi

extern "C" int sbi_b200_nll_stats(const float* d_logp, int64_t n, float* d_out2, void* stream) {
  sbi::DeviceGuard dev_guard_(d_logp);
  if (!d_logp || !d_out2 || n < 0) return SBI_EINVAL;
  sbi::nll_stats_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(d_logp, n, d_out2);
  return (int)cudaGetLastError();
}

extern "C" int sbi_b200_reduce_partials(const float* d_gpart, int n_part, int64_t n_params,
                                        float* d_grad, void* stream) {
  sbi::DeviceGuard dev_guard_(d_gpart);
  return sbi_b200_reduce_partials_norm(d_gpart, n_part, n_params, d_grad, nullptr, nullptr, stream);
}

extern "C" int sbi_b200_sumsq_blocks(int64_t n_params) { return (int)((n_params / 4 + 63) / 64); }

extern "C" int sbi_b200_reduce_partials_norm(const float* d_gpart, int n_part, int64_t n_params,
                                             float* d_grad, const uint8_t* d_mask, float* d_sumsq_part,
                                             void* stream) {
  sbi::DeviceGuard dev_guard_(d_gpart);
  if (!d_gpart || !d_grad || n_part < 1 || n_params < 4 || (n_params & 3)) return SBI_EINVAL;
  const int64_t n4 = n_params / 4;
  const int grid = (int)((n4 + 63) / 64);
  sbi::reduce_partials_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_gpart, n_part, n4, d_grad, d_mask,
                                                                   d_sumsq_part);
  return (int)cudaGetLastError();
}

extern "C" int sbi_b200_adam_clip_step(float* d_params, const float* d_grad, float* d_state,
                                       int32_t* d_step, const uint8_t* d_mask, int64_t n, float lr,
                                       float beta1, float beta2, float eps, float max_norm,
                                       float grad_scale, void* stream) {
  sbi::DeviceGuard dev_guard_(d_params);
  return sbi_b200_adam_clip_step_norm(d_params, d_grad, d_state, d_step, d_mask, n, lr, beta1, beta2, eps,
                                      max_norm, grad_scale, nullptr, 0, stream);
}

extern "C" int sbi_b200_adam_clip_step_norm(float* d_params, const float* d_grad, float* d_state,
                                            int32_t* d_step, const uint8_t* d_mask, int64_t n, float lr,
                                            float beta1, float beta2, float eps, float max_norm,
                                            float grad_scale, const float* d_sumsq_part, int n_sumsq,
                                            void* stream) {
  sbi::DeviceGuard dev_guard_(d_params);
  if (!d_params || !d_grad || !d_state || !d_step || n < 1) return SBI_EINVAL;
  if (d_sumsq_part != nullptr && n_sumsq < 1) return SBI_EINVAL;
  int grid = (int)((n + 1023) / 1024);
  if (grid > sbi::dev_num_sms()) grid = sbi::dev_num_sms();
  sbi::adam_clip_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      d_params, d_grad, d_state, d_step, d_mask, n, lr, beta1, beta2, eps, max_norm, grad_scale,
      d_sumsq_part, n_sumsq);
  return (int)cudaGetLastError();
}
