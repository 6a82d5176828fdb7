// Lock-step vectorized slice sampler: the per-chain state machine of the reference's
// SliceSamplerVectorized.run (/root/reference/sbi/samplers/mcmc/slice_numpy.py:412-587) as one
// kernel launch per lock-step.  One thread per chain; chain state (position, bracket, widths,
// dimension order, Philox RNG) lives in HBM in float64 like the reference's numpy state; the
// potential is evaluated between steps by the estimator kernels on the (C, D) float32 `params`.
// The bracket arithmetic is written with explicit round-to-nearest intrinsics so that nvcc does not
// contract it into FMAs: every bracket end and proposal is then the float64 value numpy computes from
// the same draws, which lets the tests compare a chain with the reference draw for draw.
//
// Reference semantics kept: BEGIN evaluates at the current point and draws the slice height
// logu = logp + log(1 - u); the bracket is placed randomly, stepped out below then above while the
// ends are inside the slice (and narrower than max_width), then shrunk around rejected proposals;
// during the first `tuning` sweeps width_i <- running mean of the bracket sizes; a fresh random
// dimension order is drawn for every sweep; sweep t >= tuning is recorded in samples[t - tuning].
#include <cuda_runtime.h>
#include <curand_kernel.h>
#include <math.h>

#include "../../include/sbi_b200.h"
#include "device.cuh"

namespace sbi {

typedef curandStatePhilox4_32_10_t Rng;
static_assert(sizeof(Rng) <= 64, "rng state slot");

__device__ __forceinline__ double rand01(Rng* r) {   // [0, 1) like numpy's rand()
  return 1.0 - curand_uniform_double(r);
}

__device__ __forceinline__ void shuffle_order(int32_t* ord, int D, Rng* r) {
  for (int i = 0; i < D; ++i) ord[i] = i;
  for (int i = D - 1; i > 0; --i) {   // Fisher-Yates
    int j = (int)(rand01(r) * (i + 1));
    if (j > i) j = i;
    const int t = ord[i]; ord[i] = ord[j]; ord[j] = t;
  }
}

__device__ __forceinline__ void write_params(const sbi_slice_chains& s, int c, float* params, int dim,
                                             double val) {
  const double* x = s.d_x + (size_t)c * s.D;
  float* p = params + (size_t)c * s.D;
  for (int d = 0; d < s.D; ++d) p[d] = (float)(d == dim ? val : x[d]);
}

__global__ void slice_init_kernel(const sbi_slice_chains s, float* params) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= s.C) return;
  Rng* rng = reinterpret_cast<Rng*>(reinterpret_cast<char*>(s.d_rng) + (size_t)c * 64);
  Rng r;
  curand_init(s.seed, (unsigned long long)c, 0ULL, &r);
  int32_t* ord = s.d_order + (size_t)c * s.D;
  shuffle_order(ord, s.D, &r);
  int32_t* is = s.d_istate + (size_t)c * 4;
  is[0] = SBI_SLICE_BEGIN; is[1] = 0; is[2] = 0; is[3] = 0;
  double* fs = s.d_fstate + (size_t)c * 8;
  const int dim = ord[0];
  fs[0] = s.d_x[(size_t)c * s.D + dim];              // cxi
  fs[1] = s.d_width[(size_t)c * s.D + dim];          // wi (the caller's initial widths)
  write_params(s, c, params, dim, fs[0]);
  *rng = r;
}

__global__ void slice_step_kernel(const sbi_slice_chains s, const float* __restrict__ logp,
                                  float* params, int32_t* n_done) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= s.C) return;
  int32_t* is = s.d_istate + (size_t)c * 4;
  int state = is[0];
  if (state == SBI_SLICE_DONE) { atomicAdd(n_done, 1); return; }
  Rng* rng = reinterpret_cast<Rng*>(reinterpret_cast<char*>(s.d_rng) + (size_t)c * 64);
  Rng r = *rng;
  double* fs = s.d_fstate + (size_t)c * 8;
  int32_t* ord = s.d_order + (size_t)c * s.D;
  double* x = s.d_x + (size_t)c * s.D;
  double* width = s.d_width + (size_t)c * s.D;
  int i = is[1], t = is[2];
  const int dim = ord[i];
  double cxi = fs[0], wi = fs[1], lx = fs[2], ux = fs[3], xi = fs[4], logu = fs[5];
  const double lp = (double)logp[c];
  double next = cxi;

  if (state == SBI_SLICE_BEGIN) {
    logu = lp + log(1.0 - rand01(&r));
    lx = __dsub_rn(cxi, __dmul_rn(wi, rand01(&r)));
    ux = lx + wi;
    next = lx;
    state = SBI_SLICE_LOWER;
  } else if (state == SBI_SLICE_LOWER) {
    if (lp >= logu && cxi - lx < s.max_width) {
      lx -= wi;
      next = lx;
    } else {
      next = ux;
      state = SBI_SLICE_UPPER;
    }
  } else if (state == SBI_SLICE_UPPER) {
    if (lp >= logu && ux - cxi < s.max_width) {
      ux += wi;
      next = ux;
    } else {
      xi = __dadd_rn(__dmul_rn(ux - lx, rand01(&r)), lx);
      next = xi;
      state = SBI_SLICE_SAMPLE;
    }
  } else {   // SAMPLE_SLICE
    if (lp < logu) {   // rejected: shrink the bracket
      if (xi < cxi) lx = xi; else ux = xi;
      xi = __dadd_rn(__dmul_rn(ux - lx, rand01(&r)), lx);
      next = xi;
    } else if (t < s.num_samples + s.tuning) {
      x[dim] = xi;     // accept
      if (t < s.tuning) width[dim] += ((ux - lx) - width[dim]) / (double)(t + 1);
      if (i < s.D - 1) {
        i += 1;
      } else {
        if (t >= s.tuning) {
          double* dst = s.d_samples + ((size_t)c * s.num_samples + (t - s.tuning)) * s.D;
          for (int d = 0; d < s.D; ++d) dst[d] = x[d];
        }
        t += 1;
        i = 0;
        shuffle_order(ord, s.D, &r);
      }
      state = SBI_SLICE_BEGIN;
      const int nd = ord[i];
      cxi = x[nd];
      wi = width[nd];
      fs[0] = cxi; fs[1] = wi;
      is[0] = state; is[1] = i; is[2] = t;
      write_params(s, c, params, nd, cxi);
      *rng = r;
      return;
    } else {
      state = SBI_SLICE_DONE;
      atomicAdd(n_done, 1);
    }
  }
  fs[2] = lx; fs[3] = ux; fs[4] = xi; fs[5] = logu;
  is[0] = state;
  if (state != SBI_SLICE_DONE) write_params(s, c, params, dim, next);
  *rng = r;
}

}  // namespace sbi

static int slice_check(const sbi_slice_chains* s) {
  if (!s || s->C < 1 || s->D < 1 || s->num_samples < 0 || s->tuning < 0) return SBI_EINVAL;
  if (!s->d_x || !s->d_width || !s->d_order || !s->d_istate || !s->d_fstate || !s->d_rng) return SBI_EINVAL;
  if (s->num_samples > 0 && !s->d_samples) return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_slice_init(const sbi_slice_chains* s, float* d_params, void* stream) {
  sbi::DeviceGuard dev_guard_(s ? s->d_x : nullptr);
  int rc = slice_check(s);
  if (rc || !d_params) return SBI_EINVAL;
  sbi::slice_init_kernel<<<(s->C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*s, d_params);
  return (int)cudaGetLastError();
}

extern "C" int sbi_b200_slice_step(const sbi_slice_chains* s, const float* d_logp, float* d_params,
                                   int32_t* d_n_done, void* stream) {
  sbi::DeviceGuard dev_guard_(s ? s->d_x : nullptr);
  int rc = slice_check(s);
  if (rc || !d_logp || !d_params || !d_n_done) return SBI_EINVAL;
  cudaError_t e = cudaMemsetAsync(d_n_done, 0, sizeof(int32_t), (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  sbi::slice_step_kernel<<<(s->C + 127) / 128, 128, 0, (cudaStream_t)stream>>>(*s, d_logp, d_params, d_n_done);
  return (int)cudaGetLastError();
}
