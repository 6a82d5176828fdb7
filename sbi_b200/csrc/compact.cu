// Accept / reject + order-preserving compaction of one batch of rejection-sampling proposals
// (/root/reference/sbi/samplers/rejection/rejection.py:170-200: `target_proposal_ratio = exp(potential -
// scaled proposal log-prob); keep = ratio > u; samples = candidates[keep]`): the accepted candidates are
// written, in proposal order, behind the ones already collected, together with their global proposal
// index; the running count stays on the device.  Three launches (flags + block counts, scan of the block
// counts, scatter) replace exp / compare / boolean-index (whose `nonzero` synchronises the host) -- the
// accepted set and its order are exactly those of the reference's boolean indexing.  The accept decision is a
// predicate functor, the ratio test above.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/sbi_b200.h"
#include "device.cuh"

namespace sbi {
namespace compact {

constexpr int kThreads = 256;
constexpr int kPer = 4;                       // consecutive candidates per thread
constexpr int kTile = kThreads * kPer;        // candidates per block

// Accept predicate of count_kernel / scatter_kernel: keep(i) says whether candidate i is accepted.
struct RatioAccept {
  const float* __restrict__ lt;
  const float* __restrict__ ls;
  const float* __restrict__ u;
  // same expression as the reference: exp(a - b) > u  (NaN compares false -> rejected)
  __device__ __forceinline__ bool operator()(int64_t i) const { return expf(lt[i] - ls[i]) > u[i]; }
};

template <class Accept>
__global__ void count_kernel(Accept keep_flag, int64_t n, int32_t* __restrict__ block_count) {
  __shared__ int sh[kThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kTile + (int64_t)threadIdx.x * kPer;
  int c = 0;
#pragma unroll
  for (int j = 0; j < kPer; ++j)
    if (base + j < n && keep_flag(base + j)) ++c;
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += sh[w];
    block_count[blockIdx.x] = t;
  }
}

// exclusive scan of the block counts (in place), shifted by the number already collected; *count += total
__global__ void scan_kernel(int32_t* __restrict__ block_count, int nb, int32_t* __restrict__ count) {
  __shared__ int sh[kThreads];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = *count;
  __syncthreads();
  for (int b0 = 0; b0 < nb; b0 += kThreads) {
    const int i = b0 + threadIdx.x;
    const int v = i < nb ? block_count[i] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < kThreads; o <<= 1) {          // Hillis-Steele inclusive scan
      const int t = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    if (i < nb) block_count[i] = carry + sh[threadIdx.x] - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += sh[kThreads - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *count = carry;
}

template <class Accept>
__global__ void scatter_kernel(const float* __restrict__ cand, int D, Accept keep_flag, int64_t n, int64_t index_base, const int32_t* __restrict__ block_off, float* __restrict__ out,
                               int64_t* __restrict__ out_idx, int64_t cap) {
  __shared__ int sh[kThreads / 32];
  const int64_t base = (int64_t)blockIdx.x * kTile + (int64_t)threadIdx.x * kPer;
  bool k[kPer];
  int c = 0;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    k[j] = base + j < n && keep_flag(base + j);
    c += k[j] ? 1 : 0;
  }
  // exclusive prefix of c over the block (threads own consecutive candidates, so thread order = proposal order)
  int incl = c;
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += t;
  }
  if ((threadIdx.x & 31) == 31) sh[threadIdx.x >> 5] = incl;
  __syncthreads();
  int woff = 0;
  for (int w = 0; w < (threadIdx.x >> 5); ++w) woff += sh[w];
  int64_t pos = (int64_t)block_off[blockIdx.x] + woff + incl - c;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    if (!k[j]) continue;
    if (pos < cap) {
      for (int d = 0; d < D; ++d) out[pos * D + d] = cand[(base + j) * D + d];
      if (out_idx != nullptr) out_idx[pos] = index_base + base + j;
    }
    ++pos;
  }
}

// count -> scan -> scatter for one batch of n candidates under the accept predicate `keep`
template <class Accept>
int compact(Accept keep, const float* cand, int D, int64_t n, int64_t index_base, float* out, int64_t* out_idx,
            int64_t cap, int32_t* count, int32_t* scratch, cudaStream_t s) {
  if (n == 0) return 0;
  const int64_t nb64 = (n + kTile - 1) / kTile;
  if (nb64 > (1 << 30)) return SBI_EINVAL;
  const int nb = (int)nb64;
  count_kernel<<<nb, kThreads, 0, s>>>(keep, n, scratch);
  scan_kernel<<<1, kThreads, 0, s>>>(scratch, nb, count);
  scatter_kernel<<<nb, kThreads, 0, s>>>(cand, D, keep, n, index_base, scratch, out, out_idx, cap);
  return (int)cudaGetLastError();
}

// ---- sampling-importance-resampling: one categorical draw per group of K candidates ----------------------------
// (/root/reference/sbi/samplers/importance/sir.py:59-63: `w = softmax(lw).cumsum(-1); mask = cumsum(w >= u) == 1;
// thetas.reshape(b, K, D)[mask]`).  One warp per group, kGroups groups per block; lanes walk the group in
// 32-candidate chunks, so any K >= 1 works.  The select kernel writes the chosen index of every group (-1: none)
// and the block's selection count; scan_kernel above turns the counts into output offsets; the scatter kernel
// copies the selected rows.
constexpr int kGroups = kThreads / 32;        // groups per block

__device__ __forceinline__ float log_weight(const float* lt, const float* lp, int64_t i) {
  return lt[i] - lp[i];                       // fp32 subtraction, as importance_sample computes it
}

__global__ void sir_select_kernel(const float* __restrict__ lt, const float* __restrict__ lp,
                                  const float* __restrict__ u, int64_t groups, int K, int32_t* __restrict__ sel,
                                  int32_t* __restrict__ block_count) {
  __shared__ int sh[kGroups];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t g = (int64_t)blockIdx.x * kGroups + w;
  int pick = -1;
  if (g < groups) {
    const int64_t row0 = g * K;
    // pass 1: max; a NaN or +inf anywhere (or all -inf) makes torch's softmax NaN, which selects nothing
    float m = -INFINITY;
    bool bad = false;
    for (int k0 = 0; k0 < K; k0 += 32) {
      const int k = k0 + lane;
      if (k < K) {
        const float v = log_weight(lt, lp, row0 + k);
        bad |= isnan(v) || v == INFINITY;
        m = fmaxf(m, v);
      }
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    bad = __any_sync(0xffffffffu, bad) || m == -INFINITY;
    if (!bad) {
      // pass 2: softmax denominator
      float s = 0.f;
      for (int k0 = 0; k0 < K; k0 += 32) {
        const int k = k0 + lane;
        if (k < K) s += expf(log_weight(lt, lp, row0 + k) - m);
      }
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      // pass 3: inclusive cumulative weights in index order; the first k with cumw_k >= u_g
      const float ug = u[g];
      float carry = 0.f;
      for (int k0 = 0; k0 < K; k0 += 32) {
        const int k = k0 + lane;
        float c = k < K ? expf(log_weight(lt, lp, row0 + k) - m) / s : 0.f;
        for (int o = 1; o < 32; o <<= 1) {
          const float t = __shfl_up_sync(0xffffffffu, c, o);
          if (lane >= o) c += t;
        }
        c += carry;
        const unsigned hit = __ballot_sync(0xffffffffu, k < K && c >= ug);
        if (hit) {
          pick = k0 + __ffs(hit) - 1;
          break;
        }
        carry = __shfl_sync(0xffffffffu, c, 31);
      }
    }
    if (lane == 0) sel[g] = pick;
  }
  if (lane == 0) sh[w] = pick >= 0 ? 1 : 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int j = 0; j < kGroups; ++j) t += sh[j];
    block_count[blockIdx.x] = t;
  }
}

__global__ void sir_scatter_kernel(const float* __restrict__ cand, int D, int64_t groups, int K, int64_t index_base,
                                   const int32_t* __restrict__ sel, const int32_t* __restrict__ block_off,
                                   float* __restrict__ out, int64_t* __restrict__ out_idx, int64_t cap) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t g0 = (int64_t)blockIdx.x * kGroups;
  const int64_t g = g0 + w;
  const int pick = g < groups ? sel[g] : -1;
  if (pick < 0) return;
  // groups before this one in the block that selected a row (warps own consecutive groups: warp order = group order)
  int64_t pos = block_off[blockIdx.x];
  for (int j = 0; j < w; ++j) pos += (g0 + j < groups && sel[g0 + j] >= 0) ? 1 : 0;
  if (pos >= cap) return;
  const float* src = cand + (g * K + pick) * (int64_t)D;
  for (int d = lane; d < D; d += 32) out[pos * D + d] = src[d];
  if (lane == 0 && out_idx != nullptr) out_idx[pos] = index_base + g;
}

}  // namespace compact
}  // namespace sbi

using namespace sbi;

extern "C" int64_t sbi_b200_reject_scratch_ints(int64_t n) {
  return n < 1 ? 1 : (n + compact::kTile - 1) / compact::kTile;
}

extern "C" int sbi_b200_reject_compact(const float* d_cand, int32_t D, const float* d_log_target,
                                       const float* d_log_scaled, const float* d_u, int64_t n, int64_t index_base,
                                       float* d_out, int64_t* d_out_idx, int64_t cap, int32_t* d_count,
                                       int32_t* d_scratch, void* stream) {
  sbi::DeviceGuard dev_guard_(d_cand);
  if (!d_cand || !d_log_target || !d_log_scaled || !d_u || !d_out || !d_count || !d_scratch || D < 1 || n < 0 ||
      cap < 0)
    return SBI_EINVAL;
  return compact::compact(compact::RatioAccept{d_log_target, d_log_scaled, d_u}, d_cand, D, n, index_base, d_out,
                          d_out_idx, cap, d_count, d_scratch, (cudaStream_t)stream);
}

// scratch: one count per block of kGroups groups, then the selected index of every group
extern "C" int64_t sbi_b200_sir_scratch_ints(int64_t groups) {
  if (groups < 1) return 1;
  return (groups + compact::kGroups - 1) / compact::kGroups + groups;
}

extern "C" int sbi_b200_sir_select(const float* d_cand, int32_t D, const float* d_log_target,
                                   const float* d_log_proposal, const float* d_u, int64_t groups, int32_t K,
                                   int64_t index_base, float* d_out, int64_t* d_out_idx, int64_t cap,
                                   int32_t* d_count, int32_t* d_scratch, void* stream) {
  if (!d_cand || !d_log_target || !d_log_proposal || !d_u || !d_out || !d_count || !d_scratch || D < 1 || K < 1 ||
      groups < 0 || cap < 0)
    return SBI_EINVAL;
  sbi::DeviceGuard dev_guard_(d_cand);
  if (groups == 0) return 0;
  const int64_t nb64 = (groups + compact::kGroups - 1) / compact::kGroups;
  if (nb64 > (1 << 30) || groups > INT64_MAX / K) return SBI_EINVAL;
  const int nb = (int)nb64;
  int32_t* block_count = d_scratch;
  int32_t* sel = d_scratch + nb;
  cudaStream_t s = (cudaStream_t)stream;
  compact::sir_select_kernel<<<nb, compact::kThreads, 0, s>>>(d_log_target, d_log_proposal, d_u, groups, K, sel,
                                                               block_count);
  compact::scan_kernel<<<1, compact::kThreads, 0, s>>>(block_count, nb, d_count);
  compact::sir_scatter_kernel<<<nb, compact::kThreads, 0, s>>>(d_cand, D, groups, K, index_base, sel, block_count,
                                                                d_out, d_out_idx, cap);
  return (int)cudaGetLastError();
}
