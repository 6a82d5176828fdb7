// Tensor-core bulk evaluation of the NRE `resnet` classifier: RatioEstimator.forward /
// unnormalized_log_ratio (/root/reference/sbi/neural_nets/ratio_estimators.py:132-154; network
// built at /root/reference/sbi/neural_nets/net_builders/classifier.py:172-235: nflows
// ResidualNet(in = D_theta + D_x, out = 1, hidden 50, 2 blocks, relu, no context)) for large
// numbers of (theta, x) pairs — the potential of rejection sampling and MCMC at a fixed x_o.
//
// Same machinery as nsf_tc.cu (tc_common.cuh): 128 pairs per CTA = 128 lanes of the accumulator
// store, two threads per pair splitting the hidden columns, wgmma kind tf32 with the 3xTF32 split on
// both warpgroups, A from the store, weights streamed by TMA in the no-swizzle K-major layout.
//   stages: initial layer (A = [theta | x] standardised, K = round8(Dt + Dx)),
//           per block W_1 relu(h), W_2 relu(.), final layer as an N = 16 MMA whose column 0 is
//           the logit.
// Arithmetic outside the linears follows ratio.cu (standardisation, bias adds, residual order).
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>

#include "tc_common.cuh"
#include "device.cuh"

namespace sbi {
namespace tc {

struct RatioTcSmem {
  int us, bias, ring;     // float offsets
  int bar_bytes, total_bytes;
};
__host__ __device__ inline RatioTcSmem ratio_tc_smem_layout(const sbi_ratio_model& m, int stage_cap) {
  RatioTcSmem L;
  int fl = 0;
  L.us = fl;   fl += (m.Dtp + m.Dxp) * kRows;
  L.bias = fl; fl += 64 + m.NB * 128 + 4;       // b0 | per block b1, b2 | bf
  fl = (fl + 31) & ~31;
  L.ring = fl; fl += kSlots * stage_cap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + kSlots * 8;
  return L;
}

template <int H>
__global__ void __launch_bounds__(kThreads, 2)
ratio_forward_tc_kernel(const __grid_constant__ sbi_ratio_model m, const __grid_constant__ sbi_nsf_tc tc,
                        const __grid_constant__ sbi_pairs pr, float* __restrict__ logits, const StoreArgs sa) {
  constexpr int HP8 = (H + 7) & ~7;
  constexpr int NCH = HP8 / 8;
  constexpr int NC = HP8 / 2;       // hidden columns per thread
  constexpr int NG = NC / 4;
  static_assert(HP8 % 8 == 0 && NC % 4 == 0 && H <= 64, "hidden width");
  extern __shared__ __align__(128) float sm[];
  const RatioTcSmem L = ratio_tc_smem_layout(m, tc.stage_cap);
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(sm) + L.bar_bytes);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int64_t ntiles = (pr.R + kRows - 1) / kRows;

  Issuer iss = tc_begin<kSlots>(full, sm + L.ring, tc, 1, ntiles, false, kCols, sa);

  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  float* us = sm + L.us;
  const int half = warp >> 2;
  const int row = ((warp & 3) << 5) | (tid & 31);
  const int cbase = half * NC;
  const int K0 = m.Dt + m.Dx;
  const int k0p8 = __ldg(tc.d_tab + 1);

  // biases once per CTA (zero beyond the real width): [b0 64 | per block b1 64, b2 64 | bf]
  {
    float* bs = sm + L.bias;
    for (int e = tid; e < 64 + m.NB * 128 + 1; e += kThreads) {
      float v = 0.f;
      if (e < 64) {
        if (e < H) v = __ldg(P + __ldg(T + SBI_R_B0) + e);
      } else if (e < 64 + m.NB * 128) {
        const int b = (e - 64) / 128, w = ((e - 64) % 128) / 64, j = (e - 64) % 64;
        if (j < H) v = __ldg(P + __ldg(T + SBI_R_BLK0 + 4 * b + 2 * w + 1) + j);
      } else {
        v = __ldg(P + __ldg(T + SBI_R_BF));
      }
      bs[e] = v;
    }
  }
  const float* bl = sm + L.bias + cbase;

  auto write_a = [&](const float (&act)[NC]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      float a[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = act[4 * g + i];
      store_a4(row, cbase + 4 * g, a);
    }
  };
  auto read_acc = [&](float (&d)[NC]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) ld4(row, cD + cbase + 4 * g, d + 4 * g);
  };
  auto run_stage = [&](int stage, int nk, int N) {
    uint32_t acc = 0u;
    iss.begin(__ldg(tc.d_tab + 5 + 4 * stage));
    iss.block(cD, 0, nk, 0, N, acc);
    iss.end();
  };

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * kRows;
    // ---- load + standardise the pairs (arithmetic of ratio_load, ratio.cu): us[k][row] ----
    {
      const float* __restrict__ st = m.d_stats;
      const int Dt = m.Dt, Dx = m.Dx, Dtp = m.Dtp, Dxp = m.Dxp;
      for (int e = tid; e < kRows * Dtp; e += kThreads) {
        const int r = e / Dtp, d = e % Dtp;
        const int64_t gr = row0 + r;
        float val = 0.f;
        if (d < Dt && gr < pr.R) {
          const int64_t src = pr.d_theta_index ? __ldg(pr.d_theta_index + gr) : gr;
          val = (__ldg(pr.d_theta + src * Dt + d) - __ldg(st + d)) / __ldg(st + Dtp + d);
        }
        if (d < Dt) us[d * kRows + r] = val;
      }
      for (int e = tid; e < kRows * Dxp; e += kThreads) {
        const int r = e / Dxp, d = e % Dxp;
        const int64_t gr = row0 + r;
        float val = 0.f;
        if (d < Dx && gr < pr.R) {
          const int64_t src = pr.x_shared ? 0 : (pr.d_x_index ? __ldg(pr.d_x_index + gr) : gr);
          val = (__ldg(pr.d_x + src * Dx + d) - __ldg(st + 2 * Dtp + d)) / __ldg(st + 2 * Dtp + Dxp + d);
        }
        if (d < Dx) us[(Dt + d) * kRows + r] = val;
      }
      group_sync();
    }
    // ---- initial layer: A columns [theta | x | 0], 8-column chunks alternate between the halves
    for (int c = half; c < k0p8 / 8; c += 2) {
      float a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int j = 8 * c + i;
        a[i] = (j < K0) ? us[j * kRows + row] : 0.f;
      }
      store_a8(row, 8 * c, a);
    }
    group_sync();
    run_stage(0, k0p8 / 8, 64);
    float h[NC];
    {
      float d[NC];
      read_acc(d);
#pragma unroll
      for (int q = 0; q < NC; ++q) h[q] = d[q] + bl[q];
    }
    int stage = 1;
    for (int b = 0; b < m.NB; ++b) {
      const float* b1 = bl + 64 + b * 128;
      const float* b2 = b1 + 64;
      {
        float a[NC];
#pragma unroll
        for (int q = 0; q < NC; ++q) a[q] = relu_f(h[q]);
        write_a(a);
      }
      group_sync();
      run_stage(stage++, NCH, 64);
      {
        float d[NC];
        read_acc(d);
#pragma unroll
        for (int q = 0; q < NC; ++q) d[q] = relu_f(d[q] + b1[q]);
        write_a(d);
      }
      group_sync();
      run_stage(stage++, NCH, 64);
      {
        float d[NC];
        read_acc(d);
#pragma unroll
        for (int q = 0; q < NC; ++q) h[q] = h[q] + d[q] + b2[q];     // hin + acc + bias, as ratio.cu
      }
    }
    // ---- final layer: logit = w_f . h + b_f as column 0 of an N = 16 MMA ----
    write_a(h);
    group_sync();
    run_stage(stage, NCH, 16);
    if (half == 0) {
      float d[4];
      ld4(row, cD, d);
      if (row0 + row < pr.R) logits[row0 + row] = d[0] + sm[L.bias + 64 + m.NB * 128];
    }
    group_sync();   // us and the accumulators are reused by the next tile
  }

  tc_end(kCols, sa);
}

}  // namespace tc
}  // namespace sbi

using namespace sbi;

extern "C" int sbi_b200_ratio_tc_supported(const sbi_ratio_model* m, const sbi_nsf_tc* tc) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc) return 0;
  if (m->H != 50) return 0;
  if (m->Dt + m->Dx > 56 || m->NB < 1 || m->NB > 8) return 0;
  if (tc->stage_cap <= 0 || (tc->stage_cap & 31) || tc->n_words <= 0) return 0;
  const tc::RatioTcSmem L = tc::ratio_tc_smem_layout(*m, tc->stage_cap);
  return L.total_bytes <= 112 * 1024 ? 1 : 0;
}

extern "C" int sbi_b200_ratio_tc_pack(const sbi_ratio_model* m, const sbi_nsf_tc* tc, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  return m ? tc::pack_weights(m->d_params, tc, (cudaStream_t)stream) : SBI_EINVAL;
}

extern "C" int sbi_b200_ratio_forward_tc(const sbi_ratio_model* m, const sbi_nsf_tc* tc,
                                         const sbi_pairs* pairs, float* d_logits, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc || !pairs || !pairs->d_theta || !pairs->d_x || pairs->R < 0 || !d_logits) return SBI_EINVAL;
  if (!tc->d_tab || !tc->d_tcw) return SBI_EINVAL;
  if (!sbi_b200_ratio_tc_supported(m, tc)) return SBI_ESMEM;
  if (pairs->R == 0) return 0;
  tc::StoreArgs sa;
  if (int e = tc::store_args(&sa)) return e;
  return launch(tc::ratio_forward_tc_kernel<50>, tile_grid(pairs->R, tc::kRows, 2), tc::kThreads,
                tc::ratio_tc_smem_layout(*m, tc->stage_cap).total_bytes, (cudaStream_t)stream, *m, *tc, *pairs,
                d_logits, sa);
}
