// Ratio-estimator kernels: the NRE `resnet` classifier logit and its VJP.
//   logit(theta, x) = ResidualNet( [ (theta-mu_t)/sd_t ; (x-mu_x)/sd_x ] )      (1 output)
// restating nflows ResidualNet without context (oracle/nflows_port/nn/nets/resnet.py) behind
// sbi's RatioEstimator (/root/reference/sbi/neural_nets/ratio_estimators.py:132-150).
// Same CTA structure as the flow kernels (stages.cuh).  The net is small enough to keep every
// activation of the tile in shared memory, so the VJP is one forward with saves + one backward.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>

#include "stages.cuh"
#include "device.cuh"

namespace sbi {

struct RatioSmem {
  int LD;
  int U, HB, A0, A1S, OUT;
  int dH, dA, dU, dOUT;
  int ring, bar_bytes, total_bytes;
};

__host__ __device__ inline RatioSmem ratio_smem_layout(const sbi_ratio_model& m, int TM, bool train) {
  RatioSmem L;
  L.LD = TM + 4;
  int rows = 0;
  auto take = [&](int n) { int o = rows * L.LD; rows += n; return o; };
  const int K0p = m.Dtp + m.Dxp;
  L.U = take(K0p);
  L.HB = take((train ? m.NB + 1 : 1) * m.Hp);
  L.A0 = take(m.Hp);
  L.A1S = take((train ? std::max(m.NB, 1) : 1) * m.Hp);
  L.OUT = take(4);
  L.dH = L.dA = L.dU = L.dOUT = 0;
  if (train) {
    L.dH = take(m.Hp);
    L.dA = take(m.Hp);
    L.dU = take(K0p);
    L.dOUT = take(4);
  }
  int fl = rows * L.LD;
  fl = (fl + 31) & ~31;
  L.ring = fl;
  fl += m.nbuf * m.wcap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + 2 * m.nbuf * 8 + 16;
  return L;
}

template <int TM>
__device__ __forceinline__ void ratio_load(const sbi_ratio_model& m, const sbi_pairs& pr, int64_t row0,
                                           float* U) {
  pairs_load<TM>(m.Dt, m.Dx, m.Dtp, m.Dxp, m.d_stats, pr, row0, U);
  consumer_sync();
}

// forward; SAVE keeps H_0..H_NB and the hidden relu activations A1_b for the backward
template <Role R, int TM, int RN, bool SAVE>
__device__ __forceinline__ void ratio_net_forward(const sbi_ratio_model& m, WPipe& pipe, float* sm,
                                                  const RatioSmem& L) {
  constexpr int LD = Tile<TM>::LD;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const int Hp = m.Hp, K0p = m.Dtp + m.Dxp;
  float* Hout = sm + L.HB;
  float* A0 = sm + L.A0;
  {
    const float* b0 = P + __ldg(T + SBI_R_B0);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_R_W0), Hp, K0p, m.rpc0, sm + L.U,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float b = __ldg(b0 + n);
                             const float4 h = make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b);
                             st4(Hout + n * LD + r0, h);
                             st4(A0 + n * LD + r0, relu4(h));
                           }
                         });
  }
  for (int b = 0; b < m.NB; ++b) {
    const int* BT = T + SBI_R_BLK0 + 4 * b;
    float* Hin = Hout;
    if (SAVE) Hout = Hin + Hp * LD;
    float* A1 = sm + L.A1S + (SAVE ? b : 0) * Hp * LD;
    const float* b1 = P + __ldg(BT + 1);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(BT + 0), Hp, Hp, m.rpc1, A0,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float c = __ldg(b1 + n);
                             st4(A1 + n * LD + r0, make_float4(relu_f(acc[i][0] + c), relu_f(acc[i][1] + c),
                                                               relu_f(acc[i][2] + c), relu_f(acc[i][3] + c)));
                           }
                         });
    const float* b2 = P + __ldg(BT + 3);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(BT + 2), Hp, Hp, m.rpc1, A1,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float c = __ldg(b2 + n);
                             const float4 hin = ld4(Hin + n * LD + r0);
                             const float4 h = make_float4(hin.x + acc[i][0] + c, hin.y + acc[i][1] + c,
                                                          hin.z + acc[i][2] + c, hin.w + acc[i][3] + c);
                             st4(Hout + n * LD + r0, h);
                             st4(A0 + n * LD + r0, relu4(h));
                           }
                         });
  }
  const float* bf = P + __ldg(T + SBI_R_BF);
  float* OUT = sm + L.OUT;
  fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_R_WF), 4, Hp, 4, Hout,
                       [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                         for (int i = 0; i < RN; ++i) {
                           const int n = n0 + g + i * ng;
                           const float c = __ldg(bf + n);
                           st4(OUT + n * LD + r0, make_float4(acc[i][0] + c, acc[i][1] + c, acc[i][2] + c,
                                                              acc[i][3] + c));
                         }
                       });
}

template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
ratio_forward_kernel(const __grid_constant__ sbi_ratio_model m, const __grid_constant__ sbi_pairs pr,
                     float* __restrict__ logits) {
  extern __shared__ __align__(128) float sm[];
  const RatioSmem L = ratio_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (pr.R + TM - 1) / TM;
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        ratio_net_forward<kProducer, TM, RN, false>(m, pipe, sm, L);
    return;
  }
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    ratio_load<TM>(m, pr, row0, sm + L.U);
    ratio_net_forward<kConsumer, TM, RN, false>(m, pipe, sm, L);
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads)
      if (row0 + r < pr.R) logits[row0 + r] = sm[L.OUT + r];
    consumer_sync();
  }
}

template <int TM, int RN, int RK>
__global__ void __launch_bounds__(kThreads, 1)
ratio_vjp_kernel(const __grid_constant__ sbi_ratio_model m, const __grid_constant__ sbi_pairs pr,
                 const float* __restrict__ gout, float* __restrict__ logits, float* __restrict__ gpart,
                 float* __restrict__ gtheta, float* __restrict__ gx) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const RatioSmem L = ratio_smem_layout(m, TM, true);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (pr.R + TM - 1) / TM;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const int Hp = m.Hp, K0p = m.Dtp + m.Dxp;
  // the W0 dX stage yields dU for every input column; it runs when either side's gradient is wanted
  const bool need_du = (gtheta != nullptr) || (gx != nullptr);

  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      auto noop = [](int, int, float(&)[RK][4], bool) {};
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        ratio_net_forward<kProducer, TM, RN, true>(m, pipe, sm, L);
        dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + SBI_R_WF), 4, Hp, 4, nullptr, Hp, noop);
        for (int b = m.NB - 1; b >= 0; --b) {
          const int* BT = T + SBI_R_BLK0 + 4 * b;
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(BT + 2), Hp, Hp, m.rpc1, nullptr, Hp, noop);
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(BT + 0), Hp, Hp, m.rpc1, nullptr, Hp, noop);
        }
        if (need_du) dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + SBI_R_W0), Hp, K0p, m.rpc0, nullptr, K0p, noop);
      }
    }
    return;
  }

  float* gp = gpart + (size_t)blockIdx.x * m.n_params;
  float* dH = sm + L.dH;
  float* dA = sm + L.dA;
  float* dU = sm + L.dU;
  float* dOUT = sm + L.dOUT;
  float* A0 = sm + L.A0;
  const float* __restrict__ st = m.d_stats;
  for (int e = threadIdx.x; e < 4 * LD; e += kConsumerThreads) dOUT[e] = 0.f;
  int iter = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const bool accum = iter > 0;
    const int64_t row0 = tile * TM;
    ratio_load<TM>(m, pr, row0, sm + L.U);
    ratio_net_forward<kConsumer, TM, RN, true>(m, pipe, sm, L);
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
      const bool ok = row0 + r < pr.R;
      if (ok && logits != nullptr) logits[row0 + r] = sm[L.OUT + r];
      dOUT[r] = ok ? __ldg(gout + row0 + r) : 0.f;
    }
    consumer_sync();
    const float* Hf = sm + L.HB + m.NB * Hp * LD;
    gemm_dw<TM>(dOUT, 1, Hf, m.H, Hp, gp + __ldg(T + SBI_R_WF), gp + __ldg(T + SBI_R_BF), accum);
    dx_stage<kConsumer, TM, RK>(pipe, nullptr, 4, Hp, 4, dOUT, Hp, [&](int k0, int r0, float(&acc)[RK][4], bool) {
#pragma unroll
      for (int j = 0; j < RK; ++j)
        st4(dH + (k0 + j) * LD + r0, make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]));
    });
    for (int b = m.NB - 1; b >= 0; --b) {
      const int* BT = T + SBI_R_BLK0 + 4 * b;
      const float* Hb = sm + L.HB + b * Hp * LD;
      const float* A1 = sm + L.A1S + b * Hp * LD;
      for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
        const int o = (e / TM) * LD + (e % TM);
        A0[o] = relu_f(Hb[o]);
      }
      gemm_dw<TM>(dH, m.H, A1, m.H, Hp, gp + __ldg(BT + 2), gp + __ldg(BT + 3), accum);
      dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, Hp, m.rpc1, dH, Hp,
                                  [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                                    for (int j = 0; j < RK; ++j) {
                                      const int o = (k0 + j) * LD + r0;
                                      const float4 a1 = ld4(A1 + o);
                                      float4 val = make_float4(a1.x > 0.f ? acc[j][0] : 0.f, a1.y > 0.f ? acc[j][1] : 0.f,
                                                               a1.z > 0.f ? acc[j][2] : 0.f, a1.w > 0.f ? acc[j][3] : 0.f);
                                      if (!first) {
                                        const float4 c = ld4(dA + o);
                                        val.x += c.x; val.y += c.y; val.z += c.z; val.w += c.w;
                                      }
                                      st4(dA + o, val);
                                    }
                                  });
      gemm_dw<TM>(dA, m.H, A0, m.H, Hp, gp + __ldg(BT + 0), gp + __ldg(BT + 1), accum);
      dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, Hp, m.rpc1, dA, Hp,
                                  [&](int k0, int r0, float(&acc)[RK][4], bool) {
#pragma unroll
                                    for (int j = 0; j < RK; ++j) {
                                      const int o = (k0 + j) * LD + r0;
                                      const float4 hb = ld4(Hb + o);
                                      const float4 c = ld4(dH + o);
                                      st4(dH + o, make_float4(c.x + (hb.x > 0.f ? acc[j][0] : 0.f),
                                                              c.y + (hb.y > 0.f ? acc[j][1] : 0.f),
                                                              c.z + (hb.z > 0.f ? acc[j][2] : 0.f),
                                                              c.w + (hb.w > 0.f ? acc[j][3] : 0.f)));
                                    }
                                  });
    }
    gemm_dw<TM>(dH, m.H, sm + L.U, K0p, K0p, gp + __ldg(T + SBI_R_W0), gp + __ldg(T + SBI_R_B0), accum);
    if (need_du) {
      dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, K0p, m.rpc0, dH, K0p,
                                  [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                                    for (int j = 0; j < RK; ++j) {
                                      if (k0 + j >= K0p) continue;
                                      float* p = dU + (k0 + j) * LD + r0;
                                      float4 o = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                                      if (!first) {
                                        const float4 c = ld4(p);
                                        o.x += c.x; o.y += c.y; o.z += c.z; o.w += c.w;
                                      }
                                      st4(p, o);
                                    }
                                  });
      if (gtheta != nullptr)
        for (int e = threadIdx.x; e < TM * m.Dt; e += kConsumerThreads) {
          const int r = e / m.Dt, d = e % m.Dt;
          if (row0 + r < pr.R) gtheta[(row0 + r) * m.Dt + d] = dU[d * LD + r] / __ldg(st + m.Dtp + d);
        }
      if (gx != nullptr)
        for (int e = threadIdx.x; e < TM * m.Dx; e += kConsumerThreads) {
          const int r = e / m.Dx, d = e % m.Dx;
          if (row0 + r < pr.R)
            gx[(row0 + r) * m.Dx + d] = dU[(m.Dtp + d) * LD + r] / __ldg(st + 2 * m.Dtp + m.Dxp + d);
        }
    }
    consumer_sync();
  }
}

// out[j] = sum_{k in [row_ptr[j], row_ptr[j+1])} gpair[order ? order[k] : k], summed in k order by the one
// thread that owns out[j][c]: no atomics, so repeated calls are bit-identical.
__global__ void pair_rows_sum_kernel(const float* __restrict__ gpair, int width, const int64_t* __restrict__ order,
                                     const int64_t* __restrict__ row_ptr, int64_t n_rows, float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_rows * width) return;
  const int64_t j = e / width;
  const int c = (int)(e % width);
  const int64_t k1 = __ldg(row_ptr + j + 1);
  float acc = 0.f;
  for (int64_t k = __ldg(row_ptr + j); k < k1; ++k) {
    const int64_t src = order ? __ldg(order + k) : k;
    acc += __ldg(gpair + src * width + c);
  }
  out[e] = acc;
}

}  // namespace sbi

using namespace sbi;

static int ratio_check(const sbi_ratio_model* m) {
  if (!m || !m->d_params || !m->d_tab || !m->d_stats) return SBI_EINVAL;
  if (m->Dt < 1 || m->Dx < 1 || m->H < 1 || m->NB < 0 || m->NB > 8) return SBI_EINVAL;
  if (m->Dtp != round4(m->Dt) || m->Dxp != round4(m->Dx) || m->Hp != round4(m->H)) return SBI_EINVAL;
  if (!ring_ok({{m->rpc0, m->Dtp + m->Dxp}, {m->rpc1, m->Hp}, {4, m->Hp}}, m->nbuf, m->wcap)) return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_ratio_forward(const sbi_ratio_model* m, const sbi_pairs* pairs, float* d_logits,
                                      void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = ratio_check(m);
  if (rc) return rc;
  if (!pairs || !pairs->d_theta || !pairs->d_x || pairs->R < 0 || !d_logits) return SBI_EINVAL;
  if (pairs->R == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int bytes64 = ratio_smem_layout(*m, 64, false).total_bytes;
  if (use_64_rows(pairs->R, bytes64))
    return launch(ratio_forward_kernel<64, 4>, tile_grid(pairs->R, 64, per_sm_110k(bytes64)), kThreads, bytes64, s,
                  *m, *pairs, d_logits);
  const int bytes = ratio_smem_layout(*m, 32, false).total_bytes;
  return launch(ratio_forward_kernel<32, 2>, tile_grid(pairs->R, 32, per_sm_110k(bytes)), kThreads, bytes, s, *m,
                *pairs, d_logits);
}

extern "C" int sbi_b200_ratio_vjp_parts(int64_t R) { return vjp_parts(R, 32); }

extern "C" int sbi_b200_ratio_vjp_inputs(const sbi_ratio_model* m, const sbi_pairs* pairs, const float* d_gout,
                                         float* d_logits, float* d_gpart, float* d_gtheta, float* d_gx,
                                         void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = ratio_check(m);
  if (rc) return rc;
  if (!pairs || !pairs->d_theta || !pairs->d_x || pairs->R < 1 || !d_gpart || !d_gout) return SBI_EINVAL;
  return launch(ratio_vjp_kernel<32, 2, 2>, sbi_b200_ratio_vjp_parts(pairs->R), kThreads,
                ratio_smem_layout(*m, 32, true).total_bytes, (cudaStream_t)stream, *m, *pairs, d_gout, d_logits,
                d_gpart, d_gtheta, d_gx);
}

extern "C" int sbi_b200_ratio_vjp(const sbi_ratio_model* m, const sbi_pairs* pairs, const float* d_gout,
                                  float* d_logits, float* d_gpart, float* d_gtheta, void* stream) {
  return sbi_b200_ratio_vjp_inputs(m, pairs, d_gout, d_logits, d_gpart, d_gtheta, nullptr, stream);
}

extern "C" int sbi_b200_pair_rows_sum(const float* d_gpair, int32_t width, const int64_t* d_order,
                                      const int64_t* d_row_ptr, int64_t n_rows, float* d_out, void* stream) {
  if (width < 1 || n_rows < 0 || !d_row_ptr || !d_out || (n_rows > 0 && !d_gpair)) return SBI_EINVAL;
  if (n_rows == 0) return 0;
  sbi::DeviceGuard dev_guard_(d_out);
  const int64_t n = n_rows * width;
  pair_rows_sum_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_gpair, width, d_order,
                                                                                   d_row_ptr, n_rows, d_out);
  return (int)cudaGetLastError();
}
