// Ratio-estimator kernels for the NRE `mlp` and `linear` classifiers: the logit and its VJP.
//   mlp:    logit = w_f . relu(N_1(W_1 relu(N_0(W_0 u + b_0)) + b_1)) + b_f
//   linear: logit = w_f . u + b_f
// with u = [ (theta-mu_t)/sd_t ; (x-mu_x)/sd_x ] and N_l = LayerNorm over the H features of a row (or
// the identity), restating sbi/neural_nets/net_builders/classifier.py:49-169 (sbi) behind
// sbi's RatioEstimator.  Same CTA structure as csrc/ratio.cu (stages.cuh): 8 consumer warps run the
// row-tile GEMMs on feature-major activations in shared memory while one producer lane streams the
// weights.  LayerNorm statistics are per row, so a tile needs nothing from any other tile; the VJP is
// one forward with saves (normalised pre-activations x^, 1/sigma per row, the relu outputs) plus one
// backward.  Every partial-gradient address is written by one thread in tile order (no atomics), so a
// repeated call gives bit-identical gradients.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>

#include "stages.cuh"
#include "device.cuh"

namespace sbi {

// Float offsets into shared memory.  Hidden layer l keeps XH_l (pre-activation, normalised in place) and
// A_l (relu output); without saves A_l overwrites XH_l.  STAT: per layer [mean(TM) | rstd(TM)];
// RED: row-reduction scratch, 2 x (kConsumerThreads / TM) partial sums per row, then one spare row sum.
struct MlpSmem {
  int U, H0, OUT, STAT, RED;
  int dP, dQ, dU, dOUT;
  int ring, bar_bytes, total_bytes;
};

__host__ __device__ inline MlpSmem mlp_smem_layout(const sbi_ratio_mlp_model& m, int TM, bool train) {
  MlpSmem L;
  const int LD = TM + 4;
  int fl = 0;
  auto take = [&](int n) { int o = fl; fl += n; return o; };
  const int K0p = m.Dtp + m.Dxp;
  L.U = take(K0p * LD);
  L.H0 = take((train ? 2 : 1) * m.NL * m.Hp * LD);
  L.OUT = take(4 * LD);
  L.STAT = take(2 * m.NL * TM);
  L.RED = take(2 * kConsumerThreads + TM);
  L.dP = L.dQ = L.dU = L.dOUT = 0;
  if (train) {
    L.dP = take(m.Hp * LD);
    L.dQ = take(m.Hp * LD);
    L.dU = take(K0p * LD);
    L.dOUT = take(4 * LD);
  }
  fl = (fl + 31) & ~31;
  L.ring = fl;
  fl += m.nbuf * m.wcap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + 2 * m.nbuf * 8 + 16;
  return L;
}

// For every tile row r: out0[r] = sum_{f<F} p(f, r), out1[r] = sum_{f<F} q(f, r).  Each row is summed by
// kConsumerThreads / TM threads over interleaved features, then combined in a fixed order.
template <int TM, class Fn>
__device__ __forceinline__ void row_sums(int F, float* red, float* out0, float* out1, Fn&& pq) {
  constexpr int P = kConsumerThreads / TM;
  const int r = threadIdx.x % TM, part = threadIdx.x / TM;
  float s0 = 0.f, s1 = 0.f;
  for (int f = part; f < F; f += P) {
    const float2 v = pq(f, r);
    s0 += v.x;
    s1 += v.y;
  }
  red[part * TM + r] = s0;
  red[(P + part) * TM + r] = s1;
  consumer_sync();
  if (threadIdx.x < TM) {
    float t0 = 0.f, t1 = 0.f;
#pragma unroll
    for (int q = 0; q < P; ++q) {
      t0 += red[q * TM + threadIdx.x];
      t1 += red[(P + q) * TM + threadIdx.x];
    }
    out0[threadIdx.x] = t0;
    out1[threadIdx.x] = t1;
  }
  consumer_sync();
}

// hidden layer l of the forward: Z = W_l X + b_l into XH, then (LayerNorm) and relu into A
template <Role R, int TM, int RN, bool SAVE>
__device__ __forceinline__ void mlp_layer_forward(const sbi_ratio_mlp_model& m, WPipe& pipe, float* sm,
                                                  const MlpSmem& L, int l, const float* X, int Kp, int rpc) {
  constexpr int LD = Tile<TM>::LD;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab + 4 * l;
  const int H = m.H, Hp = m.Hp;
  float* XH = sm + L.H0 + (SAVE ? 2 * l : l) * Hp * LD;
  float* A = XH + (SAVE ? Hp * LD : 0);
  const float* b = P + __ldg(T + SBI_RM_B0);
  fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_RM_W0), Hp, Kp, rpc, X,
                       [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                         for (int i = 0; i < RN; ++i) {
                           const int n = n0 + g + i * ng;
                           const float c = __ldg(b + n);
                           st4(XH + n * LD + r0, make_float4(acc[i][0] + c, acc[i][1] + c, acc[i][2] + c,
                                                             acc[i][3] + c));
                         }
                       });
  if (R == kProducer) return;
  if (m.norm == SBI_RM_NORM_LAYER) {
    float* mean = sm + L.STAT + 2 * l * TM;
    float* rstd = mean + TM;
    float* red = sm + L.RED;
    const float invH = 1.f / (float)H;
    row_sums<TM>(H, red, mean, rstd, [&](int f, int r) { return make_float2(XH[f * LD + r], 0.f); });
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads) mean[r] *= invH;
    consumer_sync();
    row_sums<TM>(H, red, rstd, red + 2 * kConsumerThreads, [&](int f, int r) {
      const float d = XH[f * LD + r] - mean[r];
      return make_float2(d * d, 0.f);
    });
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads) rstd[r] = rsqrtf(rstd[r] * invH + m.ln_eps);
    consumer_sync();
    const float* gam = P + __ldg(T + SBI_RM_G0);
    const float* bet = P + __ldg(T + SBI_RM_BE0);
    for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
      const int f = e / TM, r = e % TM, o = f * LD + r;
      float xh = 0.f, a = 0.f;
      if (f < H) {
        xh = (XH[o] - mean[r]) * rstd[r];
        a = relu_f(fmaf(xh, __ldg(gam + f), __ldg(bet + f)));
      }
      if (SAVE) XH[o] = xh;
      A[o] = a;
    }
  } else {
    for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
      const int o = (e / TM) * LD + e % TM;
      A[o] = relu_f(XH[o]);
    }
  }
  consumer_sync();
}

// forward; returns the input of the output layer (A of the last hidden layer, or U)
template <Role R, int TM, int RN, bool SAVE>
__device__ __forceinline__ const float* mlp_net_forward(const sbi_ratio_mlp_model& m, WPipe& pipe, float* sm,
                                                        const MlpSmem& L) {
  constexpr int LD = Tile<TM>::LD;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const float* X = sm + L.U;
  int Kp = m.Dtp + m.Dxp;
  for (int l = 0; l < m.NL; ++l) {
    mlp_layer_forward<R, TM, RN, SAVE>(m, pipe, sm, L, l, X, Kp, l == 0 ? m.rpc0 : m.rpc1);
    X = sm + L.H0 + (SAVE ? 2 * l + 1 : l) * m.Hp * LD;
    Kp = m.Hp;
  }
  const float* bf = P + __ldg(T + SBI_RM_BF);
  float* OUT = sm + L.OUT;
  fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_RM_WF), 4, Kp, 4, X,
                       [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                         for (int i = 0; i < RN; ++i) {
                           const int n = n0 + g + i * ng;
                           const float c = __ldg(bf + n);
                           st4(OUT + n * LD + r0, make_float4(acc[i][0] + c, acc[i][1] + c, acc[i][2] + c,
                                                              acc[i][3] + c));
                         }
                       });
  return X;
}

template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
ratio_mlp_forward_kernel(const __grid_constant__ sbi_ratio_mlp_model m, const __grid_constant__ sbi_pairs pr,
                         float* __restrict__ logits) {
  extern __shared__ __align__(128) float sm[];
  const MlpSmem L = mlp_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (pr.R + TM - 1) / TM;
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        mlp_net_forward<kProducer, TM, RN, false>(m, pipe, sm, L);
    return;
  }
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    pairs_load<TM>(m.Dt, m.Dx, m.Dtp, m.Dxp, m.d_stats, pr, row0, sm + L.U);
    consumer_sync();
    mlp_net_forward<kConsumer, TM, RN, false>(m, pipe, sm, L);
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads)
      if (row0 + r < pr.R) logits[row0 + r] = sm[L.OUT + r];
    consumer_sync();
  }
}

// hidden layer l of the backward, dY = dL/dA_l in place in D (relu mask already applied):
// LayerNorm gamma / beta gradients, then D <- dL/dZ_l = rstd (dx^ - mean_f dx^ - x^ mean_f(dx^ x^)), dx^ = gamma dY
template <int TM>
__device__ __forceinline__ void mlp_norm_backward(const sbi_ratio_mlp_model& m, float* sm, const MlpSmem& L,
                                                  int l, float* D, float* gp, bool accum) {
  constexpr int LD = Tile<TM>::LD;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab + 4 * l;
  const int H = m.H, Hp = m.Hp;
  const float* XH = sm + L.H0 + 2 * l * Hp * LD;
  const float* rstd = sm + L.STAT + (2 * l + 1) * TM;
  float* red = sm + L.RED;
  float* s_dx = sm + L.STAT + 2 * l * TM;      // the layer's row means are not needed any more
  float* s_dxx = red + 2 * kConsumerThreads;
  const float* gam = P + __ldg(T + SBI_RM_G0);
  for (int e = threadIdx.x; e < 2 * H; e += kConsumerThreads) {
    const bool beta = e >= H;
    const int f = beta ? e - H : e;
    const float* dy = D + f * LD;
    const float* xh = XH + f * LD;
    float s = 0.f;
    for (int r = 0; r < TM; ++r) s = beta ? s + dy[r] : fmaf(dy[r], xh[r], s);
    grad_out(gp + __ldg(T + (beta ? SBI_RM_BE0 : SBI_RM_G0)) + f, s, accum);
  }
  row_sums<TM>(H, red, s_dx, s_dxx, [&](int f, int r) {
    const float dxh = D[f * LD + r] * __ldg(gam + f);
    return make_float2(dxh, dxh * XH[f * LD + r]);
  });
  const float invH = 1.f / (float)H;
  for (int e = threadIdx.x; e < H * TM; e += kConsumerThreads) {
    const int f = e / TM, r = e % TM, o = f * LD + r;
    const float dxh = D[o] * __ldg(gam + f);
    D[o] = rstd[r] * (dxh - s_dx[r] * invH - XH[o] * (s_dxx[r] * invH));
  }
  consumer_sync();
}

template <int TM, int RN, int RK>
__global__ void __launch_bounds__(kThreads, 1)
ratio_mlp_vjp_kernel(const __grid_constant__ sbi_ratio_mlp_model m, const __grid_constant__ sbi_pairs pr,
                     const float* __restrict__ gout, float* __restrict__ logits, float* __restrict__ gpart,
                     float* __restrict__ gtheta) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const MlpSmem L = mlp_smem_layout(m, TM, true);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (pr.R + TM - 1) / TM;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const int H = m.H, Hp = m.Hp, K0p = m.Dtp + m.Dxp;
  const int KFp = m.NL > 0 ? Hp : K0p;
  const bool need_dth = (gtheta != nullptr);

  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      auto noop = [](int, int, float(&)[RK][4], bool) {};
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        mlp_net_forward<kProducer, TM, RN, true>(m, pipe, sm, L);
        if (m.NL > 0 || need_dth) dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + SBI_RM_WF), 4, KFp, 4, nullptr, KFp, noop);
        for (int l = m.NL - 1; l >= 0; --l) {
          if (l == 0 && !need_dth) break;
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + 4 * l + SBI_RM_W0), Hp, l == 0 ? K0p : Hp,
                                      l == 0 ? m.rpc0 : m.rpc1, nullptr, l == 0 ? K0p : Hp, noop);
        }
      }
    }
    return;
  }

  float* gp = gpart + (size_t)blockIdx.x * m.n_params;
  float* dOUT = sm + L.dOUT;
  float* dU = sm + L.dU;
  const float* __restrict__ st = m.d_stats;
  for (int e = threadIdx.x; e < 4 * LD; e += kConsumerThreads) dOUT[e] = 0.f;
  int iter = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const bool accum = iter > 0;
    const int64_t row0 = tile * TM;
    pairs_load<TM>(m.Dt, m.Dx, m.Dtp, m.Dxp, st, pr, row0, sm + L.U);
    consumer_sync();
    const float* XF = mlp_net_forward<kConsumer, TM, RN, true>(m, pipe, sm, L);
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
      const bool ok = row0 + r < pr.R;
      if (ok && logits != nullptr) logits[row0 + r] = sm[L.OUT + r];
      dOUT[r] = ok ? __ldg(gout + row0 + r) : 0.f;
    }
    consumer_sync();
    gemm_dw<TM>(dOUT, 1, XF, m.NL > 0 ? H : K0p, KFp, gp + __ldg(T + SBI_RM_WF), gp + __ldg(T + SBI_RM_BF), accum);
    // dY: gradient at the current layer's output, one of the two ping-pong buffers
    float* dY = sm + L.dP;
    float* dN = sm + L.dQ;
    const float* dZ = dOUT;   // gradient at the input of the weight stage being walked back through
    int N = 4, Kp = KFp, rpc = 4;
    for (int l = m.NL - 1; l >= -1; --l) {
      if (l < 0 && !need_dth) break;
      float* out = l >= 0 ? dY : dU;
      const float* A = l >= 0 ? sm + L.H0 + (2 * l + 1) * Hp * LD : nullptr;
      dx_stage<kConsumer, TM, RK>(pipe, nullptr, N, Kp, rpc, dZ, Kp,
                                  [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                                    for (int j = 0; j < RK; ++j) {
                                      if (k0 + j >= Kp) continue;
                                      const int o = (k0 + j) * LD + r0;
                                      float4 v = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                                      if (A != nullptr) {
                                        const float4 a = ld4(A + o);
                                        v = make_float4(a.x > 0.f ? v.x : 0.f, a.y > 0.f ? v.y : 0.f,
                                                        a.z > 0.f ? v.z : 0.f, a.w > 0.f ? v.w : 0.f);
                                      }
                                      if (!first) {
                                        const float4 c = ld4(out + o);
                                        v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w;
                                      }
                                      st4(out + o, v);
                                    }
                                  });
      if (l < 0) break;
      if (m.norm == SBI_RM_NORM_LAYER) mlp_norm_backward<TM>(m, sm, L, l, dY, gp, accum);
      const int* LT = T + 4 * l;
      const float* X = l > 0 ? sm + L.H0 + (2 * l - 1) * Hp * LD : sm + L.U;
      const int K = l > 0 ? H : K0p;
      N = Hp;
      Kp = l > 0 ? Hp : K0p;
      rpc = l > 0 ? m.rpc1 : m.rpc0;
      gemm_dw<TM>(dY, H, X, K, Kp, gp + __ldg(LT + SBI_RM_W0), gp + __ldg(LT + SBI_RM_B0), accum);
      dZ = dY;
      dY = dN;
      dN = const_cast<float*>(dZ);
    }
    if (need_dth) {
      for (int e = threadIdx.x; e < TM * m.Dt; e += kConsumerThreads) {
        const int r = e / m.Dt, d = e % m.Dt;
        if (row0 + r < pr.R) gtheta[(row0 + r) * m.Dt + d] = dU[d * LD + r] / __ldg(st + m.Dtp + d);
      }
    }
    consumer_sync();
  }
}

}  // namespace sbi

using namespace sbi;

static int ratio_mlp_check(const sbi_ratio_mlp_model* m) {
  if (!m || !m->d_params || !m->d_tab || !m->d_stats) return SBI_EINVAL;
  if (m->Dt < 1 || m->Dx < 1 || m->H < 1 || (m->NL != 0 && m->NL != 2)) return SBI_EINVAL;
  if (m->norm != SBI_RM_NORM_NONE && m->norm != SBI_RM_NORM_LAYER) return SBI_EINVAL;
  if (m->norm == SBI_RM_NORM_LAYER && !(m->ln_eps > 0.f)) return SBI_EINVAL;
  if (m->Dtp != round4(m->Dt) || m->Dxp != round4(m->Dx) || m->Hp != round4(m->H)) return SBI_EINVAL;
  const int K0p = m->Dtp + m->Dxp;
  if (!ring_ok({{m->rpc0, K0p}, {m->rpc1, m->Hp}, {4, m->NL > 0 ? m->Hp : K0p}}, m->nbuf, m->wcap)) return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_ratio_mlp_forward(const sbi_ratio_mlp_model* m, const sbi_pairs* pairs, float* d_logits,
                                          void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = ratio_mlp_check(m);
  if (rc) return rc;
  if (!pairs || !pairs->d_theta || !pairs->d_x || pairs->R < 0 || !d_logits) return SBI_EINVAL;
  if (pairs->R == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int bytes64 = mlp_smem_layout(*m, 64, false).total_bytes;
  if (use_64_rows(pairs->R, bytes64))
    return launch(ratio_mlp_forward_kernel<64, 4>, tile_grid(pairs->R, 64, per_sm_110k(bytes64)), kThreads, bytes64,
                  s, *m, *pairs, d_logits);
  const int bytes = mlp_smem_layout(*m, 32, false).total_bytes;
  return launch(ratio_mlp_forward_kernel<32, 2>, tile_grid(pairs->R, 32, per_sm_110k(bytes)), kThreads, bytes, s,
                *m, *pairs, d_logits);
}

extern "C" int sbi_b200_ratio_mlp_vjp_parts(int64_t R) { return vjp_parts(R, 32); }

extern "C" int sbi_b200_ratio_mlp_vjp(const sbi_ratio_mlp_model* m, const sbi_pairs* pairs, const float* d_gout,
                                      float* d_logits, float* d_gpart, float* d_gtheta, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = ratio_mlp_check(m);
  if (rc) return rc;
  if (!pairs || !pairs->d_theta || !pairs->d_x || pairs->R < 1 || !d_gpart || !d_gout) return SBI_EINVAL;
  return launch(ratio_mlp_vjp_kernel<32, 2, 2>, sbi_b200_ratio_mlp_vjp_parts(pairs->R), kThreads,
                mlp_smem_layout(*m, 32, true).total_bytes, (cudaStream_t)stream, *m, *pairs, d_gout, d_logits, d_gpart,
                d_gtheta);
}
