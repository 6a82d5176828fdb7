// Masked autoregressive flow kernels (log_prob, forward+backward VJP, inverse/sampling) for the
// flow sbi's `build_maf` assembles (/root/reference/sbi/neural_nets/net_builders/flow.py:115-209):
//
//   z-score -> T x [ affine autoregressive transform (MADE conditioner, feed-forward masked blocks,
//   tanh, context added after the first masked layer) -> fixed random permutation ] -> N(0, I)
//
// and, with head == SBI_MAF_RQS, for `build_maf_rqs` (flow.py:212-330): the same MADE emits 3K-1 raw
// spline parameters per feature and the element-wise map is the monotone rational-quadratic spline
// with linear tails (rqs.cuh; MaskedPiecewiseRationalQuadraticAutoregressiveTransform),
// restating nflows 0.14 MaskedAffineAutoregressiveTransform / MADE / RandomPermutation
// (oracle/nflows_port/transforms/{autoregressive,made,permutations}.py; SURVEY App. A.6).
// Same CTA structure as the NSF kernels (stages.cuh): 8 consumer warps + 1 TMA producer warp, a
// tile of TM rows resident in shared memory, weights streamed with cp.async.bulk.  Masks are
// folded into the packed weights (W .* M), so every layer is an ordinary row-tile GEMM.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>

#include "stages.cuh"
#include "device.cuh"
#include "rqs.cuh"

namespace sbi {

struct MafSmem {
  int LD;
  int ZA, ZB, CTX, HB, OUT, LDF, LDACC;
  int ZS, dZ, dZ2, dHa, dHb, dOUT, GR, dCTX;
  int ring, bar_bytes, total_bytes;
};

__host__ __device__ inline MafSmem maf_smem_layout(const sbi_maf_model& m, int TM, bool train) {
  MafSmem L;
  L.LD = TM + 4;
  int rows = 0;
  auto take = [&](int n) { int o = rows * L.LD; rows += n; return o; };
  L.ZA = take(m.Dp);
  L.ZB = take(m.Dp);
  L.CTX = take(m.Cp);
  L.HB = take((m.NB + 1) * m.Hp);
  L.OUT = take(m.OUTp);
  L.LDF = take(m.Dp);
  L.LDACC = take(1);
  L.ZS = L.dZ = L.dZ2 = L.dHa = L.dHb = L.dOUT = L.GR = L.dCTX = 0;
  if (train) {
    L.ZS = take(m.T * m.Dp);
    L.dZ = take(m.Dp);
    L.dZ2 = take(m.Dp);
    L.dHa = take(m.Hp);
    L.dHb = take(m.Hp);
    L.dOUT = take(m.OUTp);
    L.GR = take(1);
    L.dCTX = take(m.Cp);
  }
  int fl = rows * L.LD;
  fl = (fl + 31) & ~31;
  L.ring = fl;
  fl += m.nbuf * m.wcap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + 2 * m.nbuf * 8 + 16;
  return L;
}

struct MafLayerView {
  const int* LT;
  const int* perm;
  const int* iperm;
};
__device__ __forceinline__ MafLayerView maf_layer(const sbi_maf_model& m, int l) {
  MafLayerView v;
  v.LT = m.d_layer_tab + l * SBI_MAF_LAYER_STRIDE;
  v.perm = m.d_perm_tab + __ldg(v.LT + SBI_M_PERM);
  v.iperm = v.perm + m.D;
  return v;
}

__device__ __forceinline__ float maf_scale(const sbi_maf_model& m, float s) {
  return (m.scale_softplus ? softplus_f(s) : sigmoid_f(s + 2.f)) + 1e-3f;
}
// d scale / d s
__device__ __forceinline__ float maf_dscale(const sbi_maf_model& m, float s) {
  if (m.scale_softplus) return sigmoid_f(s);
  const float g = sigmoid_f(s + 2.f);
  return g * (1.f - g);
}

__device__ __forceinline__ RqsConst maf_rqs_const(const sbi_maf_model& m) {
  RqsConst c;
  c.K = m.KB; c.B = m.tail_bound; c.isq = m.isq;
  c.min_w = m.min_w; c.min_h = m.min_h; c.min_d = m.min_d;
  c.edge_raw = logf(expf(1.f - m.min_d) - 1.f);
  return c;
}

// MADE conditioner: OUT = Wf tanh(... tanh(W1 (W0 z + b0 + Wc ctx + bc) + b1) ...) + bf.
// Writes H_0 .. H_NB into sm+L.HB and the 2D autoregressive parameters into sm+L.OUT.
template <Role R, int TM, int RN>
__device__ __forceinline__ void made_forward(const sbi_maf_model& m, const MafLayerView& v, WPipe& pipe,
                                             float* sm, const MafSmem& L, const float* Zin) {
  constexpr int LD = Tile<TM>::LD;
  const float* __restrict__ P = m.d_params;
  const int Hp = m.Hp;
  float* H0 = sm + L.HB;
  const float* b0 = P + __ldg(v.LT + SBI_M_B0);
  const float* bc = P + __ldg(v.LT + SBI_M_BC);
  glu_stage<R, TM, RN>(pipe, P + __ldg(v.LT + SBI_M_W0), m.Dp, P + __ldg(v.LT + SBI_M_WC), m.Cp, Hp,
                       m.rpc0, Zin, sm + L.CTX,
                       [&](int n0, int g, int ng, int r0, float(&at)[RN][4], float(&ag)[RN][4]) {
#pragma unroll
                         for (int i = 0; i < RN; ++i) {
                           const int n = n0 + g + i * ng;
                           const float b = __ldg(b0 + n) + __ldg(bc + n);
                           st4(H0 + n * LD + r0, make_float4(at[i][0] + ag[i][0] + b, at[i][1] + ag[i][1] + b,
                                                             at[i][2] + ag[i][2] + b, at[i][3] + ag[i][3] + b));
                         }
                       });
  for (int b = 0; b < m.NB; ++b) {
    const float* Hin = sm + L.HB + b * Hp * LD;
    float* Hout = sm + L.HB + (b + 1) * Hp * LD;
    const float* bb = P + __ldg(v.LT + SBI_M_BLK0 + 2 * b + 1);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(v.LT + SBI_M_BLK0 + 2 * b), Hp, Hp, m.rpc1, Hin,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float c = __ldg(bb + n);
                             st4(Hout + n * LD + r0, make_float4(tanhf(acc[i][0] + c), tanhf(acc[i][1] + c),
                                                                 tanhf(acc[i][2] + c), tanhf(acc[i][3] + c)));
                           }
                         });
  }
  const float* Hf = sm + L.HB + m.NB * Hp * LD;
  float* OUT = sm + L.OUT;
  const float* bf = P + __ldg(v.LT + SBI_M_BF);
  fwd_stage<R, TM, RN>(pipe, P + __ldg(v.LT + SBI_M_WF), m.OUTp, Hp, m.rpcf, Hf,
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

// z' = scale * z + shift, permuted; LDACC += sum_d log scale_d (fixed order)
template <int TM>
__device__ __forceinline__ void maf_affine_forward(const sbi_maf_model& m, const MafLayerView& v, float* sm,
                                                   const MafSmem& L, const float* Zin, float* Zout) {
  constexpr int LD = Tile<TM>::LD;
  const float* OUT = sm + L.OUT;
  float* LDF = sm + L.LDF;
  if (m.head == SBI_MAF_RQS) {
    const RqsConst rc = maf_rqs_const(m);
    for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
      const int d = t / TM, r = t % TM;
      float y, ld;
      rqs_forward(OUT + (m.OUTM * d) * LD + r, LD, rc, Zin[d * LD + r], y, ld);
      Zout[__ldg(v.iperm + d) * LD + r] = y;
      LDF[d * LD + r] = ld;
    }
  } else {
    for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
      const int d = t / TM, r = t % TM;
      const float sc = maf_scale(m, OUT[(2 * d) * LD + r]);
      Zout[__ldg(v.iperm + d) * LD + r] = sc * Zin[d * LD + r] + OUT[(2 * d + 1) * LD + r];
      LDF[d * LD + r] = logf(sc);
    }
  }
  consumer_sync();
  for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
    float a = 0.f;
    for (int d = 0; d < m.D; ++d) a += LDF[d * LD + r];
    sm[L.LDACC + r] += a;
  }
  consumer_sync();
}

template <int TM>
__device__ __forceinline__ void maf_load(const sbi_maf_model& m, const sbi_rows& rows, int64_t row0,
                                         float* sm, const MafSmem& L, bool raw) {
  constexpr int LD = Tile<TM>::LD;
  load_rows<TM>(m.D, m.Dp, m.C, m.Cp, m.d_stats, rows, row0, sm + L.ZA, sm + L.CTX, raw);
  for (int e = threadIdx.x; e < m.Dp * LD; e += kConsumerThreads) sm[L.ZB + e] = 0.f;
  for (int r = threadIdx.x; r < TM; r += kConsumerThreads) sm[L.LDACC + r] = 0.f;
  consumer_sync();
}

// =================================================================================================
template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
maf_logprob_kernel(const __grid_constant__ sbi_maf_model m, const __grid_constant__ sbi_rows rows,
                   float* __restrict__ logp, float* __restrict__ noise) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const MafSmem L = maf_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int l = 0; l < m.T; ++l) made_forward<kProducer, TM, RN>(m, maf_layer(m, l), pipe, sm, L, nullptr);
    return;
  }
  const float ld_const = m.ld_zscore - 0.5f * (float)m.D * 1.8378770664093453f;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    maf_load<TM>(m, rows, row0, sm, L, false);
    float* Zin = sm + L.ZA;
    float* Zout = sm + L.ZB;
    for (int l = 0; l < m.T; ++l) {
      const MafLayerView v = maf_layer(m, l);
      made_forward<kConsumer, TM, RN>(m, v, pipe, sm, L, Zin);
      maf_affine_forward<TM>(m, v, sm, L, Zin, Zout);
      float* t = Zin; Zin = Zout; Zout = t;
    }
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads)
      if (row0 + r < rows.R) {
        float ss = 0.f;
        for (int d = 0; d < m.D; ++d) ss = fmaf(Zin[d * LD + r], Zin[d * LD + r], ss);
        logp[row0 + r] = -0.5f * ss + sm[L.LDACC + r] + ld_const;
      }
    if (noise != nullptr)
      for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
        const int r = e / m.D, d = e % m.D;
        if (row0 + r < rows.R) noise[(row0 + r) * m.D + d] = Zin[d * LD + r];
      }
    consumer_sync();
  }
}

// =================================================================================================
// inverse: D sequential MADE passes per layer (restating AutoregressiveTransform.inverse)
template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
maf_inverse_kernel(const __grid_constant__ sbi_maf_model m, const __grid_constant__ sbi_rows rows,
                   float* __restrict__ out, float* __restrict__ logabsdet) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const MafSmem L = maf_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int l = m.T - 1; l >= 0; --l)
          for (int it = 0; it < m.D; ++it)
            made_forward<kProducer, TM, RN>(m, maf_layer(m, l), pipe, sm, L, nullptr);
    return;
  }
  const float* __restrict__ st = m.d_stats;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    maf_load<TM>(m, rows, row0, sm, L, true);
    float* Y = sm + L.ZA;     // layer output (pre-inverse), holds the current flow state
    float* X = sm + L.ZB;     // autoregressive iterate
    float* Yp = sm + L.LDF;   // un-permuted layer output
    const float* OUT = sm + L.OUT;
    for (int l = m.T - 1; l >= 0; --l) {
      const MafLayerView v = maf_layer(m, l);
      for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
        const int d = t / TM, r = t % TM;
        Yp[d * LD + r] = Y[__ldg(v.iperm + d) * LD + r];
        X[d * LD + r] = 0.f;
      }
      consumer_sync();
      for (int it = 0; it < m.D; ++it) {
        made_forward<kConsumer, TM, RN>(m, v, pipe, sm, L, X);
        const bool last = (it == m.D - 1);
        if (m.head == SBI_MAF_RQS) {
          const RqsConst rc = maf_rqs_const(m);
          for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
            const int d = t / TM, r = t % TM;
            float xv, ld;
            rqs_inverse(OUT + (m.OUTM * d) * LD + r, LD, rc, Yp[d * LD + r], xv, ld);
            X[d * LD + r] = xv;
            if (last) Y[d * LD + r] = -ld;      // forward log-derivative (ld = log dx/dy)
          }
        } else {
          for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
            const int d = t / TM, r = t % TM;
            const float sc = maf_scale(m, OUT[(2 * d) * LD + r]);
            X[d * LD + r] = (Yp[d * LD + r] - OUT[(2 * d + 1) * LD + r]) / sc;
            if (last) Y[d * LD + r] = logf(sc);   // Y is free now: stash log scale
          }
        }
        consumer_sync();
      }
      for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
        float a = 0.f;
        for (int d = 0; d < m.D; ++d) a += Y[d * LD + r];
        sm[L.LDACC + r] -= a;
      }
      consumer_sync();
      for (int e = threadIdx.x; e < m.D * TM; e += kConsumerThreads) {
        const int d = e / TM, r = e % TM;
        Y[d * LD + r] = X[d * LD + r];
      }
      consumer_sync();
    }
    for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
      const int r = e / m.D, d = e % m.D;
      if (row0 + r < rows.R)
        out[(row0 + r) * m.D + d] = (Y[d * LD + r] - __ldg(st + d)) / __ldg(st + m.Dp + d);
    }
    if (logabsdet != nullptr)
      for (int r = threadIdx.x; r < TM; r += kConsumerThreads)
        if (row0 + r < rows.R) logabsdet[row0 + r] = sm[L.LDACC + r] - m.ld_zscore;
    consumer_sync();
  }
}

// =================================================================================================
template <int TM, int RN, int RK>
__global__ void __launch_bounds__(kThreads, 1)
maf_vjp_kernel(const __grid_constant__ sbi_maf_model m, const __grid_constant__ sbi_rows rows,
               const float* __restrict__ gout, float g_const, float* __restrict__ logp,
               float* __restrict__ gpart, float* __restrict__ ginput, float* __restrict__ gcond,
               float* __restrict__ loss_acc) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const MafSmem L = maf_smem_layout(m, TM, true);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  const bool need_dctx = (gcond != nullptr);
  const float* __restrict__ P = m.d_params;
  const int Hp = m.Hp, Dp = m.Dp, Cp = m.Cp;
  const int rpcc = max(4, min(Hp, (m.wcap / Cp) & ~3));
  const int rpcd = max(4, min(Hp, (m.wcap / Dp) & ~3));

  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      auto noop = [](int, int, float(&)[RK][4], bool) {};
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        for (int l = 0; l < m.T; ++l) made_forward<kProducer, TM, RN>(m, maf_layer(m, l), pipe, sm, L, nullptr);
        for (int l = m.T - 1; l >= 0; --l) {
          const MafLayerView v = maf_layer(m, l);
          made_forward<kProducer, TM, RN>(m, v, pipe, sm, L, nullptr);
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_M_WF), m.OUTp, Hp, m.rpcf, nullptr, Hp, noop);
          for (int b = m.NB - 1; b >= 0; --b)
            dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_M_BLK0 + 2 * b), Hp, Hp, m.rpc1, nullptr, Hp, noop);
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_M_W0), Hp, Dp, rpcd, nullptr, Dp, noop);
          if (need_dctx)
            dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_M_WC), Hp, Cp, rpcc, nullptr, Cp, noop);
        }
      }
    }
    return;
  }

  const float ld_const = m.ld_zscore - 0.5f * (float)m.D * 1.8378770664093453f;
  float* gp = gpart + (size_t)blockIdx.x * m.n_params;
  float* GR = sm + L.GR;
  float* dCTX = sm + L.dCTX;
  float* dOUT = sm + L.dOUT;
  const float* OUT = sm + L.OUT;
  const float* __restrict__ st = m.d_stats;
  for (int e = threadIdx.x; e < m.OUTp * LD; e += kConsumerThreads) dOUT[e] = 0.f;

  int iter = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const bool accum = iter > 0;
    const int64_t row0 = tile * TM;
    maf_load<TM>(m, rows, row0, sm, L, false);
    float* Zin = sm + L.ZA;
    float* Zout = sm + L.ZB;
    for (int l = 0; l < m.T; ++l) {
      const MafLayerView v = maf_layer(m, l);
      for (int e = threadIdx.x; e < Dp * LD; e += kConsumerThreads) sm[L.ZS + l * Dp * LD + e] = Zin[e];
      made_forward<kConsumer, TM, RN>(m, v, pipe, sm, L, Zin);
      maf_affine_forward<TM>(m, v, sm, L, Zin, Zout);
      float* t = Zin; Zin = Zout; Zout = t;
    }
    {
      float nll = 0.f, bad = 0.f;
      for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
        float g = 0.f;
        if (row0 + r < rows.R) {
          float ss = 0.f;
          for (int d = 0; d < m.D; ++d) ss = fmaf(Zin[d * LD + r], Zin[d * LD + r], ss);
          const float lp = -0.5f * ss + sm[L.LDACC + r] + ld_const;
          if (logp != nullptr) logp[row0 + r] = lp;
          g = gout ? __ldg(gout + row0 + r) : g_const;
          if (isfinite(lp)) nll -= lp; else bad += 1.f;
        }
        GR[r] = g;
      }
      if (loss_acc != nullptr && threadIdx.x < ((TM + 31) / 32) * 32) {
        nll = warp_sum(nll);
        bad = warp_sum(bad);
        if ((threadIdx.x & 31) == 0) {
          atomicAdd(loss_acc + 0, nll);
          if (bad != 0.f) atomicAdd(loss_acc + 1, bad);
        }
      }
    }
    consumer_sync();
    float* dZ = sm + L.dZ;
    float* dZ2 = sm + L.dZ2;
    for (int e = threadIdx.x; e < Dp * TM; e += kConsumerThreads) {
      const int d = e / TM, r = e % TM;
      dZ[d * LD + r] = -GR[r] * Zin[d * LD + r];
      dZ2[d * LD + r] = 0.f;
    }
    if (need_dctx)
      for (int e = threadIdx.x; e < Cp * LD; e += kConsumerThreads) dCTX[e] = 0.f;
    consumer_sync();

    for (int l = m.T - 1; l >= 0; --l) {
      const MafLayerView v = maf_layer(m, l);
      const float* ZSl = sm + L.ZS + l * Dp * LD;
      made_forward<kConsumer, TM, RN>(m, v, pipe, sm, L, ZSl);
      // affine + permutation backward
      if (m.head == SBI_MAF_RQS) {
        const RqsConst rc = maf_rqs_const(m);
        for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
          const int d = t / TM, r = t % TM;
          const float dzn = dZ[__ldg(v.iperm + d) * LD + r];
          dZ2[d * LD + r] = rqs_backward(OUT + (m.OUTM * d) * LD + r, LD, rc, ZSl[d * LD + r], dzn, GR[r],
                                         dOUT + (m.OUTM * d) * LD + r, LD);
        }
      } else {
        for (int t = threadIdx.x; t < m.D * TM; t += kConsumerThreads) {
          const int d = t / TM, r = t % TM;
          const float dzn = dZ[__ldg(v.iperm + d) * LD + r];
          const float s = OUT[(2 * d) * LD + r];
          const float sc = maf_scale(m, s);
          dOUT[(2 * d) * LD + r] = (dzn * ZSl[d * LD + r] + GR[r] / sc) * maf_dscale(m, s);
          dOUT[(2 * d + 1) * LD + r] = dzn;
          dZ2[d * LD + r] = dzn * sc;
        }
      }
      consumer_sync();
      float* dHa = sm + L.dHa;
      float* dHb = sm + L.dHb;
      // final layer
      {
        const float* Hf = sm + L.HB + m.NB * Hp * LD;
        gemm_dw<TM>(dOUT, m.OUTM * m.D, Hf, m.H, Hp, gp + __ldg(v.LT + SBI_M_WF), gp + __ldg(v.LT + SBI_M_BF), accum);
        const bool act = m.NB > 0;   // H_NB = tanh(.) iff there is at least one block
        dx_stage<kConsumer, TM, RK>(pipe, nullptr, m.OUTp, Hp, m.rpcf, dOUT, Hp,
                                    [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                                      for (int j = 0; j < RK; ++j) {
                                        const int o = (k0 + j) * LD + r0;
                                        float4 val = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                                        if (!first) {
                                          const float4 c = ld4(dHa + o);
                                          val.x += c.x; val.y += c.y; val.z += c.z; val.w += c.w;
                                        }
                                        st4(dHa + o, val);
                                      }
                                    });
        if (act) {   // tanh'(.) = 1 - h^2, applied once all chunks are accumulated
          for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
            const int o = (e / TM) * LD + (e % TM);
            const float h = Hf[o];
            dHa[o] *= (1.f - h * h);
          }
          consumer_sync();
        }
      }
      for (int b = m.NB - 1; b >= 0; --b) {
        const float* Hb = sm + L.HB + b * Hp * LD;      // input of block b
        gemm_dw<TM>(dHa, m.H, Hb, m.H, Hp, gp + __ldg(v.LT + SBI_M_BLK0 + 2 * b),
                    gp + __ldg(v.LT + SBI_M_BLK0 + 2 * b + 1), accum);
        dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, Hp, m.rpc1, dHa, Hp,
                                    [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                                      for (int j = 0; j < RK; ++j) {
                                        const int o = (k0 + j) * LD + r0;
                                        float4 val = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                                        if (!first) {
                                          const float4 c = ld4(dHb + o);
                                          val.x += c.x; val.y += c.y; val.z += c.z; val.w += c.w;
                                        }
                                        st4(dHb + o, val);
                                      }
                                    });
        if (b > 0) {   // H_b = tanh(.) for b >= 1; H_0 is the raw pre-activation
          for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
            const int o = (e / TM) * LD + (e % TM);
            const float h = Hb[o];
            dHb[o] *= (1.f - h * h);
          }
          consumer_sync();
        }
        float* t = dHa; dHa = dHb; dHb = t;
      }
      // initial (masked) layer + context layer; dHa = grad wrt H_0
      gemm_dw<TM>(dHa, m.H, ZSl, m.D, Dp, gp + __ldg(v.LT + SBI_M_W0), gp + __ldg(v.LT + SBI_M_B0), accum);
      gemm_dw<TM>(dHa, m.H, sm + L.CTX, m.C, Cp, gp + __ldg(v.LT + SBI_M_WC), gp + __ldg(v.LT + SBI_M_BC), accum);
      dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, Dp, rpcd, dHa, Dp,
                                  [&](int k0, int r0, float(&acc)[RK][4], bool) {
#pragma unroll
                                    for (int j = 0; j < RK; ++j) {
                                      if (k0 + j >= Dp) continue;
                                      float* p = dZ2 + (k0 + j) * LD + r0;
                                      const float4 c = ld4(p);
                                      st4(p, make_float4(c.x + acc[j][0], c.y + acc[j][1], c.z + acc[j][2],
                                                         c.w + acc[j][3]));
                                    }
                                  });
      if (need_dctx)
        dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, Cp, rpcc, dHa, Cp,
                                    [&](int k0, int r0, float(&acc)[RK][4], bool) {
#pragma unroll
                                      for (int j = 0; j < RK; ++j) {
                                        if (k0 + j >= Cp) continue;
                                        float* p = dCTX + (k0 + j) * LD + r0;
                                        const float4 c = ld4(p);
                                        st4(p, make_float4(c.x + acc[j][0], c.y + acc[j][1], c.z + acc[j][2],
                                                           c.w + acc[j][3]));
                                      }
                                    });
      float* t = dZ; dZ = dZ2; dZ2 = t;
    }
    if (ginput != nullptr)
      for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
        const int r = e / m.D, d = e % m.D;
        if (row0 + r < rows.R) ginput[(row0 + r) * m.D + d] = dZ[d * LD + r] * __ldg(st + Dp + d);
      }
    if (need_dctx)
      for (int e = threadIdx.x; e < TM * m.C; e += kConsumerThreads) {
        const int r = e / m.C, c = e % m.C;
        if (row0 + r < rows.R) gcond[(row0 + r) * m.C + c] = dCTX[c * LD + r] / __ldg(st + 2 * Dp + Cp + c);
      }
    consumer_sync();
  }
}

}  // namespace sbi

// =================================================================================================
using namespace sbi;

static int maf_check(const sbi_maf_model* m) {
  if (!m || !m->d_params || !m->d_layer_tab || !m->d_perm_tab || !m->d_stats) return SBI_EINVAL;
  if (m->D < 1 || m->C < 1 || m->H < 1 || m->T < 1 || m->NB < 0 || m->NB > 8) return SBI_EINVAL;
  if (m->head != SBI_MAF_AFFINE && m->head != SBI_MAF_RQS) return SBI_EINVAL;
  if (m->OUTM != (m->head == SBI_MAF_AFFINE ? 2 : 3 * m->KB - 1)) return SBI_EINVAL;
  if (m->head == SBI_MAF_RQS && (m->KB < 2 || m->KB > kRqsMaxBins || !(m->tail_bound > 0.f))) return SBI_EINVAL;
  if (m->Dp != round4(m->D) || m->Cp != round4(m->C) || m->Hp != round4(m->H) ||
      m->OUTp != round4(m->OUTM * m->D))
    return SBI_EINVAL;
  if (!ring_ok({{m->rpc0, m->Dp + m->Cp}, {m->rpc1, m->Hp}, {m->rpcf, m->Hp}, {4, m->Cp}, {4, m->Dp}}, m->nbuf,
               m->wcap))
    return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_maf_logprob(const sbi_maf_model* m, const sbi_rows* rows, float* d_logp,
                                    float* d_noise, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = maf_check(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_logp) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int bytes64 = maf_smem_layout(*m, 64, false).total_bytes;
  if (use_64_rows(rows->R, bytes64))
    return launch(maf_logprob_kernel<64, 4>, tile_grid(rows->R, 64, per_sm_110k(bytes64)), kThreads, bytes64, s,
                  *m, *rows, d_logp, d_noise);
  const int bytes = maf_smem_layout(*m, 32, false).total_bytes;
  return launch(maf_logprob_kernel<32, 2>, tile_grid(rows->R, 32, per_sm_110k(bytes)), kThreads, bytes, s, *m,
                *rows, d_logp, d_noise);
}

extern "C" int sbi_b200_maf_inverse(const sbi_maf_model* m, const sbi_rows* rows, float* d_out,
                                    float* d_logabsdet, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = maf_check(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_out) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int bytes64 = maf_smem_layout(*m, 64, false).total_bytes;
  if (use_64_rows(rows->R, bytes64))
    return launch(maf_inverse_kernel<64, 4>, tile_grid(rows->R, 64, per_sm_110k(bytes64)), kThreads, bytes64, s,
                  *m, *rows, d_out, d_logabsdet);
  const int bytes = maf_smem_layout(*m, 32, false).total_bytes;
  return launch(maf_inverse_kernel<32, 2>, tile_grid(rows->R, 32, per_sm_110k(bytes)), kThreads, bytes, s, *m,
                *rows, d_out, d_logabsdet);
}

extern "C" int sbi_b200_maf_vjp_parts(int64_t R) { return vjp_parts(R, 32); }

extern "C" int sbi_b200_maf_vjp(const sbi_maf_model* m, const sbi_rows* rows, const float* d_gout,
                                float g_const, float* d_logp, float* d_gpart, float* d_ginput,
                                float* d_gcond, float* d_loss_acc, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = maf_check(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 1 || !d_gpart) return SBI_EINVAL;
  return launch(maf_vjp_kernel<32, 2, 2>, sbi_b200_maf_vjp_parts(rows->R), kThreads,
                maf_smem_layout(*m, 32, true).total_bytes, (cudaStream_t)stream, *m, *rows, d_gout, g_const, d_logp,
                d_gpart, d_ginput, d_gcond, d_loss_acc);
}
