// NSF kernels + their C-ABI entry points (see include/sbi_b200.h).
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>

#include "nsf.cuh"
#include "device.cuh"

namespace sbi {

// =================================================================================================
// log_prob:  persistent over row tiles
// =================================================================================================
template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
nsf_logprob_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_rows rows,
                   float* __restrict__ logp, float* __restrict__ noise) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const NsfSmem L = nsf_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m, sm, L);
  const int64_t ntiles = (rows.R + TM - 1) / TM;

  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        for (int l = 0; l < m.T; ++l) {
          const NsfLayerView v = layer_view(m, l);
          float* hf = cond_forward<kProducer, TM, RN, false>(m, v, pipe, sm, L);
          spline_forward<kProducer, TM, RN, false>(m, v, pipe, sm, L, hf);
        }
      }
    }
    return;
  }

  const bool mog = m.head == SBI_NSF_MOG;          // no base density: the mixture terms are the likelihood
  const float ld_const = mog ? m.ld_zscore
                             : lu_logdet_total(m, sm + L.PRM) + m.ld_zscore - 0.5f * (float)m.D * 1.8378770664093453f;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    load_tile<TM>(m, rows, row0, sm, L, false);
    for (int l = 0; l < m.T; ++l) {
      const NsfLayerView v = layer_view(m, l);
      lu_prepare(m, v, sm, L);
      gather_identity<TM>(m, v, sm + L.Z, sm + L.U);
      float* hf = cond_forward<kConsumer, TM, RN, false>(m, v, pipe, sm, L);
      spline_forward<kConsumer, TM, RN, false>(m, v, pipe, sm, L, hf);
      fold_ldf<TM>(v, sm, L);
      lu_forward<TM>(m, v, sm, L);
    }
    consumer_sync();
    const float* Z = sm + L.Z;
    for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
      if (row0 + r < rows.R) {
        float ss = 0.f;
        if (!mog)
          for (int d = 0; d < m.D; ++d) ss = fmaf(Z[d * LD + r], Z[d * LD + r], ss);
        logp[row0 + r] = -0.5f * ss + sm[L.LDACC + r] + ld_const;
      }
    }
    if (noise != nullptr) {
      for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
        const int r = e / m.D, d = e % m.D;
        if (row0 + r < rows.R) noise[(row0 + r) * m.D + d] = Z[d * LD + r];
      }
    }
    consumer_sync();
  }
}

// =================================================================================================
// inverse (sampling):  x = T^{-1}(noise | cond)
// =================================================================================================
template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
nsf_inverse_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_rows rows,
                   float* __restrict__ out, float* __restrict__ logabsdet) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const NsfSmem L = nsf_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m, sm, L);
  const int64_t ntiles = (rows.R + TM - 1) / TM;

  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        for (int l = m.T - 1; l >= 0; --l) {
          const NsfLayerView v = layer_view(m, l);
          float* hf = cond_forward<kProducer, TM, RN, false>(m, v, pipe, sm, L);
          spline_forward<kProducer, TM, RN, true>(m, v, pipe, sm, L, hf);
        }
      }
    }
    return;
  }

  const float ld_const = -lu_logdet_total(m, sm + L.PRM) - m.ld_zscore;
  const float* __restrict__ st = m.d_stats;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    load_tile<TM>(m, rows, row0, sm, L, true);
    for (int l = m.T - 1; l >= 0; --l) {
      const NsfLayerView v = layer_view(m, l);
      lu_prepare(m, v, sm, L);
      consumer_sync();
      lu_inverse<TM>(m, v, sm, L);
      gather_identity<TM>(m, v, sm + L.Z, sm + L.U);
      float* hf = cond_forward<kConsumer, TM, RN, false>(m, v, pipe, sm, L);
      spline_forward<kConsumer, TM, RN, true>(m, v, pipe, sm, L, hf);
      fold_ldf<TM>(v, sm, L);
      consumer_sync();
    }
    const float* Z = sm + L.Z;
    for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
      const int r = e / m.D, d = e % m.D;
      if (row0 + r < rows.R)
        out[(row0 + r) * m.D + d] = (Z[d * LD + r] - __ldg(st + d)) / __ldg(st + m.Dp + d);
    }
    if (logabsdet != nullptr) {
      for (int r = threadIdx.x; r < TM; r += kConsumerThreads)
        if (row0 + r < rows.R) logabsdet[row0 + r] = sm[L.LDACC + r] + ld_const;
    }
    consumer_sync();
  }
}

// =================================================================================================
// VJP: forward + backward of  sum_r g_r log q_r  in one kernel (per-layer recompute)
// =================================================================================================
// LU backward for one layer.  In: dZ = grad wrt LU output, VS_l = LU input v.  Out: dZ = grad
// wrt v; parameter gradients -> gp.
template <int TM>
__device__ __forceinline__ void lu_backward(const sbi_nsf_model& m, const NsfLayerView& v,
                                            float* sm, const NsfSmem& L, const float* V,
                                            float* __restrict__ gp, bool accumulate) {
  constexpr int LD = Tile<TM>::LD;
  if (!__ldg(v.LT + SBI_L_HAS_LU)) return;
  const int D = m.D;
  const LuView w = lu_view(m, sm, L);
  float* dZ = sm + L.dZ;
  float* Y = sm + L.Y;     // y = U v
  float* DY = sm + L.Y2;   // dy = L^T dz
  const float* GR = sm + L.GR;
  const int o_lo = __ldg(v.LT + SBI_L_LU_LOWER), o_up = __ldg(v.LT + SBI_L_LU_UPPER);
  const int o_dg = __ldg(v.LT + SBI_L_LU_DIAG), o_bi = __ldg(v.LT + SBI_L_LU_BIAS);
  for (int t = threadIdx.x; t < D * TM; t += kConsumerThreads) {
    const int i = t / TM, r = t % TM;
    float a = 0.f;
    for (int j = i; j < D; ++j) a = fmaf(w.U[i * D + j], V[j * LD + r], a);
    Y[i * LD + r] = a;
    float b = dZ[i * LD + r];
    for (int k = i + 1; k < D; ++k) b = fmaf(w.Lw[k * D + i], dZ[k * LD + r], b);
    DY[i * LD + r] = b;
  }
  consumer_sync();
  // parameter gradients: one (i,j) pair per thread, reduction over the tile rows
  for (int t = threadIdx.x; t < D * D + D; t += kConsumerThreads) {
    float a = 0.f;
    float* dst;
    if (t < D * D) {
      const int i = t / D, j = t % D;
      if (i > j) {          // dL_ij = sum_r dz_i y_j
        for (int r = 0; r < TM; ++r) a = fmaf(dZ[i * LD + r], Y[j * LD + r], a);
        dst = gp + o_lo + i * (i - 1) / 2 + j;
      } else if (i < j) {   // dU_ij = sum_r dy_i v_j
        for (int r = 0; r < TM; ++r) a = fmaf(DY[i * LD + r], V[j * LD + r], a);
        dst = gp + o_up + i * D - i * (i + 1) / 2 + (j - i - 1);
      } else {              // raw diag: (dU_ii + G / U_ii) * sigmoid(raw_i)
        float gs = 0.f;
        for (int r = 0; r < TM; ++r) {
          a = fmaf(DY[i * LD + r], V[i * LD + r], a);
          gs += GR[r];
        }
        a = (a + gs / w.diag[i]) * sigmoid_f(__ldg(m.d_params + o_dg + i));
        dst = gp + o_dg + i;
      }
    } else {
      const int i = t - D * D;
      for (int r = 0; r < TM; ++r) a += dZ[i * LD + r];
      dst = gp + o_bi + i;
    }
    grad_out(dst, a, accumulate);
  }
  consumer_sync();
  for (int t = threadIdx.x; t < D * TM; t += kConsumerThreads) {
    const int j = t / TM, r = t % TM;
    float a = 0.f;
    for (int i = 0; i <= j; ++i) a = fmaf(w.U[i * D + j], DY[i * LD + r], a);
    dZ[j * LD + r] = a;
  }
  consumer_sync();
}

template <int TM, int RN, int RK, bool SPILL>
__global__ void __launch_bounds__(kThreads, 1)
nsf_vjp_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_rows rows,
               const float* __restrict__ gout, float g_const, float* __restrict__ logp,
               float* __restrict__ gpart, float* __restrict__ ginput, float* __restrict__ gcond,
               float* __restrict__ loss_acc, float* __restrict__ scratch) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const NsfSmem L = nsf_smem_layout(m, TM, true);
  WPipe pipe = make_pipe(m, sm, L);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  const bool need_dctx = (gcond != nullptr);
  // Activation spill: with a scratch buffer (one slab per CTA and layer, L2-resident) the forward
  // sweep keeps every conditioner intermediate and the spline parameters of each layer, and the
  // backward sweep reads them back instead of recomputing the conditioner (a quarter of the GEMM
  // work of this kernel).  Without it (scratch == nullptr) the layer is recomputed.
  constexpr bool spill = SPILL;      // compile-time: the unused path costs instruction cache
  const int sv_rows = (4 * m.NB + 1) * m.Hp;           // HS | A1S | T2S | SS, contiguous
  const int prm_rows = m.TRmax * m.PR;
  const int slab = (sv_rows + prm_rows) * LD;          // floats per (CTA, layer)
  const float* __restrict__ P = m.d_params;
  const int Hp = m.Hp, Cp = m.Cp, K0p = m.Cp + m.IDp;

  // ------------------------------------------------------------------ producer
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        for (int l = 0; l < m.T; ++l) {
          const NsfLayerView v = layer_view(m, l);
          float* hf = cond_forward<kProducer, TM, RN, true>(m, v, pipe, sm, L);
          spline_forward<kProducer, TM, RN, false>(m, v, pipe, sm, L, hf);
        }
        for (int l = m.T - 1; l >= 0; --l) {
          const NsfLayerView v = layer_view(m, l);
          if (!spill) {
            float* hf = cond_forward<kProducer, TM, RN, true>(m, v, pipe, sm, L);
            final_layer<kProducer, TM, RN>(m, v, pipe, sm, L, hf);
          }
          auto noop2 = [](int, int, float(&)[RK][4], bool) {};
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_L_WF), v.n_tr * m.PR, Hp,
                                      m.nf_chunk * m.PR, nullptr, Hp, noop2);
          if (m.cond_mlp) {
            for (int k = m.NB; k >= 1; --k)
              dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_L_BLK0), Hp, Hp, m.rpc1, nullptr, Hp, noop2);
          } else
          for (int b = m.NB - 1; b >= 0; --b) {
            const int* BT = v.LT + SBI_L_BLK0 + 6 * b;
            dx_stage<kProducer, TM, RK>(pipe, P + __ldg(BT + 2), Hp, Hp, m.rpc1, nullptr, Hp, noop2);
            if (need_dctx)
              dx_stage<kProducer, TM, RK>(pipe, P + __ldg(BT + 4), Hp, Cp, m.rpc1, nullptr, Cp, noop2);
            dx_stage<kProducer, TM, RK>(pipe, P + __ldg(BT + 0), Hp, Hp, m.rpc1, nullptr, Hp, noop2);
          }
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(v.LT + SBI_L_W0), Hp, K0p, m.rpc0, nullptr, K0p,
                                      noop2);
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers
  const RqsConst rc = rqs_const(m);
  const bool mog = m.head == SBI_NSF_MOG;
  const float ld_const = mog ? m.ld_zscore
                             : lu_logdet_total(m, sm + L.PRM) + m.ld_zscore - 0.5f * (float)m.D * 1.8378770664093453f;
  float* gp = gpart + (size_t)blockIdx.x * m.n_params;
  float* Z = sm + L.Z;
  float* U = sm + L.U;
  float* dZ = sm + L.dZ;
  float* dU = sm + L.dU;
  float* dH = sm + L.dH;
  float* dT = sm + L.dT;
  float* dG = sm + L.dG;
  float* dA = sm + L.A1;        // free in SAVE mode
  float* A0 = sm + L.A0;
  float* PRM = sm + L.PRM;
  float* dPRM = sm + L.dPRM;
  float* GR = sm + L.GR;
  float* dCTX = sm + L.dCTX;
  const float* __restrict__ st = m.d_stats;

  for (int e = threadIdx.x; e < m.TRmax * m.PR * LD; e += kConsumerThreads) dPRM[e] = 0.f;

  int iter = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const bool accum = iter > 0;
    const int64_t row0 = tile * TM;
    load_tile<TM>(m, rows, row0, sm, L, false);
    // ---------------- forward sweep (keeps only layer inputs z_l and coupling outputs v_l)
    for (int l = 0; l < m.T; ++l) {
      const NsfLayerView v = layer_view(m, l);
      for (int e = threadIdx.x; e < m.Dp * LD; e += kConsumerThreads)
        sm[L.ZS + l * m.Dp * LD + e] = Z[e];
      lu_prepare(m, v, sm, L);
      gather_identity<TM>(m, v, Z, U);
      float* hf = cond_forward<kConsumer, TM, RN, true>(m, v, pipe, sm, L);
      spline_forward<kConsumer, TM, RN, false>(m, v, pipe, sm, L, hf);
      if (spill) {
        // (spline_forward ended with a barrier; nothing below touches these regions before the
        // barriers inside lu_forward, so every thread's part is out before they are rewritten)
        float4* dst = reinterpret_cast<float4*>(scratch + ((size_t)blockIdx.x * m.T + l) * slab);
        const float4* s0 = reinterpret_cast<const float4*>(sm + L.HS);
        const float4* s1 = reinterpret_cast<const float4*>(sm + L.PRM);
        const int n0 = sv_rows * LD / 4, n1 = prm_rows * LD / 4;
        for (int e = threadIdx.x; e < n0; e += kConsumerThreads) __stcg(dst + e, s0[e]);
        for (int e = threadIdx.x; e < n1; e += kConsumerThreads) __stcg(dst + n0 + e, s1[e]);
      }
      fold_ldf<TM>(v, sm, L);
      for (int e = threadIdx.x; e < m.Dp * LD; e += kConsumerThreads)
        sm[L.VS + l * m.Dp * LD + e] = Z[e];
      lu_forward<TM>(m, v, sm, L);
    }
    consumer_sync();
    // ---------------- log-prob, upstream gradient, loss statistics
    {
      float nll = 0.f, bad = 0.f;
      for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
        float g = 0.f;
        if (row0 + r < rows.R) {
          float ss = 0.f;
          if (!mog)
            for (int d = 0; d < m.D; ++d) ss = fmaf(Z[d * LD + r], Z[d * LD + r], ss);
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
    // d(sum g logp)/dz_T = -g z_T
    for (int e = threadIdx.x; e < m.Dp * TM; e += kConsumerThreads) {
      const int d = e / TM, r = e % TM;
      dZ[d * LD + r] = mog ? 0.f : -GR[r] * Z[d * LD + r];
    }
    if (need_dctx)
      for (int e = threadIdx.x; e < Cp * LD; e += kConsumerThreads) dCTX[e] = 0.f;
    consumer_sync();

    // ---------------- backward sweep
    for (int l = m.T - 1; l >= 0; --l) {
      const NsfLayerView v = layer_view(m, l);
      const float* ZSl = sm + L.ZS + l * m.Dp * LD;
      const float* VSl = sm + L.VS + l * m.Dp * LD;
      lu_prepare(m, v, sm, L);
      consumer_sync();
      lu_backward<TM>(m, v, sm, L, VSl, gp, accum);
      // the conditioner's intermediates of this layer: read back, or recomputed from the saved
      // layer input
      gather_identity<TM>(m, v, ZSl, U);
      float* hf;
      if (spill) {
        const float4* src = reinterpret_cast<const float4*>(scratch + ((size_t)blockIdx.x * m.T + l) * slab);
        float4* d0 = reinterpret_cast<float4*>(sm + L.HS);
        float4* d1 = reinterpret_cast<float4*>(sm + L.PRM);
        const int n0 = sv_rows * LD / 4, n1 = prm_rows * LD / 4;
        for (int e = threadIdx.x; e < n0; e += kConsumerThreads) d0[e] = __ldcg(src + e);
        for (int e = threadIdx.x; e < n1; e += kConsumerThreads) d1[e] = __ldcg(src + n0 + e);
        hf = sm + L.HS + m.NB * Hp * LD;
        consumer_sync();
      } else {
        hf = cond_forward<kConsumer, TM, RN, true>(m, v, pipe, sm, L);
      }
      // final layer (all features) -> spline backward -> dW, dH
      {
        const int oWF = __ldg(v.LT + SBI_L_WF), oBF = __ldg(v.LT + SBI_L_BF);
        const int N = v.n_tr * m.PR;
        if (!spill) final_layer<kConsumer, TM, RN>(m, v, pipe, sm, L, hf);
        if (mog) {
          for (int t = threadIdx.x; t < v.n_tr * TM; t += kConsumerThreads) {
            const int f = t / TM, r = t % TM;
            const int j = __ldg(v.trf + f);
            // the dummy feature has no likelihood term; dPRM of its rows stays zero
            dZ[j * LD + r] = j == 0 ? 0.f
                                    : mog_backward(PRM + f * m.PR * LD + r, LD, m.M, m.mog_eps, ZSl[j * LD + r], GR[r],
                                                   dPRM + f * m.PR * LD + r, LD);
          }
        } else {
          for (int t = threadIdx.x; t < v.n_tr * TM; t += kConsumerThreads) {
            const int f = t / TM, r = t % TM;
            const int j = __ldg(v.trf + f);
            const float gx = rqs_backward(PRM + f * m.PR * LD + r, LD, rc, ZSl[j * LD + r],
                                          dZ[j * LD + r], GR[r], dPRM + f * m.PR * LD + r, LD);
            dZ[j * LD + r] = gx;
          }
        }
        consumer_sync();
        gemm_dw<TM>(dPRM, N, hf, m.H, Hp, gp + oWF, gp + oBF, accum);
        dx_stage<kConsumer, TM, RK>(
            pipe, nullptr, N, Hp, m.nf_chunk * m.PR, dPRM, Hp,
            [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
              for (int j = 0; j < RK; ++j) {
                float* p = dH + (k0 + j) * LD + r0;
                float4 o = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                if (!first) {
                  const float4 c = ld4(p);
                  o.x += c.x; o.y += c.y; o.z += c.z; o.w += c.w;
                }
                st4(p, o);
              }
            });
      }
      if (m.cond_mlp) {
        // context-only MLP (1-D flow): dH = grad wrt the last relu output HS[NB]; the hidden layer is shared,
        // so its weight gradient accumulates over its NB applications; ends with dH = grad wrt the
        // pre-activation of the initial layer, which the common code below turns into dW0 / dU
        const int oWh = __ldg(v.LT + SBI_L_BLK0), oBh = __ldg(v.LT + SBI_L_BLK0 + 1);
        for (int k = m.NB; k >= 1; --k) {
          const float* Hk = sm + L.HS + k * Hp * LD;
          const float* Hkm1 = sm + L.HS + (k - 1) * Hp * LD;
          for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
            const int o = (e / TM) * LD + (e % TM);
            dT[o] = Hk[o] > 0.f ? dH[o] : 0.f;
          }
          consumer_sync();
          gemm_dw<TM>(dT, m.H, Hkm1, m.H, Hp, gp + oWh, gp + oBh, accum || k < m.NB);
          dx_stage<kConsumer, TM, RK>(
              pipe, nullptr, Hp, Hp, m.rpc1, dT, Hp, [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                for (int j = 0; j < RK; ++j) {
                  float* p = dH + (k0 + j) * LD + r0;
                  float4 o4 = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                  if (!first) {
                    const float4 c = ld4(p);
                    o4.x += c.x; o4.y += c.y; o4.z += c.z; o4.w += c.w;
                  }
                  st4(p, o4);
                }
              });
        }
        const float* H0 = sm + L.HS;
        for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
          const int o = (e / TM) * LD + (e % TM);
          dH[o] = H0[o] > 0.f ? dH[o] : 0.f;
        }
        consumer_sync();
      } else
      // residual blocks, last to first.  dH = grad wrt HS[b+1]
      for (int b = m.NB - 1; b >= 0; --b) {
        const int* BT = v.LT + SBI_L_BLK0 + 6 * b;
        const float* Hb = sm + L.HS + b * Hp * LD;
        const float* A1b = sm + L.A1S + b * Hp * LD;
        const float* T2b = sm + L.T2S + b * Hp * LD;
        const float* Sb = sm + L.SS + b * Hp * LD;
        for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
          const int n = e / TM, r = e % TM, o = n * LD + r;
          const float s = Sb[o], dh = dH[o];
          dT[o] = dh * s;
          dG[o] = dh * T2b[o] * s * (1.f - s);
          A0[o] = relu_f(Hb[o]);
        }
        consumer_sync();
        gemm_dw<TM>(dT, m.H, A1b, m.H, Hp, gp + __ldg(BT + 2), gp + __ldg(BT + 3), accum);
        gemm_dw<TM>(dG, m.H, U, m.C, Cp, gp + __ldg(BT + 4), gp + __ldg(BT + 5), accum);
        dx_stage<kConsumer, TM, RK>(
            pipe, nullptr, Hp, Hp, m.rpc1, dT, Hp, [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
              for (int j = 0; j < RK; ++j) {
                const int o = (k0 + j) * LD + r0;
                const float4 a1 = ld4(A1b + o);
                float4 val = make_float4(a1.x > 0.f ? acc[j][0] : 0.f, a1.y > 0.f ? acc[j][1] : 0.f,
                                         a1.z > 0.f ? acc[j][2] : 0.f, a1.w > 0.f ? acc[j][3] : 0.f);
                if (!first) {
                  const float4 c = ld4(dA + o);
                  val.x += c.x; val.y += c.y; val.z += c.z; val.w += c.w;
                }
                st4(dA + o, val);
              }
            });
        if (need_dctx) {
          dx_stage<kConsumer, TM, RK>(
              pipe, nullptr, Hp, Cp, m.rpc1, dG, Cp, [&](int k0, int r0, float(&acc)[RK][4], bool) {
#pragma unroll
                for (int j = 0; j < RK; ++j) {
                  if (k0 + j >= Cp) continue;
                  float* p = dCTX + (k0 + j) * LD + r0;
                  const float4 c = ld4(p);
                  st4(p, make_float4(c.x + acc[j][0], c.y + acc[j][1], c.z + acc[j][2],
                                     c.w + acc[j][3]));
                }
              });
        }
        gemm_dw<TM>(dA, m.H, A0, m.H, Hp, gp + __ldg(BT + 0), gp + __ldg(BT + 1), accum);
        dx_stage<kConsumer, TM, RK>(
            pipe, nullptr, Hp, Hp, m.rpc1, dA, Hp, [&](int k0, int r0, float(&acc)[RK][4], bool) {
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
      // initial layer
      gemm_dw<TM>(dH, m.H, U, Cp + v.n_id, K0p, gp + __ldg(v.LT + SBI_L_W0),
                  gp + __ldg(v.LT + SBI_L_B0), accum);
      if (mog) {   // context_layer.bias enters the same sum as initial_layer.bias: same gradient
        float* gbc = gp + __ldg(v.LT + SBI_L_BC0);
        for (int n = threadIdx.x; n < m.H; n += kConsumerThreads) {
          float a = 0.f;
          for (int r = 0; r < TM; ++r) a += dH[n * LD + r];
          grad_out(gbc + n, a, accum);
        }
      }
      dx_stage<kConsumer, TM, RK>(
          pipe, nullptr, Hp, K0p, m.rpc0, dH, K0p, [&](int k0, int r0, float(&acc)[RK][4], bool first) {
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
      for (int e = threadIdx.x; e < v.n_id * TM; e += kConsumerThreads) {
        const int i = e / TM, r = e % TM;
        dZ[__ldg(v.idf + i) * LD + r] += dU[(Cp + i) * LD + r];
      }
      if (need_dctx)
        for (int e = threadIdx.x; e < m.C * TM; e += kConsumerThreads) {
          const int c = e / TM, r = e % TM;
          dCTX[c * LD + r] += dU[c * LD + r];
        }
      consumer_sync();
    }
    // ---------------- input / condition gradients (through the z-scoring)
    if (ginput != nullptr)
      for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
        const int r = e / m.D, d = e % m.D;
        if (row0 + r < rows.R) ginput[(row0 + r) * m.D + d] = dZ[d * LD + r] * __ldg(st + m.Dp + d);
      }
    if (need_dctx)
      for (int e = threadIdx.x; e < TM * m.C; e += kConsumerThreads) {
        const int r = e / m.C, c = e % m.C;
        if (row0 + r < rows.R)
          gcond[(row0 + r) * m.C + c] = dCTX[c * LD + r] / __ldg(st + 2 * m.Dp + Cp + c);
      }
    consumer_sync();
  }
}

// =================================================================================================
// `made` sampling: D sequential passes of the masked conditioner (MixtureOfGaussiansMADE.sample,
// oracle/nflows_port/nn/nde/made.py); feature f is drawn from its mixture given features < f.
// =================================================================================================
template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 2)
made_sample_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_rows rows,
                   const float* __restrict__ uniform, float* __restrict__ out) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const NsfSmem L = nsf_smem_layout(m, TM, false);
  WPipe pipe = make_pipe(m, sm, L);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  const NsfLayerView v = layer_view(m, 0);
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        for (int f = 0; f < m.D; ++f) {
          float* hf = cond_forward<kProducer, TM, RN, false>(m, v, pipe, sm, L);
          final_layer<kProducer, TM, RN>(m, v, pipe, sm, L, hf);
        }
    return;
  }
  const float* __restrict__ st = m.d_stats;
  float* Z = sm + L.Z;
  float* NZ = sm + L.Y;       // the normal draws of the tile (Y / Y2 are free: no LU here)
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    load_tile<TM>(m, rows, row0, sm, L, true);          // Z = normal draws (raw), U[0:C] = context
    for (int e = threadIdx.x; e < m.Dp * LD; e += kConsumerThreads) { NZ[e] = Z[e]; Z[e] = 0.f; }
    consumer_sync();
    for (int f = 0; f < m.D; ++f) {
      gather_identity<TM>(m, v, Z, sm + L.U);
      float* hf = cond_forward<kConsumer, TM, RN, false>(m, v, pipe, sm, L);
      final_layer<kConsumer, TM, RN>(m, v, pipe, sm, L, hf);
      consumer_sync();
      for (int r = threadIdx.x; r < TM; r += kConsumerThreads) {
        const int64_t gr = row0 + r;
        const float u = gr < rows.R ? __ldg(uniform + gr * m.D + f) : 0.f;
        Z[f * LD + r] = mog_sample(sm + L.PRM + f * m.PR * LD + r, LD, m.M, m.mog_eps, u, NZ[f * LD + r]);
      }
      consumer_sync();
    }
    for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
      const int r = e / m.D, d = e % m.D;
      if (row0 + r < rows.R)
        out[(row0 + r) * m.D + d] = (Z[d * LD + r] - __ldg(st + d)) / __ldg(st + m.Dp + d);
    }
    consumer_sync();
  }
}

}  // namespace sbi

// =================================================================================================
// C ABI
// =================================================================================================
using namespace sbi;

static int check_model(const sbi_nsf_model* m) {
  if (!m || !m->d_params || !m->d_layer_tab || !m->d_feat_tab || !m->d_stats) return SBI_EINVAL;
  if (m->D < 1 || m->C < 1 || m->H < 1 || m->T < 1 || m->KB < 2 || m->NB < 0) return SBI_EINVAL;
  if (m->KB > kRqsMaxBins) return SBI_EINVAL;
  if (m->NB > SBI_NSF_MAX_BLOCKS) return SBI_EINVAL;
  if (m->Dp != round4(m->D) || m->Cp != round4(m->C) || m->Hp != round4(m->H)) return SBI_EINVAL;
  if (m->head != SBI_NSF_SPLINE && m->head != SBI_NSF_MOG) return SBI_EINVAL;
  if (m->cond_mlp && (m->head != SBI_NSF_SPLINE || m->TRmax * m->PR > m->Hp)) return SBI_EINVAL;
  if (m->head == SBI_NSF_MOG && (m->M < 1 || m->M > kMogMax || m->T != 1 || !(m->mog_eps > 0.f))) return SBI_EINVAL;
  if (m->PR != (m->head == SBI_NSF_MOG ? round4(3 * m->M) : round4(3 * m->KB - 1)) || (m->IDp & 3) || m->nf_chunk < 1)
    return SBI_EINVAL;
  if (!ring_ok({{m->rpc0, m->Cp + m->IDp}, {m->rpc1, m->Hp}, {m->rpc2, m->Hp + m->Cp}, {m->nf_chunk * m->PR, m->Hp}},
               m->nbuf, m->wcap))
    return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_abi_version(void) { return SBI_B200_ABI_VERSION; }

extern "C" int sbi_b200_device_ok(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n < 1) return 0;
  cudaDeviceProp p;
  if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) return 0;
  return (p.major == 9 && p.minor == 0) ? 1 : 0;
}

extern "C" int sbi_b200_nsf_logprob(const sbi_nsf_model* m, const sbi_rows* rows, float* d_logp,
                                    float* d_noise, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = check_model(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_logp) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int bytes64 = nsf_smem_layout(*m, 64, false).total_bytes;
  if (use_64_rows(rows->R, bytes64))
    return launch(nsf_logprob_kernel<64, 4>, tile_grid(rows->R, 64, per_sm_110k(bytes64)), kThreads,
                  bytes64, s, *m, *rows, d_logp, d_noise);
  const int bytes = nsf_smem_layout(*m, 32, false).total_bytes;
  const int per_sm = std::max(1, std::min(2, kMaxSmemBytes / (bytes + 1024)));
  return launch(nsf_logprob_kernel<32, 2>, tile_grid(rows->R, 32, per_sm), kThreads, bytes, s, *m, *rows, d_logp,
                d_noise);
}

extern "C" int sbi_b200_made_sample(const sbi_nsf_model* m, const sbi_rows* rows, const float* d_uniform,
                                    float* d_out, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = check_model(m);
  if (rc) return rc;
  if (m->head != SBI_NSF_MOG) return SBI_EINVAL;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_uniform || !d_out) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  const int bytes = nsf_smem_layout(*m, 32, false).total_bytes;
  return launch(made_sample_kernel<32, 2>, tile_grid(rows->R, 32, per_sm_110k(bytes)), kThreads, bytes,
                (cudaStream_t)stream, *m, *rows, d_uniform, d_out);
}

extern "C" int sbi_b200_nsf_inverse(const sbi_nsf_model* m, const sbi_rows* rows, float* d_out,
                                    float* d_logabsdet, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = check_model(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_out) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  cudaStream_t s = (cudaStream_t)stream;
  const int bytes64 = nsf_smem_layout(*m, 64, false).total_bytes;
  if (use_64_rows(rows->R, bytes64))
    return launch(nsf_inverse_kernel<64, 4>, tile_grid(rows->R, 64, per_sm_110k(bytes64)), kThreads,
                  bytes64, s, *m, *rows, d_out, d_logabsdet);
  const int bytes = nsf_smem_layout(*m, 32, false).total_bytes;
  return launch(nsf_inverse_kernel<32, 2>, tile_grid(rows->R, 32, per_sm_110k(bytes)), kThreads, bytes, s,
                *m, *rows, d_out, d_logabsdet);
}

extern "C" int sbi_b200_nsf_vjp_parts(int64_t R) { return vjp_parts(R, 32); }

// Whether the VJP of `m` runs on 32-row tiles.  Deep conditioners (`made`: five residual blocks) keep too many
// intermediates for a 32-row tile and take 16-row tiles that recompute each layer's conditioner (no spill).
static bool vjp_32_rows(const sbi_nsf_model& m) { return nsf_smem_layout(m, 32, true).total_bytes <= kMaxSmemBytes; }

extern "C" int64_t sbi_b200_nsf_vjp_save_bytes(const sbi_nsf_model* m, int64_t R) {
  if (check_model(m) || R < 1 || !vjp_32_rows(*m)) return 0;
  // the slab nsf_vjp_kernel spills per (CTA, layer): HS | A1S | T2S | SS and the spline parameters
  const int64_t slab = (int64_t)((4 * m->NB + 1) * m->Hp + m->TRmax * m->PR) * Tile<32>::LD;
  return (int64_t)sizeof(float) * slab * m->T * sbi_b200_nsf_vjp_parts(R);
}

extern "C" int sbi_b200_nsf_vjp(const sbi_nsf_model* m, const sbi_rows* rows, const float* d_gout,
                                float g_const, float* d_logp, float* d_gpart, float* d_ginput,
                                float* d_gcond, float* d_loss_acc, float* d_save, int64_t save_bytes,
                                void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = check_model(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 1 || !d_gpart) return SBI_EINVAL;
  if (d_save && save_bytes < sbi_b200_nsf_vjp_save_bytes(m, rows->R)) return SBI_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = sbi_b200_nsf_vjp_parts(rows->R);
  if (!vjp_32_rows(*m)) {
    // every CTA walks its 16-row tiles and accumulates into its slab (the grid keeps the 32-row part count: the
    // caller sized its slabs from sbi_b200_nsf_vjp_parts)
    return launch(nsf_vjp_kernel<16, 2, 2, false>, grid, kThreads, nsf_smem_layout(*m, 16, true).total_bytes, s, *m,
                  *rows, d_gout, g_const, d_logp, d_gpart, d_ginput, d_gcond, d_loss_acc, nullptr);
  }
  auto k = d_save ? nsf_vjp_kernel<32, 2, 2, true> : nsf_vjp_kernel<32, 2, 2, false>;
  return launch(k, grid, kThreads, nsf_smem_layout(*m, 32, true).total_bytes, s, *m, *rows, d_gout, g_const, d_logp,
                d_gpart, d_ginput, d_gcond, d_loss_acc, d_save);
}
