// Flow-matching (FMPE) kernels: the VectorFieldMLP forward (ODE right-hand side) and the fused
// flow-matching loss forward+backward.
//
// Reference: /root/reference/sbi/neural_nets/net_builders/vector_field_nets.py:610-719
//   a = W_i theta_n + b_i ; c = W_c ctx + b_c ; h = gelu( W_m gelu([a ; c]) + b_m )
//   t_emb = W_t [sin(t f_j), cos(t f_j)]_interleaved + b_t
//   L x:  h = LayerNorm( gelu(W_l h + b_l) + t_emb + h )
//   v_out = W_o h + b_o
// and /root/reference/sbi/neural_nets/estimators/flowmatching_estimator.py:120-347:
//   theta_t = (1-t) theta + (t + 1e-3) eps ; mu_t = (1-t) mu_0 ; sd_t = sqrt(((1-t) sd_0)^2 + t^2 + 1e-6)
//   theta_n = (theta_t - mu_t) / sd_t ; target = ((eps - theta) + mu_0) / sqrt(1 + sd_0^2)
//   loss = mean_d (v_out - target)^2 ; forward(): v = v_out * sqrt(1 + sd_0^2) - mu_0.
// Same CTA structure as the other kernels (stages.cuh).  Every activation of the tile is kept
// in shared memory, so the backward is one pass (no recompute); TM = 16 rows for the VJP.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>

#include "stages.cuh"
#include "device.cuh"

namespace sbi {

__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float dgelu_f(float x) {
  return 0.5f * (1.f + erff(x * 0.70710678118654752f)) + x * 0.3989422804014327f * expf(-0.5f * x * x);
}

struct FmSmem {
  int LD;
  int TN, CTX, SC, TGT, ABP, AB, HMP, HS, ZS, TEB, X1, X2, STAT, RED, OUT;
  int dH, dTE;
  int UH, dAB, dHt, dUt, DIV;     // trace mode: normalised LayerNorm inputs per layer, tangent buffers, divergence
  int ring, bar_bytes, total_bytes;
};

// mode 0: evaluation; 1: training (everything the backward needs); 2: exact-trace evaluation (keeps what
// the forward-mode tangents need: pre-activations of every gelu, the normalised LayerNorm inputs and 1/std)
enum { kFmEval = 0, kFmTrain = 1, kFmTrace = 2 };

__host__ __device__ inline FmSmem fm_smem_layout(const sbi_fm_model& m, int TM, int mode) {
  const bool train = mode == kFmTrain, trace = mode == kFmTrace;
  FmSmem L;
  L.LD = TM + 4;
  int rows = 0;
  auto take = [&](int n) { int o = rows * L.LD; rows += n; return o; };
  L.TN = take(m.Dp);
  L.CTX = take(m.Cp);
  L.SC = take(m.TEp);
  L.TGT = take(trace ? 0 : m.Dp);
  L.ABP = take(train || trace ? 2 * m.Hp : 0);
  L.AB = take(2 * m.Hp);
  L.HMP = take(train || trace ? m.Hp : 0);
  L.HS = take((train ? m.NL + 1 : 1) * m.Hp);
  L.ZS = take((train || trace ? m.NL : 1) * m.Hp);
  L.TEB = take(m.Hp);
  L.X1 = take(m.Hp);
  L.X2 = take(train ? m.Hp : 0);
  L.STAT = take(round4(2 * m.NL));
  L.RED = take(32);
  L.OUT = take(m.Dp);
  L.dH = take(train ? m.Hp : 0);
  L.dTE = take(train ? m.Hp : 0);
  L.UH = take(trace ? m.NL * m.Hp : 0);
  L.dAB = take(trace ? 2 * m.Hp : 0);
  L.dHt = take(trace ? m.Hp : 0);
  L.dUt = take(trace ? m.Hp : 0);
  L.DIV = take(trace ? 1 : 0);
  int fl = rows * L.LD;
  fl = (fl + 31) & ~31;
  L.ring = fl;
  fl += m.nbuf * m.wcap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + 2 * m.nbuf * 8 + 16;
  return L;
}

// per-row reduction over H features: every consumer thread (r, part) sums its features into RED,
// then reads the `parts` partials of its row.  Returns the row total to all threads of the row.
template <int TM, class F>
__device__ __forceinline__ float row_reduce(int H, float* RED, F&& f) {
  constexpr int LD = Tile<TM>::LD;
  constexpr int PARTS = kConsumerThreads / TM;
  const int r = threadIdx.x % TM, p = threadIdx.x / TM;
  float a = 0.f;
  for (int k = p; k < H; k += PARTS) a += f(k, r);
  RED[p * LD + r] = a;
  consumer_sync();
  float t = 0.f;
#pragma unroll 4
  for (int q = 0; q < PARTS; ++q) t += RED[q * LD + r];
  consumer_sync();
  return t;
}

// tile prologue: theta_n, ctx, sin/cos features, regression target
template <int TM, bool TRAIN>
__device__ __forceinline__ void fm_load(const sbi_fm_model& m, const sbi_rows& rows, const float* time,
                                        int time_shared, const float* eps, int64_t row0, float* sm,
                                        const FmSmem& L) {
  constexpr int LD = Tile<TM>::LD;
  const float* __restrict__ st = m.d_stats;
  const int D = m.D, Dp = m.Dp, C = m.C, Cp = m.Cp;
  float* TN = sm + L.TN;
  float* TGT = sm + L.TGT;
  for (int e = threadIdx.x; e < TM * Dp; e += kConsumerThreads) {
    const int r = e / Dp, d = e % Dp;
    const int64_t gr = row0 + r;
    float tn = 0.f, tg = 0.f;
    if (d < D && gr < rows.R) {
      const int64_t src = rows.d_index ? __ldg(rows.d_index + gr) : gr;
      const float th = __ldg(rows.d_input + src * D + d);
      const float t = __ldg(time + (time_shared ? 0 : gr));
      const float mu0 = __ldg(st + d), sd0 = __ldg(st + Dp + d);
      if (m.raw) {            // bare network (score estimators): the caller prepared the network input
        tn = th;
      } else {
        float tht = th;
        if (TRAIN) {
          const float e1 = __ldg(eps + gr * D + d);
          tht = (1.f - t) * th + (t + m.noise_scale) * e1;
          tg = ((e1 - th) + mu0) / sqrtf(1.f + sd0 * sd0);
        }
        const float a = (1.f - t) * sd0;
        const float sdt = sqrtf(a * a + t * t + 1e-6f);
        tn = (tht - (1.f - t) * mu0) / sdt;
      }
    }
    TN[d * LD + r] = tn;
    if (TRAIN) TGT[d * LD + r] = tg;
  }
  float* CTX = sm + L.CTX;
  for (int e = threadIdx.x; e < TM * Cp; e += kConsumerThreads) {
    const int r = e / Cp, c = e % Cp;
    const int64_t gr = row0 + r;
    float val = 0.f;
    if (c < C && gr < rows.R) {
      const int64_t src = rows.cond_shared ? 0 : (rows.d_index ? __ldg(rows.d_index + gr) : gr);
      val = (__ldg(rows.d_cond + src * C + c) - __ldg(st + 2 * Dp + c)) / __ldg(st + 2 * Dp + Cp + c);
    }
    CTX[c * LD + r] = val;
  }
  float* SC = sm + L.SC;
  const float* freq = st + 2 * Dp + 2 * Cp;
  for (int e = threadIdx.x; e < TM * m.TEp; e += kConsumerThreads) {
    const int r = e / m.TEp, k = e % m.TEp;
    const int64_t gr = row0 + r;
    float val = 0.f;
    if (k < m.TE && gr < rows.R) {
      const float t = __ldg(time + (time_shared ? 0 : gr));
      const float arg = t * __ldg(freq + (k >> 1));
      val = (k & 1) ? cosf(arg) : sinf(arg);
    }
    SC[k * LD + r] = val;
  }
  consumer_sync();
}

// network forward.  MODE kFmTrain keeps pre-activations / per-layer states for the backward, kFmTrace what
// the forward-mode tangents of the exact trace need (fm_trace_kernel).
template <Role R, int TM, int RN, int MODE>
__device__ __forceinline__ void fm_net_forward(const sbi_fm_model& m, WPipe& pipe, float* sm, const FmSmem& L) {
  constexpr int LD = Tile<TM>::LD;
  constexpr bool TRAIN = MODE == kFmTrain;
  constexpr bool KEEP = MODE != kFmEval;       // pre-activations are kept
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const int Hp = m.Hp, H = m.H;
  float* AB = sm + L.AB;
  float* ABP = sm + L.ABP;
  {   // a = gelu(W_i theta_n + b_i), c = gelu(W_c ctx + b_c)
    const float* bi = P + __ldg(T + SBI_F_BI);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_F_WI), Hp, m.Dp, m.rpc_i, sm + L.TN,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float b = __ldg(bi + n);
                             const float4 z = make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b);
                             if (KEEP) st4(ABP + n * LD + r0, z);
                             st4(AB + n * LD + r0, make_float4(gelu_f(z.x), gelu_f(z.y), gelu_f(z.z), gelu_f(z.w)));
                           }
                         });
    const float* bc = P + __ldg(T + SBI_F_BC);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_F_WC), Hp, m.Cp, m.rpc_c, sm + L.CTX,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = Hp + n0 + g + i * ng;
                             const float b = __ldg(bc + n - Hp);
                             const float4 z = make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b);
                             if (KEEP) st4(ABP + n * LD + r0, z);
                             st4(AB + n * LD + r0, make_float4(gelu_f(z.x), gelu_f(z.y), gelu_f(z.z), gelu_f(z.w)));
                           }
                         });
  }
  float* Hcur = sm + L.HS;
  {   // h0 = gelu(W_m [a ; c] + b_m)
    const float* bm = P + __ldg(T + SBI_F_BM);
    float* HMP = sm + L.HMP;
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_F_WM), Hp, 2 * Hp, m.rpc_m, AB,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float b = __ldg(bm + n);
                             const float4 z = make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b);
                             if (KEEP) st4(HMP + n * LD + r0, z);
                             st4(Hcur + n * LD + r0, make_float4(gelu_f(z.x), gelu_f(z.y), gelu_f(z.z), gelu_f(z.w)));
                           }
                         });
  }
  float* TEB = sm + L.TEB;
  {   // t_emb = W_t sc + b_t
    const float* bt = P + __ldg(T + SBI_F_BT);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_F_WT), Hp, m.TEp, m.rpc_t, sm + L.SC,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float b = __ldg(bt + n);
                             st4(TEB + n * LD + r0, make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b));
                           }
                         });
  }
  float* U = sm + L.X1;
  for (int l = 0; l < m.NL; ++l) {
    const int* LT = T + SBI_F_LAYER0 + 4 * l;
    float* Hin = Hcur;
    float* Hout = TRAIN ? Hin + Hp * LD : Hin;
    float* Z = sm + L.ZS + (KEEP ? l : 0) * Hp * LD;
    const float* bl = P + __ldg(LT + 1);
    fwd_stage<R, TM, RN>(pipe, P + __ldg(LT + 0), Hp, Hp, m.rpc_h, Hin,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float b = __ldg(bl + n);
                             const float4 z = make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b);
                             const float4 te = ld4(TEB + n * LD + r0);
                             const float4 ho = ld4(Hin + n * LD + r0);
                             if (KEEP) st4(Z + n * LD + r0, z);
                             st4(U + n * LD + r0, make_float4(gelu_f(z.x) + te.x + ho.x, gelu_f(z.y) + te.y + ho.y,
                                                              gelu_f(z.z) + te.z + ho.z, gelu_f(z.w) + te.w + ho.w));
                           }
                         });
    if (R == kConsumer) {   // LayerNorm over the H features of every row (two-pass, biased variance)
      float* RED = sm + L.RED;
      const float mean = row_reduce<TM>(H, RED, [&](int k, int r) { return U[k * LD + r]; }) / (float)H;
      const float var = row_reduce<TM>(H, RED, [&](int k, int r) {
        const float d = U[k * LD + r] - mean;
        return d * d;
      }) / (float)H;
      const float rstd = rsqrtf(var + m.ln_eps);
      const int r = threadIdx.x % TM, p = threadIdx.x / TM;
      constexpr int PARTS = kConsumerThreads / TM;
      const float* ga = P + __ldg(LT + 2);
      const float* be = P + __ldg(LT + 3);
      for (int k = p; k < Hp; k += PARTS) {
        const float uh = k < H ? (U[k * LD + r] - mean) * rstd : 0.f;
        Hout[k * LD + r] = k < H ? uh * __ldg(ga + k) + __ldg(be + k) : 0.f;
        if (MODE == kFmTrace) sm[L.UH + (l * Hp + k) * LD + r] = uh;
      }
      if (KEEP && p == 0) {
        sm[L.STAT + (2 * l) * LD + r] = mean;
        sm[L.STAT + (2 * l + 1) * LD + r] = rstd;
      }
      consumer_sync();
    }
    Hcur = Hout;
  }
  {   // v_out = W_o h + b_o
    const float* bo = P + __ldg(T + SBI_F_BO);
    float* OUT = sm + L.OUT;
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_F_WO), m.Dp, Hp, m.rpc_o, Hcur,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int i = 0; i < RN; ++i) {
                             const int n = n0 + g + i * ng;
                             const float b = __ldg(bo + n);
                             st4(OUT + n * LD + r0, make_float4(acc[i][0] + b, acc[i][1] + b, acc[i][2] + b, acc[i][3] + b));
                           }
                         });
  }
}

template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 1)
fm_forward_kernel(const __grid_constant__ sbi_fm_model m, const __grid_constant__ sbi_rows rows,
                  const float* __restrict__ time, int time_shared, float* __restrict__ v) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const FmSmem L = fm_smem_layout(m, TM, kFmEval);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
        fm_net_forward<kProducer, TM, RN, kFmEval>(m, pipe, sm, L);
    return;
  }
  const float* __restrict__ st = m.d_stats;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    fm_load<TM, false>(m, rows, time, time_shared, nullptr, row0, sm, L);
    fm_net_forward<kConsumer, TM, RN, kFmEval>(m, pipe, sm, L);
    for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
      const int r = e / m.D, d = e % m.D;
      if (row0 + r < rows.R) {
        const float sd0 = __ldg(st + m.Dp + d);
        v[(row0 + r) * m.D + d] = m.raw ? sm[L.OUT + d * LD + r]
                                          : sm[L.OUT + d * LD + r] * sqrtf(1.f + sd0 * sd0) - __ldg(st + d);
      }
    }
    consumer_sync();
  }
}

// =================================================================================================
// v(theta, t; x) AND its exact divergence  sum_i d v_i / d theta_i  (the integrand of the neural-ODE
// log-probability: zuko FreeFormJacobianTransform(exact=True) computes the same diagonal with D reverse-mode
// passes through autograd, /root/reference/sbi/samplers/ode_solvers/zuko_ode.py:80-124,
// /root/reference/sbi/inference/potentials/vector_field_potential.py:145-212).  Here: one forward that keeps
// every gelu pre-activation and the normalised LayerNorm inputs in shared memory, then D forward-mode
// tangents e_i through the same linears (the time embedding and the condition branch do not depend on
// theta):   d a = gelu'(.) W_i[:, i] / sd_t,i  ->  W_m  ->  NL x [ gelu'(z) (W_l dh) + dh -> LayerNorm tangent ]
// -> row i of W_o.  Tangent i only needs output i, so the last linear is one dot product per row.
template <Role R, int TM, int RN>
__device__ __forceinline__ void fm_tangent_pass(const sbi_fm_model& m, WPipe& pipe, float* sm, const FmSmem& L,
                                                int i, const float* inv_sdt /* [TM] */) {
  constexpr int LD = Tile<TM>::LD;
  constexpr int PARTS = kConsumerThreads / TM;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const int Hp = m.Hp, H = m.H;
  float* dAB = sm + L.dAB;
  float* dH = sm + L.dHt;
  float* dU = sm + L.dUt;
  if (R == kConsumer) {
    const float* wi = P + __ldg(T + SBI_F_WI);
    const float* ABP = sm + L.ABP;
    for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
      const int n = e / TM, r = e % TM;
      dAB[n * LD + r] = n < H ? dgelu_f(ABP[n * LD + r]) * __ldg(wi + n * m.Dp + i) * inv_sdt[r] : 0.f;
    }
    consumer_sync();
  }
  {
    const float* HMP = sm + L.HMP;
    fwd_stage<R, TM, RN>(pipe, P + __ldg(T + SBI_F_WM), Hp, 2 * Hp, m.rpc_m, dAB,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int q = 0; q < RN; ++q) {
                             const int n = n0 + g + q * ng;
                             const float4 z = ld4(HMP + n * LD + r0);
                             st4(dH + n * LD + r0, make_float4(dgelu_f(z.x) * acc[q][0], dgelu_f(z.y) * acc[q][1],
                                                               dgelu_f(z.z) * acc[q][2], dgelu_f(z.w) * acc[q][3]));
                           }
                         });
  }
  for (int l = 0; l < m.NL; ++l) {
    const int* LT = T + SBI_F_LAYER0 + 4 * l;
    const float* Z = sm + L.ZS + l * Hp * LD;
    fwd_stage<R, TM, RN>(pipe, P + __ldg(LT + 0), Hp, Hp, m.rpc_h, dH,
                         [&](int n0, int g, int ng, int r0, float(&acc)[RN][4]) {
#pragma unroll
                           for (int q = 0; q < RN; ++q) {
                             const int n = n0 + g + q * ng;
                             const float4 z = ld4(Z + n * LD + r0);
                             const float4 h = ld4(dH + n * LD + r0);
                             st4(dU + n * LD + r0, make_float4(fmaf(dgelu_f(z.x), acc[q][0], h.x), fmaf(dgelu_f(z.y), acc[q][1], h.y),
                                                               fmaf(dgelu_f(z.z), acc[q][2], h.z), fmaf(dgelu_f(z.w), acc[q][3], h.w)));
                           }
                         });
    if (R == kConsumer) {   // d LayerNorm(u) = gamma / std * (du - mean(du) - u_hat mean(u_hat du))
      float* RED = sm + L.RED;
      const float* UH = sm + L.UH + l * Hp * LD;
      const float m1 = row_reduce<TM>(H, RED, [&](int k, int r) { return dU[k * LD + r]; }) / (float)H;
      const float m2 = row_reduce<TM>(H, RED, [&](int k, int r) { return UH[k * LD + r] * dU[k * LD + r]; }) / (float)H;
      const int r = threadIdx.x % TM, p = threadIdx.x / TM;
      const float rstd = sm[L.STAT + (2 * l + 1) * LD + r];
      const float* ga = P + __ldg(LT + 2);
      for (int k = p; k < Hp; k += PARTS)
        dH[k * LD + r] = k < H ? __ldg(ga + k) * rstd * (dU[k * LD + r] - m1 - UH[k * LD + r] * m2) : 0.f;
      consumer_sync();
    }
  }
  if (R == kConsumer) {
    float* RED = sm + L.RED;
    const float* wo = P + __ldg(T + SBI_F_WO) + (size_t)i * Hp;
    const float dv = row_reduce<TM>(H, RED, [&](int k, int r) { return __ldg(wo + k) * dH[k * LD + r]; });
    if (threadIdx.x < TM) {
      const float sd0 = __ldg(m.d_stats + m.Dp + i);
      sm[L.DIV + threadIdx.x] += dv * (m.raw ? 1.f : sqrtf(1.f + sd0 * sd0));
    }
    consumer_sync();
  }
}

template <int TM, int RN>
__global__ void __launch_bounds__(kThreads, 1)
fm_trace_kernel(const __grid_constant__ sbi_fm_model m, const __grid_constant__ sbi_rows rows,
                const float* __restrict__ time, int time_shared, float* __restrict__ v,
                float* __restrict__ div) {
  constexpr int LD = Tile<TM>::LD;
  extern __shared__ __align__(128) float sm[];
  const FmSmem L = fm_smem_layout(m, TM, kFmTrace);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads)
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        fm_net_forward<kProducer, TM, RN, kFmTrace>(m, pipe, sm, L);
        for (int i = 0; i < m.D; ++i) fm_tangent_pass<kProducer, TM, RN>(m, pipe, sm, L, i, nullptr);
      }
    return;
  }
  const float* __restrict__ st = m.d_stats;
  __shared__ float s_inv[TM];
  // the condition half of the merge layer's input never carries a tangent
  for (int e = threadIdx.x; e < m.Hp * LD; e += kConsumerThreads) sm[L.dAB + m.Hp * LD + e] = 0.f;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t row0 = tile * TM;
    fm_load<TM, false>(m, rows, time, time_shared, nullptr, row0, sm, L);
    fm_net_forward<kConsumer, TM, RN, kFmTrace>(m, pipe, sm, L);
    if (v != nullptr)
      for (int e = threadIdx.x; e < TM * m.D; e += kConsumerThreads) {
        const int r = e / m.D, d = e % m.D;
        if (row0 + r < rows.R) {
          const float sd0 = __ldg(st + m.Dp + d);
          v[(row0 + r) * m.D + d] = m.raw ? sm[L.OUT + d * LD + r]
                                          : sm[L.OUT + d * LD + r] * sqrtf(1.f + sd0 * sd0) - __ldg(st + d);
        }
      }
    if (threadIdx.x < TM) sm[L.DIV + threadIdx.x] = 0.f;
    for (int i = 0; i < m.D; ++i) {
      if (threadIdx.x < TM) {       // 1 / sd_t,i of the row (fm_load's standardisation)
        const int64_t gr = row0 + threadIdx.x;
        float inv = 0.f;
        if (gr < rows.R) {
          const float t = __ldg(time + (time_shared ? 0 : gr));
          const float a = (1.f - t) * __ldg(st + m.Dp + i);
          inv = m.raw ? 1.f : rsqrtf(a * a + t * t + 1e-6f);
        }
        s_inv[threadIdx.x] = inv;
      }
      consumer_sync();
      fm_tangent_pass<kConsumer, TM, RN>(m, pipe, sm, L, i, s_inv);
      if (m.raw && threadIdx.x < TM) {   // bare network: the Jacobian's diagonal, entry by entry
        if (row0 + threadIdx.x < rows.R) div[(row0 + threadIdx.x) * m.D + i] = sm[L.DIV + threadIdx.x];
        sm[L.DIV + threadIdx.x] = 0.f;
      }
    }
    if (!m.raw && threadIdx.x < TM && row0 + threadIdx.x < rows.R) div[row0 + threadIdx.x] = sm[L.DIV + threadIdx.x];
    consumer_sync();
  }
}


template <int TM, int RN, int RK>
__global__ void __launch_bounds__(kThreads, 1)
fm_vjp_kernel(const __grid_constant__ sbi_fm_model m, const __grid_constant__ sbi_rows rows,
              const float* __restrict__ time, const float* __restrict__ eps, const float* __restrict__ gout,
              float g_const, float* __restrict__ loss, float* __restrict__ gpart, float* __restrict__ loss_acc,
              const float* __restrict__ dout, float* __restrict__ dcond) {
  constexpr int LD = Tile<TM>::LD;
  constexpr int PARTS = kConsumerThreads / TM;
  extern __shared__ __align__(128) float sm[];
  const FmSmem L = fm_smem_layout(m, TM, kFmTrain);
  WPipe pipe = make_pipe(m.nbuf, m.wcap, sm, L.ring, L.bar_bytes);
  const int64_t ntiles = (rows.R + TM - 1) / TM;
  const float* __restrict__ P = m.d_params;
  const int* T = m.d_tab;
  const int Hp = m.Hp, H = m.H;
  // no upstream gradient at all (validation, the autograd Function's forward): the loss values only -- the
  // backward sweep and its weight stream are skipped and the gradient slab is left untouched
  const bool loss_only = dout == nullptr && gout == nullptr && g_const == 0.f;

  if (threadIdx.x >= kConsumerThreads) {
    if (threadIdx.x == kConsumerThreads) {
      auto noop = [](int, int, float(&)[RK][4], bool) {};
      for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        fm_net_forward<kProducer, TM, RN, kFmTrain>(m, pipe, sm, L);
        if (loss_only) continue;
        dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + SBI_F_WO), m.Dp, Hp, m.rpc_o, nullptr, Hp, noop);
        for (int l = m.NL - 1; l >= 0; --l)
          dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + SBI_F_LAYER0 + 4 * l), Hp, Hp, m.rpc_h, nullptr, Hp, noop);
        dx_stage<kProducer, TM, RK>(pipe, P + __ldg(T + SBI_F_WM), Hp, 2 * Hp, m.rpc_m, nullptr, 2 * Hp, noop);
      }
    }
    return;
  }

  float* gp = gpart + (size_t)blockIdx.x * m.n_params;
  float* dH = sm + L.dH;
  float* dTE = sm + L.dTE;
  float* X1 = sm + L.X1;
  float* X2 = sm + L.X2;
  float* RED = sm + L.RED;
  float* OUT = sm + L.OUT;
  const float* TGT = sm + L.TGT;
  const float* TEB = sm + L.TEB;
  const int r_ = threadIdx.x % TM, p_ = threadIdx.x / TM;

  int iter = 0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++iter) {
    const bool accum = iter > 0;
    const int64_t row0 = tile * TM;
    fm_load<TM, true>(m, rows, time, 0, eps, row0, sm, L);
    fm_net_forward<kConsumer, TM, RN, kFmTrain>(m, pipe, sm, L);
    if (dout != nullptr) {
      // bare network: the upstream gradient of the outputs is given (score estimators, sbi_b200_fm_net_vjp)
      for (int e = threadIdx.x; e < m.Dp * TM; e += kConsumerThreads) {
        const int d = e / TM, r = e % TM;
        OUT[d * LD + r] = (d < m.D && row0 + r < rows.R) ? __ldg(dout + (row0 + r) * m.D + d) : 0.f;
      }
      consumer_sync();
    } else
    // loss_r = mean_d (v_out - target)^2 ; dOUT = g_r * 2/D * (v_out - target)   (in place in OUT)
    {
      float lsum = 0.f, bad = 0.f;
      if (p_ == 0) {
        const bool ok = row0 + r_ < rows.R;
        float a = 0.f;
        for (int d = 0; d < m.D; ++d) {
          const float df = OUT[d * LD + r_] - TGT[d * LD + r_];
          a = fmaf(df, df, a);
        }
        a /= (float)m.D;
        const float g = ok ? (gout ? __ldg(gout + row0 + r_) : g_const) : 0.f;
        if (ok) {
          if (loss != nullptr) loss[row0 + r_] = a;
          if (isfinite(a)) lsum = a; else bad = 1.f;
        }
        RED[r_] = g * 2.f / (float)m.D;
      }
      if (loss_acc != nullptr && threadIdx.x < 32) {   // TM <= 32: the p_ == 0 threads sit in warp 0
        lsum = warp_sum(lsum);
        bad = warp_sum(bad);
        if (threadIdx.x == 0) {
          atomicAdd(loss_acc + 0, lsum);
          if (bad != 0.f) atomicAdd(loss_acc + 1, bad);
        }
      }
      consumer_sync();
      if (loss_only) continue;
      for (int e = threadIdx.x; e < m.Dp * TM; e += kConsumerThreads) {
        const int d = e / TM, r = e % TM;
        OUT[d * LD + r] = d < m.D ? RED[r] * (OUT[d * LD + r] - TGT[d * LD + r]) : 0.f;
      }
      consumer_sync();
    }
    for (int e = threadIdx.x; e < Hp * LD; e += kConsumerThreads) dTE[e] = 0.f;
    // output layer
    const float* HL = sm + L.HS + m.NL * Hp * LD;
    gemm_dw<TM>(OUT, m.D, HL, H, Hp, gp + __ldg(T + SBI_F_WO), gp + __ldg(T + SBI_F_BO), accum);
    dx_stage<kConsumer, TM, RK>(pipe, nullptr, m.Dp, Hp, m.rpc_o, OUT, Hp,
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
    for (int l = m.NL - 1; l >= 0; --l) {
      const int* LT = T + SBI_F_LAYER0 + 4 * l;
      const float* Hin = sm + L.HS + l * Hp * LD;
      const float* Z = sm + L.ZS + l * Hp * LD;
      const float* ga = P + __ldg(LT + 2);
      const float mean = sm[L.STAT + (2 * l) * LD + r_];
      const float rstd = sm[L.STAT + (2 * l + 1) * LD + r_];
      // xhat -> X1 ; dxhat = dH * gamma -> X2
      for (int k = p_; k < Hp; k += PARTS) {
        const int o = k * LD + r_;
        const float u = gelu_f(Z[o]) + TEB[o] + Hin[o];
        X1[o] = k < H ? (u - mean) * rstd : 0.f;
        X2[o] = k < H ? dH[o] * __ldg(ga + k) : 0.f;
      }
      consumer_sync();
      // LN affine gradients (reduction over the tile rows, one feature per thread)
      for (int k = threadIdx.x; k < H; k += kConsumerThreads) {
        float sg = 0.f, sb = 0.f;
        for (int r = 0; r < TM; ++r) {
          const float dy = dH[k * LD + r];
          sg = fmaf(dy, X1[k * LD + r], sg);
          sb += dy;
        }
        grad_out(gp + __ldg(LT + 2) + k, sg, accum);
        grad_out(gp + __ldg(LT + 3) + k, sb, accum);
      }
      const float m1 = row_reduce<TM>(H, RED, [&](int k, int r) { return X2[k * LD + r]; }) / (float)H;
      const float m2 = row_reduce<TM>(H, RED, [&](int k, int r) { return X2[k * LD + r] * X1[k * LD + r]; }) / (float)H;
      // du = rstd (dxhat - m1 - xhat m2): -> dTE += du ; dH (skip path) = du ; dZ = du gelu'(Z) -> X1
      for (int k = p_; k < Hp; k += PARTS) {
        const int o = k * LD + r_;
        const float du = k < H ? rstd * (X2[o] - m1 - X1[o] * m2) : 0.f;
        dTE[o] += du;
        dH[o] = du;
        X1[o] = du * dgelu_f(Z[o]);
      }
      consumer_sync();
      gemm_dw<TM>(X1, H, Hin, H, Hp, gp + __ldg(LT + 0), gp + __ldg(LT + 1), accum);
      dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, Hp, m.rpc_h, X1, Hp,
                                  [&](int k0, int r0, float(&acc)[RK][4], bool) {
#pragma unroll
                                    for (int j = 0; j < RK; ++j) {
                                      float* p = dH + (k0 + j) * LD + r0;
                                      const float4 c = ld4(p);
                                      st4(p, make_float4(c.x + acc[j][0], c.y + acc[j][1], c.z + acc[j][2],
                                                         c.w + acc[j][3]));
                                    }
                                  });
    }
    // time embedding layer
    gemm_dw<TM>(dTE, H, sm + L.SC, m.TE, m.TEp, gp + __ldg(T + SBI_F_WT), gp + __ldg(T + SBI_F_BT), accum);
    // merge layer: dH = grad wrt h0 = gelu(HMP)
    const float* HMP = sm + L.HMP;
    for (int e = threadIdx.x; e < Hp * TM; e += kConsumerThreads) {
      const int o = (e / TM) * LD + (e % TM);
      X1[o] = dH[o] * dgelu_f(HMP[o]);
    }
    consumer_sync();
    gemm_dw<TM>(X1, H, sm + L.AB, 2 * Hp, 2 * Hp, gp + __ldg(T + SBI_F_WM), gp + __ldg(T + SBI_F_BM), accum);
    float* dAB = sm + L.ZS;   // layer pre-activations are dead now (needs NL >= 2 for 2*Hp rows)
    dx_stage<kConsumer, TM, RK>(pipe, nullptr, Hp, 2 * Hp, m.rpc_m, X1, 2 * Hp,
                                [&](int k0, int r0, float(&acc)[RK][4], bool first) {
#pragma unroll
                                  for (int j = 0; j < RK; ++j) {
                                    float* p = dAB + (k0 + j) * LD + r0;
                                    float4 o = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
                                    if (!first) {
                                      const float4 c = ld4(p);
                                      o.x += c.x; o.y += c.y; o.z += c.z; o.w += c.w;
                                    }
                                    st4(p, o);
                                  }
                                });
    const float* ABP = sm + L.ABP;
    for (int e = threadIdx.x; e < 2 * Hp * TM; e += kConsumerThreads) {
      const int o = (e / TM) * LD + (e % TM);
      dAB[o] *= dgelu_f(ABP[o]);
    }
    consumer_sync();
    gemm_dw<TM>(dAB, H, sm + L.TN, m.D, m.Dp, gp + __ldg(T + SBI_F_WI), gp + __ldg(T + SBI_F_BI), accum);
    gemm_dw<TM>(dAB + Hp * LD, H, sm + L.CTX, m.C, m.Cp, gp + __ldg(T + SBI_F_WC), gp + __ldg(T + SBI_F_BC), accum);
    if (dcond != nullptr) {
      // condition gradient of the row: W_c^T dc through the in-kernel z-score, one thread per (row, feature)
      const float* wc = P + __ldg(T + SBI_F_WC);
      const float* csd = m.d_stats + 2 * m.Dp + m.Cp;
      const float* dC = dAB + Hp * LD;
      for (int e = threadIdx.x; e < TM * m.C; e += kConsumerThreads) {
        const int r = e / m.C, c = e % m.C;
        if (row0 + r >= rows.R) continue;
        float a = 0.f;
        for (int n = 0; n < H; ++n) a = fmaf(dC[n * LD + r], __ldg(wc + n * m.Cp + c), a);
        dcond[(row0 + r) * m.C + c] = a / __ldg(csd + c);
      }
    }
    consumer_sync();
  }
}

}  // namespace sbi

using namespace sbi;

// Launch-side tuning of the weight pipeline (the kernels read nbuf / wcap / rpc_* from the model struct, the
// packed weights do not depend on them).  Measured on cfg4 (FMPE dim 20, batch 16384, trainer level, M samples/s;
// profiles/r02_bench_cfg4*.json), in two steps:
//  * Re-chunk per kernel.  A forward chunk of `cnt` weight rows occupies cnt / RN of the 256 / (TM / 4)
//    output-thread groups, so the caller's 32-row chunks of a 100-wide layer kept 25 % (16-row tiles) to 50 %
//    (32-row tiles) of the consumer threads busy, the 16-row chunks of the merge layer half of that.  Two stages of
//    the largest chunk that fits (60 rows in training, whole layers in evaluation) with RN = kFmRN = 1 output row
//    per thread fill them.  (RN = 1 with the 32-row chunks is SLOWER, 7.67: five shared-memory wavefronts per
//    16 FMAs without the extra parallelism.)
//  * Deepen the ring to what the 227 KB of shared memory leave after the activation tile.  ncu attributes ~25 % of
//    fm_vjp's stall samples to the ring's `full` barrier (profiles/r02_fm_vjp.md).
// Deepening alone moved 9.80 -> 9.99, re-chunking on top of it 9.99 -> 12.5.
constexpr int kFmRN = 1;
static sbi_fm_model fm_tune(const sbi_fm_model& m, int TM, int mode) {
  sbi_fm_model c = m;
  constexpr int kBudget = kMaxSmemBytes - 1024;   // static shared memory of the kernels stays below 1 KB
  {
    sbi_fm_model z = m;
    z.nbuf = 0;
    z.wcap = 0;
    const int act = fm_smem_layout(z, TM, mode).total_bytes;          // activation tile
    int cap = (kBudget - act - 2 * 8 * 8) / 4 / 2;                    // floats per stage with two stages
    cap = std::min(cap, 2 * m.Hp * m.Hp);                             // the merge layer is the largest matrix
    cap &= ~31;
    if (cap >= 4 * 2 * m.Hp) {
      auto rows = [&](int rowlen, int nmax) { return std::max(4, std::min(nmax, (cap / rowlen) & ~3)); };
      c.rpc_i = rows(m.Dp, m.Hp);
      c.rpc_c = rows(m.Cp, m.Hp);
      c.rpc_m = rows(2 * m.Hp, m.Hp);
      c.rpc_t = rows(m.TEp, m.Hp);
      c.rpc_h = rows(m.Hp, m.Hp);
      c.rpc_o = rows(m.Hp, m.Dp);
      const int used = std::max({c.rpc_i * m.Dp, c.rpc_c * m.Cp, c.rpc_m * 2 * m.Hp, c.rpc_t * m.TEp,
                                 c.rpc_h * m.Hp, c.rpc_o * m.Hp});
      c.wcap = (used + 31) & ~31;
      c.nbuf = 2;
      if (fm_smem_layout(c, TM, mode).total_bytes > kBudget) c = m;   // (cannot happen; keep the caller's plan)
    }
  }
  const int nb0 = c.nbuf;
  for (int nb = 8; nb > nb0; --nb) {
    c.nbuf = nb;
    if (fm_smem_layout(c, TM, mode).total_bytes <= kBudget) return c;
  }
  c.nbuf = nb0;
  return c;
}

static int fm_check(const sbi_fm_model* m) {
  if (!m || !m->d_params || !m->d_tab || !m->d_stats) return SBI_EINVAL;
  if (m->D < 1 || m->C < 1 || m->H < 1 || m->NL < 2 || m->NL > SBI_FM_MAX_LAYERS || m->TE < 2 || (m->TE & 1)) return SBI_EINVAL;
  if (m->Dp != round4(m->D) || m->Cp != round4(m->C) || m->Hp != round4(m->H) || m->TEp != round4(m->TE)) return SBI_EINVAL;
  if (!ring_ok({{m->rpc_i, m->Dp}, {m->rpc_c, m->Cp}, {m->rpc_m, 2 * m->Hp}, {m->rpc_t, m->TEp}, {m->rpc_h, m->Hp},
                {m->rpc_o, m->Hp}},
               m->nbuf, m->wcap))
    return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_fm_forward(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                                   int32_t time_shared, float* d_v, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = fm_check(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_time || !d_v) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  constexpr int TM = 32;
  const sbi_fm_model md = fm_tune(*m, TM, kFmEval);
  return launch(fm_forward_kernel<TM, kFmRN>, tile_grid(rows->R, TM, 1), kThreads,
                fm_smem_layout(md, TM, kFmEval).total_bytes, (cudaStream_t)stream, md, *rows, d_time, time_shared, d_v);
}

extern "C" int sbi_b200_fm_forward_div(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                                       int32_t time_shared, float* d_v, float* d_div, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = fm_check(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_time || !d_div) return SBI_EINVAL;
  if (rows->R == 0) return 0;
  constexpr int TM = 16;
  const sbi_fm_model md = fm_tune(*m, TM, kFmTrace);
  return launch(fm_trace_kernel<TM, kFmRN>, tile_grid(rows->R, TM, 1), kThreads,
                fm_smem_layout(md, TM, kFmTrace).total_bytes, (cudaStream_t)stream, md, *rows, d_time, time_shared, d_v,
                d_div);
}

extern "C" int sbi_b200_fm_plan(const sbi_fm_model* m, int32_t kernel, int32_t* out10) {
  // introspection (no device work): the weight-pipeline plan a launch of `kernel` (0 forward, 1 loss / parameter
  // gradient, 2 forward + divergence) would use: [nbuf, wcap, rpc_i, rpc_c, rpc_m, rpc_t, rpc_h, rpc_o,
  // dynamic shared memory bytes, output rows per thread]
  if (!m || !out10 || kernel < 0 || kernel > 2) return SBI_EINVAL;
  const int TM = kernel == 0 ? 32 : 16;
  const int mode = kernel == 0 ? kFmEval : (kernel == 1 ? kFmTrain : kFmTrace);
  const sbi_fm_model c = fm_tune(*m, TM, mode);
  const int v[10] = {c.nbuf, c.wcap, c.rpc_i, c.rpc_c, c.rpc_m, c.rpc_t, c.rpc_h, c.rpc_o,
                     fm_smem_layout(c, TM, mode).total_bytes, kFmRN};
  for (int i = 0; i < 10; ++i) out10[i] = v[i];
  return 0;
}

extern "C" int sbi_b200_fm_vjp_parts(int64_t R) { return vjp_parts(R, 16); }

extern "C" int sbi_b200_fm_loss_vjp(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                                    const float* d_eps, const float* d_gout, float g_const, float* d_loss,
                                    float* d_gpart, float* d_loss_acc, void* stream) {
  return sbi_b200_fm_loss_vjp_cond(m, rows, d_time, d_eps, d_gout, g_const, d_loss, d_gpart, d_loss_acc, nullptr,
                                   stream);
}

extern "C" int sbi_b200_fm_loss_vjp_cond(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                                         const float* d_eps, const float* d_gout, float g_const, float* d_loss,
                                         float* d_gpart, float* d_loss_acc, float* d_gcond, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = fm_check(m);
  if (rc) return rc;
  if (!rows || !rows->d_input || !rows->d_cond || rows->R < 1 || !d_time || !d_eps || !d_gpart) return SBI_EINVAL;
  if (d_gcond != nullptr && d_gout == nullptr && g_const == 0.f) {
    // no upstream gradient: the kernel skips the backward sweep, so the condition gradient is zero
    cudaError_t e = cudaMemsetAsync(d_gcond, 0, (size_t)rows->R * m->C * sizeof(float), (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
  }
  constexpr int TM = 16;
  const sbi_fm_model md = fm_tune(*m, TM, kFmTrain);
  return launch(fm_vjp_kernel<TM, kFmRN, 2>, sbi_b200_fm_vjp_parts(rows->R), kThreads,
                fm_smem_layout(md, TM, kFmTrain).total_bytes, (cudaStream_t)stream, md, *rows, d_time, d_eps, d_gout,
                g_const, d_loss, d_gpart, d_loss_acc, nullptr, d_gcond);
}

extern "C" int sbi_b200_fm_net_vjp(const sbi_fm_model* m, const sbi_rows* rows, const float* d_time,
                                   const float* d_dout, float* d_gpart, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  int rc = fm_check(m);
  if (rc) return rc;
  if (!m->raw || !rows || !rows->d_input || !rows->d_cond || rows->R < 1 || !d_time || !d_dout || !d_gpart)
    return SBI_EINVAL;
  constexpr int TM = 16;
  const sbi_fm_model md = fm_tune(*m, TM, kFmTrain);
  return launch(fm_vjp_kernel<TM, kFmRN, 2>, sbi_b200_fm_vjp_parts(rows->R), kThreads,
                fm_smem_layout(md, TM, kFmTrain).total_bytes, (cudaStream_t)stream, md, *rows, d_time, nullptr, nullptr,
                0.f, nullptr, d_gpart, nullptr, d_dout, nullptr);
}
