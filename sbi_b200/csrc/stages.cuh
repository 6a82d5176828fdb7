// Stage helpers shared by all model families: the warp-specialised weight pipeline driving the
// row-tile GEMMs of tile_gemm.cuh.  Both roles (producer lane / consumer warps) call the same
// helpers in the same order; the producer only issues the TMA bulk copies.
#pragma once
#include "../../include/sbi_b200.h"
#include "tile_gemm.cuh"

namespace sbi {

enum Role { kProducer = 0, kConsumer = 1 };

__device__ __forceinline__ float4 relu4(float4 v) {
  return make_float4(relu_f(v.x), relu_f(v.y), relu_f(v.z), relu_f(v.w));
}

// ---- stage helpers (both roles) -----------------------------------------------------------
// forward GEMM stage: Y = W X, streamed in chunks of `rpc` rows.
// epi(n0, g, ng, r0, acc): chunk first row n0, thread rows n0 + g + i*ng, tile rows r0..r0+3
template <Role R, int TM, int RN, class Epi>
__device__ __forceinline__ void fwd_stage(WPipe& pipe, const float* __restrict__ Wg, int N,
                                          int Kp, int rpc, const float* X, Epi&& epi) {
  for (int n0 = 0; n0 < N; n0 += rpc) {
    const int cnt = min(rpc, N - n0);
    if (R == kProducer) {
      pipe.produce(Wg + (size_t)n0 * Kp, cnt * Kp);
    } else {
      const float* w = pipe.acquire();
      gemm_fwd_chunk<TM, RN>(X, Kp >> 2, w, Kp, cnt,
                             [&](int g, int ng, int r0, float(&acc)[RN][4]) {
                               epi(n0, g, ng, r0, acc);
                             });
      pipe.release();
    }
  }
  if (R == kConsumer) consumer_sync();
}

// GLU stage: t = W2 X1, gt = Wc X2 for the same output rows; one chunk = [W2 rows | Wc rows]
template <Role R, int TM, int RN, class Epi>
__device__ __forceinline__ void glu_stage(WPipe& pipe, const float* __restrict__ W2g, int Kp2,
                                          const float* __restrict__ Wcg, int Kpc, int N, int rpc,
                                          const float* X1, const float* X2, Epi&& epi) {
  constexpr int NRG = Tile<TM>::NRG, NOG = Tile<TM>::NOG;
  for (int n0 = 0; n0 < N; n0 += rpc) {
    const int cnt = min(rpc, N - n0);
    if (R == kProducer) {
      pipe.produce(W2g + (size_t)n0 * Kp2, cnt * Kp2, Wcg + (size_t)n0 * Kpc, cnt * Kpc);
    } else {
      const float* w2 = pipe.acquire();
      const float* wc = w2 + cnt * Kp2;
      const int rg = threadIdx.x % NRG, og = threadIdx.x / NRG;
      const int ng = cnt / RN;
      for (int g = og; g < ng; g += NOG) {
        float at[RN][4], ag[RN][4];
#pragma unroll
        for (int i = 0; i < RN; ++i)
#pragma unroll
          for (int c = 0; c < 4; ++c) at[i][c] = ag[i][c] = 0.f;
        gemm_fwd_acc<TM, RN>(at, X1, Kp2 >> 2, w2, Kp2, g, ng, rg);
        gemm_fwd_acc<TM, RN>(ag, X2, Kpc >> 2, wc, Kpc, g, ng, rg);
        epi(n0, g, ng, 4 * rg, at, ag);
      }
      pipe.release();
    }
  }
  if (R == kConsumer) consumer_sync();
}

// backward-x stage over a weight matrix of N rows: dX = W^T dY (accumulated over chunks).
// epi(k0, r0, acc, first) ; `first` = first chunk (overwrite vs. add is up to the epilogue).
template <Role R, int TM, int RK, class Epi>
__device__ __forceinline__ void dx_stage(WPipe& pipe, const float* __restrict__ Wg, int N, int Kp,
                                         int rpc, const float* dY, int Kout, Epi&& epi) {
  for (int n0 = 0; n0 < N; n0 += rpc) {
    const int cnt = min(rpc, N - n0);
    if (R == kProducer) {
      pipe.produce(Wg + (size_t)n0 * Kp, cnt * Kp);
    } else {
      const float* w = pipe.acquire();
      gemm_dx_chunk<TM, RK>(dY, n0, cnt, w, Kp, Kout,
                            [&](int k0, int r0, float(&acc)[RK][4]) { epi(k0, r0, acc, n0 == 0); });
      pipe.release();
    }
  }
  if (R == kConsumer) consumer_sync();
}

// Z[d][r] = input[row][d] * scale[d] + shift[d] (or raw), CTX[c][r] = (cond[row][c]-mean[c])/std[c];
// stats = [shift(Dp) | scale(Dp) | mean(Cp) | std(Cp)]; pad rows / rows beyond R are zero.
// No barrier inside.
template <int TM>
__device__ __forceinline__ void load_rows(int D, int Dp, int C, int Cp, const float* __restrict__ st,
                                          const sbi_rows& rows, int64_t row0, float* Z, float* CTX,
                                          bool raw_input) {
  constexpr int LD = Tile<TM>::LD;
  for (int e = threadIdx.x; e < TM * Dp; e += kConsumerThreads) {
    const int r = e / Dp, d = e % Dp;
    const int64_t gr = row0 + r;
    float val = 0.f;
    if (d < D && gr < rows.R) {
      const int64_t src = rows.d_index ? __ldg(rows.d_index + gr) : gr;
      const float x = __ldg(rows.d_input + src * D + d);
      val = raw_input ? x : __fadd_rn(__fmul_rn(x, __ldg(st + Dp + d)), __ldg(st + d));
    }
    Z[d * LD + r] = val;
  }
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
}

// classifier input U = [theta | pad | x | pad] (Dtp + Dxp feature rows) of the pairs row0 .. row0+TM-1,
// standardised by stats = [theta_mean(Dtp) | theta_std(Dtp) | x_mean(Dxp) | x_std(Dxp)] (include/sbi_b200.h
// sbi_pairs); pad rows / rows beyond R are zero.  No barrier inside.
template <int TM>
__device__ __forceinline__ void pairs_load(int Dt, int Dx, int Dtp, int Dxp, const float* __restrict__ st,
                                           const sbi_pairs& pr, int64_t row0, float* U) {
  constexpr int LD = Tile<TM>::LD;
  for (int e = threadIdx.x; e < TM * Dtp; e += kConsumerThreads) {
    const int r = e / Dtp, d = e % Dtp;
    const int64_t gr = row0 + r;
    float val = 0.f;
    if (d < Dt && gr < pr.R) {
      const int64_t src = pr.d_theta_index ? __ldg(pr.d_theta_index + gr) : gr;
      val = (__ldg(pr.d_theta + src * Dt + d) - __ldg(st + d)) / __ldg(st + Dtp + d);
    }
    U[d * LD + r] = val;
  }
  for (int e = threadIdx.x; e < TM * Dxp; e += kConsumerThreads) {
    const int r = e / Dxp, d = e % Dxp;
    const int64_t gr = row0 + r;
    float val = 0.f;
    if (d < Dx && gr < pr.R) {
      const int64_t src = pr.x_shared ? 0 : (pr.d_x_index ? __ldg(pr.d_x_index + gr) : gr);
      val = (__ldg(pr.d_x + src * Dx + d) - __ldg(st + 2 * Dtp + d)) / __ldg(st + 2 * Dtp + Dxp + d);
    }
    U[(Dtp + d) * LD + r] = val;
  }
}

// carve the weight ring + its mbarriers out of shared memory (all threads call this)
__device__ __forceinline__ WPipe make_pipe(int nbuf, int wcap, float* sm, int ring_off, int bar_bytes) {
  WPipe p;
  p.buf = sm + ring_off;
  p.full = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(sm) + bar_bytes);
  p.empty = p.full + nbuf;
  p.cap = wcap;
  p.nbuf = nbuf;
  p.it = 0;
  if (threadIdx.x == 0) {
    for (int s = 0; s < nbuf; ++s) {
      mbar_init(&p.full[s], 1);
      mbar_init(&p.empty[s], kConsumerThreads / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  return p;
}

}  // namespace sbi
