// Tensor-core bulk evaluation and sampling of the neural spline flow: NFlowsFlow.log_prob /
// inverse_transform / sample (/root/reference/sbi/neural_nets/estimators/nflows_flow.py:42-128)
// from 1024 rows.
//
// Same function, same parameter buffer and same evaluation order outside the linears as
// nsf_logprob_kernel (nsf.cu); the ResidualNet linears (nflows ResidualNet, restated in
// oracle/nflows_port/nn/nets/resnet.py; built at flow.py:411-419) run on the tensor cores:
//
//   * one CTA = 8 warps (128 rows = 128 lanes of the accumulator store, two threads per row
//     splitting the columns of every epilogue), two CTAs per SM (256 store columns each); the
//     warps take turns issuing the TMA copies of the weight stages (tc_common.cuh);
//   * wgmma.mma_async kind tf32, both warpgroups together (64 rows each), synchronously (the training forward
//     keeps two K-steps in flight, tc_common.cuh): the row
//     threads put A (activations) into the accumulator store (tc_common.cuh) after splitting every
//     fp32 value into hi = tf32(x) and lo = x - hi, the warpgroups load their A fragments from it;
//     B (weights, pre-split hi/lo and pre-arranged in the K-major no-swizzle layout by
//     tc_pack_kernel) is streamed by TMA bulk copies into a shared-memory ring;
//     D = A_hi B_hi + A_lo B_hi + A_hi B_lo (3xTF32) accumulates in fp32 registers and goes back
//     to the store for the bias / relu / GLU / spline epilogues;
//   * the context is a K-extension of the hidden operand: A columns are
//     [ hidden (H) | context (C) | 0 ], so the GLU gate W_c ctx is one more small MMA on the
//     same operand and the context never has to be re-staged;
//   * spline, LU (register-resident row against zero-padded 16x16 factors) and base density are
//     per-thread code on the thread's own row;
//   * the same kernel template runs the sampling direction (layers T-1..0, LU^-1, inverse spline).
//
// Store columns of a CTA:  [0,64) A_hi | [64,128) A_lo | [128,192) D | [192,256) G (GLU gate);
// the final layer's spline parameters P (32 columns per feature, 2 features per pass)
// alternate between D and G.  The training forward (SAVE) runs one CTA per SM (one tile each), keeps
// A_hi / A_lo in shared memory (tc_common.cuh) and reserves only [0,64) D | [64,128) G of the store.
// When a chunk of tiles would leave SMs idle, the training forward runs two CTAs per tile, one per 64-row
// half (RPC = 64): four threads per row, both warpgroups on the CTA's 64 rows (tc_common.cuh), D | G in shared
// memory instead of the store, and the tile's save slab at lanes [64 r, 64 r + 64) for half r.
#include <cuda_runtime.h>
#include <math.h>
#include <algorithm>
#include <cstdlib>

#include "nsf.cuh"

#include "tc_common.cuh"
#include "nsf_tc_save.cuh"
#include "rqs_fast.cuh"
#include "device.cuh"

namespace sbi {
namespace tc {

// ---- shared memory plan -------------------------------------------------------------------------
struct TcSmem {
  int zs, ctx, lds, ldf, lum, bias, bias_stride, a, acc, ring;   // float offsets
  int bar_bytes, total_bytes;
};
// a_smem: the training forward (SAVE) also keeps its A operands in shared memory (tc_common.cuh), and on half
// tiles its accumulator columns; rpc: rows per CTA (128, or 64 for the training forward's half tiles)
__host__ __device__ inline TcSmem tc_smem_layout(const sbi_nsf_model& m, int stage_cap, bool a_smem, int rpc = kRows) {
  TcSmem L;
  int fl = 0;
  L.zs = fl;  fl += m.Dp * rpc;
  L.ctx = fl; fl += m.Cp * rpc;
  L.lds = fl; fl += rpc;
  L.ldf = fl; fl += rpc < kRows ? kLuMax * rpc : 0;     // half tiles: log|det| per spline feature of a layer
  L.lum = fl; fl += 2 * kLuMax * kLuMax + 2 * kLuMax;   // [U 16x16 | L 16x16 | bias 16 | diag 16]
  L.bias_stride = 64 + m.NB * 192 + m.TRmax * 32;
  L.bias = fl; fl += m.T * L.bias_stride;
  fl = (fl + 31) & ~31;
  L.a = fl;   fl += a_smem ? a_smem_floats(rpc) : 0;
  L.acc = fl; fl += a_smem && rpc < kRows ? acc_smem_floats() : 0;
  L.ring = fl; fl += kSlots * stage_cap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + kSlots * 8;
  return L;
}

// Two threads share a row: part `tq` 0 owns hidden columns [0, HP8/2), part 1 owns [HP8/2, HP8)
// (which end in the first context columns).  All epilogues are column-wise, so the
// parts never exchange activations; the spline features of a layer alternate between them.
// Half tiles (RPC = 64, training forward only) have four threads per row, part tq owning columns
// [16 tq, 16 tq + 16); part 3 holds the last hidden columns, the context and the zero tail.  The spline
// features go round-robin over the four parts, which leave each feature's log|det| in shared memory;
// parts 0 and 1 add them up in the order of the two-part split, so every row's result is bit-identical.
//
// Per coupling layer the tensor core sees these stages (result columns after the arrow):
//   initial layer -> D
//   per block:  W_c ctx -> G,  W_1 relu(h) -> D,  W_2 relu(.) -> D
//   final layer in passes of <= 2 spline features, pass p -> P_(p&1) (two result regions, so
//               pass p + 1 may be computed before the spline of pass p has read its parameters).
//
// INV = false: log_prob (logp (R,), optional base-space point `noise` (R,D)).
// INV = true : sampling direction x = T^{-1}(noise | cond): rows.d_input holds the noise, the
//              layers run T-1 .. 0 with LU^{-1} first and the inverse spline; `noise` receives x
//              (R,D) and `logp` (optional) log|det dx/dnoise|  (sbi_b200_nsf_inverse).
//
// SAVE = true (training forward, INV = false): every layer's conditioner intermediates, raw spline
// parameters, layer input and coupling output of the tile go to the activation scratch `save`
// (layout: nsf_tc_save.cuh) for the tensor-core backward and weight-gradient kernels (nsf_vjp_tc.cu),
// together with the final base-space point and the row's log-density.
template <int H, int KB, bool INV, bool SAVE = false, int RPC = kRows>
__global__ void __launch_bounds__(kThreads, SAVE ? 1 : 2)
nsf_logprob_tc_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_nsf_tc tc,
                      const __grid_constant__ sbi_rows rows, float* __restrict__ logp,
                      float* __restrict__ noise, float* __restrict__ save, const StoreArgs sa) {
  constexpr int HP8 = (H + 7) & ~7;
  constexpr int NCH = HP8 / 8;      // K-steps / 8-column chunks of the hidden operand
  constexpr int KC0 = H / 8;        // first chunk that holds context columns
  constexpr int TPR = kThreads / RPC;                   // threads per row
  constexpr int UPT = kRows / RPC;                      // CTAs per tile
  constexpr int NC = TPR == 2 ? HP8 / 2 : 16;           // hidden columns per thread ([tq NC, tq NC + NC))
  constexpr int NG = NC / 4;        // groups of 4 columns
  constexpr int QC = H - (TPR - 1) * NC;                // first column offset of the last part that is context
  static_assert(HP8 % 8 == 0 && NC % 4 == 0 && QC > 0 && QC <= NC && H <= 64, "hidden width");
  static_assert(!(RPC < kRows) || (SAVE && !INV), "half tiles are a layout of the training forward");
  extern __shared__ __align__(128) float sm[];
  const TcSmem L = tc_smem_layout(m, tc.stage_cap, SAVE, RPC);
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(sm) + L.bar_bytes);
  const int tid = threadIdx.x, warp = tid >> 5;
  const int C = m.C;
  const int nkc = (H + C + 7) / 8 - KC0;     // K-steps that cover the context columns
  const int64_t nunits = (rows.R + kRows - 1) / kRows * UPT;     // CTA tiles of RPC rows
  const TcSave SV = tc_save_layout(m.NB, m.TRmax, m.T);

  // SAVE: A in shared memory, the store holds D | G only; half tiles keep D | G in shared memory too
  constexpr int ncols = RPC < kRows ? 0 : SAVE ? kColsDG : kCols;
  constexpr int kD = SAVE ? cDs : cD, kG = SAVE ? cGs : cG;
  float* as = sm + L.a;
  float* accs = sm + L.acc;
  SBI_TL(1);
  IssuerT<kSlots, SAVE, RPC> iss =
      tc_begin<kSlots, SAVE, RPC>(full, sm + L.ring, tc, m.T, nunits, INV, ncols, sa, as, accs);

  const float* __restrict__ P = m.d_params;
  float* zs = sm + L.zs;
  float* ctx_s = sm + L.ctx;
  float* lds = sm + L.lds;
  float* ldf = sm + L.ldf;
  const float* bias_s = sm + L.bias;
  const int tq = RPC == kRows ? warp >> 2 : warp >> 1;                      // which column part of the row
  const int row = ((RPC == kRows ? warp & 3 : warp & 1) << 5) | (tid & 31);  // row of the CTA = store lane
  const int cbase = tq * NC;                               // first hidden column of this thread
  const int last = TPR == 2 ? tq : tq == TPR - 1;          // nonzero: the part that holds the context columns
  RqsConst rc = rqs_const(m);
  rc.K = KB;
  const int D = m.D;

  // all biases of the conditioners, once per CTA (zero beyond the real widths):
  //   per layer [b0 64 | per block: b1 64, b2 64, bc 64 | bf TRmax*32]
  // kBatch entries per thread at a time: the layer-table loads of all of them, then their parameter loads, then
  // the stores, so that a batch waits for two loads rather than two per entry (the evaluation kernels, 128
  // registers, take one entry at a time)
  {
    constexpr int kBatch = SAVE ? 8 : 1;
    float* bs = sm + L.bias;
    const int n = m.T * L.bias_stride;
    for (int e0 = tid; e0 < n; e0 += kBatch * kThreads) {
      int src[kBatch];     // parameter index of the entry, or -1: zero
#pragma unroll
      for (int k = 0; k < kBatch; ++k) {
        const int e = min(e0 + k * kThreads, n - 1);
        const int l = e / L.bias_stride, o = e % L.bias_stride;
        const int* LT = m.d_layer_tab + l * SBI_NSF_LAYER_STRIDE;
        const int b = (o - 64) / 192, w = ((o - 64) % 192) / 64, j = (o - 64) % 64;
        const int q = o - 64 - m.NB * 192, f = q / 32, i = q % 32;
        const int slot = o < 64 ? SBI_L_B0 : o < 64 + m.NB * 192 ? SBI_L_BLK0 + 6 * b + 1 + 2 * w : SBI_L_BF;
        const int base = __ldg(LT + slot), ntr = __ldg(LT + SBI_L_NTR);
        const bool ok = o < 64 ? o < H : o < 64 + m.NB * 192 ? j < H : f < ntr && i < 3 * KB - 1;
        const int off = o < 64 ? o : o < 64 + m.NB * 192 ? j : f * m.PR + i;
        src[k] = ok ? base + off : -1;
      }
      float v[kBatch];
#pragma unroll
      for (int k = 0; k < kBatch; ++k) v[k] = src[k] >= 0 ? __ldg(P + src[k]) : 0.f;
#pragma unroll
      for (int k = 0; k < kBatch; ++k)
        if (e0 + k * kThreads < n) bs[e0 + k * kThreads] = v[k];
    }
  }
  SBI_TL(2);
  // batch-constant part of the log-density, summed in the order of lu_logdet_total (nsf.cuh).  The training forward
  // runs one tile per CTA, so this sits on its critical path: each warp of part 1 takes the layer-table entries of
  // up to 32 layers at once (lane k: layer l0 + k), then per layer lane i < D the term of diagonal entry i, and the
  // terms are added in feature order, the layer sums in layer order.  The evaluation kernels loop over many tiles
  // per CTA and keep the serial loop, which needs fewer registers under their 128-register bound.
  float ld_const = 0.f;
  if (tq == 1) {
    float tot = 0.f;
    if constexpr (SAVE) {
      const int lane = tid & 31;
      for (int l0 = 0; l0 < m.T; l0 += 32) {
        int has = 0, od = 0;
        if (l0 + lane < m.T) {
          const int* LT = m.d_layer_tab + (l0 + lane) * SBI_NSF_LAYER_STRIDE;
          has = __ldg(LT + SBI_L_HAS_LU);
          od = __ldg(LT + SBI_L_LU_DIAG);
        }
        for (int k = 0; k < 32 && l0 + k < m.T; ++k) {
          const int hk = __shfl_sync(0xffffffffu, has, k), ok = __shfl_sync(0xffffffffu, od, k);
          float term = 0.f;
          if (hk && lane < D) term = logf(softplus_f(__ldg(P + ok + lane)) + 1e-3f);
          float sacc = 0.f;
          if (hk)
            for (int i = 0; i < D; ++i) sacc += __shfl_sync(0xffffffffu, term, i);
          tot += sacc;
        }
      }
    } else {
      for (int l = 0; l < m.T; ++l) {
        const int* LT = m.d_layer_tab + l * SBI_NSF_LAYER_STRIDE;
        float sacc = 0.f;
        if (__ldg(LT + SBI_L_HAS_LU))
          for (int i = 0; i < D; ++i)
            sacc += logf(softplus_f(__ldg(P + __ldg(LT + SBI_L_LU_DIAG) + i)) + 1e-3f);
        tot += sacc;
      }
    }
    ld_const = INV ? (-tot - m.ld_zscore) : (tot + m.ld_zscore - 0.5f * (float)D * 1.8378770664093453f);
  }
  SBI_TL(3);

  auto put_a4 = [&](int col, const float (&a)[4]) {
    if constexpr (SAVE) smem_a4<RPC>(as, row, col, a);
    else store_a4(row, col, a);
  };
  auto put_a8 = [&](int col, const float (&a)[8]) {
    if constexpr (SAVE) smem_a8<RPC>(as, row, col, a);
    else store_a8(row, col, a);
  };
  // operands written: hand them over to the MMAs
  auto hand_over = [&]() {
    if constexpr (SAVE) fence_async_smem();
    group_sync();
  };
  // A-operand column j of a hidden layer: activation (j < H), context (H <= j < H+C), zero
  auto acol = [&](int j, float act) -> float {
    const int c = j - H;
    return j < H ? act : ((c < C) ? ctx_s[c * RPC + row] : 0.f);
  };
  // this thread's NC columns of a hidden-layer A operand; the last part's last columns are context
  // (columns from HP8 on are the tail, written once per tile)
  auto write_a = [&](const float (&act)[NC]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      if (TPR * NC > HP8 && cbase + 4 * g >= HP8) continue;
      float a[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int q = 4 * g + i;
        if (q < QC) a[i] = act[q];
        else a[i] = last ? ((q - QC < C) ? ctx_s[(q - QC) * RPC + row] : 0.f) : act[q];
      }
      put_a4(cbase + 4 * g, a);
    }
  };
  auto read_acc = [&](int region, float (&d)[NC]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) ld4<RPC>(row, region + cbase + 4 * g, d + 4 * g, accs);
  };

  for (int64_t unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
    const int64_t tile = unit / UPT;                        // 128-row tile (save slab)
    const int srow = (int)(unit % UPT) * RPC + row;         // lane of the row in the tile's save slab
    const int64_t row0 = unit * RPC;
    // the tile's ready counters of the weight-gradient units start at zero (nsf_tc_save.cuh)
    if constexpr (SAVE) {
      if (unit % UPT == 0)
        for (int e = tid; e < m.T * SV.units(); e += kThreads)
          reinterpret_cast<unsigned*>(save + (size_t)tile * SV.tile_stride + (size_t)(e / SV.units()) * SV.layer_stride +
                                      SV.ready())[e % SV.units()] = 0u;
    }
    // ---- load + standardise the CTA's rows (arithmetic of load_rows, stages.cuh) ----
    {
      const float* st = m.d_stats;
      const int Dp = m.Dp, Cp = m.Cp;
      if constexpr (SAVE) {
        // the training forward has one tile per CTA, so the gather sits on its critical path: each thread takes
        // one row and every TPR-th input and context feature of it (Dp, Cp <= 16: sbi_b200_nsf_tc_supported); the
        // row's index first, then all of its loads, then the stores.  (The evaluation kernels keep the loop below,
        // which needs fewer registers under their 128-register bound.)
        constexpr int kF = 16 / TPR;
        const int r = tid % RPC, part = tid / RPC;
        const int64_t gr = row0 + r;
        const bool live = gr < rows.R;
        const int64_t src = live && rows.d_index ? __ldg(rows.d_index + gr) : gr;
        const int64_t csrc = rows.cond_shared ? 0 : src;
        float xv[kF], xs[kF], xm[kF], cv[kF], cm[kF], cs[kF];
#pragma unroll
        for (int k = 0; k < kF; ++k) {
          const int d = part + TPR * k;
          const bool dok = live && d < D, cok = live && d < C;
          xv[k] = dok ? __ldg(rows.d_input + src * D + d) : 0.f;
          xs[k] = dok ? __ldg(st + Dp + d) : 0.f;
          xm[k] = dok ? __ldg(st + d) : 0.f;
          cv[k] = cok ? __ldg(rows.d_cond + csrc * C + d) : 0.f;
          cm[k] = cok ? __ldg(st + 2 * Dp + d) : 0.f;
          cs[k] = cok ? __ldg(st + 2 * Dp + Cp + d) : 1.f;
        }
#pragma unroll
        for (int k = 0; k < kF; ++k) {
          const int d = part + TPR * k;
          if (d < Dp) zs[d * RPC + r] = live && d < D ? __fadd_rn(__fmul_rn(xv[k], xs[k]), xm[k]) : 0.f;
          if (d < Cp) ctx_s[d * RPC + r] = live && d < C ? (cv[k] - cm[k]) / cs[k] : 0.f;
        }
      } else {
        for (int e = tid; e < RPC * Dp; e += kThreads) {
          const int r = e / Dp, d = e % Dp;
          const int64_t gr = row0 + r;
          float val = 0.f;
          if (d < D && gr < rows.R) {
            const int64_t src = rows.d_index ? __ldg(rows.d_index + gr) : gr;
            const float x = __ldg(rows.d_input + src * D + d);
            val = INV ? x : __fadd_rn(__fmul_rn(x, __ldg(st + Dp + d)), __ldg(st + d));
          }
          zs[d * RPC + r] = val;
        }
        for (int e = tid; e < RPC * Cp; e += kThreads) {
          const int r = e / Cp, c = e % Cp;
          const int64_t gr = row0 + r;
          float val = 0.f;
          if (c < C && gr < rows.R) {
            const int64_t src = rows.cond_shared ? 0 : (rows.d_index ? __ldg(rows.d_index + gr) : gr);
            val = (__ldg(rows.d_cond + src * C + c) - __ldg(st + 2 * Dp + c)) / __ldg(st + 2 * Dp + Cp + c);
          }
          ctx_s[c * RPC + r] = val;
        }
      }
      SBI_TL(4);
      if (INV) prep_lu(m, m.T - 1, sm + L.lum);
      group_sync();
    }
    // context tail columns [HP8, 64) never change within a tile
    if (tq == 0) {
#pragma unroll
      for (int c = NCH; c < 8; ++c) {
        float v[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = acol(8 * c + i, 0.f);
        put_a8(8 * c, v);
      }
    }
    float ldacc = 0.f;

    for (int li = 0; li < m.T; ++li) {
      SBI_TL(1000 * (li + 1));
      const int l = INV ? m.T - 1 - li : li;
      const NsfLayerView v = layer_view(m, l);
      const int32_t* tab = tc.d_tab + l * SBI_NSF_TC_STRIDE;
      const float* bl = bias_s + l * L.bias_stride;
      const int kid8 = __ldg(tab + 1);
      int stage = 0;
      float h[NC];
      float* svl = SAVE ? save + (size_t)tile * SV.tile_stride + (size_t)l * SV.layer_stride : nullptr;
      if (SAVE && tq == 1) tc_save_row16<RPC>(svl + SV.zin, srow, zs, row, D);      // layer input z_l

      // ---- sampling: z <- U^{-1} L^{-1} (z - b) on the thread's row (order of lu_inverse, nsf.cuh)
      if (INV && tq == 1 && __ldg(v.LT + SBI_L_HAS_LU)) {
        const float4* U4 = reinterpret_cast<const float4*>(sm + L.lum);
        const float4* L4 = U4 + kLuMax * kLuMax / 4;
        const float* bias = sm + L.lum + 2 * kLuMax * kLuMax;
        const float* diag = bias + kLuMax;
        float zr[kLuMax];
#pragma unroll
        for (int j = 0; j < kLuMax; ++j) zr[j] = (j < D) ? zs[j * RPC + row] : 0.f;
#pragma unroll
        for (int i = 0; i < kLuMax; ++i) {
          if (i < D) {
            float a = zr[i] - bias[i];
#pragma unroll
            for (int j4 = 0; j4 <= (i - 1) / 4 && i > 0; ++j4) {
              const float4 w = L4[i * (kLuMax / 4) + j4];
              if (4 * j4 + 0 < i) a -= w.x * zr[4 * j4 + 0];
              if (4 * j4 + 1 < i) a -= w.y * zr[4 * j4 + 1];
              if (4 * j4 + 2 < i) a -= w.z * zr[4 * j4 + 2];
              if (4 * j4 + 3 < i) a -= w.w * zr[4 * j4 + 3];
            }
            zr[i] = a;
          }
        }
#pragma unroll
        for (int i = kLuMax - 1; i >= 0; --i) {
          if (i < D) {
            float a = zr[i];
#pragma unroll
            for (int j4 = (i + 1) / 4; j4 < kLuMax / 4; ++j4) {
              const float4 w = U4[i * (kLuMax / 4) + j4];      // padded entries are zero
              if (4 * j4 + 0 > i) a -= w.x * zr[4 * j4 + 0];
              if (4 * j4 + 1 > i) a -= w.y * zr[4 * j4 + 1];
              if (4 * j4 + 2 > i) a -= w.z * zr[4 * j4 + 2];
              if (4 * j4 + 3 > i) a -= w.w * zr[4 * j4 + 3];
            }
            zr[i] = a / diag[i];
            zs[i * RPC + row] = zr[i];
          }
        }
      }
      // ---- initial layer: A = [identity features | 0 ... | context] ----
      // (part 1 ran the LU on this row, so it also writes the identity columns)
      if (tq == 1) {
        for (int kk = 0; kk < kid8 / 8; ++kk) {
          float a[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int j = 8 * kk + i;
            a[i] = (j < v.n_id) ? zs[__ldg(v.idf + j) * RPC + row] : 0.f;
          }
          put_a8(8 * kk, a);
        }
      } else if (TPR == 2 || tq == 0) {
#pragma unroll
        for (int c = KC0; c < NCH; ++c) {
          float a[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) a[i] = acol(8 * c + i, 0.f);
          put_a8(8 * c, a);
        }
      }
      hand_over();
      {
        iss.begin(__ldg(tab + 5 + 4 * stage));
        if (li == 0) SBI_TL(6);
        uint32_t acc = 0u;
        iss.block(kD, 0, kid8 / 8, 0, 64, acc);
        iss.block(kD, 8 * KC0, nkc, 64 * kid8, 64, acc);
        iss.end();
      }
      ++stage;
      SBI_TL(1000 * (li + 1) + 1);
      // dense LU factors: forward needs this layer's after the spline, sampling needs the next
      // processed layer's before its conditioner; either way the previous contents were last
      // read before the barrier above
      if (!INV) prep_lu(m, l, sm + L.lum);
      else if (l > 0) prep_lu(m, l - 1, sm + L.lum);
      const float* blh = bl + cbase;
      {
        float d[NC];
        read_acc(kD, d);
#pragma unroll
        for (int q = 0; q < NC; ++q) h[q] = d[q] + blh[q];     // columns >= H: zero weights + zero bias
      }
      SBI_TL(1000 * (li + 1) + 2);

      // ---- residual blocks ----
      for (int b = 0; b < m.NB; ++b) {
        const float* b1 = blh + 64 + b * 192;
        const float* b2 = b1 + 64;
        const float* bc = b1 + 128;
        // A = [relu(h) | ctx]
        if (SAVE) tc_save_cols<NC>(svl + SV.h(b), srow, tq, h);
        {
          float a[NC];
#pragma unroll
          for (int q = 0; q < NC; ++q) a[q] = relu_f(h[q]);
          write_a(a);
        }
        hand_over();
        {
          uint32_t accg = 0u;
          iss.begin(__ldg(tab + 5 + 4 * stage));
          iss.block(kG, 8 * KC0, nkc, 0, 64, accg);
          iss.end();
          uint32_t acc = 0u;
          iss.begin(__ldg(tab + 5 + 4 * (stage + 1)));
          iss.block(kD, 0, NCH, 0, 64, acc);
          iss.end();
        }
        stage += 2;
        SBI_TL(1000 * (li + 1) + 10 * b + 13);
        // gate = sigmoid(Wc ctx + bc)
        float sg[NC];
        {
          float g[NC];
          read_acc(kG, g);
#pragma unroll
          for (int q = 0; q < NC; ++q) sg[q] = sigmoid_fast(g[q] + bc[q]);
          if (SAVE) tc_save_cols<NC>(svl + SV.s(b), srow, tq, sg);
        }
        SBI_TL(1000 * (li + 1) + 10 * b + 14);
        {
          float d[NC];
          read_acc(kD, d);
#pragma unroll
          for (int q = 0; q < NC; ++q) d[q] = relu_f(d[q] + b1[q]);
          if (SAVE) tc_save_cols<NC>(svl + SV.a1(b), srow, tq, d);
          write_a(d);
        }
        hand_over();
        {
          uint32_t acc = 0u;
          iss.begin(__ldg(tab + 5 + 4 * stage));
          iss.block(kD, 0, NCH, 0, 64, acc);
          iss.end();
        }
        ++stage;
        SBI_TL(1000 * (li + 1) + 10 * b + 15);
        {
          // h += (W2 a + b2) * gate
          float d[NC];
          read_acc(kD, d);
          if (SAVE) {
#pragma unroll
            for (int q = 0; q < NC; ++q) d[q] += b2[q];
            tc_save_cols<NC>(svl + SV.t2(b), srow, tq, d);
#pragma unroll
            for (int q = 0; q < NC; ++q) h[q] = fmaf(d[q], sg[q], h[q]);
          } else {
#pragma unroll
            for (int q = 0; q < NC; ++q) h[q] = fmaf(d[q] + b2[q], sg[q], h[q]);
          }
        }
        SBI_TL(1000 * (li + 1) + 10 * b + 16);
      }

      // ---- final layer passes + spline on the transformed features ----
      {
        if (SAVE) tc_save_cols<NC>(svl + SV.hf, srow, tq, h);
        write_a(h);
        const float* bf = bl + 64 + m.NB * 192;
        const int ns = __ldg(tab);
        const int np = ns - stage;            // passes
        hand_over();
        {
          for (int p = 0; p < 2 && p < np; ++p) {
            uint32_t acc = 0u;
            iss.begin(__ldg(tab + 5 + 4 * (stage + p)));
            iss.block(kD + 64 * p, 0, NCH, 0, __ldg(tab + 6 + 4 * (stage + p)), acc);
            iss.end();
          }
        }
        SBI_TL(1000 * (li + 1) + 40);
        for (int p = 0; p < np; ++p) {
          const int aux = __ldg(tab + 7 + 4 * (stage + p));
          const int f0 = aux & 0xffff, nf = aux >> 16;
          for (int f = 0; f < nf; ++f) {
            if (((f0 + f) & (TPR - 1)) != tq) continue;     // warp-uniform: features go round-robin over the parts
            float q[32];
            ld_cols<4, RPC>(row, kD + 64 * (p & 1) + 32 * f, q, accs);
            const float* bff = bf + (f0 + f) * 32;
#pragma unroll
            for (int i = 0; i < 32; ++i) q[i] = (i < 3 * KB - 1) ? q[i] + bff[i] : 0.f;
            if (SAVE) tc_save_prm(svl + SV.prm, srow, m.TRmax, f0 + f, q);
            const int j = __ldg(v.trf + f0 + f);
            const float x = zs[j * RPC + row];
            float y, ld;
            if (INV) rqs_inverse_fast<KB>(q, rc, x, y, ld);
            else rqs_forward_fast<KB>(q, rc, x, y, ld);
            zs[j * RPC + row] = y;
            if (TPR == 2) ldacc += ld;
            else ldf[(f0 + f) * RPC + row] = ld;
          }
          SBI_TL(1000 * (li + 1) + 41 + p);
          if (p + 2 < np) {
            // region p&1 has been read by everyone: pass p+2 may overwrite it
            group_sync();
            {
              uint32_t acc = 0u;
              iss.begin(__ldg(tab + 5 + 4 * (stage + p + 2)));
              iss.block(kD + 64 * (p & 1), 0, NCH, 0, __ldg(tab + 6 + 4 * (stage + p + 2)), acc);
              iss.end();
            }
          }
        }
      }

      // ---- LULinear on the row (part 1: it has one spline feature less, and it also writes the
      //      next layer's identity columns):  z <- L (U z) + b, in place ----
      group_sync();      // all parts' spline outputs are in zs
      SBI_TL(1000 * (li + 1) + 50);
      if (TPR > 2 && tq < 2)      // parts 0 / 1 take the even / odd features' log|det|, in feature order
        for (int k = tq; k < v.n_tr; k += 2) ldacc += ldf[k * RPC + row];
      if (SAVE && tq == 1) tc_save_row16<RPC>(svl + SV.v, srow, zs, row, D);         // coupling output v_l
      if (!INV && tq == 1 && __ldg(v.LT + SBI_L_HAS_LU)) {
        const float4* U4 = reinterpret_cast<const float4*>(sm + L.lum);
        const float4* L4 = U4 + kLuMax * kLuMax / 4;
        const float* bias = sm + L.lum + 2 * kLuMax * kLuMax;
        float zr[kLuMax];
#pragma unroll
        for (int j = 0; j < kLuMax; ++j) zr[j] = (j < D) ? zs[j * RPC + row] : 0.f;
        // y = U z (upper triangular incl. diagonal; padded entries are zero), same j order as
        // lu_forward (nsf.cuh)
#pragma unroll
        for (int i = 0; i < kLuMax; ++i) {
          if (i < D) {
            float a = 0.f;
#pragma unroll
            for (int j4 = i / 4; j4 < kLuMax / 4; ++j4) {
              const float4 w = U4[i * (kLuMax / 4) + j4];
              if (4 * j4 + 0 >= i) a = fmaf(w.x, zr[4 * j4 + 0], a);
              if (4 * j4 + 1 >= i) a = fmaf(w.y, zr[4 * j4 + 1], a);
              if (4 * j4 + 2 >= i) a = fmaf(w.z, zr[4 * j4 + 2], a);
              if (4 * j4 + 3 >= i) a = fmaf(w.w, zr[4 * j4 + 3], a);
            }
            zr[i] = a;
          }
        }
        // z = L y + b (strictly lower), rows from the bottom so that y_j (j < i) is still intact
#pragma unroll
        for (int i = kLuMax - 1; i >= 0; --i) {
          if (i < D) {
            float a = zr[i];
#pragma unroll
            for (int j4 = 0; j4 <= (i - 1) / 4 && i > 0; ++j4) {
              const float4 w = L4[i * (kLuMax / 4) + j4];
              if (4 * j4 + 0 < i) a = fmaf(w.x, zr[4 * j4 + 0], a);
              if (4 * j4 + 1 < i) a = fmaf(w.y, zr[4 * j4 + 1], a);
              if (4 * j4 + 2 < i) a = fmaf(w.z, zr[4 * j4 + 2], a);
              if (4 * j4 + 3 < i) a = fmaf(w.w, zr[4 * j4 + 3], a);
            }
            zr[i] = a + bias[i];
            zs[i * RPC + row] = zr[i];
          }
        }
      }
    }

    // ---- base density ----
    SBI_TL(9000);
    if (tq == 0) lds[row] = ldacc;
    group_sync();
    if (tq == 1 && row0 + row < rows.R) {
      if (!INV) {
        float ss = 0.f;
        for (int d = 0; d < D; ++d) ss = fmaf(zs[d * RPC + row], zs[d * RPC + row], ss);
        const float lp = -0.5f * ss + (lds[row] + ldacc) + ld_const;
        if (logp != nullptr) logp[row0 + row] = lp;
        if (SAVE) {
          tc_save_row16<RPC>(save + (size_t)tile * SV.tile_stride + SV.zt, srow, zs, row, D);
          float* lpt = save + (size_t)tile * SV.tile_stride + SV.lp;
          lpt[srow] = lp;
        }
        if (noise != nullptr)
          for (int d = 0; d < D; ++d) noise[(row0 + row) * D + d] = zs[d * RPC + row];
      } else {
        const float* st = m.d_stats;
        for (int d = 0; d < D; ++d)
          noise[(row0 + row) * D + d] = (zs[d * RPC + row] - __ldg(st + d)) / __ldg(st + m.Dp + d);
        if (logp != nullptr) logp[row0 + row] = (lds[row] + ldacc) + ld_const;
      }
    }
    group_sync();   // rows of the next tile are written cooperatively
  }

  tc_end(ncols, sa);
}

// the accumulator store of every tensor-core kernel of the library (tc_common.cuh)
static __device__ float g_store[kStoreSlots][kStoreCols * kStoreLanes];
static __device__ unsigned int g_store_mask[kStoreSlots];

int store_args(StoreArgs* out) {
  static StoreArgs cache[kMaxDev];
  static bool ready[kMaxDev] = {false};
  const int d = cur_dev();
  if (!ready[d]) {
    cudaError_t e = cudaGetSymbolAddress(reinterpret_cast<void**>(&cache[d].slab), g_store);
    if (e == cudaSuccess) e = cudaGetSymbolAddress(reinterpret_cast<void**>(&cache[d].mask), g_store_mask);
    if (e != cudaSuccess) return (int)e;
    ready[d] = true;
  }
  *out = cache[d];
  return 0;
}

}  // namespace tc
}  // namespace sbi

// =================================================================================================
// C ABI
// =================================================================================================
using namespace sbi;

extern "C" int sbi_b200_nsf_tc_supported(const sbi_nsf_model* m, const sbi_nsf_tc* tc) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc) return 0;
  if (m->head != SBI_NSF_SPLINE || m->cond_mlp) return 0;   // spline coupling flow with the ResidualNet conditioner
  if (m->H != 50 || m->KB != 10) return 0;        // instantiated hidden width / bin count
  if (m->H + m->C > 64) return 0;                 // context rides in the hidden operand's K range
  if (m->IDp > 48 || m->PR > 32 || m->D > tc::kLuMax) return 0;
  if (m->NB < 1 || m->NB > SBI_NSF_MAX_BLOCKS) return 0;
  if (tc->stage_cap <= 0 || (tc->stage_cap & 31) || tc->n_words <= 0) return 0;
  // the weight ring has to fit next to a second CTA on the SM
  return tc::tc_smem_layout(*m, tc->stage_cap, false).total_bytes <= 112 * 1024 ? 1 : 0;
}

extern "C" int sbi_b200_nsf_tc_pack(const sbi_nsf_model* m, const sbi_nsf_tc* tc, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  return m ? tc::pack_weights(m->d_params, tc, (cudaStream_t)stream) : SBI_EINVAL;
}

extern "C" int sbi_b200_nsf_logprob_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc,
                                       const sbi_rows* rows, float* d_logp, float* d_noise,
                                       void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc || !rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_logp)
    return SBI_EINVAL;
  if (!tc->d_tab || !tc->d_tcw) return SBI_EINVAL;
  if (!sbi_b200_nsf_tc_supported(m, tc)) return SBI_ESMEM;
  if (rows->R == 0) return 0;
  tc::StoreArgs sa;
  if (int e = tc::store_args(&sa)) return e;
  return launch(tc::nsf_logprob_tc_kernel<50, 10, false>, tile_grid(rows->R, tc::kRows, 2), tc::kThreads,
                tc::tc_smem_layout(*m, tc->stage_cap, false).total_bytes, (cudaStream_t)stream, *m, *tc, *rows, d_logp,
                d_noise, nullptr, sa);
}

int sbi::tc::launch_forward_save(const sbi_nsf_model* m, const sbi_nsf_tc* tc, const sbi_rows* rows, float* d_logp,
                                 float* d_save, bool half_tiles, cudaStream_t s) {
  tc::StoreArgs sa;
  if (int e = tc::store_args(&sa)) return e;
  // one tile per CTA (`d_save` slab = blockIdx), or two CTAs per tile (slab = blockIdx / 2)
  const int tiles = (int)((rows->R + tc::kRows - 1) / tc::kRows);
  if (half_tiles)
    return launch(tc::nsf_logprob_tc_kernel<50, 10, false, true, 64>, 2 * tiles, tc::kThreads,
                  tc::forward_save_smem_bytes(*m, *tc, 64), s, *m, *tc, *rows, d_logp, nullptr, d_save, sa);
  return launch(tc::nsf_logprob_tc_kernel<50, 10, false, true>, tiles, tc::kThreads,
                tc::forward_save_smem_bytes(*m, *tc, tc::kRows), s, *m, *tc, *rows, d_logp, nullptr, d_save, sa);
}

int sbi::tc::forward_save_smem_bytes(const sbi_nsf_model& m, const sbi_nsf_tc& tc, int rpc) {
  return tc::tc_smem_layout(m, tc.stage_cap, true, rpc).total_bytes;
}

extern "C" int sbi_b200_nsf_inverse_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc,
                                       const sbi_rows* rows, float* d_out, float* d_logabsdet,
                                       void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc || !rows || !rows->d_input || !rows->d_cond || rows->R < 0 || !d_out)
    return SBI_EINVAL;
  if (!tc->d_tab || !tc->d_tcw) return SBI_EINVAL;
  if (!sbi_b200_nsf_tc_supported(m, tc)) return SBI_ESMEM;
  if (rows->R == 0) return 0;
  tc::StoreArgs sa;
  if (int e = tc::store_args(&sa)) return e;
  return launch(tc::nsf_logprob_tc_kernel<50, 10, true>, tile_grid(rows->R, tc::kRows, 2), tc::kThreads,
                tc::tc_smem_layout(*m, tc->stage_cap, false).total_bytes, (cudaStream_t)stream, *m, *tc, *rows, d_logabsdet,
                d_out, nullptr, sa);
}

#ifdef SBI_TC_TIMELINE
// tuning builds only: copy out and reset the phase timeline of CTA 0; returns the number of (id, clock) pairs
extern "C" int sbi_b200_debug_timeline_fwd(unsigned long long* out, int cap) {
  int n = 0;
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(&n, sbi::tc::g_tl_n, sizeof(int));
  if (n > cap) n = cap;
  cudaMemcpyFromSymbol(out, sbi::tc::g_tl, (size_t)n * 2 * sizeof(unsigned long long));
  const int zero = 0;
  cudaMemcpyToSymbol(sbi::tc::g_tl_n, &zero, sizeof(int));
  return n;
}
#endif
