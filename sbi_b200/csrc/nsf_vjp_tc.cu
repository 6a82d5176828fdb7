// Tensor-core training step of the neural spline flow: backward sweep of
//   loss = sum_r g_r log q(theta_r | x_r)      (NFlowsFlow.loss + autograd backward,
//   /root/reference/sbi/neural_nets/estimators/nflows_flow.py:99-109,
//   /root/reference/sbi/inference/trainers/base.py:1171-1180)
// for the parameter gradients, on the activations the tensor-core forward sweep
// (nsf_logprob_tc_kernel<..., SAVE = true>, nsf_tc.cu) left in the activation scratch
// (nsf_tc_save.cuh).  Replaces nsf_vjp_kernel (nsf.cu, FP32 SIMT) when only parameter gradients
// are asked for -- the trainer's case.  Two kernels per chunk of rows, after the forward sweep:
//
// nsf_vjp_tc_kernel: the chain of the backward sweep, which each layer waits on.  One CTA = 8 warps owns a
// tile of 128 rows (row = store lane, two threads per row splitting the columns), walks the layers
// T-1 .. 0 and, per layer, the linears of the conditioner (nflows ResidualNet, restated in
// oracle/nflows_port/nn/nets/resnet.py) in reverse:
//
//   * input-gradient chain  dX = dY W  on wgmma kind tf32 (both warpgroups, 64 rows each): A = dY from
//     the shared-memory A region of tc_common.cuh (written by the row threads, 3xTF32 hi/lo split), two
//     K-steps in flight, the accumulators in the accumulator store (in shared memory on half tiles); B = W^T
//     streamed by TMA bulk copies from the
//     pre-transposed operand blocks (pack.NsfLayout.tc_bwd_plan) through a 2-slot ring; relu / GLU
//     masks, the spline backward (rqs.cuh) and the LULinear input gradient are per-thread code on the
//     thread's own row between the MMAs;
//   * the output gradient dY of every linear goes to the dY region of the activation scratch, and the gradient
//     dz at every LULinear output below the top layer to the prm region of the layer above (nsf_tc_save.cuh),
//     where the weight-gradient kernel picks them up;
//   * COND instantiation only: the condition gradient d(sum g log q)/d ctx in raw condition space, accumulated
//     per row over the T layers from the context columns of the initial layer (dh W0[:, :C]) and the GLU
//     context layer of every residual block (dG Wc).  dh / dG of the whole row are read back from the dY region
//     after the CTA barrier that follows their write, so each of the row's threads takes its share of the C
//     features over all H columns, on the CUDA cores from the fp32 parameters (C is small next to H), and
//     accumulates them in place in d_gcond: every entry has one owner thread and a fixed summation order.
//
// nsf_dw_tc_kernel: the weight gradients  dW = dY^T X  (K = the 128 rows of a tile), which no layer waits on,
// so they run on every SM instead of the one SM per tile of the chain.  One CTA per (tile, layer, linear):
// the row threads write dY^T (dY region) and X^T (saved activations, the context, the identity features)
// into K-major staging buffers ([row/4][feature][row%4], one padding row per slab so that the 32 rows of a
// warp hit 32 banks) and one M = 64 MMA chain of 16 K-steps multiplies them (single TF32 pass: the sum over
// rows averages the operand rounding; the two warpgroups split N); a ones row appended to X^T yields the bias
// gradient in the same MMA.  The accumulators are written into a shared-memory image laid out like the block
// in the parameter buffer, and ONE thread sends it to the tile's partial-gradient slab with two TMA bulk
// copies (a reducing copy for every chunk after the first).  One more CTA per (tile, layer) takes the LULinear
// parameter gradients: dot products over the tile's 128 rows of dz, y = U v, dy = dz + L^T dz and v, on the
// CUDA cores (D^2 + D sums of 128 terms).
//
// Accumulator columns of the backward (128): [0,64) D | [64,128) G, in the store on whole tiles and in shared
// memory on half tiles.  One A set serves every MMA: each pass's MMAs complete (wgmma wait) before the CTA
// barrier of Issuer::end(), and the next operands are written after it.
//
// Half tiles (RPC = 64, when a chunk of tiles would leave SMs idle): two CTAs per tile, CTA r owning tile rows
// [64 r, 64 r + 64) with four threads per row (the layout of the forward's half tiles, nsf_tc.cu).  Everything
// the backward computes is per row, so the two CTAs never talk to each other.
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

constexpr int kBwdSlots = 2;
constexpr int kStLd = 65;                       // feature rows per K-slab of a staging buffer (64 + 1 pad)
constexpr int kStFloats = 32 * kStLd * 4;       // [128 rows / 4][65][4]

struct BwdSmem {
  int dz, gr, lum, a, acc, ring;   // float offsets
  int bar_bytes, total_bytes;
};
// rpc: rows per CTA (128, or 64 for half tiles, which also keep their accumulator columns here)
__host__ __device__ inline BwdSmem bwd_smem_layout(int stage_cap, int rpc) {
  BwdSmem L;
  int fl = 0;
  L.dz = fl;  fl += 16 * rpc;
  L.gr = fl;  fl += rpc;
  L.lum = fl; fl += 2 * kLuMax * kLuMax + 2 * kLuMax;
  fl = (fl + 31) & ~31;
  L.a = fl;   fl += a_smem_floats(rpc);           // A_hi | A_lo (tc_common.cuh)
  L.acc = fl; fl += rpc < kRows ? acc_smem_floats() : 0;
  L.ring = fl; fl += kBwdSlots * stage_cap;
  L.bar_bytes = fl * 4;
  L.total_bytes = L.bar_bytes + kBwdSlots * 8;
  return L;
}
// ldmax: longest packed weight row (floats) of the model, max(Hp, Cp + IDp, Cp)
__host__ __device__ inline int dw_ldmax(const sbi_nsf_model& m) {
  int a = m.Hp > m.Cp + m.IDp ? m.Hp : m.Cp + m.IDp;
  return a > m.Cp ? a : m.Cp;
}
// weight-gradient kernel: staging buffers A' | B', then the output image [<= 64 rows][ld] + its bias row
__host__ __device__ inline int dw_smem_bytes(const sbi_nsf_model& m) {
  return (2 * kStFloats + 64 * dw_ldmax(m) + 64) * 4;
}
// work units of the weight-gradient kernel per (tile, layer) (TcSave::units)
__host__ __device__ inline int dw_units(const sbi_nsf_model& m) { return tc_save_layout(m.NB, m.TRmax, m.T).units(); }

// where the accumulators of one weight-gradient MMA go in the partial-gradient slab
struct DwGeo {
  int oW, ldw;     // weight block: entry (m, n) at oW + m * ldw + n for n < nX   (ldw % 4 == 0, oW % 4 == 0)
  int oB;          // bias: entry m at oB + m   (column `ones` of the accumulator)
  int nX, ones;    // X columns that are weight columns; index of the ones column
  int Mv, N;       // rows of the block incl. zero padding rows (Mv % 4 == 0); accumulator columns (multiple of 16)
};

// dW = A'^T-staged dY (M = 64 feature rows) x B'-staged X (N = 2 NH feature rows), K = 128 tile rows ->
// the shared-memory image of the block, laid out exactly like the block in the parameter buffer ([Mv][ldw]
// weights, then the Mv bias entries).  Columns >= nX of a row are padding and take a zero gradient.
template <int NH>
__device__ __forceinline__ void dw_mma_image(const float* As, const float* Bs, const DwGeo& g, float* obuf) {
  const uint64_t da = make_bdesc(smem_u32(As), kStLd * 16u, 128u);
  const uint64_t db = make_bdesc(smem_u32(Bs), kStLd * 16u, 128u);
  float d[NH / 2];
  mma_ss64_n<NH>(d, da, db, (uint64_t)((2u * kStLd * 16u) >> 4), kRows / 8);
  const int lane = threadIdx.x & 31;
  const int m0 = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  const int n0 = (threadIdx.x >> 7) * NH + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < NH / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int mr = m0 + 8 * (e >> 1), n = n0 + 8 * j + (e & 1);
      const float val = d[4 * j + e];
      if (mr < g.Mv) {
        if (n < g.ldw) obuf[mr * g.ldw + n] = n < g.nX ? val : 0.f;
        if (n == g.ones) obuf[g.Mv * g.ldw + mr] = val;
      }
    }
  }
}

__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void red_add_gpu(unsigned* p, unsigned v) {
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// On half tiles (the chunk leaves SMs idle) it is launched right behind the backward sweep with programmatic
// stream serialization: it may start once every backward CTA has run griddepcontrol.launch_dependents, and
// each CTA waits for its own unit's dY instead of for the whole backward grid.  Its CTAs are then numbered in
// the order the backward produces their dY: layer T-1 .. 0, then the unit in write order (the LULinear, whose dz
// the backward publishes after the layer's LU section, final-layer passes, blocks NB-1 .. 0 with GLU context,
// W2, W1, the initial linear), then the tile, so the CTAs dispatched first are the first to find their unit
// ready.  On whole tiles every SM runs a backward CTA, so it is an ordinary launch after the backward (`upt` = 0:
// no wait) with the CTAs tile-major.  Every unit writes a disjoint block of its tile's partial-gradient slab, so
// neither order changes a value.
// The wait cannot deadlock:
//   * the grid launches only after every backward CTA has run launch_dependents, so the whole backward
//     grid is resident (one CTA per SM: the chunk never has more backward CTAs than SMs);
//   * the backward never waits on this kernel, so every counter reaches its count.
// A backward CTA takes its SM's whole register file (255 registers x 256 threads), so these CTAs run only on
// SMs the backward does not use, or after its CTA there has exited: they never take issue slots from it.
// The dY loads are ld.global.cg (L2, coherent) after an acquire of the counter and a CTA barrier; nothing
// the backward writes is read through the non-coherent path.  The counters start at zero in every run --
// graph replays included -- because the forward sweep of the same chunk zeroes them, and stream order puts
// that forward after the previous chunk's (or step's) weight-gradient kernel and before this backward.
// `upt`: the count at which a unit is ready (2, one per CTA of the tile, on half tiles; 0 on whole tiles).
// `gout` / `g_const`: the row weights of the chunk's rows, as given to the backward sweep.
template <int H>
__global__ void __launch_bounds__(kThreads, 2)
nsf_dw_tc_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_rows rows,
                 const float* __restrict__ save, float* __restrict__ gpart, int accum, unsigned upt,
                 const float* __restrict__ gout, float g_const) {
  constexpr int HP8 = (H + 7) & ~7;
  constexpr int NC = HP8 / 2;
  static_assert(HP8 <= kDyCols, "the dY columns from kDyCols on hold the ready counters");
  extern __shared__ __align__(128) float sm[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int half = warp >> 2;
  const int row = ((warp & 3) << 5) | lane;
  const int cbase = half * NC;
  const int q_one = H - cbase;                 // this thread's column that is X column H (the ones column)
  const int C = m.C, Cp = m.Cp, Hp = m.Hp;
  const TcSave SV = tc_save_layout(m.NB, m.TRmax, m.T);
  const int nu = SV.units(), npm = SV.npm;
  int64_t tile;
  int l, u;
  if (upt > 0) {
    const int ntiles = gridDim.x / (nu * m.T);
    const int j = (blockIdx.x / ntiles) % nu - 1;  // unit in write order, the LULinear (-1) first
    tile = blockIdx.x % ntiles;
    l = m.T - 1 - (int)(blockIdx.x / (ntiles * nu));
    u = j < 0 ? SV.lu_unit()
              : j < npm || j == npm + 3 * m.NB ? j : npm + 3 * (m.NB - 1 - (j - npm) / 3) + (j - npm) % 3;
  } else {
    // after the backward: tile-major, so that the CTAs running together read and write one tile's slabs
    tile = blockIdx.x / (nu * m.T);
    l = (blockIdx.x / nu) % m.T;
    u = blockIdx.x % nu;
  }
  const NsfLayerView v = layer_view(m, l);
  if (u < npm && v.n_tr <= 2 * u) return;      // (CTA-uniform) this layer has fewer final-layer passes
  const float* svl = save + (size_t)tile * SV.tile_stride + (size_t)l * SV.layer_stride;
  const int64_t gr = tile * kRows + row;
  const bool live = gr < rows.R;               // rows past the end of the batch contribute nothing
  float* As = sm;
  float* Bs = sm + kStFloats;
  float* obuf = sm + 2 * kStFloats;
  auto st_put = [&](float* buf, int n, float val) { buf[((row >> 2) * kStLd + n) * 4 + (row & 3)] = val; };
  // context feature n < C of the row, standardised like load_rows (stages.cuh)
  auto ctx = [&](int n) {
    const int64_t src = rows.cond_shared ? 0 : (rows.d_index ? __ldg(rows.d_index + gr) : gr);
    return (__ldg(rows.d_cond + src * C + n) - __ldg(m.d_stats + 2 * m.Dp + n)) / __ldg(m.d_stats + 2 * m.Dp + Cp + n);
  };
  // A' = dY^T: the thread's NC hidden columns
  auto put_dy = [&](int off) {
    float a[NC];
    tc_load_cols<NC>(svl + off, row, half, a);
#pragma unroll
    for (int q = 0; q < NC; ++q) st_put(As, cbase + q, live ? a[q] : 0.f);
  };
  // B' = X^T from a saved [128][64] activation array, ones column at H
  auto put_x = [&](int off, bool relu) {
    float x[NC];
    tc_load_cols<NC>(svl + off, row, half, x);
#pragma unroll
    for (int q = 0; q < NC; ++q) st_put(Bs, cbase + q, !live ? 0.f : q == q_one ? 1.f : relu ? relu_f(x[q]) : x[q]);
  };

  // X comes from the forward sweep and the condition; dY only after the backward has counted the unit ready
  auto wait_ready = [&]() {
    if (tid == 0 && upt > 0) {
      const unsigned* rdy = reinterpret_cast<const unsigned*>(svl + SV.ready()) + u;
      unsigned ns = 32;
      while (ld_acquire_gpu(rdy) < upt) {
        __nanosleep(ns);
        ns = min(2 * ns, 512u);
      }
    }
    __syncthreads();
  };

  if (u == SV.lu_unit()) {
    // ---- LULinear (y = U v, z' = L y + b): parameter gradients summed over the tile's 128 rows, each in the
    //      order of lu_backward (nsf.cu).  It returns before the end of the kernel: in production order it is
    //      never the grid's last CTA, and on whole tiles (tile-major, an ordinary launch) that CTA waits for nothing.
    if (!__ldg(v.LT + SBI_L_HAS_LU)) return;
    static_assert(4 * kLuMax * kRows + kRows + 2 * kLuMax * kLuMax + 2 * kLuMax <= 2 * kStFloats, "LU unit");
    const int D = m.D;
    float* DZ = sm;                  // feature-major [16][128]: dz, y, dy, v; then the row weights and U | L
    float* Y = DZ + kLuMax * kRows;
    float* DY = Y + kLuMax * kRows;
    float* V = DY + kLuMax * kRows;
    float* GR = V + kLuMax * kRows;
    float* U = GR + kRows;
    const float* Lw = U + kLuMax * kLuMax;
    const float g = live ? (gout ? __ldg(gout + gr) : g_const) : 0.f;
    prep_lu(m, l, U);
    // dz of the top layer is d(sum g log q)/dz_T = -g z_T; below it, the backward writes dz as it enters the layer
    if (l < m.T - 1) wait_ready();
    else __syncthreads();
    if (half == 0) {
      float vr[kLuMax];
      tc_load_row16(svl + SV.v, row, vr);
#pragma unroll
      for (int i = 0; i < kLuMax; ++i) {
        float y = 0.f;
#pragma unroll
        for (int j = 0; j < kLuMax; ++j)
          if (j >= i) y = fmaf(U[i * kLuMax + j], vr[j], y);        // padded entries are zero
        if (i < D) {
          V[i * kRows + row] = vr[i];
          Y[i * kRows + row] = y;
        }
      }
      GR[row] = g;
    } else {
      float dzr[kLuMax];
      if (l == m.T - 1) {
        tc_load_row16(save + (size_t)tile * SV.tile_stride + SV.zt, row, dzr);
#pragma unroll
        for (int i = 0; i < kLuMax; ++i) dzr[i] = live ? -g * dzr[i] : 0.f;
      } else {
        tc_load_row16(svl + SV.layer_stride + SV.dz_below(), row, dzr);
      }
#pragma unroll
      for (int i = 0; i < kLuMax; ++i) dzr[i] = (i < D) ? dzr[i] : 0.f;
      // dy = dz + L^T dz (strictly lower part)
#pragma unroll
      for (int i = 0; i < kLuMax; ++i) {
        float dy = dzr[i];
#pragma unroll
        for (int j = 0; j < kLuMax; ++j)
          if (j > i) dy = fmaf(Lw[j * kLuMax + i], dzr[j], dy);
        if (i < D) {
          DZ[i * kRows + row] = dzr[i];
          DY[i * kRows + row] = dy;
        }
      }
    }
    __syncthreads();
    // one (i,j) pair per thread; four independent partial sums; the lanes of a warp read different feature rows
    // (same bank at the same offset), so entry t starts 4 (t % 32) rows in
    float* gp = gpart + (size_t)tile * m.n_params;
    const int o_lo = __ldg(v.LT + SBI_L_LU_LOWER), o_up = __ldg(v.LT + SBI_L_LU_UPPER);
    const int o_dg = __ldg(v.LT + SBI_L_LU_DIAG), o_bi = __ldg(v.LT + SBI_L_LU_BIAS);
    for (int t = tid; t < D * D + D; t += kThreads) {
      const int rot = 4 * (t & 31);
      auto dot = [&](const float* p, const float* q) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
        for (int r = 0; r < kRows; r += 4) {
          const int rr = (r + rot) & (kRows - 1);
          const float4 x4 = *reinterpret_cast<const float4*>(p + rr);
          const float4 y4 = *reinterpret_cast<const float4*>(q + rr);
          a0 = fmaf(x4.x, y4.x, a0); a1 = fmaf(x4.y, y4.y, a1);
          a2 = fmaf(x4.z, y4.z, a2); a3 = fmaf(x4.w, y4.w, a3);
        }
        return (a0 + a1) + (a2 + a3);
      };
      auto rsum = [&](const float* p) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
        for (int r = 0; r < kRows; r += 4) {
          const float4 x4 = *reinterpret_cast<const float4*>(p + ((r + rot) & (kRows - 1)));
          a0 += x4.x; a1 += x4.y; a2 += x4.z; a3 += x4.w;
        }
        return (a0 + a1) + (a2 + a3);
      };
      float a;
      float* dst;
      if (t < D * D) {
        const int i = t / D, j = t % D;
        if (i > j) {
          a = dot(DZ + i * kRows, Y + j * kRows);
          dst = gp + o_lo + i * (i - 1) / 2 + j;
        } else if (i < j) {
          a = dot(DY + i * kRows, V + j * kRows);
          dst = gp + o_up + i * D - i * (i + 1) / 2 + (j - i - 1);
        } else {
          a = dot(DY + i * kRows, V + i * kRows);
          const float gs = rsum(GR);
          a = (a + gs / U[i * kLuMax + i]) * sigmoid_f(__ldg(m.d_params + o_dg + i));
          dst = gp + o_dg + i;
        }
      } else {
        const int i = t - D * D;
        a = rsum(DZ + i * kRows);
        dst = gp + o_bi + i;
      }
      *dst = accum ? (*dst + a) : a;
    }
    // the arrays are padded to a multiple of 4 entries: padding takes a zero gradient (every entry of the slab is
    // written by this kernel; nothing is zero-filled beforehand)
    if (!accum && tid >= kThreads - 4) {
      const int k = tid - (kThreads - 4);
      const int ntri = D * (D - 1) / 2;
      const int o = k == 0 ? o_lo : k == 1 ? o_up : k == 2 ? o_dg : o_bi;
      const int n = k < 2 ? ntri : D;
      for (int e = n; e < ((n + 3) & ~3); ++e) gp[o + e] = 0.f;
    }
    return;
  }
  DwGeo g;
  if (u < npm) {
    // ---- final layer, pass u: dW of the parameter rows of features 2u, 2u+1; X = the final-layer input
    const int nf = min(2, v.n_tr - 2 * u);
    put_x(SV.hf, false);
    wait_ready();
    if (half < nf) {
      float a[32];
      tc_load_prm(svl + SV.dy_fin(u), row, 0, half, a);
#pragma unroll
      for (int i = 0; i < 32; ++i) st_put(As, 32 * half + i, live ? a[i] : 0.f);
    }
    g.oW = __ldg(v.LT + SBI_L_WF) + 2 * u * m.PR * Hp; g.ldw = Hp; g.oB = __ldg(v.LT + SBI_L_BF) + 2 * u * m.PR;
    g.nX = H; g.ones = H; g.Mv = 32 * nf; g.N = 64;
  } else if (u < npm + 3 * m.NB) {
    const int b = (u - npm) / 3, k = (u - npm) % 3;
    const int* BT = v.LT + SBI_L_BLK0 + 6 * b;
    if (k == 0) {
      // ---- dWc = dG^T ctx  (GLU gate)
      const int Nc = (Cp + 1 + 15) & ~15;
      for (int n = half * (Nc / 2); n < (half + 1) * (Nc / 2); ++n)
        st_put(Bs, n, !live ? 0.f : n < C ? ctx(n) : (n == Cp ? 1.f : 0.f));
      g.oW = __ldg(BT + 4); g.ldw = Cp; g.oB = __ldg(BT + 5); g.nX = Cp; g.ones = Cp; g.Mv = Hp; g.N = Nc;
    } else if (k == 1) {
      // ---- dW2 = dT^T a1
      put_x(SV.a1(b), false);
      g.oW = __ldg(BT + 2); g.ldw = Hp; g.oB = __ldg(BT + 3); g.nX = H; g.ones = H; g.Mv = Hp; g.N = 64;
    } else {
      // ---- dW1 = dA1^T relu(h_b)
      put_x(SV.h(b), true);
      g.oW = __ldg(BT + 0); g.ldw = Hp; g.oB = __ldg(BT + 1); g.nX = H; g.ones = H; g.Mv = Hp; g.N = 64;
    }
    wait_ready();
    put_dy(SV.dy_blk(b, k));
  } else {
    // ---- initial layer: dW0 = dh^T [ctx | id | 1]
    const int K0p = Cp + m.IDp;
    const int N0 = (K0p + 1 + 15) & ~15;
    for (int n = half * (N0 / 2); n < (half + 1) * (N0 / 2); ++n) {
      float val = 0.f;
      if (!live) val = 0.f;
      else if (n < Cp) val = n < C ? ctx(n) : 0.f;
      else if (n < K0p) {
        const int i = n - Cp;
        if (i < v.n_id) val = tc_load_row16_at(svl + SV.zin, row, __ldg(v.idf + i));
      } else if (n == K0p) val = 1.f;
      st_put(Bs, n, val);
    }
    g.oW = __ldg(v.LT + SBI_L_W0); g.ldw = K0p; g.oB = __ldg(v.LT + SBI_L_B0); g.nX = K0p; g.ones = K0p;
    g.Mv = Hp; g.N = N0;
    wait_ready();
    put_dy(SV.dy_init());
  }
  fence_async_smem();
  __syncthreads();
  switch (g.N) {
    case 16: dw_mma_image<8>(As, Bs, g, obuf); break;
    case 32: dw_mma_image<16>(As, Bs, g, obuf); break;
    case 48: dw_mma_image<24>(As, Bs, g, obuf); break;
    case 64: dw_mma_image<32>(As, Bs, g, obuf); break;
    default: __trap();      // weight-gradient blocks are planned with N in {16, 32, 48, 64}
  }
  fence_async_smem();
  __syncthreads();
  if (tid == 0) {
    float* gp = gpart + (size_t)tile * m.n_params;
    bulk_s2g(gp + g.oW, obuf, (uint32_t)(g.Mv * g.ldw) * 4u, accum != 0);
    bulk_s2g(gp + g.oB, obuf + g.Mv * g.ldw, (uint32_t)g.Mv * 4u, accum != 0);
    bulk_commit();
    bulk_wait_all();
  }
  // the last CTA (its unit is among the last the backward writes) holds the grid open until the backward grid
  // has completed, so that stream work after this kernel also finds the backward's other outputs (condition
  // gradients, loss statistics) in memory
  if (blockIdx.x == gridDim.x - 1) asm volatile("griddepcontrol.wait;" ::: "memory");
}

template <int H, int RPC, int KB, bool COND>
__global__ void __launch_bounds__(kThreads, 1)
nsf_vjp_tc_kernel(const __grid_constant__ sbi_nsf_model m, const __grid_constant__ sbi_nsf_tc tcb,
                  const __grid_constant__ sbi_rows rows, const float* __restrict__ gout, float g_const,
                  float* __restrict__ loss_acc, float* __restrict__ save, const StoreArgs sa,
                  float* __restrict__ dcond) {
  constexpr int HP8 = (H + 7) & ~7;
  constexpr int NCH = HP8 / 8;
  constexpr int TPR = kThreads / RPC;                   // threads per row
  constexpr int UPT = kRows / RPC;                      // CTAs per tile
  constexpr int NC = TPR == 2 ? HP8 / 2 : 16;           // columns per thread ([tq NC, tq NC + NC))
  constexpr int NG = NC / 4;
  static_assert(HP8 % 8 == 0 && NC % 4 == 0 && H > (TPR - 1) * NC && H < HP8 + 1 && HP8 <= kDyCols, "hidden width");
  extern __shared__ __align__(128) float sm[];
  const BwdSmem L = bwd_smem_layout(tcb.stage_cap, RPC);
  uint64_t* full = reinterpret_cast<uint64_t*>(reinterpret_cast<char*>(sm) + L.bar_bytes);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int C = m.C, D = m.D;
  const int64_t nunits = (rows.R + kRows - 1) / kRows * UPT;     // CTA tiles of RPC rows
  const TcSave SV = tc_save_layout(m.NB, m.TRmax, m.T);

  // whole tiles: D | G in the store; half tiles: in shared memory
  constexpr int ncols = RPC < kRows ? 0 : kColsDG;
  float* as = sm + L.a;
  float* accs = sm + L.acc;
  SBI_TL(10);
  IssuerT<kBwdSlots, true, RPC> iss =
      tc_begin<kBwdSlots, true, RPC>(full, sm + L.ring, tcb, m.T, nunits, true, ncols, sa, as, accs);
  // half tiles: the weight-gradient kernel may start once every CTA of this grid is resident (it waits per unit)
  if constexpr (UPT > 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  SBI_TL(100);

  const float* __restrict__ P = m.d_params;
  float* dzs = sm + L.dz;
  float* GRs = sm + L.gr;
  const int tq = warp / (RPC / 32);                        // which column part of the row
  const int row = ((warp % (RPC / 32)) << 5) | lane;       // row of the CTA = store lane
  const int cbase = tq * NC;
  RqsConst rc = rqs_const(m);
  rc.K = KB;
  // condition gradient: features [c_lo, c_hi) of this thread's row; dY = the row's dY columns at `dy`
  // (written by all threads of the row before the CTA barrier that precedes the call)
  const int c_part = (C + TPR - 1) / TPR;
  const int c_lo = tq * c_part, c_hi = min(C, c_lo + c_part);
  auto dctx_add = [&](const float* dy, const float* W, int ldw, int64_t row0, int srow) {
    if (row0 + row >= rows.R) return;
    const float* csd = m.d_stats + 2 * m.Dp + m.Cp;
    float* out = dcond + (row0 + row) * C;
    for (int c = c_lo; c < c_hi; ++c) {
      float a = 0.f;
      for (int n = 0; n < H; ++n) a = fmaf(__ldcg(dy + ((n >> 2) * kRows + srow) * 4 + (n & 3)), __ldg(W + n * ldw + c), a);
      out[c] += a / __ldg(csd + c);
    }
  };

  // operands written: hand them over to the MMAs
  auto hand_over = [&]() {
    fence_async_smem();
    group_sync();
  };
  auto write_a = [&](const float (&act)[NC], int col0) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      if (TPR * NC > HP8 && cbase + 4 * g >= HP8) continue;     // no MMA reads columns from HP8 on
      float a[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = act[4 * g + i];
      smem_a4<RPC>(as, row, col0 + cbase + 4 * g, a);
    }
  };
  auto read_acc = [&](int region, float (&d)[NC]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) ld4<RPC>(row, region + cbase + 4 * g, d + 4 * g, accs);
  };
  // the thread's dY columns of a [128][64] dY array (none from kDyCols on: they hold the ready counters)
  auto save_dy = [&](float* q, int srow, const float (&d)[NC]) {
#pragma unroll
    for (int g = 0; g < NG; ++g) {
      if (TPR * NC > kDyCols && cbase + 4 * g >= kDyCols) continue;
      __stcg(tc_grp(q, tq * NG + g, srow), make_float4(d[4 * g], d[4 * g + 1], d[4 * g + 2], d[4 * g + 3]));
    }
  };
  // half tiles, after the CTA barrier that follows the write-out of units [u0, u0 + n) of the layer at svl:
  // count this CTA in their ready counters (release at gpu scope, which the CTA barrier makes cover every
  // thread's dY).  Releasing unit by unit spreads the weight-gradient work over the chain.  Whole tiles leave
  // no SM idle and release nothing: their weight-gradient kernel is an ordinary launch after the backward.
  auto publish = [&](float* svl, int u0, int n) {
    if constexpr (UPT > 1) {
      if (tid == 0) {
        unsigned* rdy = reinterpret_cast<unsigned*>(svl + SV.ready());
        fence_acq_rel_gpu();
        for (int i = 0; i < n; ++i) red_add_gpu(rdy + u0 + i, 1u);
      }
    }
  };

  for (int64_t unit = blockIdx.x; unit < nunits; unit += gridDim.x) {
    const int64_t tile = unit / UPT;                        // 128-row tile (save slab)
    const int srow = (int)(unit % UPT) * RPC + row;         // lane of the row in the tile's save slab
    const int64_t row0 = unit * RPC;
    float* svt = save + (size_t)tile * SV.tile_stride;
    // ---- per-tile setup: upstream gradient, loss statistics, d(sum g log q)/dz_T = -g z_T
    {
      const bool live = row0 + row < rows.R;
      const float g = live ? (gout ? __ldg(gout + row0 + row) : g_const) : 0.f;
      if (tq == 0) {
        GRs[row] = g;
        float nll = 0.f, bad = 0.f;
        if (live) {
          const float lp = __ldcg(svt + SV.lp + srow);
          if (isfinite(lp)) nll = -lp; else bad = 1.f;
        }
        if (loss_acc != nullptr) {
          nll = warp_sum(nll);
          bad = warp_sum(bad);
          if (lane == 0) {
            atomicAdd(loss_acc + 0, nll);
            if (bad != 0.f) atomicAdd(loss_acc + 1, bad);
          }
        }
      } else if (TPR == 2 || tq == 1) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 t = __ldcg(tc_grp(svt + SV.zt, i, srow));
          // (rows past the end of the batch were never saved: their gradient is exactly zero)
          dzs[(4 * i + 0) * RPC + row] = live ? -g * t.x : 0.f;
          dzs[(4 * i + 1) * RPC + row] = live ? -g * t.y : 0.f;
          dzs[(4 * i + 2) * RPC + row] = live ? -g * t.z : 0.f;
          dzs[(4 * i + 3) * RPC + row] = live ? -g * t.w : 0.f;
        }
      }
      if (COND && live)
        for (int c = c_lo; c < c_hi; ++c) dcond[(row0 + row) * C + c] = 0.f;
      prep_lu(m, m.T - 1, sm + L.lum);
      group_sync();
    }
    SBI_TL(101);

    for (int li = 0; li < m.T; ++li) {
      const int l = m.T - 1 - li;
      const NsfLayerView v = layer_view(m, l);
      const int32_t* tab = tcb.d_tab + l * SBI_NSF_TC_STRIDE;
      float* svl = svt + (size_t)l * SV.layer_stride;
      int stage = 0;
      SBI_TL(1000 * (li + 1));

      // the spline parameters of this thread's first feature (the features go round-robin over the row's
      // parts), requested before the LU section
      float qn[32], xn = 0.f;
      int jn = 0;
#pragma unroll
      for (int i = 0; i < 32; ++i) qn[i] = 0.f;
      if (tq < v.n_tr) {
        tc_load_prm(svl + SV.prm, srow, m.TRmax, tq, qn);
        jn = __ldg(v.trf + tq);
        xn = tc_load_row16_at(svl + SV.zin, srow, jn);
      }

      // ================= LULinear backward (y = U v, z' = L y + b): dv = U^T (dz + L^T dz) =================
      // (the dense factors of this layer were built a layer ago: prep_lu below; the parameter gradients are the
      // weight-gradient kernel's LULinear unit, which reads the dz written here)
      if (__ldg(v.LT + SBI_L_HAS_LU)) {
        if (tq == 1) {
          const float* U = sm + L.lum;
          const float* Lw = U + kLuMax * kLuMax;
          float dzr[kLuMax], dyr[kLuMax];
#pragma unroll
          for (int i = 0; i < kLuMax; ++i) dzr[i] = (i < D) ? dzs[i * RPC + row] : 0.f;
          // dy = dz + L^T dz (strictly lower part)
#pragma unroll
          for (int i = 0; i < kLuMax; ++i) {
            float dy = dzr[i];
#pragma unroll
            for (int j = 0; j < kLuMax; ++j)
              if (j > i) dy = fmaf(Lw[j * kLuMax + i], dzr[j], dy);
            dyr[i] = dy;
          }
          // dv = U^T dy
#pragma unroll
          for (int j = 0; j < kLuMax; ++j) {
            if (j < D) {
              float a = 0.f;
#pragma unroll
              for (int i = 0; i < kLuMax; ++i)
                if (i <= j) a = fmaf(U[i * kLuMax + j], dyr[i], a);
              dzs[j * RPC + row] = a;
            }
          }
        }
        group_sync();
        if (l < m.T - 1) publish(svl, SV.lu_unit(), 1);
      }
      if (l > 0) prep_lu(m, l - 1, sm + L.lum);     // next layer's dense factors: first read a whole layer of barriers later
      SBI_TL(1000 * (li + 1) + 1);

      // ================= final layer + spline backward, passes of <= 2 features =================
      const int np = __ldg(tab + 1);
      {
        for (int p = 0; p < np; ++p) {
          // feature f of pass p is feature f & 1 of the pass, taken by part f % TPR (warp-uniform)
          const int f = 2 * p + (tq & 1);
          const int nf = min(2, v.n_tr - 2 * p);
          const bool mine = TPR == 2 || ((p ^ (tq >> 1)) & 1) == 0;
          const bool has = mine && f < v.n_tr;
          // this feature's parameters were requested a feature (or the LU section) ago; request the next
          float q[32];
          const float x = xn;
          const int j = jn;
#pragma unroll
          for (int i = 0; i < 32; ++i) q[i] = qn[i];
          if (mine && f + TPR < v.n_tr) {
            tc_load_prm(svl + SV.prm, srow, m.TRmax, f + TPR, qn);
            jn = __ldg(v.trf + f + TPR);
            xn = tc_load_row16_at(svl + SV.zin, srow, jn);
          }
          if (has) {
            float dq[32];
            const float gx = rqs_backward_fast<KB>(q, rc, x, dzs[j * RPC + row], GRs[row], dq);
            dzs[j * RPC + row] = gx;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              float a[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) a[i] = dq[8 * c + i];
              smem_a8<RPC>(as, row, 32 * (tq & 1) + 8 * c, a);
            }
            tc_save_prm(svl + SV.dy_fin(p), srow, 0, tq & 1, dq);
          }
          hand_over();
          publish(svl, p, 1);
          {
            uint32_t acc = p > 0 ? 1u : 0u;
            iss.begin(__ldg(tab + 5 + 4 * (stage + p)));
            iss.block(cDs, 0, 4 * nf, 0, 64, acc);
            iss.end();
          }
          SBI_TL(1000 * (li + 1) + 10 + p);
        }
        stage += np;
      }
      // (loads of saved activations are requested one wait ahead of their use throughout the blocks)
      float sv[NC], t2[NC];
      if (m.NB > 0) {
        tc_load_cols<NC>(svl + SV.s(m.NB - 1), srow, tq, sv);
        tc_load_cols<NC>(svl + SV.t2(m.NB - 1), srow, tq, t2);
      }
      float dh[NC];
      read_acc(cDs, dh);
      SBI_TL(1000 * (li + 1) + 20);

      // ================= residual blocks, last to first =================
      for (int b = m.NB - 1; b >= 0; --b) {
        const int* BT = v.LT + SBI_L_BLK0 + 6 * b;
        float dT[NC], a1[NC];
        tc_load_cols<NC>(svl + SV.a1(b), srow, tq, a1);
        {
          // ---- dG = dh t2 s (1 - s): output gradient of the GLU context linear (the COND instantiation
          //      also takes dctx += dG Wc)
          float dG[NC];
#pragma unroll
          for (int q = 0; q < NC; ++q) {
            const float dhq = dh[q], s = sv[q];
            dT[q] = dhq * s;
            dG[q] = dhq * t2[q] * s * (1.f - s);
          }
          save_dy(svl + SV.dy_blk(b, 0), srow, dG);
          if (COND) {
            group_sync();
            publish(svl, SV.npm + 3 * b, 1);
            dctx_add(svl + SV.dy_blk(b, 0), P + __ldg(BT + 4), m.Cp, row0, srow);     // dG Wc
          }
        }
        SBI_TL(1000 * (li + 1) + 30 + 10 * b);
        // ---- dA1 = (dT W2) * [a1 > 0]
        {
          save_dy(svl + SV.dy_blk(b, 1), srow, dT);
          write_a(dT, 0);
          SBI_TL(1000 * (li + 1) + 72 + 10 * b);
          hand_over();
          if (COND) publish(svl, SV.npm + 3 * b + 1, 1);
          else publish(svl, SV.npm + 3 * b, 2);
          SBI_TL(1000 * (li + 1) + 73 + 10 * b);
          {
            uint32_t acc = 0u;
            iss.begin(__ldg(tab + 5 + 4 * stage));
            iss.block(cDs, 0, NCH, 0, 64, acc);
            iss.end();
          }
          SBI_TL(1000 * (li + 1) + 74 + 10 * b);
          ++stage;
        }
        SBI_TL(1000 * (li + 1) + 31 + 10 * b);
        float hb[NC];
        tc_load_cols<NC>(svl + SV.h(b), srow, tq, hb);
        float dA[NC];
        read_acc(cDs, dA);
#pragma unroll
        for (int q = 0; q < NC; ++q) dA[q] = a1[q] > 0.f ? dA[q] : 0.f;
        SBI_TL(1000 * (li + 1) + 32 + 10 * b);
        // ---- dh += (dA1 W1) * [h_b > 0]
        {
          save_dy(svl + SV.dy_blk(b, 2), srow, dA);
          write_a(dA, 0);
          hand_over();
          publish(svl, SV.npm + 3 * b + 2, 1);
          {
            uint32_t acc = 0u;
            iss.begin(__ldg(tab + 5 + 4 * stage));
            iss.block(cGs, 0, NCH, 0, 64, acc);
            iss.end();
          }
          ++stage;
        }
        SBI_TL(1000 * (li + 1) + 33 + 10 * b);
        if (b > 0) {
          tc_load_cols<NC>(svl + SV.s(b - 1), srow, tq, sv);
          tc_load_cols<NC>(svl + SV.t2(b - 1), srow, tq, t2);
        }
        {
          float d[NC];
          read_acc(cGs, d);
#pragma unroll
          for (int q = 0; q < NC; ++q) dh[q] += hb[q] > 0.f ? d[q] : 0.f;
        }
        SBI_TL(1000 * (li + 1) + 34 + 10 * b);
      }

      // ================= initial layer: d(identity features) = dh W0[:, C:] =================
      {
        const int K0p = m.Cp + m.IDp;
        save_dy(svl + SV.dy_init(), srow, dh);
        write_a(dh, 0);
        hand_over();
        publish(svl, SV.npm + 3 * m.NB, 1);
        if (COND) dctx_add(svl + SV.dy_init(), P + __ldg(v.LT + SBI_L_W0), K0p, row0, srow);     // the context columns of dh W0
        {
          uint32_t acc = 0u;
          iss.begin(__ldg(tab + 5 + 4 * stage));
          iss.block(cDs, 0, NCH, 0, 16, acc);
          iss.end();
        }
        ++stage;
        SBI_TL(1000 * (li + 1) + 60);
        if (tq == 0) {
          float d[16];
          ld8<RPC>(row, cDs, d, accs);
          ld8<RPC>(row, cDs + 8, d + 8, accs);
#pragma unroll
          for (int j = 0; j < 16; ++j)
            if (j < v.n_id) dzs[__ldg(v.idf + j) * RPC + row] += d[j];
          // the row's dz at layer l - 1's LULinear output, for the weight-gradient kernel's LULinear unit of that
          // layer, in this layer's spline parameters, whose last reader is done (nsf_tc_save.cuh).  Before the
          // barrier: after it, part 1 of the row overwrites dz with dv.  The LU section of layer l - 1
          // publishes it after its CTA barrier.
          if (l > 0) tc_save_row16<RPC>(svl + SV.dz_below(), srow, dzs, row, D);
        }
        group_sync();
      }
    }
    SBI_TL(9000);
  }
  SBI_TL(9001);

  tc_end(ncols, sa);
}

}  // namespace tc
}  // namespace sbi

// =================================================================================================
// C ABI
// =================================================================================================
using namespace sbi;

static int vjp_tc_ok(const sbi_nsf_model* m, const sbi_nsf_tc* tcf, const sbi_nsf_tc* tcb) {
  if (!sbi_b200_nsf_tc_supported(m, tcf)) return 0;
  if (!tcb || !tcb->d_tab || !tcb->d_tcw || tcb->stage_cap <= 0 || (tcb->stage_cap & 31)) return 0;
  if (m->IDp > 16 || m->Cp + m->IDp + 1 > 64 || m->Cp + 1 > 64) return 0;
  // the training pair runs one CTA per SM: the forward with activation save and the backward sweep may each
  // opt into a whole SM's shared memory, on whole tiles and on half tiles
  for (int rpc : {tc::kRows, 64})
    if (tc::forward_save_smem_bytes(*m, *tcf, rpc) > kMaxSmemBytes ||
        tc::bwd_smem_layout(tcb->stage_cap, rpc).total_bytes > kMaxSmemBytes)
      return 0;
  return tc::dw_smem_bytes(*m) <= kMaxSmemBytes ? 1 : 0;
}

extern "C" int sbi_b200_nsf_vjp_tc_supported(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd,
                                             const sbi_nsf_tc* tc_bwd) {
  if (!m || !tc_fwd || !tc_bwd) return 0;
  return vjp_tc_ok(m, tc_fwd, tc_bwd);
}

// rows of one forward + backward launch pair (one tile per CTA, every SM busy once)
static int64_t vjp_tc_chunk_rows() { return (int64_t)tc::kRows * sbi::dev_num_sms(); }

extern "C" int sbi_b200_nsf_vjp_tc_parts(int64_t R) { return vjp_parts(R, tc::kRows); }

extern "C" int64_t sbi_b200_nsf_vjp_tc_save_bytes(const sbi_nsf_model* m, int64_t R) {
  if (!m || R < 1) return 0;
  const tc::TcSave SV = tc::tc_save_layout(m->NB, m->TRmax, m->T);
  return (int64_t)sizeof(float) * SV.tile_stride * sbi_b200_nsf_vjp_tc_parts(R);
}

template <bool COND>
static int vjp_tc_launch(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd,
                         const sbi_rows* rows, const float* d_gout, float g_const, float* d_logp, float* d_gpart,
                         float* d_loss_acc, float* d_gcond, float* d_save, int64_t save_bytes, void* stream) {
  sbi::DeviceGuard dev_guard_(m ? m->d_params : nullptr);
  if (!m || !tc_fwd || !tc_bwd || !rows || !rows->d_input || !rows->d_cond || rows->R < 1 || !d_gpart ||
      !d_save || (COND && !d_gcond))
    return SBI_EINVAL;
  if (!vjp_tc_ok(m, tc_fwd, tc_bwd)) return SBI_ESMEM;
  if (save_bytes < sbi_b200_nsf_vjp_tc_save_bytes(m, rows->R)) return SBI_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int bwd_bytes = tc::bwd_smem_layout(tc_bwd->stage_cap, tc::kRows).total_bytes;
  const int bwd_bytes_half = tc::bwd_smem_layout(tc_bwd->stage_cap, 64).total_bytes;
  const int dw_bytes = tc::dw_smem_bytes(*m);
  // opt the backward kernels in before anything is launched: a failed opt-in leaves no forward sweep behind
  if (int e = set_smem(reinterpret_cast<const void*>(tc::nsf_vjp_tc_kernel<50, tc::kRows, 10, COND>), bwd_bytes))
    return e;
  if (int e = set_smem(reinterpret_cast<const void*>(tc::nsf_vjp_tc_kernel<50, 64, 10, COND>), bwd_bytes_half))
    return e;
  if (int e = set_smem(reinterpret_cast<const void*>(tc::nsf_dw_tc_kernel<50>), dw_bytes)) return e;
  // chunks of one tile per SM: forward sweep (saves activations), backward sweep of the same rows (tile t
  // writes partial-gradient slab t), then their weight gradients (one CTA per tile, layer and linear), which on
  // half tiles start while the backward runs and take each unit as soon as its dY is written; later chunks accumulate
  // into the partial-gradient slabs.  A chunk of at most half as many tiles as SMs runs the two sweeps on
  // half tiles (two CTAs per tile), so that twice as many SMs take part.
  tc::StoreArgs sa;
  if (int e = tc::store_args(&sa)) return e;
  const int64_t chunk = vjp_tc_chunk_rows();
  for (int64_t r0 = 0; r0 < rows->R; r0 += chunk) {
    sbi_rows rr = *rows;
    rr.R = std::min<int64_t>(chunk, rows->R - r0);
    if (rows->d_index) rr.d_index = rows->d_index + r0;
    else {
      rr.d_input = rows->d_input + r0 * m->D;
      if (!rows->cond_shared) rr.d_cond = rows->d_cond + r0 * m->C;
    }
    const int grid = (int)((rr.R + tc::kRows - 1) / tc::kRows);
    const bool half_tiles = 2 * grid <= sbi::dev_num_sms();
    if (int rc = tc::launch_forward_save(m, tc_fwd, &rr, d_logp ? d_logp + r0 : nullptr, d_save, half_tiles, s))
      return rc;
    const float* gout = d_gout ? d_gout + r0 : nullptr;
    if (int rc = half_tiles ? launch(tc::nsf_vjp_tc_kernel<50, 64, 10, COND>, 2 * grid, tc::kThreads, bwd_bytes_half,
                                     s, *m, *tc_bwd, rr, gout, g_const, d_loss_acc, d_save, sa,
                                     COND ? d_gcond + r0 * m->C : nullptr)
                            : launch(tc::nsf_vjp_tc_kernel<50, tc::kRows, 10, COND>, grid, tc::kThreads, bwd_bytes, s, *m,
                                     *tc_bwd, rr, gout, g_const, d_loss_acc, d_save, sa,
                                     COND ? d_gcond + r0 * m->C : nullptr))
      return rc;
    if (int rc = launch(tc::nsf_dw_tc_kernel<50>, Grid(grid * m->T * tc::dw_units(*m), half_tiles), tc::kThreads,
                        dw_bytes, s, *m, rr, d_save, d_gpart, r0 > 0 ? 1 : 0, half_tiles ? 2u : 0u, gout, g_const))
      return rc;
  }
  return 0;
}

extern "C" int sbi_b200_nsf_vjp_tc(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd,
                                   const sbi_rows* rows, const float* d_gout, float g_const, float* d_logp,
                                   float* d_gpart, float* d_loss_acc, float* d_save, int64_t save_bytes,
                                   void* stream) {
  return vjp_tc_launch<false>(m, tc_fwd, tc_bwd, rows, d_gout, g_const, d_logp, d_gpart, d_loss_acc, nullptr, d_save,
                              save_bytes, stream);
}

extern "C" int sbi_b200_nsf_vjp_tc_cond(const sbi_nsf_model* m, const sbi_nsf_tc* tc_fwd, const sbi_nsf_tc* tc_bwd,
                                        const sbi_rows* rows, const float* d_gout, float g_const, float* d_logp,
                                        float* d_gpart, float* d_loss_acc, float* d_gcond, float* d_save,
                                        int64_t save_bytes, void* stream) {
  return vjp_tc_launch<true>(m, tc_fwd, tc_bwd, rows, d_gout, g_const, d_logp, d_gpart, d_loss_acc, d_gcond, d_save,
                             save_bytes, stream);
}

#ifdef SBI_TC_TIMELINE
// tuning builds only: copy out and reset the phase timeline of CTA 0; returns the number of (id, clock) pairs
extern "C" int sbi_b200_debug_timeline_bwd(unsigned long long* out, int cap) {
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
