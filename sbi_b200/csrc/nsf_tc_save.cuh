// Activation scratch shared by the tensor-core training kernels: the forward sweep
// (nsf_logprob_tc_kernel<.., SAVE = true>, nsf_tc.cu) writes the activations, the backward sweep
// (nsf_vjp_tc_kernel, nsf_vjp_tc.cu) reads them and writes the output gradients dY, the weight-gradient
// kernel (nsf_dw_tc_kernel, nsf_vjp_tc.cu) reads both.  One slab per 128-row tile:
//
//   per layer l (layer_stride floats):
//     for each residual block b:  h_b | a1_b | t2_b | s_b     each [128 rows][64 columns]
//         h_b  = input of block b (pre-activation)            (relu mask of dW1's dX, X of dW1)
//         a1_b = relu(W1 relu(h_b) + b1)                      (relu mask, X of dW2)
//         t2_b = W2 a1_b + b2        s_b = sigmoid(Wc ctx + bc)   (GLU: block output = t2 * s)
//     hf   = input of the final layer                         [128][64]
//     prm  = raw spline parameters incl. bias                 [128][TRmax][32]
//     zin  = layer input z_l,  v = coupling output (LULinear input)   each [128][16]
//     dy   = output gradients dY of the layer's linears, written by the backward sweep and read by the
//            weight-gradient kernel (nsf_dw_tc_kernel)        [128][64 npm + 192 NB + 64]:
//            final-layer pass p (features 2p, 2p+1: 32 parameter rows each) at column 64p (npm passes),
//            block b: dG (GLU context linear) | dT (W2) | dA (W1) at 64 npm + 192b, then dh (initial linear)
//     ready = one counter per weight-gradient unit of the layer (u32, indexed like nsf_dw_tc_kernel's units),
//            in columns [kDyCols, 64) of dh, which hold no gradient: the backward sweep adds 1 per CTA of
//            the tile once the unit's dY is written, the weight-gradient kernel waits for the unit's count
//            and the forward sweep zeroes the counters of its tile
//     dz of layer l-1 (l > 0): the gradient at layer l-1's LULinear output, [128][16], in columns [0, 16) of
//            THIS layer's prm (prm has >= 32 columns).  The backward sweep writes it at the end of layer l,
//            after layer l's spline backward -- the only reader of prm_l after the forward sweep; the
//            weight-gradient kernel never reads prm -- and the weight-gradient kernel's LULinear unit of
//            layer l-1 reads it.  The top layer's dz is -g z_T, which that unit computes from zt.
//   then per tile:  zt = base-space point z_T [128][16],  lp = log q [128]
//
// Every array of a slab is stored as float4 groups with the ROW index fastest: group g of row r sits at
// float offset (g * 128 + r) * 4, so the 32 rows of a warp write / read 512 contiguous bytes per
// instruction (4 full lines instead of 32 partial sectors).  Groups: 4 adjacent columns of the
// [128][64] arrays (16 groups), parameter quadruple i of feature f (group f * 8 + i) of prm, and
// components 4i..4i+3 of the [128][16] arrays.
// (what the reference keeps as autograd-saved tensors of nflows' ResidualNet / spline transform,
// /root/reference/sbi/neural_nets/net_builders/flow.py:411-432)
#pragma once
#include <cuda_runtime.h>

#include "../../include/sbi_b200.h"

namespace sbi {
namespace tc {

// dY columns that are written and read (hidden width <= 56); columns [kDyCols, 64) of the dY arrays are free
constexpr int kDyCols = 56;
// a layer's counters (<= 8 final-layer passes of <= 16 features, 3 per block, the initial linear, the LULinear)
// fit them
static_assert(8 + 3 * SBI_NSF_MAX_BLOCKS + 2 <= (64 - kDyCols) * 128, "ready counters");

struct TcSave {
  int NB;
  int npm;                    // final-layer passes of the widest layer, (TRmax + 1) / 2
  int hf, prm, zin, v, dy;    // float offsets inside a layer slab
  int layer_stride;
  int zt, lp;                 // float offsets inside a tile slab (after the T layer slabs)
  int64_t tile_stride;
  __host__ __device__ int h(int b) const { return (4 * b + 0) * 64 * 128; }
  __host__ __device__ int a1(int b) const { return (4 * b + 1) * 64 * 128; }
  __host__ __device__ int t2(int b) const { return (4 * b + 2) * 64 * 128; }
  __host__ __device__ int s(int b) const { return (4 * b + 3) * 64 * 128; }
  // dY of final-layer pass p, of linear k (0: GLU context, 1: W2, 2: W1) of block b, of the initial linear
  __host__ __device__ int dy_fin(int p) const { return dy + 64 * p * 128; }
  __host__ __device__ int dy_blk(int b, int k) const { return dy + (64 * npm + 192 * b + 64 * k) * 128; }
  __host__ __device__ int dy_init() const { return dy + (64 * npm + 192 * NB) * 128; }
  // weight-gradient units of a layer: the final-layer passes, three linears per residual block (GLU context,
  // W2, W1), the initial linear, the LULinear parameters
  __host__ __device__ int units() const { return npm + 3 * NB + 2; }
  __host__ __device__ int lu_unit() const { return npm + 3 * NB + 1; }
  // dz at the LULinear output of layer l - 1, in layer l's slab (l > 0)
  __host__ __device__ int dz_below() const { return prm; }
  // ready counters of the layer, units() of the (64 - kDyCols) * 128 free words
  __host__ __device__ int ready() const { return dy_init() + kDyCols * 128; }
};

__host__ __device__ inline TcSave tc_save_layout(int NB, int TRmax, int T) {
  TcSave L;
  L.NB = NB;
  L.npm = (TRmax + 1) / 2;
  L.hf = 4 * NB * 64 * 128;
  L.prm = L.hf + 64 * 128;
  L.zin = L.prm + TRmax * 32 * 128;
  L.v = L.zin + 16 * 128;
  L.dy = L.v + 16 * 128;
  L.layer_stride = L.dy + (64 * L.npm + 192 * NB + 64) * 128;
  L.zt = T * L.layer_stride;
  L.lp = L.zt + 16 * 128;
  L.tile_stride = (int64_t)L.lp + 128;
  return L;
}

__device__ __forceinline__ float4* tc_grp(float* q, int g, int row) {
  return reinterpret_cast<float4*>(q) + g * 128 + row;
}
__device__ __forceinline__ const float4* tc_grp(const float* q, int g, int row) {
  return reinterpret_cast<const float4*>(q) + g * 128 + row;
}

// the thread's NC columns (column half `half`: columns [half*NC, half*NC + NC)) of its row; NC % 4 == 0
template <int NC>
__device__ __forceinline__ void tc_save_cols(float* q, int row, int half, const float (&v)[NC]) {
#pragma unroll
  for (int i = 0; i < NC / 4; ++i)
    __stcg(tc_grp(q, half * (NC / 4) + i, row), make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]));
}
template <int NC>
__device__ __forceinline__ void tc_load_cols(const float* q, int row, int half, float (&v)[NC]) {
#pragma unroll
  for (int i = 0; i < NC / 4; ++i) {
    const float4 t = __ldcg(tc_grp(q, half * (NC / 4) + i, row));
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
  }
}
// 32 raw spline parameters of feature f of the row
__device__ __forceinline__ void tc_save_prm(float* q, int row, int TRmax, int f, const float (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
    __stcg(tc_grp(q, f * 8 + i, row), make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]));
}
__device__ __forceinline__ void tc_load_prm(const float* q, int row, int TRmax, int f, float (&v)[32]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 t = __ldcg(tc_grp(q, f * 8 + i, row));
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
  }
}
// the D <= 16 values of row `row` of a feature-major shared array zs[d][RPC], into lane `lane`
template <int RPC>
__device__ __forceinline__ void tc_save_row16(float* q, int lane, const float* zs, int row, int D) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float t[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) t[j] = (4 * i + j < D) ? zs[(4 * i + j) * RPC + row] : 0.f;
    __stcg(tc_grp(q, i, lane), make_float4(t[0], t[1], t[2], t[3]));
  }
}
__device__ __forceinline__ void tc_load_row16(const float* q, int row, float (&v)[16]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 t = __ldcg(tc_grp(q, i, row));
    v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
  }
}
// component j of the row in a [128][16] array
__device__ __forceinline__ float tc_load_row16_at(const float* q, int row, int j) {
  return __ldcg(q + ((j >> 2) * 128 + row) * 4 + (j & 3));
}

// forward sweep of a training step: nsf_logprob_tc_kernel<50, 10, false, SAVE = true>, one tile per CTA, or
// with `half_tiles` two CTAs of 64 rows per tile (defined in nsf_tc.cu; returns a C-ABI status code)
int launch_forward_save(const sbi_nsf_model* m, const sbi_nsf_tc* tc, const sbi_rows* rows, float* d_logp,
                        float* d_save, bool half_tiles, cudaStream_t s);
// dynamic shared memory of that launch with `rpc` rows per CTA (its A operands live in shared memory)
int forward_save_smem_bytes(const sbi_nsf_model& m, const sbi_nsf_tc& tc, int rpc);

}  // namespace tc
}  // namespace sbi
