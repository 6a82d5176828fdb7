// Building blocks of the tensor-core (wgmma) row-tile kernels: the accumulator store, the MMAs, the
// 3xTF32 split, the weight-stage ring and its issuing logic.  Used by nsf_tc.cu, nsf_vjp_tc.cu and
// ratio_tc.cu; see the header of nsf_tc.cu for the design.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/sbi_b200.h"
#include "common.cuh"
#include "wgmma.cuh"

namespace sbi {
namespace tc {

// Phase timeline of CTA 0 (tuning builds only: -DSBI_TC_TIMELINE, profiles/tc_timeline.py): thread 0
// appends (id, clock64) pairs to a global buffer read back through sbi_b200_debug_timeline_{fwd,bwd}().
#ifdef SBI_TC_TIMELINE
static __device__ unsigned long long g_tl[4096];     // one copy per translation unit
static __device__ int g_tl_n;
#define SBI_TL(id)                                                                        \
  do {                                                                                    \
    if (blockIdx.x == 0 && threadIdx.x == 0 && g_tl_n < 2047) {                           \
      g_tl[2 * g_tl_n] = (unsigned long long)(id);                                        \
      g_tl[2 * g_tl_n + 1] = clock64();                                                   \
      ++g_tl_n;                                                                           \
    }                                                                                     \
  } while (0)
#else
#define SBI_TL(id) do { } while (0)
#endif

constexpr int kRows = 128;        // rows per tile
constexpr int kThreads = 256;     // 8 warps, two threads per row (column halves); all issue the MMAs
constexpr int kLuMax = 16;        // LULinear runs on register-resident rows of <= 16 features
constexpr int kSlots = 3;         // weight ring: up to two stages in use + one prefetched
constexpr int kCols = 256;        // accumulator-store columns per CTA
constexpr int cAhi = 0, cAlo = 64, cD = 128, cG = 192;
// kernels that keep A in shared memory (the training pair, below) reserve the accumulator columns only
constexpr int kColsDG = 128;
constexpr int cDs = 0, cGs = 64;
// On half tiles (RPC = 64, below) the training pair keeps those columns in shared memory instead of the
// store: kColsDG columns of kAccLd floats, column-major like the store.  64 lanes + 4 of padding: in the
// fragment write-back the 4 threads of a quad write columns 2t apart, which a stride of 64 would put in
// one bank.
constexpr int kAccLd = 64 + 4;
__host__ __device__ constexpr int acc_smem_floats() { return kColsDG * kAccLd; }

// ---- accumulator store --------------------------------------------------------------------------
// The kernels keep their MMA accumulators, and all but the training pair (A in shared memory, below) their
// A operands, in columns of 128 lanes, lane = tile row.
// Hopper keeps wgmma accumulators in registers, and an SM's shared memory is taken by the weight ring
// and the staging buffers (except on the training pair's half tiles, above), so the columns live in global memory: kStoreSlots slabs of kStoreCols
// columns x 128 lanes (lane-contiguous, so the 32 threads of a warp touch one 128-byte line per column;
// 34.6 MB per device, defined once in nsf_tc.cu and mostly L2-resident while a kernel runs), handed out
// in 64-column units through one mask per slab.  A CTA picks the slab of the SM it starts on (for
// locality only) and records the slab and its first column in s_store / s_store_col; every later address
// comes from that record, so a CTA that resumes on another SM keeps its columns.  The kernels index
// columns relative to their first column.
constexpr int kStoreCols = 512;
constexpr int kStoreLanes = 128;
constexpr int kStoreSlots = 132;  // one per H100 SXM SM; SMs with larger ids share slabs through the masks
struct StoreArgs {
  float* slab;              // [kStoreSlots][kStoreCols * kStoreLanes]
  unsigned int* mask;       // [kStoreSlots]: bit u = columns [64u, 64u + 64) are taken
};
// the device's slabs and masks (host; defined in nsf_tc.cu); returns a cudaError_t
int store_args(StoreArgs* out);

static __shared__ float* s_store;          // this CTA's slab, set by store_alloc
static __shared__ uint32_t s_store_col;    // first column of this CTA in its slab, set by store_alloc

// element (row, column) of this CTA's columns
__device__ __forceinline__ float* store_at(uint32_t row, uint32_t col) {
  return s_store + ((s_store_col + col) * kStoreLanes + row);
}
// warp 0 of the CTA, before the CTA barrier that publishes s_store / s_store_col: reserve `ncols`
// (multiple of 64, <= kStoreCols) columns of a slab.  Spins while other CTAs hold the columns.  A
// waiting CTA holds no columns (a reservation is one CAS of all its units), and a holder waits on no
// other CTA before it releases, so the wait cannot form a cycle.
__device__ __forceinline__ void store_alloc(int ncols, const StoreArgs& sa) {
  if ((threadIdx.x & 31) == 0) {
    uint32_t sm;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    const uint32_t slot = sm % kStoreSlots;
    unsigned int* mk = sa.mask + slot;
    const int units = ncols / 64;
    const unsigned int want = (1u << units) - 1u;
    for (;;) {
      const unsigned int cur = atomicAdd(mk, 0u);
      int pos = -1;
      for (int p = 0; p + units <= kStoreCols / 64; p += units)
        if (!(cur & (want << p))) { pos = p; break; }
      if (pos >= 0 && atomicCAS(mk, cur, cur | (want << pos)) == cur) {
        __threadfence();
        s_store = sa.slab + (size_t)slot * kStoreCols * kStoreLanes;
        s_store_col = (uint32_t)pos * 64u;
        break;
      }
      __nanosleep(200);
    }
  }
  __syncwarp();
}
// warp 0 of the CTA, after the CTA barrier that ends the last use of the columns: release them
__device__ __forceinline__ void store_dealloc(int ncols, const StoreArgs& sa) {
  if ((threadIdx.x & 31) == 0) {
    const size_t slot = (size_t)(s_store - sa.slab) / ((size_t)kStoreCols * kStoreLanes);
    __threadfence();
    atomicAnd(sa.mask + slot, ~(((1u << (ncols / 64)) - 1u) << (s_store_col / 64)));
  }
  __syncwarp();
}

// shared-memory operand descriptor of wgmma, no swizzle (interleave), K-major: core matrix = 8 rows x
// 16 B contiguous; LBO = byte distance of K-adjacent core matrices, SBO = byte distance of 8-row groups
__device__ __forceinline__ uint64_t make_bdesc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3fff) << 32;
  return d;
}
// 8 / 4 consecutive columns [col, col + 8 / 4) of tile row `row`
__device__ __forceinline__ void st8(uint32_t row, uint32_t col, const float (&v)[8]) {
  float* p = store_at(row, col);
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i * kStoreLanes] = v[i];
}
// accumulator reads of an RPC-row CTA: from the store, or on half tiles from the shared-memory columns `accs`
template <int RPC = kRows>
__device__ __forceinline__ void ld8(uint32_t row, uint32_t col, float* v, const float* accs = nullptr) {
  constexpr int ld = RPC < kRows ? kAccLd : kStoreLanes;
  const float* p = RPC < kRows ? accs + col * kAccLd + row : store_at(row, col);
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = p[i * ld];
}
__device__ __forceinline__ void st4(uint32_t row, uint32_t col, const float (&v)[4]) {
  float* p = store_at(row, col);
#pragma unroll
  for (int i = 0; i < 4; ++i) p[i * kStoreLanes] = v[i];
}
template <int RPC = kRows>
__device__ __forceinline__ void ld4(uint32_t row, uint32_t col, float* v, const float* accs = nullptr) {
  constexpr int ld = RPC < kRows ? kAccLd : kStoreLanes;
  const float* p = RPC < kRows ? accs + col * kAccLd + row : store_at(row, col);
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = p[i * ld];
}

// ---- A operands in shared memory ------------------------------------------------------------------
// The training pair (nsf_logprob_tc_kernel<..., SAVE>, nsf_vjp_tc_kernel) runs one CTA per SM, which leaves
// room for A_hi | A_lo (RPC rows x 64 K-columns each) in shared memory, so the MMAs read A through a
// descriptor instead of waiting for fragment loads from the L2-resident store in every K-step.  RPC, the
// rows of a CTA, is 128 (a whole tile) or 64 (half a tile, when a chunk of tiles would leave SMs idle).
// Layout: wgmma's K-major no-swizzle canonical layout [k/4][RPC rows][4], the convention of make_bdesc for
// B: a core matrix (8 rows x 4 K-columns) is 128 contiguous bytes, 8-row groups are 128 B apart (SBO),
// K-adjacent core matrices RPC x 16 B apart (LBO); a K-step of 8 columns advances RPC x 32 B, and with
// RPC = 128 warpgroup 1 (rows 64 ..) starts 1024 B in.  A row thread writes 4 consecutive columns as one
// float4, so the 32 rows of a warp cover 512 contiguous bytes.
__host__ __device__ constexpr int a_smem_floats(int rpc) { return 2 * 64 * rpc; }   // A_hi | A_lo

// ---- the MMAs: both warpgroups of the CTA, complete on return ------------------------------------
// Accumulator fragment of wgmma m64nNk8 (f32): warp w of the warpgroup holds rows 16w + g and
// 16w + g + 8 (g = lane / 4), columns 8j + 2t and 8j + 2t + 1 (t = lane % 4) in d[4j .. 4j+3].
//
// D[M = RPC] (+)= A * B[smem]^T over nk K-steps, 3xTF32 (A_hi B_hi + A_lo B_hi + A_hi B_lo):
// RPC = 128: warpgroup wg computes rows 64 wg .. 64 wg + 63; RPC = 64: both warpgroups compute the CTA's
// 64 rows, each its own N columns (the caller offsets dcol and the B descriptors).  ASMEM = false: ah / al
// are the A_hi / A_lo store columns of the first K-step and the fragments come straight from the store;
// ASMEM = true: ah / al are the shared-memory descriptors of the warpgroup's first K-step.  Same products in
// the same order.  D is in the store, or on half tiles (RPC = 64) in the shared-memory columns `accs`.
// ASMEM keeps the next K-step's MMAs in flight while the running sum takes the current one.
template <int N, bool ASMEM, int RPC = kRows>
__device__ __forceinline__ void mma_rows_n(uint32_t dcol, uint64_t ah, uint64_t al, uint64_t dh,
                                           uint64_t dl, uint64_t dstep, int nk, uint32_t acc, float* accs) {
  constexpr uint64_t kAStep = (RPC * 32u) >> 4;       // descriptor start-address advance per K-step
  constexpr bool kDSmem = RPC < kRows;
  constexpr uint32_t kLd = kDSmem ? kAccLd : kStoreLanes;
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const uint32_t r0 = (RPC == kRows ? (threadIdx.x >> 7) * 64 : 0) + ((threadIdx.x >> 5) & 3) * 16 + g;
  const uint32_t c0 = kDSmem ? 0u : s_store_col;
  dcol += c0;
  const uint32_t ahcol = (uint32_t)ah + c0, alcol = (uint32_t)al + c0;
  float* slab = kDSmem ? accs : s_store;
  float d[N / 2];
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const uint32_t c = dcol + 8 * j + 2 * t;
    d[4 * j + 0] = acc ? slab[c * kLd + r0] : 0.f;
    d[4 * j + 1] = acc ? slab[(c + 1) * kLd + r0] : 0.f;
    d[4 * j + 2] = acc ? slab[c * kLd + r0 + 8] : 0.f;
    d[4 * j + 3] = acc ? slab[(c + 1) * kLd + r0 + 8] : 0.f;
  }
  if constexpr (ASMEM) {
    // each K-step into a fresh accumulator (two alternate), correction terms first; K-step k + 1 is issued
    // before the running sum takes K-step k, with the round-to-nearest adds of the synchronous loop below in
    // the same order
    float p0[N / 2], p1[N / 2];
    auto issue = [&](float (&p)[N / 2]) {
      wgmma_fence();
      wgmma_ss<N>(p, al, dh, 0u);
      wgmma_ss<N>(p, ah, dl, 1u);
      wgmma_ss<N>(p, ah, dh, 1u);
      wgmma_commit();
      ah += kAStep; al += kAStep;
      dh += dstep; dl += dstep;
    };
    auto take = [&](float (&p)[N / 2]) {
      wgmma_fence_operand(p);
#pragma unroll
      for (int i = 0; i < N / 2; ++i) d[i] += p[i];
    };
    issue(p0);
    int kk = 1;
    for (; kk + 1 < nk; kk += 2) {
      issue(p1);
      wgmma_wait<1>();
      take(p0);
      issue(p0);
      wgmma_wait<1>();
      take(p1);
    }
    if (kk < nk) {
      issue(p1);
      wgmma_wait<1>();
      take(p0);
      wgmma_wait<0>();
      take(p1);
    } else {
      wgmma_wait<0>();
      take(p0);
    }
  } else {
    for (int kk = 0; kk < nk; ++kk) {
      // each K-step into a fresh accumulator, correction terms first; the running sum is then carried
      // with round-to-nearest adds (the tensor core's own fp32 accumulation truncates)
      float p[N / 2];
#pragma unroll
      for (int i = 0; i < N / 2; ++i) p[i] = 0.f;
      uint32_t fh[4], fl[4];
      const uint32_t ch = ahcol + 8 * kk + t, cl = alcol + 8 * kk + t;
      fh[0] = __float_as_uint(slab[ch * kStoreLanes + r0]);
      fh[1] = __float_as_uint(slab[ch * kStoreLanes + r0 + 8]);
      fh[2] = __float_as_uint(slab[(ch + 4) * kStoreLanes + r0]);
      fh[3] = __float_as_uint(slab[(ch + 4) * kStoreLanes + r0 + 8]);
      fl[0] = __float_as_uint(slab[cl * kStoreLanes + r0]);
      fl[1] = __float_as_uint(slab[cl * kStoreLanes + r0 + 8]);
      fl[2] = __float_as_uint(slab[(cl + 4) * kStoreLanes + r0]);
      fl[3] = __float_as_uint(slab[(cl + 4) * kStoreLanes + r0 + 8]);
      wgmma_fence();
      wgmma_rs<N>(p, fl, dh, 0u);
      wgmma_rs<N>(p, fh, dl, 1u);
      wgmma_rs<N>(p, fh, dh, 1u);
      wgmma_commit();
      wgmma_wait_all();
#pragma unroll
      for (int i = 0; i < N / 2; ++i) d[i] += p[i];
      dh += dstep; dl += dstep;
    }
  }
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const uint32_t c = dcol + 8 * j + 2 * t;
    slab[c * kLd + r0] = d[4 * j + 0];
    slab[(c + 1) * kLd + r0] = d[4 * j + 1];
    slab[c * kLd + r0 + 8] = d[4 * j + 2];
    slab[(c + 1) * kLd + r0 + 8] = d[4 * j + 3];
  }
}
template <bool ASMEM, int RPC = kRows>
__device__ __forceinline__ void mma_rows(int N, uint32_t dcol, uint64_t ah, uint64_t al, uint64_t dh,
                                         uint64_t dl, uint64_t dstep, int nk, uint32_t acc, float* accs) {
  switch (N) {
    case 8: mma_rows_n<8, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 16: mma_rows_n<16, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 24: mma_rows_n<24, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 32: mma_rows_n<32, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 40: mma_rows_n<40, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 48: mma_rows_n<48, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 56: mma_rows_n<56, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    case 64: mma_rows_n<64, ASMEM, RPC>(dcol, ah, al, dh, dl, dstep, nk, acc, accs); break;
    default: __trap();      // operand blocks are planned with N in {8, ..., 64}
  }
}

// D[M = 64, N = 2 NH] = A[smem]^T-staged * B[smem]^T over nk K-steps, single TF32 pass, into registers:
// warpgroup wg computes columns [wg NH, (wg + 1) NH); d holds the accumulator fragment of the
// warpgroup's m64nNHk8 MMA (rows 16w + g and 16w + g + 8 of warp w, columns wg NH + 8j + 2t, + 1).
template <int NH>
__device__ __forceinline__ void mma_ss64_n(float (&d)[NH / 2], uint64_t da, uint64_t db, uint64_t dstep, int nk) {
  const int wg = threadIdx.x >> 7;
  db += (uint64_t)((wg * NH / 8) * 128 >> 4);      // 8-row groups of B are 128 B apart
#pragma unroll
  for (int i = 0; i < NH / 2; ++i) d[i] = 0.f;
  for (int kk = 0; kk < nk; ++kk) {
    float p[NH / 2];
#pragma unroll
    for (int i = 0; i < NH / 2; ++i) p[i] = 0.f;
    wgmma_fence();
    wgmma_ss<NH>(p, da, db, 0u);
    wgmma_commit();
    wgmma_wait_all();
#pragma unroll
    for (int i = 0; i < NH / 2; ++i) d[i] += p[i];
    da += dstep; db += dstep;
  }
}
template <int NCHUNK, int RPC = kRows>
__device__ __forceinline__ void ld_cols(uint32_t row, uint32_t col, float* v, const float* accs = nullptr) {
#pragma unroll
  for (int c = 0; c < NCHUNK; ++c) ld8<RPC>(row, col + 8 * c, v + 8 * c, accs);
}

// hi = x rounded to tf32 (10 explicit mantissa bits, round half away in the integer domain),
// lo = x - hi (exact in fp32).  Same hi as cvt.rna.tf32.f32.
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
  lo = x - hi;
}
// split 8 values and put them into A_hi / A_lo columns [col, col+8) of tile row `row`
__device__ __forceinline__ void store_a8(uint32_t row, int col, const float (&v)[8]) {
  float hi[8], lo[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) split_tf32(v[i], hi[i], lo[i]);
  st8(row, cAhi + col, hi);
  st8(row, cAlo + col, lo);
}
__device__ __forceinline__ void store_a4(uint32_t row, int col, const float (&v)[4]) {
  float hi[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_tf32(v[i], hi[i], lo[i]);
  st4(row, cAhi + col, hi);
  st4(row, cAlo + col, lo);
}
// the same into the shared-memory A region `as` of an RPC-row CTA (col % 4 == 0); the writer issues
// fence_async_smem() before the CTA barrier that hands the operands to the MMAs
template <int RPC>
__device__ __forceinline__ void smem_a4(float* as, uint32_t row, int col, const float (&v)[4]) {
  float hi[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split_tf32(v[i], hi[i], lo[i]);
  float4* p = reinterpret_cast<float4*>(as + ((col >> 2) * RPC + row) * 4);
  p[0] = make_float4(hi[0], hi[1], hi[2], hi[3]);
  p[a_smem_floats(RPC) / 8] = make_float4(lo[0], lo[1], lo[2], lo[3]);
}
template <int RPC>
__device__ __forceinline__ void smem_a8(float* as, uint32_t row, int col, const float (&v)[8]) {
  smem_a4<RPC>(as, row, col, {v[0], v[1], v[2], v[3]});
  smem_a4<RPC>(as, row, col + 4, {v[4], v[5], v[6], v[7]});
}
__device__ __forceinline__ void group_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
// dense LU factors of NSF layer l, zero-padded to 16x16, into lum = [U | L | bias 16 | diag 16]
// (all threads; the unit diagonal of L is implicit)
__device__ __forceinline__ void prep_lu(const sbi_nsf_model& m, int l, float* lum) {
  const int* LT = m.d_layer_tab + l * SBI_NSF_LAYER_STRIDE;
  if (!__ldg(LT + SBI_L_HAS_LU)) return;
  const int D = m.D;
  const float* lo = m.d_params + __ldg(LT + SBI_L_LU_LOWER);
  const float* up = m.d_params + __ldg(LT + SBI_L_LU_UPPER);
  const float* dg = m.d_params + __ldg(LT + SBI_L_LU_DIAG);
  const float* bi = m.d_params + __ldg(LT + SBI_L_LU_BIAS);
  float* U = lum;
  float* Lw = U + kLuMax * kLuMax;
  for (int t = threadIdx.x; t < kLuMax * kLuMax; t += kThreads) {
    const int i = t / kLuMax, j = t % kLuMax;
    float u = 0.f, lv = 0.f;
    if (i < D && j < D) {
      if (j > i) u = __ldg(up + i * D - i * (i + 1) / 2 + (j - i - 1));
      else if (j < i) lv = __ldg(lo + i * (i - 1) / 2 + j);
      else u = softplus_f(__ldg(dg + i)) + 1e-3f;
    }
    U[t] = u;
    Lw[t] = lv;
    if (j == 0) Lw[kLuMax * kLuMax + i] = (i < D) ? __ldg(bi + i) : 0.f;
    if (j == i) Lw[kLuMax * kLuMax + kLuMax + i] = (i < D) ? u : 1.f;
  }
}

// ---- weight re-pack: flat fp32 parameters -> [hi | lo] wgmma operand blocks --------------------
static __global__ void tc_pack_kernel(const float* __restrict__ params, const int32_t* __restrict__ src,
                                   float* __restrict__ tcw, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = __ldg(src + i);
  float v = 0.f;
  if (s >= 0) {
    float hi, lo;
    split_tf32(__ldg(params + s), hi, lo);
    v = hi;
  } else if (s <= -2) {
    float hi, lo;
    split_tf32(__ldg(params + (-2 - s)), hi, lo);
    v = lo;
  }
  tcw[i] = v;
}

// host: re-pack `params` into the operand blocks of `tc`; returns a C-ABI status code
static int pack_weights(const float* params, const sbi_nsf_tc* tc, cudaStream_t s) {
  if (!params || !tc || !tc->d_src || !tc->d_tcw || tc->n_words <= 0) return SBI_EINVAL;
  const int threads = 256, blocks = (tc->n_words + threads - 1) / threads;
  tc_pack_kernel<<<blocks, threads, 0, s>>>(params, tc->d_src, tc->d_tcw, tc->n_words);
  return (int)cudaGetLastError();
}

// ---- the kernel ------------------------------------------------------------------------------------
// Every thread runs begin / block / end: the MMAs of a stage take both warpgroups and are complete
// once end() returns.  The weight stream rotates between the warps (stage k is fetched by the
// elected lane of warp (k + 4) % 8).  Stage k lives in ring slot k % NSLOT.  A stage is fetched
// (TMA bulk copy, completion on full[slot]) by the end() of the stage that used its slot NSLOT stages
// earlier.  ASMEM: A comes from the shared-memory A region of an RPC-row CTA at `abase`, else from the store;
// half tiles (RPC = 64) keep D | G in the shared-memory columns `accs`.
template <int NSLOT, bool ASMEM = false, int RPC = kRows>
struct IssuerT {
  bool leader;          // the elected lane of this warp
  int warp;             // this warp; stage k is fetched by warp (k+4) % 8
  uint32_t abase;       // ASMEM: shared address of the A region
  float* accs;          // half tiles: the shared-memory accumulator columns (acc_smem_floats() floats)
  float* ring;
  uint64_t* full;
  const float* tcw;
  const int32_t* tab;   // stage table (all layers)
  int cap, T;
  uint32_t it;          // stages issued (and complete)
  uint32_t fetched;     // stages fetched
  uint32_t sbase, lo_off;   // current stage: shared address of the hi half, byte offset of lo half
  int64_t f_tile, ntiles, tile_step;   // next stage to fetch
  int f_l, f_s;
  bool reverse;         // layers are walked T-1 .. 0 (sampling direction)

  __device__ __forceinline__ void pump() {
    while (fetched < it + NSLOT && f_tile < ntiles) {
      const int32_t* t = tab + (reverse ? T - 1 - f_l : f_l) * SBI_NSF_TC_STRIDE;
      const int off = __ldg(t + 4 + 4 * f_s), nfl = __ldg(t + 5 + 4 * f_s);
      const uint32_t slot = fetched % NSLOT;
      if (leader && (int)((fetched + 4u) & 7u) == warp) {
        mbar_arrive_expect_tx(&full[slot], (uint32_t)nfl * 4u);
        bulk_g2s(ring + (size_t)slot * cap, tcw + off, (uint32_t)nfl * 4u, &full[slot]);
      }
      ++fetched;
      if (++f_s == __ldg(t)) {
        f_s = 0;
        if (++f_l == T) { f_l = 0; f_tile += tile_step; }
      }
    }
  }
  __device__ __forceinline__ void begin(int stage_floats) {
    const uint32_t s = it % NSLOT;
    mbar_wait(&full[s], (it / NSLOT) & 1u);
    sbase = smem_u32(ring + (size_t)s * cap);
    lo_off = (uint32_t)stage_floats * 2u;   // (floats / 2) * 4 bytes
  }
  // one operand block of N rows starting `blk_floats` into the half: nk K-steps, A columns from a0
  __device__ __forceinline__ void block(int dcol, int a0, int nk, int blk_floats, int N, uint32_t& acc) {
    const uint32_t slab = (uint32_t)N * 16u;
    const uint32_t bh = sbase + (uint32_t)blk_floats * 4u;
    const uint64_t dh = make_bdesc(bh, slab, 128u);
    const uint64_t dl = make_bdesc(bh + lo_off, slab, 128u);
    const uint64_t dstep = (uint64_t)((2u * slab) >> 4);    // start-address field advance per K-step
    if constexpr (ASMEM && RPC == kRows) {
      // column a0 (a multiple of 4) of the warpgroup's first row
      const uint32_t ah = abase + (uint32_t)a0 * (kRows * 4u) + (threadIdx.x >> 7) * 1024u;
      if (nk > 0)
        mma_rows<true>(N, dcol, make_bdesc(ah, kRows * 16u, 128u),
                       make_bdesc(ah + a_smem_floats(kRows) * 2u, kRows * 16u, 128u), dh, dl, dstep, nk, acc, accs);
    } else if constexpr (ASMEM) {
      // both warpgroups on the CTA's rows from column a0; warpgroup wg takes result columns
      // [wg N/2, (wg + 1) N/2), whose B rows start wg N/16 8-row groups (128 B each) in
      const uint32_t ah = abase + (uint32_t)a0 * (RPC * 4u);
      const uint32_t nh = (uint32_t)N / 2u, wg = threadIdx.x >> 7;
      const uint64_t boff = (uint64_t)((wg * nh / 8u) * 128u >> 4);
      if (nk > 0)
        mma_rows<true, RPC>((int)nh, dcol + wg * nh, make_bdesc(ah, RPC * 16u, 128u),
                            make_bdesc(ah + a_smem_floats(RPC) * 2u, RPC * 16u, 128u), dh + boff, dl + boff, dstep,
                            nk, acc, accs);
    } else {
      if (nk > 0) mma_rows<false>(N, dcol, cAhi + a0, cAlo + a0, dh, dl, dstep, nk, acc, nullptr);
    }
    if (nk > 0) acc = 1u;
  }
  // close the stage: after the CTA barrier its accumulators are in place and its ring slot is free
  __device__ __forceinline__ void end() {
    group_sync();
    ++it;
    pump();
  }
};
using Issuer = IssuerT<kSlots>;

// Kernel prologue, all threads: thread 0 initialises the ring's mbarriers full[0 .. NSLOT) (and any
// other mbarrier the kernel initialised before the call), warp 0 reserves `ncols` store columns (none on
// half tiles), and after the CTA barrier the issuer starts fetching the first NSLOT stages of the CTA's
// first tile.  `ntiles` counts the CTA tiles of RPC rows.  ASMEM: `as` is the shared-memory A region
// (a_smem_floats(RPC) floats, 16-byte aligned); half tiles: `accs` the shared-memory accumulator columns.
template <int NSLOT, bool ASMEM = false, int RPC = kRows>
__device__ __forceinline__ IssuerT<NSLOT, ASMEM, RPC> tc_begin(uint64_t* full, float* ring, const sbi_nsf_tc& tc, int T,
                                                          int64_t ntiles, bool reverse, int ncols, const StoreArgs& sa,
                                                          float* as = nullptr, float* accs = nullptr) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < NSLOT; ++s) mbar_init(&full[s], 1);
    fence_barrier_init();
  }
  if (ncols > 0 && threadIdx.x < 32) store_alloc(ncols, sa);
  __syncthreads();
  IssuerT<NSLOT, ASMEM, RPC> iss;
  uint32_t el = 0;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(el));
  iss.leader = el != 0;
  iss.warp = threadIdx.x >> 5;
  iss.abase = ASMEM ? smem_u32(as) : 0u;
  iss.accs = accs;
  iss.ring = ring; iss.full = full;
  iss.tcw = tc.d_tcw; iss.tab = tc.d_tab; iss.cap = tc.stage_cap; iss.T = T;
  iss.it = 0; iss.fetched = 0;
  iss.sbase = 0; iss.lo_off = 0;
  iss.f_tile = blockIdx.x; iss.ntiles = ntiles; iss.tile_step = gridDim.x; iss.f_l = 0; iss.f_s = 0;
  iss.reverse = reverse;
  iss.pump();
  return iss;
}
// Kernel epilogue, all threads: release the store columns once every thread is done with them.
__device__ __forceinline__ void tc_end(int ncols, const StoreArgs& sa) {
  group_sync();
  if (ncols > 0 && threadIdx.x < 32) store_dealloc(ncols, sa);
}

// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// TMA bulk copy shared -> global (bulk async-group of the calling thread); bytes % 16 == 0, both
// addresses 16-byte aligned.  `add`: element-wise fp32 reduction into global instead of a plain store.
__device__ __forceinline__ void bulk_s2g(float* dst_gmem, const float* src_smem, uint32_t bytes, bool add) {
  if (add)
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(dst_gmem),
                 "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
  else
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem),
                 "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the committed groups have finished READING shared memory (the source may be overwritten)
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// the committed groups are complete (their global writes are performed)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

}  // namespace tc
}  // namespace sbi
