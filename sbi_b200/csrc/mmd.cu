// MMD misspecification test (reference sbi/diagnostics/misspecification.py:19-110): for S index sets at once, the
// median-heuristic RBF MMD between an X block and a Y block of rows of one device matrix Z (R, D).
//
// Launch sequence (the same for every S): init; four (count, select) radix passes that find the exact lower median
// of each set's X-Y squared distances; sum; finalize.  Every pass recomputes distances tile by tile from Z, so no
// nx*ny distance array is ever stored.
//  * Pair tiles are 64 x 64 rows, 256 threads with 4 x 4 pairs each; features stream through shared memory in
//    chunks of KC.  d^2 = sum (a - b)^2 in fp32, one fp32 partial per chunk added to the pair's running sum.
//  * Radix select on the fp32 bit patterns of d^2 (non-negative, so bit order is value order), 8 bits per pass:
//    warp-aggregated shared histograms, flushed to a per-set global histogram with integer atomics (the counts do
//    not depend on order).  sqrt is monotone, so the median distance is sqrtf of the median d^2.
//  * A set's pairs are split over P = min(tiles, kParts) CTAs; CTA b takes tiles b, b + P, ...  Each thread sums
//    its tile's kernel values in fp32 and adds them to fp64 accumulators; the CTA reduces them in a fixed tree and
//    the finalize kernel adds the P partials in index order.  P and the tile order depend only on the set's own
//    sizes, so results are bit-identical across calls and independent of the other sets in the launch.
//  * XX and YY are symmetric: only tiles on or above the diagonal are evaluated, off-diagonal ones counted twice.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "device.cuh"

namespace sbi {
namespace mmd {

constexpr int kTile = 64;          // rows per side of a pair tile
constexpr int kThreads = 256;      // 16 x 16 threads, 4 x 4 pairs each
constexpr int kParts = 128;        // most CTAs (and fp64 partials) per set
constexpr int kBins = 256;         // 8-bit radix digit
constexpr int kPasses = 4;
constexpr double kLog2e = 1.4426950408889634;

__host__ __device__ __forceinline__ int64_t tiles(int64_t n) { return (n + kTile - 1) / kTile; }

// pair tiles of a set: X-Y, then the X-X and Y-Y squares
__host__ __device__ __forceinline__ int64_t sum_tiles(int64_t nx, int64_t ny) {
  return tiles(nx) * tiles(ny) + tiles(nx) * tiles(nx) + tiles(ny) * tiles(ny);
}

template <int KC>
struct __align__(16) TileSmem {
  float a[KC][kTile + 4];
  float b[KC][kTile + 4];
  int ra[kTile], rb[kTile];
};

// d2[r][c]: squared distance between row (ty*4 + r) of the A rows and row (tx*4 + c) of the B rows of the tile;
// rows past na / nb read as zeros.
template <int KC>
__device__ __forceinline__ void tile_d2(const float* __restrict__ z, int D, const int32_t* __restrict__ rows_a,
                                        int na, const int32_t* __restrict__ rows_b, int nb, TileSmem<KC>& sm,
                                        float (&d2)[4][4]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  __syncthreads();   // the previous tile's loads are done with ra / rb
  for (int i = threadIdx.x; i < 2 * kTile; i += kThreads) {
    if (i < kTile) sm.ra[i] = i < na ? rows_a[i] : -1;
    else sm.rb[i - kTile] = i - kTile < nb ? rows_b[i - kTile] : -1;
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) d2[r][c] = 0.f;
  for (int f0 = 0; f0 < D; f0 += KC) {
    __syncthreads();
    for (int e = threadIdx.x; e < 2 * kTile * KC; e += kThreads) {
      const int side = e / (kTile * KC), r = (e / KC) % kTile, f = e % KC;
      const int row = side ? sm.rb[r] : sm.ra[r];
      const float v = (row >= 0 && f0 + f < D) ? z[(int64_t)row * D + f0 + f] : 0.f;
      if (side) sm.b[f][r] = v;
      else sm.a[f][r] = v;
    }
    __syncthreads();
    float p[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) p[r][c] = 0.f;
#pragma unroll
    for (int f = 0; f < KC; ++f) {
      const float4 av = *reinterpret_cast<const float4*>(&sm.a[f][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&sm.b[f][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float t = aa[r] - bb[c];
          p[r][c] = fmaf(t, t, p[r][c]);
        }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) d2[r][c] += p[r][c];
  }
}

__global__ void init_kernel(const int32_t* __restrict__ nxy, uint32_t* __restrict__ hist,
                            uint32_t* __restrict__ state) {
  const int s = blockIdx.x;
  hist[(int64_t)s * kBins + threadIdx.x] = 0;
  if (threadIdx.x == 0) {
    const int64_t n = (int64_t)nxy[2 * s] * nxy[2 * s + 1];
    state[2 * s] = 0;                                       // digits decided so far
    state[2 * s + 1] = n > 0 ? (uint32_t)((n - 1) / 2) : 0; // rank still to find (torch.median: lower middle)
  }
}

// Histogram of the `pass`-th digit of d^2 over the X-Y pairs whose higher digits equal the prefix found so far.
template <int KC>
__global__ void __launch_bounds__(kThreads) count_kernel(const float* __restrict__ z, int D,
                                                         const int32_t* __restrict__ idx, int L,
                                                         const int32_t* __restrict__ nxy, int pmax,
                                                         uint32_t* __restrict__ hist,
                                                         const uint32_t* __restrict__ state, int pass) {
  __shared__ TileSmem<KC> sm;
  __shared__ uint32_t sh[kBins];
  const int s = blockIdx.x / pmax, b = blockIdx.x % pmax;
  const int nx = nxy[2 * s], ny = nxy[2 * s + 1];
  const int64_t Ty = tiles(ny), T = tiles(nx) * Ty;
  const int P = (int)(T < kParts ? T : kParts);
  if (b >= P) return;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kBins; i += kThreads) sh[i] = 0;
  const uint32_t prefix = state[2 * s];
  const uint32_t hi_mask = pass ? ~0u << (32 - 8 * pass) : 0u;
  const int shift = 24 - 8 * pass;
  const int32_t* rows = idx + (int64_t)s * L;
  for (int64_t t = b; t < T; t += P) {
    const int i = (int)(t / Ty), j = (int)(t % Ty);
    const int na = min(kTile, nx - i * kTile), nb = min(kTile, ny - j * kTile);
    float d2[4][4];
    tile_d2<KC>(z, D, rows + i * kTile, na, rows + nx + j * kTile, nb, sm, d2);
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const uint32_t bits = __float_as_uint(d2[r][c]);
        const bool ok = ty * 4 + r < na && tx * 4 + c < nb && (bits & hi_mask) == prefix;
        const int bin = ok ? (int)((bits >> shift) & (kBins - 1)) : -1;
        const unsigned peers = __match_any_sync(0xffffffffu, bin);
        if (bin >= 0 && __ffs(peers) - 1 == lane) atomicAdd(&sh[bin], (uint32_t)__popc(peers));
      }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += kThreads)
    if (sh[i]) atomicAdd(&hist[(int64_t)s * kBins + i], sh[i]);
}

// One warp per set: the digit whose bin holds the remaining rank; clears the histogram for the next pass.  After the
// last pass the prefix is the median d^2, and its square root the bandwidth.
__global__ void select_kernel(const int32_t* __restrict__ nxy, uint32_t* __restrict__ hist,
                              uint32_t* __restrict__ state, float* __restrict__ bw, int pass) {
  const int s = blockIdx.x, lane = threadIdx.x;
  uint32_t* h = hist + (int64_t)s * kBins;
  const int64_t n = (int64_t)nxy[2 * s] * nxy[2 * s + 1];
  uint32_t c[8], tot = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    c[k] = h[lane * 8 + k];
    tot += c[k];
    h[lane * 8 + k] = 0;
  }
  uint32_t incl = tot;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  const uint32_t excl = incl - tot, rank = state[2 * s + 1];
  const unsigned who = __ballot_sync(0xffffffffu, excl <= rank && rank < incl);
  if (n == 0) {
    if (lane == 0 && pass == kPasses - 1) bw[s] = __int_as_float(0x7fc00000);   // median of nothing: NaN
    return;
  }
  if (who == 0 || lane != __ffs(who) - 1) return;
  uint32_t r = rank - excl;
  int digit = -1;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (digit < 0) {
      if (r < c[k]) digit = k;
      else r -= c[k];
    }
  }
  const uint32_t prefix = state[2 * s] | ((uint32_t)(lane * 8 + digit) << (24 - 8 * pass));
  state[2 * s] = prefix;
  state[2 * s + 1] = r;
  if (pass == kPasses - 1) bw[s] = sqrtf(__uint_as_float(prefix));
}

// Kernel sums of every set: fp64 partials (sum Kxx, sum Kyy, sum Kxy) per CTA.
template <int KC>
__global__ void __launch_bounds__(kThreads) sum_kernel(const float* __restrict__ z, int D,
                                                       const int32_t* __restrict__ idx, int L,
                                                       const int32_t* __restrict__ nxy, int pmax,
                                                       const float* __restrict__ bw, double* __restrict__ parts) {
  __shared__ TileSmem<KC> sm;
  __shared__ double red[3][kThreads];
  const int s = blockIdx.x / pmax, b = blockIdx.x % pmax;
  const int nx = nxy[2 * s], ny = nxy[2 * s + 1];
  const int64_t Tx = tiles(nx), Ty = tiles(ny), Txy = Tx * Ty, T = sum_tiles(nx, ny);
  const int P = (int)(T < kParts ? T : kParts);
  if (b >= P) return;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const double h = bw[s];
  const float c2 = (float)(kLog2e / (2.0 * h * h));   // K = exp(-d^2 / (2 h^2)) = exp2(-d^2 * c2)
  const int32_t* rows = idx + (int64_t)s * L;
  double sxx = 0.0, syy = 0.0, sxy = 0.0;
  for (int64_t t = b; t < T; t += P) {
    int64_t u = t;
    int kind, i, j;   // 0: X-X, 1: Y-Y, 2: X-Y
    if (u < Txy) {
      kind = 2, i = (int)(u / Ty), j = (int)(u % Ty);
    } else if ((u -= Txy) < Tx * Tx) {
      kind = 0, i = (int)(u / Tx), j = (int)(u % Tx);
    } else {
      u -= Tx * Tx;
      kind = 1, i = (int)(u / Ty), j = (int)(u % Ty);
    }
    if (kind != 2 && j < i) continue;   // lower triangle: counted twice through its mirror
    const int32_t* ra = rows + (kind == 1 ? nx : 0) + i * kTile;
    const int32_t* rb = rows + (kind == 0 ? 0 : nx) + j * kTile;
    const int na = min(kTile, (kind == 1 ? ny : nx) - i * kTile), nb = min(kTile, (kind == 0 ? nx : ny) - j * kTile);
    float d2[4][4];
    tile_d2<KC>(z, D, ra, na, rb, nb, sm, d2);
    float acc = 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (ty * 4 + r < na && tx * 4 + c < nb) acc += exp2f(-d2[r][c] * c2);
    const double v = (double)acc * (kind != 2 && i != j ? 2.0 : 1.0);
    if (kind == 0) sxx += v;
    else if (kind == 1) syy += v;
    else sxy += v;
  }
  red[0][threadIdx.x] = sxx;
  red[1][threadIdx.x] = syy;
  red[2][threadIdx.x] = sxy;
  __syncthreads();
  for (int o = kThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o)
#pragma unroll
      for (int k = 0; k < 3; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x < 3) parts[((int64_t)s * kParts + b) * 3 + threadIdx.x] = red[threadIdx.x][0];
}

// The partials of each set in index order, then the reference's statistic (misspecification.py:28-42).
__global__ void finalize_kernel(const int32_t* __restrict__ nxy, int S, const double* __restrict__ parts,
                                int unbiased, double* __restrict__ mmd) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= S) return;
  const double nx = nxy[2 * s], ny = nxy[2 * s + 1];
  const int64_t T = sum_tiles(nxy[2 * s], nxy[2 * s + 1]);
  const int P = (int)(T < kParts ? T : kParts);
  double sxx = 0.0, syy = 0.0, sxy = 0.0;
  for (int b = 0; b < P; ++b) {
    const double* p = parts + ((int64_t)s * kParts + b) * 3;
    sxx += p[0];
    syy += p[1];
    sxy += p[2];
  }
  // torch.mean of an empty matrix and 0/0 are NaN; the unbiased form of a single row divides by zero (inf)
  const double dxx = unbiased ? nx * (nx - 1.0) : nx * nx, dyy = unbiased ? ny * (ny - 1.0) : ny * ny;
  mmd[s] = sxx / dxx + syy / dyy - 2.0 * (sxy / (nx * ny));
}

__global__ void rbf_matrix_kernel(const float* __restrict__ x, int64_t nx, const float* __restrict__ y, int64_t ny,
                                  int D, float c2, float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nx * ny) return;
  const float* a = x + (e / ny) * D;
  const float* b = y + (e % ny) * D;
  float acc = 0.f;
  for (int f = 0; f < D; ++f) {
    const float t = a[f] - b[f];
    acc = fmaf(t, t, acc);
  }
  out[e] = exp2f(-acc * c2);
}

struct Ws {
  uint32_t* hist;
  uint32_t* state;
  double* parts;
};

inline Ws carve(void* ws, int S) {
  char* p = static_cast<char*>(ws);
  Ws w;
  w.parts = reinterpret_cast<double*>(p);
  p += (size_t)S * kParts * 3 * sizeof(double);
  w.hist = reinterpret_cast<uint32_t*>(p);
  p += (size_t)S * kBins * sizeof(uint32_t);
  w.state = reinterpret_cast<uint32_t*>(p);
  return w;
}

// Feature chunk: the largest of 16, 8, 4, 2, 1 whose padding of the last chunk costs at most 1/8 of D.
inline int chunk_for(int D) {
  for (int kc = 16; kc > 1; kc >>= 1)
    if ((int64_t)((D + kc - 1) / kc) * kc * 8 <= (int64_t)D * 9) return kc;
  return 1;
}

template <int KC>
int run(const float* z, int D, const int32_t* idx, int L, const int32_t* nxy, int S, int max_nx, int max_ny,
        int unbiased, int given_bw, float* bw, double* out, const Ws& w, cudaStream_t st) {
  int e = 0;
  if (!given_bw) {
    const int64_t txy = tiles(max_nx) * tiles(max_ny);
    const int pxy = (int)(txy < kParts ? (txy > 0 ? txy : 1) : kParts);
    e = launch(init_kernel, S, kBins, 0, st, nxy, w.hist, w.state);
    for (int pass = 0; pass < kPasses && !e; ++pass) {
      e = launch(count_kernel<KC>, S * pxy, kThreads, 0, st, z, D, idx, L, nxy, pxy, w.hist,
                 (const uint32_t*)w.state, pass);
      if (!e) e = launch(select_kernel, S, 32, 0, st, nxy, w.hist, w.state, bw, pass);
    }
  }
  if (e || out == nullptr) return e;
  const int64_t t = sum_tiles(max_nx, max_ny);
  const int p = (int)(t < kParts ? (t > 0 ? t : 1) : kParts);
  e = launch(sum_kernel<KC>, S * p, kThreads, 0, st, z, D, idx, L, nxy, p, (const float*)bw, w.parts);
  if (!e) e = launch(finalize_kernel, (S + 127) / 128, 128, 0, st, nxy, S, (const double*)w.parts, unbiased, out);
  return e;
}

}  // namespace mmd
}  // namespace sbi

using namespace sbi;

extern "C" int64_t sbi_b200_mmd_ws_bytes(int32_t S) {
  if (S < 1) return 0;
  return (int64_t)S * (mmd::kParts * 3 * sizeof(double) + mmd::kBins * sizeof(uint32_t) + 2 * sizeof(uint32_t));
}

extern "C" int sbi_b200_mmd(const float* d_z, int64_t R, int32_t D, const int32_t* d_idx, int32_t L,
                            const int32_t* d_nxy, int32_t S, int32_t max_nx, int32_t max_ny, int32_t unbiased,
                            int32_t given_bw, float* d_bw, double* d_mmd, void* d_ws, void* stream) {
  if (!d_z || !d_idx || !d_nxy || !d_bw || !d_ws || R < 1 || R > INT32_MAX || D < 1 || S < 1 ||
      S > SBI_MMD_MAX_SETS || L < 1 || L > SBI_MMD_MAX_ROWS || max_nx < 0 || max_ny < 0 ||
      (int64_t)max_nx + max_ny > L || (given_bw && !d_mmd))
    return SBI_EINVAL;
  sbi::DeviceGuard dev_guard_(d_z);
  const mmd::Ws w = mmd::carve(d_ws, S);
  cudaStream_t st = (cudaStream_t)stream;
  switch (mmd::chunk_for(D)) {
    case 16: return mmd::run<16>(d_z, D, d_idx, L, d_nxy, S, max_nx, max_ny, unbiased, given_bw, d_bw, d_mmd, w, st);
    case 8: return mmd::run<8>(d_z, D, d_idx, L, d_nxy, S, max_nx, max_ny, unbiased, given_bw, d_bw, d_mmd, w, st);
    case 4: return mmd::run<4>(d_z, D, d_idx, L, d_nxy, S, max_nx, max_ny, unbiased, given_bw, d_bw, d_mmd, w, st);
    case 2: return mmd::run<2>(d_z, D, d_idx, L, d_nxy, S, max_nx, max_ny, unbiased, given_bw, d_bw, d_mmd, w, st);
    default: return mmd::run<1>(d_z, D, d_idx, L, d_nxy, S, max_nx, max_ny, unbiased, given_bw, d_bw, d_mmd, w, st);
  }
}

extern "C" int sbi_b200_rbf_matrix(const float* d_x, int64_t nx, const float* d_y, int64_t ny, int32_t D,
                                   double bandwidth, float* d_out, void* stream) {
  if (!d_x || !d_y || !d_out || nx < 0 || ny < 0 || D < 1 || (ny > 0 && nx > ((int64_t)1 << 38) / ny))
    return SBI_EINVAL;
  sbi::DeviceGuard dev_guard_(d_x);
  const int64_t n = nx * ny;
  if (n == 0) return 0;
  const float c2 = (float)(mmd::kLog2e / (2.0 * bandwidth * bandwidth));
  return launch(mmd::rbf_matrix_kernel, (int)((n + 255) / 256), 256, 0, (cudaStream_t)stream, d_x, nx, d_y, ny, D,
                c2, d_out);
}
