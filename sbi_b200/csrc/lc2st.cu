// L-C2ST classifiers (reference sbi/diagnostics/lc2st.py): train M independent ReLU-MLP binary classifiers with
// scikit-learn's `MLPClassifier(solver="adam")` algorithm in one launch, and evaluate M parameter sets on S rows.
//
// Training: one persistent CTA per model.  The model's weights and its gradient accumulator live in shared memory
// (each weight matrix with an odd row stride, so column walks are free of bank conflicts); the minibatch streams
// through in TM-row tiles; the Adam moments and the best-so-far weights live in a per-model global workspace that
// stays resident in L2.  Every gradient element is accumulated by one thread over the minibatch rows in row order,
// and every reduction has a fixed order, so a model's result is bit-reproducible and independent of the other
// models of the launch.  The per-epoch early-stopping bookkeeping (sklearn's `_update_no_improvement_count`) runs
// on the device: the host reads nothing until the launch has finished.
//
// Evaluation: one CTA per (row chunk, classifier); a classifier is `E` consecutive parameter sets (an ensemble)
// whose class-0 probabilities 1 - p are averaged, as EnsembleClassifier.predict_proba does.  The score
// sum_s (prob_s - 1/2)^2 / S is reduced in float64, per chunk in row order and then over chunks in chunk order.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

#include "device.cuh"

namespace sbi {
namespace lc2st {

constexpr int kThreads = 256;
constexpr int kMisc = 64;   // floats at the start of shared memory: 16 doubles of reduction scratch, then flags

// Per-layer geometry of the packed (sklearn) and padded (shared-memory) parameter layouts.  Layer l maps
// kin[l] -> kout[l]; packed: [W_0 (kin x kout, row-major), b_0, W_1, b_1, ...], i.e. coefs_[l] then
// intercepts_[l] per layer; padded: the same with row stride ldw[l] = kout[l] | 1.
struct Layout {
  int nl, hmax;
  int kin[SBI_LC2ST_MAX_HIDDEN + 1], kout[SBI_LC2ST_MAX_HIDDEN + 1], ldw[SBI_LC2ST_MAX_HIDDEN + 1];
  int pw[SBI_LC2ST_MAX_HIDDEN + 1], pb[SBI_LC2ST_MAX_HIDDEN + 1];   // packed offsets
  int sw[SBI_LC2ST_MAX_HIDDEN + 1], sb[SBI_LC2ST_MAX_HIDDEN + 1];   // padded offsets
  int P, Ppad, hsum;
};

__host__ __device__ inline Layout make_layout(const sbi_lc2st_net& n) {
  Layout L;
  L.nl = n.L + 1;
  L.hmax = 1;
  L.hsum = 0;
  int p = 0, s = 0;
  for (int l = 0; l < L.nl; ++l) {
    L.kin[l] = l == 0 ? n.F : n.H[l - 1];
    L.kout[l] = l == n.L ? 1 : n.H[l];
    L.ldw[l] = L.kout[l] | 1;
    L.pw[l] = p;
    p += L.kin[l] * L.kout[l];
    L.pb[l] = p;
    p += L.kout[l];
    L.sw[l] = s;
    s += L.kin[l] * L.ldw[l];
    L.sb[l] = s;
    s += L.kout[l];
    if (l < n.L) {
      L.hmax = L.hmax > n.H[l] ? L.hmax : n.H[l];
      L.hsum += n.H[l];
    }
  }
  L.P = p;
  L.Ppad = s;
  return L;
}

// Shared-memory floats of the training kernel at TM rows per tile: reduction scratch, weights, gradient,
// activations of every layer (input, hidden, output), two delta buffers, labels and per-row losses.
__host__ __device__ inline int64_t train_floats(const Layout& L, int F, int TM) {
  return kMisc + 2 * (int64_t)L.Ppad + (int64_t)TM * (F + L.hsum + 1) + 2 * (int64_t)TM * L.hmax + 2 * TM;
}

// Shared-memory floats of the evaluation kernel at TE rows per chunk: weights, input, two activation buffers,
// the class-0 probability accumulator and the output.
__host__ __device__ inline int64_t eval_floats(const Layout& L, int F, int TE) {
  return kMisc + (int64_t)L.Ppad + (int64_t)TE * F + 2 * (int64_t)TE * L.hmax + 2 * TE;
}

inline bool net_ok(const sbi_lc2st_net* n) {
  if (!n || n->F < 1 || n->F > SBI_LC2ST_MAX_F || n->L < 1 || n->L > SBI_LC2ST_MAX_HIDDEN) return false;
  for (int l = 0; l < n->L; ++l)
    if (n->H[l] < 1 || n->H[l] > SBI_LC2ST_MAX_WIDTH) return false;
  return make_layout(*n).P == n->P;
}

// Largest tile of {32, 16, 8} (training) or {64, 32, 16, 8} (evaluation) rows that fits; 0 if none does.
inline int pick_rows(const sbi_lc2st_net* n, bool train) {
  const Layout L = make_layout(*n);
  for (int t = train ? 32 : 64; t >= 8; t >>= 1) {
    const int64_t f = train ? train_floats(L, n->F, t) : eval_floats(L, n->F, t);
    if (f * 4 <= kMaxSmemBytes) return t;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// device building blocks (all threads of the CTA call them; the caller synchronises afterwards)

// out[r][j] = act(sum_k in[r][k] W[k][j] + b[j]) for r < nr; four rows per thread, k in order.
__device__ inline void dense(const float* in, int ldi, int Kin, const float* W, int ldw, const float* b, float* out,
                             int Kout, int nr, bool relu) {
  const int nrb = (nr + 3) >> 2;
  for (int it = threadIdx.x; it < nrb * Kout; it += blockDim.x) {
    const int rb = it / Kout, j = it - rb * Kout, r0 = rb * 4;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    const float* x = in + r0 * ldi;
    for (int k = 0; k < Kin; ++k) {
      const float w = W[k * ldw + j];
      a0 = fmaf(x[k], w, a0);
      a1 = fmaf(x[ldi + k], w, a1);
      a2 = fmaf(x[2 * ldi + k], w, a2);
      a3 = fmaf(x[3 * ldi + k], w, a3);
    }
    const float acc[4] = {a0, a1, a2, a3};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (r0 + q < nr) {
        const float v = acc[q] + b[j];
        out[(r0 + q) * Kout + j] = relu ? fmaxf(v, 0.f) : v;
      }
    }
  }
}

// The logistic output of sklearn (scipy.special.expit) on the float32 logit.
__device__ inline float logistic(float z) { return 1.f / (1.f + expf(-z)); }

// Forward pass of nr rows already in act[0]; leaves post-ReLU activations in act[1..L] and p in act[L+1].
__device__ inline void forward(const Layout& L, const float* W, float* const* act, int nr) {
  for (int l = 0; l < L.nl; ++l) {
    const bool last = l == L.nl - 1;
    dense(act[l], L.kin[l], L.kin[l], W + L.sw[l], L.ldw[l], W + L.sb[l], act[l + 1], L.kout[l], nr, !last);
    __syncthreads();
  }
  float* z = act[L.nl];
  for (int r = threadIdx.x; r < nr; r += blockDim.x) z[r] = logistic(z[r]);
  __syncthreads();
}

// Fixed-order block sum of one double per thread (warp tree, then warps in order by thread 0); all threads get it.
__device__ inline double block_sum(double v, double* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    red[15] = t;
  }
  __syncthreads();
  const double t = red[15];
  __syncthreads();
  return t;
}

// Keyed bijection of [0, n): a 4-round balanced Feistel network on the smallest even number of bits covering n,
// cycle-walked back into range.  Pure arithmetic: an epoch order costs no memory.
__device__ inline uint32_t mix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x7feb352du;
  h ^= h >> 15;
  h *= 0x846ca68bu;
  h ^= h >> 16;
  return h;
}

__device__ inline int feistel_index(int p, int n, uint64_t key, int epoch) {
  int bits = 2;
  while ((1 << bits) < n) bits += 2;
  const int half = bits >> 1;
  const uint32_t mask = (1u << half) - 1u;
  const uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
  const uint32_t e = mix32((uint32_t)epoch * 0x9e3779b9u ^ k1);
  uint32_t x = (uint32_t)p;
  do {
    uint32_t l = x >> half, r = x & mask;
#pragma unroll
    for (int round = 0; round < 4; ++round) {
      const uint32_t f = mix32(r ^ mix32(k0 + e + (uint32_t)round * 0x632be5abu)) & mask;
      const uint32_t nl = r;
      r = l ^ f;
      l = nl;
    }
    x = (l << half) | r;
  } while (x >= (uint32_t)n);
  return (int)x;
}

__device__ inline void load_packed(const Layout& L, const float* src, float* dst) {
  for (int l = 0; l < L.nl; ++l) {
    const int kin = L.kin[l], kout = L.kout[l], ldw = L.ldw[l];
    for (int i = threadIdx.x; i < kin * ldw; i += blockDim.x) {
      const int k = i / ldw, j = i - k * ldw;
      dst[L.sw[l] + i] = j < kout ? src[L.pw[l] + k * kout + j] : 0.f;
    }
    for (int j = threadIdx.x; j < kout; j += blockDim.x) dst[L.sb[l] + j] = src[L.pb[l] + j];
  }
}

__device__ inline void store_packed(const Layout& L, const float* src, float* dst) {
  for (int l = 0; l < L.nl; ++l) {
    const int kin = L.kin[l], kout = L.kout[l], ldw = L.ldw[l];
    for (int i = threadIdx.x; i < kin * kout; i += blockDim.x) {
      const int k = i / kout, j = i - k * kout;
      dst[L.pw[l] + i] = src[L.sw[l] + k * ldw + j];
    }
    for (int j = threadIdx.x; j < kout; j += blockDim.x) dst[L.pb[l] + j] = src[L.sb[l] + j];
  }
}

// ---------------------------------------------------------------------------------------------------------------
struct TrainArgs {
  sbi_lc2st_net net;
  sbi_lc2st_opt opt;
  const sbi_lc2st_job* jobs;
  const float* theta;
  const float* x;
  int dt, dx, TM;
  const int32_t* rows;
  const float* labels;
  const int32_t* order;
  float* params;
  float* ws;
  int32_t* n_iter;
  double* val_curve;
  double* loss_curve;
  double* best;
};

__global__ void __launch_bounds__(kThreads) train_kernel(TrainArgs a) {
  extern __shared__ __align__(16) float sm[];
  const Layout L = make_layout(a.net);
  const sbi_lc2st_opt& o = a.opt;
  const int m = blockIdx.x, TM = a.TM, F = a.net.F, tid = threadIdx.x;
  const sbi_lc2st_job J = a.jobs[m];
  const int n_train = J.n_train, n_val = J.n_val;

  double* red = reinterpret_cast<double*>(sm);
  float* W = sm + kMisc;
  float* G = W + L.Ppad;
  float* act[SBI_LC2ST_MAX_HIDDEN + 2];
  act[0] = G + L.Ppad;
  for (int l = 0; l < L.nl; ++l) act[l + 1] = act[l] + TM * L.kin[l];
  float* dbuf[2] = {act[L.nl] + TM, act[L.nl] + TM + TM * L.hmax};
  float* lab = dbuf[1] + TM * L.hmax;
  float* rowv = lab + TM;
  int* s_flag = reinterpret_cast<int*>(sm + 32);   // after the 16 doubles of `red`

  float* mom = a.ws + (int64_t)m * 3 * L.Ppad;
  float* vel = mom + L.Ppad;
  float* best = vel + L.Ppad;
  float* out = a.params + (int64_t)m * L.P;

  load_packed(L, out, W);
  for (int i = tid; i < L.Ppad; i += blockDim.x) G[i] = 0.f;
  __syncthreads();
  for (int i = tid; i < L.Ppad; i += blockDim.x) {
    mom[i] = 0.f;
    vel[i] = 0.f;
    best[i] = W[i];
  }

  const int batch = o.batch_size < 1 ? (n_train < 200 ? n_train : 200) : (o.batch_size < n_train ? o.batch_size
                                                                                                  : n_train);
  const int32_t* rows = a.rows + 2 * J.row0;
  const float* labels = a.labels + J.row0;
  const float alpha = o.alpha, b1 = o.beta1, b2 = o.beta2, omb1 = o.one_minus_beta1, omb2 = o.one_minus_beta2;
  const float eps_f = o.eps, eps_p = 1.1920928955078125e-07f;   // np.finfo(float32).eps clips the log loss

  // feature row r of the tile <- sample `s` of this model (train: s < n_train, validation: n_train + s)
  auto load_tile = [&](int nr, auto sample_of) {
    for (int i = tid; i < nr * F; i += blockDim.x) {
      const int r = i / F, c = i - r * F;
      const int s = sample_of(r);
      const int32_t ti = rows[2 * s], xi = rows[2 * s + 1];
      act[0][i] = c < a.dt ? a.theta[(int64_t)ti * a.dt + c] : a.x[(int64_t)xi * a.dx + (c - a.dt)];
    }
    for (int r = tid; r < nr; r += blockDim.x) lab[r] = labels[sample_of(r)];
    __syncthreads();
  };

  double best_score = -INFINITY, best_loss = INFINITY;
  int no_improve = 0, n_iter = 0, t = 0;
  for (int it = 0; it < o.max_iter; ++it) {
    double epoch_loss = 0.0;   // thread 0
    for (int b0 = 0; b0 < n_train; b0 += batch) {
      const int blen = n_train - b0 < batch ? n_train - b0 : batch;
      double batch_loss = 0.0;   // thread 0: sum of the rows' clipped log losses
      for (int r0 = 0; r0 < blen; r0 += TM) {
        const int nr = blen - r0 < TM ? blen - r0 : TM;
        load_tile(nr, [&](int r) {
          const int p = b0 + r0 + r;
          if (J.order0 >= 0) return a.order[J.order0 + (int64_t)it * n_train + p];
          return o.shuffle ? feistel_index(p, n_train, J.key, it) : p;
        });
        forward(L, W, act, nr);
        // output delta p - y and the per-row log loss
        const float* p = act[L.nl];
        float* d = dbuf[L.nl & 1];
        for (int r = tid; r < nr; r += blockDim.x) {
          const float y = lab[r];
          d[r] = p[r] - y;
          const float pc = fminf(fmaxf(p[r], eps_p), 1.f - eps_p);
          rowv[r] = y > 0.5f ? -logf(pc) : -logf(1.f - pc);
        }
        __syncthreads();
        if (tid == 0)
          for (int r = 0; r < nr; ++r) batch_loss += (double)rowv[r];
        // backward: layer l's gradient from its input act[l] and its delta; then the delta of layer l - 1
        for (int l = L.nl - 1; l >= 0; --l) {
          const int kin = L.kin[l], kout = L.kout[l], ldw = L.ldw[l];
          const float* dl = dbuf[(l + 1) & 1];
          const float* al = act[l];
          float* gw = G + L.sw[l];
          for (int i = tid; i < kin * kout; i += blockDim.x) {
            const int k = i / kout, j = i - k * kout;
            float g = gw[k * ldw + j];
            for (int r = 0; r < nr; ++r) g = fmaf(al[r * kin + k], dl[r * kout + j], g);
            gw[k * ldw + j] = g;
          }
          for (int j = tid; j < kout; j += blockDim.x) {
            float g = G[L.sb[l] + j];
            for (int r = 0; r < nr; ++r) g += dl[r * kout + j];
            G[L.sb[l] + j] = g;
          }
          if (l > 0) {
            // delta_{l-1}[r][k] = sum_j delta_l[r][j] W_l[k][j], zero where the ReLU output act[l][r][k] is 0
            float* dn = dbuf[l & 1];
            const float* w = W + L.sw[l];
            const int nrb = (nr + 3) >> 2;
            for (int i = tid; i < nrb * kin; i += blockDim.x) {
              const int rb = i / kin, k = i - rb * kin, q0 = rb * 4;
              float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
              for (int j = 0; j < kout; ++j) {
                const float wv = w[k * ldw + j];
                s0 = fmaf(dl[q0 * kout + j], wv, s0);
                s1 = fmaf(dl[(q0 + 1) * kout + j], wv, s1);
                s2 = fmaf(dl[(q0 + 2) * kout + j], wv, s2);
                s3 = fmaf(dl[(q0 + 3) * kout + j], wv, s3);
              }
              const float s[4] = {s0, s1, s2, s3};
#pragma unroll
              for (int q = 0; q < 4; ++q)
                if (q0 + q < nr) dn[(q0 + q) * kin + k] = al[(q0 + q) * kin + k] == 0.f ? 0.f : s[q];
            }
          }
          __syncthreads();
        }
      }
      // Adam step as numpy 2 evaluates sklearn's expressions (no contraction): the moments in float32; the step
      // size lr_t is a float64 scalar, so -lr_t * m / (sqrt(v) + eps) is a float64 array that `param += update`
      // rounds to float32 once
      ++t;
      const double lr_t = o.lr_d * sqrt(1.0 - pow(o.beta2_d, (double)t)) / (1.0 - pow(o.beta1_d, (double)t));
      const float fn = (float)blen;
      float sumsq = 0.f;
      for (int l = 0; l < L.nl; ++l) {
        const int kin = L.kin[l], kout = L.kout[l], ldw = L.ldw[l];
        for (int i = tid; i < kin * ldw + kout; i += blockDim.x) {
          const bool coef = i < kin * ldw;
          if (coef && i % ldw >= kout) continue;   // padding column
          const int at = L.sw[l] + i;               // the bias block follows the weight block
          const float w = W[at];
          const float g = coef ? __fdiv_rn(__fadd_rn(G[at], __fmul_rn(alpha, w)), fn) : __fdiv_rn(G[at], fn);
          if (coef) sumsq = fmaf(w, w, sumsq);
          const float mv = __fadd_rn(__fmul_rn(b1, mom[at]), __fmul_rn(omb1, g));
          const float vv = __fadd_rn(__fmul_rn(b2, vel[at]), __fmul_rn(omb2, __fmul_rn(g, g)));
          mom[at] = mv;
          vel[at] = vv;
          const float den = __fadd_rn(__fsqrt_rn(vv), eps_f);
          W[at] = (float)__dadd_rn((double)w, __ddiv_rn(__dmul_rn(-lr_t, (double)mv), (double)den));
          G[at] = 0.f;
        }
      }
      const double ss = block_sum((double)sumsq, red);   // ends with a barrier: W is updated everywhere
      if (tid == 0) epoch_loss += (batch_loss / blen + 0.5 * (double)alpha * ss / blen) * blen;
    }
    ++n_iter;
    // sklearn's _update_no_improvement_count, on the validation accuracy or on the epoch loss
    if (tid == 0) {
      const double loss = epoch_loss / n_train;
      a.loss_curve[(int64_t)m * o.max_iter + it] = loss;
      s_flag[0] = 0;
      if (!o.early_stopping) {
        no_improve = loss > best_loss - o.tol ? no_improve + 1 : 0;
        if (loss < best_loss) best_loss = loss;
      }
    }
    if (o.early_stopping) {
      int correct = 0;   // thread 0
      for (int r0 = 0; r0 < n_val; r0 += TM) {
        const int nr = n_val - r0 < TM ? n_val - r0 : TM;
        load_tile(nr, [&](int r) { return n_train + r0 + r; });
        forward(L, W, act, nr);
        if (tid == 0)
          for (int r = 0; r < nr; ++r) correct += ((act[L.nl][r] > 0.5f) == (lab[r] > 0.5f)) ? 1 : 0;
        __syncthreads();
      }
      if (tid == 0) {
        const double score = (double)correct / n_val;
        a.val_curve[(int64_t)m * o.max_iter + it] = score;
        no_improve = score < best_score + o.tol ? no_improve + 1 : 0;
        if (score > best_score) {
          best_score = score;
          s_flag[0] = 1;
        }
      }
    }
    if (tid == 0) s_flag[1] = no_improve > o.n_iter_no_change;
    __syncthreads();
    if (s_flag[0])
      for (int i = tid; i < L.Ppad; i += blockDim.x) best[i] = W[i];
    const bool stop = s_flag[1];
    __syncthreads();
    if (stop) break;
  }
  // the restored best weights (early stopping) or the last ones
  __syncthreads();
  store_packed(L, o.early_stopping ? best : W, out);
  if (tid == 0) {
    a.n_iter[m] = n_iter;
    a.best[m] = o.early_stopping ? best_score : best_loss;
  }
}

// ---------------------------------------------------------------------------------------------------------------
struct EvalArgs {
  sbi_lc2st_net net;
  const float* params;
  int E, dt, dx, TE, nchunk;
  int64_t S;
  const float* theta;
  const int32_t* group;
  const float* x;
  float* prob;
  double* part;
};

__global__ void __launch_bounds__(kThreads) eval_kernel(EvalArgs a) {
  extern __shared__ __align__(16) float sm[];
  const Layout L = make_layout(a.net);
  const int c = blockIdx.y, ch = blockIdx.x, TE = a.TE, F = a.net.F, tid = threadIdx.x;
  const int64_t s0 = (int64_t)ch * TE;
  const int nr = (int)(a.S - s0 < TE ? a.S - s0 : TE);
  float* W = sm + kMisc;
  float* in = W + L.Ppad;
  float* buf[2] = {in + TE * F, in + TE * F + TE * L.hmax};
  float* acc = buf[1] + TE * L.hmax;
  float* sq = acc + TE;

  const int g = a.group ? a.group[c] : 0;
  const float* th = a.theta + ((int64_t)g * a.S + s0) * a.dt;
  for (int i = tid; i < nr * F; i += blockDim.x) {
    const int r = i / F, k = i - r * F;
    in[i] = k < a.dt ? th[(int64_t)r * a.dt + k] : a.x[k - a.dt];
  }
  for (int r = tid; r < TE; r += blockDim.x) acc[r] = 0.f;
  for (int e = 0; e < a.E; ++e) {
    __syncthreads();
    load_packed(L, a.params + ((int64_t)c * a.E + e) * L.P, W);
    __syncthreads();
    const float* cur = in;
    for (int l = 0; l < L.nl; ++l) {
      float* nxt = buf[l & 1];
      dense(cur, L.kin[l], L.kin[l], W + L.sw[l], L.ldw[l], W + L.sb[l], nxt, L.kout[l], nr, l < L.nl - 1);
      __syncthreads();
      cur = nxt;
    }
    for (int r = tid; r < nr; r += blockDim.x) acc[r] += 1.f - logistic(cur[r]);
  }
  __syncthreads();
  for (int r = tid; r < nr; r += blockDim.x) {
    const float pr = a.E == 1 ? acc[r] : acc[r] / (float)a.E;
    a.prob[(int64_t)c * a.S + s0 + r] = pr;
    sq[r] = pr;
  }
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int r = 0; r < nr; ++r) {
      const double d = (double)sq[r] - 0.5;
      s += d * d;
    }
    a.part[(int64_t)c * a.nchunk + ch] = s;
  }
}

__global__ void score_kernel(const double* part, int C, int nchunk, int64_t S, double* score) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double s = 0.0;
  for (int i = 0; i < nchunk; ++i) s += part[(int64_t)c * nchunk + i];
  score[c] = s / (double)S;
}

}  // namespace lc2st
}  // namespace sbi

using namespace sbi;

extern "C" int sbi_b200_lc2st_plan(const sbi_lc2st_net* net, int32_t* out3) {
  if (!out3 || !lc2st::net_ok(net)) return SBI_EINVAL;
  const lc2st::Layout L = lc2st::make_layout(*net);
  const int tm = lc2st::pick_rows(net, true), te = lc2st::pick_rows(net, false);
  out3[0] = tm;
  out3[1] = te;
  out3[2] = L.Ppad;
  return tm > 0 && te > 0 ? 0 : SBI_ESMEM;
}

extern "C" int64_t sbi_b200_lc2st_ws_floats(const sbi_lc2st_net* net, int32_t M) {
  if (!lc2st::net_ok(net) || M < 0) return -1;
  return 3 * (int64_t)lc2st::make_layout(*net).Ppad * M;
}

extern "C" int sbi_b200_lc2st_eval_chunks(const sbi_lc2st_net* net, int64_t S) {
  if (!lc2st::net_ok(net) || S < 1) return SBI_EINVAL;
  const int te = lc2st::pick_rows(net, false);
  if (te == 0) return SBI_ESMEM;
  const int64_t n = (S + te - 1) / te;
  return n > 65535 * 1024LL ? SBI_EINVAL : (int)n;
}

extern "C" int sbi_b200_lc2st_train(const sbi_lc2st_net* net, const sbi_lc2st_opt* opt, const sbi_lc2st_job* d_jobs,
                                    int32_t M, const float* d_theta, int32_t dt, const float* d_x, int32_t dx,
                                    const int32_t* d_rows, const float* d_labels, const int32_t* d_order,
                                    float* d_params, float* d_ws, int32_t* d_n_iter, double* d_val_curve,
                                    double* d_loss_curve, double* d_best, void* stream) {
  if (!lc2st::net_ok(net) || !opt || !d_jobs || M < 0 || dt < 0 || dx < 0 || dt + dx != net->F || !d_rows ||
      !d_labels || !d_params || !d_ws || !d_n_iter || !d_val_curve || !d_loss_curve || !d_best ||
      (dt > 0 && !d_theta) || (dx > 0 && !d_x) || opt->max_iter < 1 || opt->n_iter_no_change < 0)
    return SBI_EINVAL;
  sbi::DeviceGuard dev_guard_(d_params);
  if (M == 0) return 0;
  const int tm = lc2st::pick_rows(net, true);
  if (tm == 0) return SBI_ESMEM;
  lc2st::TrainArgs a{*net,  *opt,     d_jobs,  d_theta, d_x,    dt,          dx,           tm,    d_rows,
                     d_labels, d_order, d_params, d_ws, d_n_iter, d_val_curve, d_loss_curve, d_best};
  const int smem = (int)(lc2st::train_floats(lc2st::make_layout(*net), net->F, tm) * 4);
  return launch(lc2st::train_kernel, M, lc2st::kThreads, smem, (cudaStream_t)stream, a);
}

extern "C" int sbi_b200_lc2st_eval(const sbi_lc2st_net* net, const float* d_params, int32_t C, int32_t E,
                                   const float* d_theta, int32_t dt, int64_t S, const int32_t* d_group,
                                   const float* d_x, int32_t dx, float* d_prob, double* d_part, double* d_score,
                                   void* stream) {
  if (!lc2st::net_ok(net) || !d_params || C < 0 || C > 65535 || E < 1 || dt < 0 || dx < 0 || dt + dx != net->F ||
      S < 1 || (dt > 0 && !d_theta) || (dx > 0 && !d_x) || !d_prob || !d_part || !d_score)
    return SBI_EINVAL;
  sbi::DeviceGuard dev_guard_(d_params);
  if (C == 0) return 0;
  const int nchunk = sbi_b200_lc2st_eval_chunks(net, S);
  if (nchunk < 0) return nchunk;
  const int te = lc2st::pick_rows(net, false);
  lc2st::EvalArgs a{*net, d_params, E, dt, dx, te, nchunk, S, d_theta, d_group, d_x, d_prob, d_part};
  const int smem = (int)(lc2st::eval_floats(lc2st::make_layout(*net), net->F, te) * 4);
  cudaStream_t s = (cudaStream_t)stream;
  if (int e = set_smem(reinterpret_cast<const void*>(lc2st::eval_kernel), smem)) return e;
  lc2st::eval_kernel<<<dim3(nchunk, C), lc2st::kThreads, smem, s>>>(a);
  if (int e = (int)cudaGetLastError()) return e;
  return launch(lc2st::score_kernel, (C + 127) / 128, 128, 0, s, (const double*)d_part, (int)C, nchunk, S, d_score);
}
