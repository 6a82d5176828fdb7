// Lock-step HMC and NUTS: the transition kernels of `mcmc_method="hmc_pyro"` / `"nuts_pyro"` with pyro's
// defaults (DESIGN §3.6 states the algorithm as this project's contract).  One thread per chain and one launch
// per lock-step; every lock-step is one leapfrog step of every chain, so the host evaluates log p and its
// gradient once per launch.  Chain state lives in HBM in float64, column-per-chain (include/sbi_b200.h).
//
// NUTS (Hoffman & Gelman 2014, Betancourt 2017): the trajectory doubles in a random direction until the
// generalized U-turn criterion holds, a leaf diverges or max_tree_depth doublings are done.  A doubling of
// depth j produces its 2^j leaves one per lock-step from the frontier in its direction; the completed subtrees
// of the doubling are kept in slots by size (slot k holds a 2^k-leaf subtree), like the bits of a counter, so
// leaf n closes the subtrees of its trailing one-bits, innermost first, as the recursive builder would.  Each
// slot holds the subtree's momentum sum, its first momentum, its proposal and its log-weight.  Inside a
// doubling the proposal is sampled uniformly (multinomial), at the top level with the biased rule.
// HMC: a fixed trajectory of max(1, int(trajectory_length / step_size)) leapfrog steps and a Metropolis test.
// Adaptation per chain: dual averaging of log(step size), Stan's windows for the diagonal inverse mass matrix
// (regularised Welford variance), and the step-size search at the start and after every mass-matrix window.
#include <cuda_runtime.h>
#include <math.h>

#include "../../include/sbi_b200.h"
#include "device.cuh"

namespace sbi {
namespace {

// working vectors: gradient at the chain position, the two frontier states (position, momentum, gradient),
// the momentum sum of the whole trajectory, the inverse mass diagonal, the Welford accumulators; then per
// slot k: momentum sum, first momentum, proposal position, proposal gradient
enum { V_GZ = 0, V_Z0 = 1, V_R0 = 2, V_G0 = 3, V_Z1 = 4, V_R1 = 5, V_G1 = 6, V_RSUM = 7, V_MINV = 8,
       V_WMEAN = 9, V_WM2 = 10 };
static_assert(V_WM2 + 1 == SBI_HMC_NV0, "vector count");
enum { S_RSUM = 0, S_RFIRST = 1, S_Z = 2, S_G = 3 };
// int state: phase, transitions done, completed doublings, leaf index in the doubling, direction, HMC steps
// left, leapfrog steps in the transition, adaptation window, Welford count, dual-averaging count, step-search
// direction and trials, post-warm-up divergences, divergent flag of the transition
enum { I_PHASE = 0, I_T, I_DEPTH, I_N, I_DIR, I_STEPS, I_NLF, I_WIN, I_WN, I_DAT, I_FDIR, I_FTRIAL, I_NDIV,
       I_DIVERGED };
static_assert(I_DIVERGED + 1 == SBI_HMC_NI, "int state count");
// double state: potential at the position, initial energy, step size, tree log-weight, accept-stat sum of the
// transition, dual averaging (averaged iterate, averaged statistic, prox centre), post-warm-up sums of the
// accept stat and the tree depth; then per slot k: log-weight, potential of the proposal
enum { F_PEZ = 0, F_H0, F_EPS, F_WTREE, F_SACC, F_XBAR, F_GBAR, F_MU, F_SACC_POST, F_SDEPTH_POST };
static_assert(F_SDEPTH_POST + 1 == SBI_HMC_NF0, "double state count");

constexpr double kMaxDeltaEnergy = 1000.0;   // divergence threshold on H - H0
constexpr double kDaT0 = 10.0, kDaKappa = 0.75, kDaGamma = 0.05;
constexpr double kSearchLogAccept = -0.22314355131420976;   // log(0.8): the step-size search's threshold
constexpr int kMaxSearchTrials = 100;      // the search stops 2^±100 away from where it started
constexpr double kMaxHmcSteps = 1e9;

struct Ch {
  const sbi_hmc_chains& s;
  int c;
  __device__ double& v(int vec, int d) const { return s.d_vec[((size_t)vec * s.D + d) * s.C + c]; }
  __device__ double& z(int d) const { return s.d_z[(size_t)c * s.D + d]; }
  __device__ int32_t& i(int k) const { return s.d_istate[(size_t)k * s.C + c]; }
  __device__ double& f(int k) const { return s.d_fstate[(size_t)k * s.C + c]; }
  __device__ double u(int k) const { return s.d_uniform[(size_t)k * s.C + c]; }
  __device__ double& sw(int k) const { return f(SBI_HMC_NF0 + 2 * k); }
  __device__ double& spe(int k) const { return f(SBI_HMC_NF0 + 2 * k + 1); }
  __device__ void copy(int dst, int src) const {
    for (int d = 0; d < s.D; ++d) v(dst, d) = v(src, d);
  }
};

__device__ __forceinline__ int slot(int k, int part) { return SBI_HMC_NV0 + 4 * k + part; }

__device__ __forceinline__ double logaddexp(double a, double b) {
  const double m = fmax(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + log(exp(a - m) + exp(b - m));
}

// H - H0 of a leapfrog point; not finite (NaN potential, energy or gradient) counts as +inf
__device__ __forceinline__ double delta_energy(double pe, double kin, double h0) {
  const double dh = pe + kin - h0;
  return isnan(dh) ? INFINITY : dh;
}

// fresh momentum r = M^(1/2) n in the frontier-0 state, which starts at the chain position; returns the energy
__device__ double start_at_position(const Ch& h) {
  double kin = 0.0;
  for (int d = 0; d < h.s.D; ++d) {
    const double minv = h.v(V_MINV, d);
    const double r = h.s.d_normal[(size_t)d * h.s.C + h.c] / sqrt(minv);
    h.v(V_R0, d) = r;
    h.v(V_Z0, d) = h.z(d);
    h.v(V_G0, d) = h.v(V_GZ, d);
    kin += 0.5 * minv * r * r;
  }
  return h.f(F_PEZ) + kin;
}

// first half of a leapfrog step of signed size `step` on the state (zv, zv+1, zv+2); writes the new position
__device__ void leapfrog_begin(const Ch& h, int zv, double step) {
  float* p = h.s.d_params + (size_t)h.c * h.s.D;
  for (int d = 0; d < h.s.D; ++d) {
    const double r = h.v(zv + 1, d) - 0.5 * step * h.v(zv + 2, d);
    const double z = h.v(zv, d) + step * h.v(V_MINV, d) * r;
    h.v(zv + 1, d) = r;
    h.v(zv, d) = z;
    p[d] = (float)z;
  }
}

// second half with the gradient of U = -log p evaluated by the host; returns the kinetic energy, NaN when the
// gradient is not finite
__device__ double leapfrog_end(const Ch& h, int zv, double step) {
  const float* gl = h.s.d_grad + (size_t)h.c * h.s.D;
  double kin = 0.0;
  bool finite = true;
  for (int d = 0; d < h.s.D; ++d) {
    const double g = -(double)gl[d];
    finite = finite && isfinite(g);
    const double r = h.v(zv + 1, d) - 0.5 * step * g;
    h.v(zv + 2, d) = g;
    h.v(zv + 1, d) = r;
    kin += 0.5 * h.v(V_MINV, d) * r * r;
  }
  return finite ? kin : NAN;
}

// generalized U-turn criterion (Betancourt 2017, A.4.2): rho = sum r - (ra + rb) / 2 against M^-1 ra, M^-1 rb
__device__ bool turning(const Ch& h, int rsum, int ra, int rb) {
  double la = 0.0, lb = 0.0;
  for (int d = 0; d < h.s.D; ++d) {
    const double a = h.v(ra, d), b = h.v(rb, d), minv = h.v(V_MINV, d);
    const double rho = h.v(rsum, d) - 0.5 * (a + b);
    la += minv * a * rho;
    lb += minv * b * rho;
  }
  return la <= 0.0 || lb <= 0.0;
}

// the chain position becomes the frontier state `zv` (NUTS proposal / accepted HMC end point)
__device__ void take_proposal(const Ch& h, int zv, int gv, double pe) {
  for (int d = 0; d < h.s.D; ++d) {
    h.z(d) = h.v(zv, d);
    h.v(V_GZ, d) = h.v(gv, d);
  }
  h.f(F_PEZ) = pe;
}

__device__ void search_trial(const Ch& h) {
  h.f(F_H0) = start_at_position(h);
  h.i(I_PHASE) = SBI_HMC_PHASE_FIND;
  leapfrog_begin(h, V_Z0, h.f(F_EPS));
}

__device__ void start_doubling(const Ch& h) {
  const int dir = h.u(0) < 0.5 ? 1 : -1;
  h.i(I_DIR) = dir;
  h.i(I_N) = 0;
  leapfrog_begin(h, dir > 0 ? V_Z1 : V_Z0, dir * h.f(F_EPS));
}

__device__ void start_transition(const Ch& h, int32_t* n_done) {
  if (h.i(I_T) >= h.s.warmup + h.s.num_samples) {
    h.i(I_PHASE) = SBI_HMC_PHASE_DONE;
    atomicAdd(n_done, 1);
    return;
  }
  h.i(I_PHASE) = SBI_HMC_PHASE_TRAJ;
  h.f(F_H0) = start_at_position(h);
  h.i(I_NLF) = 0;
  h.i(I_DIVERGED) = 0;
  h.i(I_DEPTH) = 0;
  h.f(F_SACC) = 0.0;
  const double eps = h.f(F_EPS);
  if (h.s.algo == SBI_HMC_HMC) {
    h.i(I_STEPS) = (int)fmax(1.0, fmin(kMaxHmcSteps, floor(h.s.trajectory_length / eps)));
    leapfrog_begin(h, V_Z0, eps);
    return;
  }
  h.copy(V_Z1, V_Z0);
  h.copy(V_R1, V_R0);
  h.copy(V_G1, V_G0);
  h.copy(V_RSUM, V_R0);
  h.f(F_WTREE) = 0.0;
  start_doubling(h);
}

// dual averaging (Nesterov 2009 as in Hoffman & Gelman 2014, Alg. 5) on log(step size), statistic g
__device__ void dual_averaging_step(const Ch& h, double g) {
  const int t = ++h.i(I_DAT);
  const double gbar = (1.0 - 1.0 / (t + kDaT0)) * h.f(F_GBAR) + g / (t + kDaT0);
  const double x = h.f(F_MU) - sqrt((double)t) / kDaGamma * gbar;
  const double w = pow((double)t, -kDaKappa);
  h.f(F_GBAR) = gbar;
  h.f(F_XBAR) = (1.0 - w) * h.f(F_XBAR) + w * x;
  h.f(F_EPS) = exp(x);
}

// warm-up transition t done with accept statistic `acc`; returns true when a step-size search has started
__device__ bool adapt(const Ch& h, int t, double acc) {
  const int w = h.i(I_WIN), nw = h.s.n_windows;
  const bool mass_phase = h.s.adapt_mass_matrix && w > 0 && w < nw - 1;
  if (h.s.adapt_step_size) dual_averaging_step(h, h.s.target_accept - acc);
  if (mass_phase) {   // Welford on the position after the transition
    const int n = ++h.i(I_WN);
    for (int d = 0; d < h.s.D; ++d) {
      const double x = h.z(d);
      const double pre = x - h.v(V_WMEAN, d);
      const double mean = h.v(V_WMEAN, d) + pre / n;
      h.v(V_WMEAN, d) = mean;
      h.v(V_WM2, d) += pre * (x - mean);
    }
  }
  if (w >= nw || t != h.s.win_end[w]) return false;
  if (w == nw - 1) {   // end of warm-up: the averaged iterate
    if (h.s.adapt_step_size) h.f(F_EPS) = exp(h.f(F_XBAR));
    h.i(I_WIN) = w + 1;
    return false;
  }
  h.i(I_WIN) = w + 1;
  if (!mass_phase) return false;
  const int n = h.i(I_WN);
  if (n >= 2) {   // regularised towards 1e-3 as in Stan
    const double a = n / (n + 5.0), b = 1e-3 * 5.0 / (n + 5.0);
    for (int d = 0; d < h.s.D; ++d) h.v(V_MINV, d) = a * h.v(V_WM2, d) / (n - 1) + b;
  }
  h.i(I_WN) = 0;
  for (int d = 0; d < h.s.D; ++d) {
    h.v(V_WMEAN, d) = 0.0;
    h.v(V_WM2, d) = 0.0;
  }
  if (!h.s.adapt_step_size) return false;
  search_trial(h);
  return true;
}

__device__ void end_transition(const Ch& h, double acc, int32_t* n_done) {
  const int t = h.i(I_T);
  const int D = h.s.D;
  if (h.s.d_trace) {
    double* tr = h.s.d_trace + ((size_t)h.c * (h.s.warmup + h.s.num_samples) + t) * (2 * D + SBI_HMC_TRACE_SCALARS);
    for (int d = 0; d < D; ++d) {
      tr[d] = h.z(d);
      tr[D + d] = h.v(V_MINV, d);
    }
    tr[2 * D] = h.i(I_DEPTH);
    tr[2 * D + 1] = h.i(I_NLF);
    tr[2 * D + 2] = h.i(I_DIVERGED);
    tr[2 * D + 3] = acc;
    tr[2 * D + 4] = h.f(F_EPS);
  }
  h.i(I_T) = t + 1;
  if (t < h.s.warmup) {
    if (adapt(h, t, acc)) return;
  } else {
    double* dst = h.s.d_samples + ((size_t)h.c * h.s.num_samples + (t - h.s.warmup)) * D;
    for (int d = 0; d < D; ++d) dst[d] = h.z(d);
    h.f(F_SACC_POST) += acc;
    h.f(F_SDEPTH_POST) += h.i(I_DEPTH);
    h.i(I_NDIV) += h.i(I_DIVERGED);
  }
  start_transition(h, n_done);
}

// a NUTS leaf has been evaluated
__device__ void nuts_leaf(const Ch& h, double pe, int32_t* n_done) {
  const int dir = h.i(I_DIR);
  const int zv = dir > 0 ? V_Z1 : V_Z0;
  const double eps = h.f(F_EPS);
  const double dh = delta_energy(pe, leapfrog_end(h, zv, dir * eps), h.f(F_H0));
  h.i(I_NLF) += 1;
  h.f(F_SACC) += dh > 0.0 ? exp(-dh) : 1.0;
  const double mean_acc = h.f(F_SACC) / h.i(I_NLF);
  if (dh > kMaxDeltaEnergy) {
    h.i(I_DIVERGED) = 1;
    end_transition(h, mean_acc, n_done);
    return;
  }
  const int n = h.i(I_N), j = h.i(I_DEPTH);
  const int L = __ffs(~n) - 1;   // subtrees closed by this leaf: the trailing one-bits of n
  const int acc = slot(L, 0);
  for (int d = 0; d < h.s.D; ++d) {
    const double r = h.v(zv + 1, d);
    h.v(acc + S_RSUM, d) = r;
    h.v(acc + S_RFIRST, d) = r;
    h.v(acc + S_Z, d) = h.v(zv, d);
    h.v(acc + S_G, d) = h.v(zv + 2, d);
  }
  h.sw(L) = -dh;
  h.spe(L) = pe;
  for (int k = 0; k < L; ++k) {   // slot k is the first half, the accumulator the second half
    const int sk = slot(k, 0);
    const double wn = logaddexp(h.sw(k), h.sw(L));
    if (!(h.u(1 + k) < exp(h.sw(L) - wn))) {
      h.copy(acc + S_Z, sk + S_Z);
      h.copy(acc + S_G, sk + S_G);
      h.spe(L) = h.spe(k);
    }
    for (int d = 0; d < h.s.D; ++d) h.v(acc + S_RSUM, d) += h.v(sk + S_RSUM, d);
    h.sw(L) = wn;
    if (turning(h, acc + S_RSUM, sk + S_RFIRST, zv + 1)) {
      end_transition(h, mean_acc, n_done);
      return;
    }
  }
  if (L > 0) h.copy(acc + S_RFIRST, slot(L - 1, S_RFIRST));
  if (L < j) {
    h.i(I_N) = n + 1;
    leapfrog_begin(h, zv, dir * eps);
    return;
  }
  // the doubling is complete: the biased top-level choice, then the U-turn test of the whole trajectory
  h.i(I_DEPTH) = j + 1;
  if (h.u(h.s.max_tree_depth) < exp(h.sw(L) - h.f(F_WTREE))) take_proposal(h, acc + S_Z, acc + S_G, h.spe(L));
  for (int d = 0; d < h.s.D; ++d) h.v(V_RSUM, d) += h.v(acc + S_RSUM, d);
  if (turning(h, V_RSUM, V_R0, V_R1) || j + 1 >= h.s.max_tree_depth) {
    end_transition(h, mean_acc, n_done);
    return;
  }
  h.f(F_WTREE) = logaddexp(h.f(F_WTREE), h.sw(L));
  start_doubling(h);
}

__device__ void hmc_leaf(const Ch& h, double pe, int32_t* n_done) {
  const double eps = h.f(F_EPS);
  const double dh = delta_energy(pe, leapfrog_end(h, V_Z0, eps), h.f(F_H0));
  h.i(I_NLF) += 1;
  const int left = h.i(I_STEPS) - 1;
  h.i(I_STEPS) = left;
  if (dh > kMaxDeltaEnergy) {   // divergent: the trajectory stops and the transition is rejected
    h.i(I_DIVERGED) = 1;
    end_transition(h, 0.0, n_done);
    return;
  }
  if (left > 0) {
    leapfrog_begin(h, V_Z0, eps);
    return;
  }
  const double acc = dh > 0.0 ? exp(-dh) : 1.0;
  if (h.u(h.s.max_tree_depth) < acc) take_proposal(h, V_Z0, V_G0, pe);
  end_transition(h, acc, n_done);
}

// one trial of the step-size search has been evaluated: double or halve until the sign of dH + log 0.8 changes
__device__ void search_result(const Ch& h, double pe, int32_t* n_done) {
  const double eps = h.f(F_EPS);
  const double dh = delta_energy(pe, leapfrog_end(h, V_Z0, eps), h.f(F_H0));
  const int dnew = (kSearchLogAccept < -dh) ? 1 : -1;
  const int fdir = h.i(I_FDIR), trials = h.i(I_FTRIAL);
  if (fdir == 0 || (dnew == fdir && trials < kMaxSearchTrials)) {
    const int dir = fdir == 0 ? dnew : fdir;
    h.i(I_FDIR) = dir;
    h.i(I_FTRIAL) = trials + 1;
    h.f(F_EPS) = dir > 0 ? 2.0 * eps : 0.5 * eps;
    search_trial(h);
    return;
  }
  h.i(I_FDIR) = 0;
  h.i(I_FTRIAL) = 0;
  h.f(F_MU) = log(10.0 * eps);
  h.f(F_XBAR) = 0.0;
  h.f(F_GBAR) = 0.0;
  h.i(I_DAT) = 0;
  start_transition(h, n_done);
}

__global__ void hmc_init_kernel(const sbi_hmc_chains s) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= s.C) return;
  const Ch h{s, c};
  for (int k = 0; k < SBI_HMC_NI; ++k) h.i(k) = 0;
  for (int k = 0; k < SBI_HMC_NF0 + 2 * s.max_tree_depth; ++k) h.f(k) = 0.0;
  h.i(I_PHASE) = SBI_HMC_PHASE_INIT;
  h.f(F_EPS) = s.step_size;
  for (int d = 0; d < s.D; ++d) {
    h.v(V_MINV, d) = 1.0;
    h.v(V_WMEAN, d) = 0.0;
    h.v(V_WM2, d) = 0.0;
    s.d_params[(size_t)c * s.D + d] = (float)h.z(d);
  }
}

__global__ void hmc_step_kernel(const sbi_hmc_chains s, int32_t* n_done) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= s.C) return;
  const Ch h{s, c};
  const int phase = h.i(I_PHASE);
  if (phase == SBI_HMC_PHASE_DONE) {
    atomicAdd(n_done, 1);
    return;
  }
  const double pe = -(double)s.d_logp[c];
  if (phase == SBI_HMC_PHASE_INIT) {
    const float* gl = s.d_grad + (size_t)c * s.D;
    for (int d = 0; d < s.D; ++d) h.v(V_GZ, d) = -(double)gl[d];
    h.f(F_PEZ) = pe;
    if (s.adapt_step_size) search_trial(h);
    else start_transition(h, n_done);
  } else if (phase == SBI_HMC_PHASE_FIND) {
    search_result(h, pe, n_done);
  } else if (s.algo == SBI_HMC_HMC) {
    hmc_leaf(h, pe, n_done);
  } else {
    nuts_leaf(h, pe, n_done);
  }
}

}  // namespace
}  // namespace sbi

static int hmc_check(const sbi_hmc_chains* s) {
  if (!s || s->C < 1 || s->D < 1 || s->warmup < 0 || s->num_samples < 0) return SBI_EINVAL;
  if (s->algo != SBI_HMC_NUTS && s->algo != SBI_HMC_HMC) return SBI_EINVAL;
  if (s->max_tree_depth < 1 || s->max_tree_depth > SBI_HMC_MAX_TREE_DEPTH) return SBI_EINVAL;
  if (s->n_windows < 0 || s->n_windows > SBI_HMC_MAX_WINDOWS) return SBI_EINVAL;
  if (!(s->step_size > 0.0) || !(s->trajectory_length > 0.0)) return SBI_EINVAL;
  if (!s->d_z || !s->d_vec || !s->d_istate || !s->d_fstate || !s->d_normal || !s->d_uniform || !s->d_logp ||
      !s->d_grad || !s->d_params)
    return SBI_EINVAL;
  if (s->num_samples > 0 && !s->d_samples) return SBI_EINVAL;
  return 0;
}

extern "C" int sbi_b200_hmc_init(const sbi_hmc_chains* s, void* stream) {
  sbi::DeviceGuard dev_guard_(s ? s->d_z : nullptr);
  if (int rc = hmc_check(s)) return rc;
  return sbi::launch(sbi::hmc_init_kernel, (s->C + 127) / 128, 128, 0, (cudaStream_t)stream, *s);
}

extern "C" int sbi_b200_hmc_step(const sbi_hmc_chains* s, int32_t* d_n_done, void* stream) {
  sbi::DeviceGuard dev_guard_(s ? s->d_z : nullptr);
  if (int rc = hmc_check(s)) return rc;
  if (!d_n_done) return SBI_EINVAL;
  cudaError_t e = cudaMemsetAsync(d_n_done, 0, sizeof(int32_t), (cudaStream_t)stream);
  if (e != cudaSuccess) return (int)e;
  return sbi::launch(sbi::hmc_step_kernel, (s->C + 127) / 128, 128, 0, (cudaStream_t)stream, *s, d_n_done);
}
