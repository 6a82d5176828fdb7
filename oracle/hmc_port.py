"""CPU float64 restatement of the NUTS and HMC transition kernels with their warm-up adaptation -- the checker of
csrc/hmc.cu (TEST INFRASTRUCTURE ONLY).

Written from the published sources, not from any implementation: Hoffman & Gelman 2014 (NUTS, dual averaging),
Betancourt 2017 (multinomial sampling, the generalized U-turn criterion of App. A.4.2) and the Stan reference
manual (windowed adaptation, the regularised variance).  The defaults are pyro's, as DESIGN §3.6 writes them
down.  Unlike the kernel, the tree is built recursively, one chain at a time.

Random numbers are not drawn here: `draws[k] = (normal (D, C), uniform (K + 1, C))` are the numbers of lock-step
k, the lock-step that follows the k-th potential evaluation (k = 0 evaluates the initial position).  A chain takes
them in the order include/sbi_b200.h documents: a fresh momentum from `normal`, the direction of a doubling from
uniform[0] (< 0.5: forward), the choice of the merge that forms a 2^(k+1)-leaf subtree from uniform[1 + k], the
top-level choice and the HMC Metropolis test from uniform[K], with K = max_tree_depth.

`run_chain` returns one record per transition: the position after it, the inverse mass diagonal and the step
size it used, its tree depth (completed doublings), leapfrog steps, divergence flag and accept statistic, and the
smallest margin of the discrete decisions taken in it or in the step-size search that preceded it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

MAX_DELTA_ENERGY = 1000.0
SEARCH_LOG_ACCEPT = math.log(0.8)
MAX_SEARCH_TRIALS = 100


def adaptation_schedule(warmup: int) -> List[Tuple[int, int]]:
    """Stan's windows (inclusive transition indices): buffers of 75 / 25 / 50 with doubling windows, the last one
    stretched to the terminal buffer; 15 % / 10 % buffers and one window when they do not fit; one window below
    20 warm-up transitions."""
    if warmup < 20:
        return [(0, warmup - 1)] if warmup > 0 else []
    start, end, init = 75, 50, 25
    if start + end + init > warmup:
        start, end = int(0.15 * warmup), int(0.1 * warmup)
        init = warmup - start - end
    out = [(0, start - 1)]
    end_start = warmup - end
    size, nxt = init, start
    while nxt < end_start:
        cur, cur_size = nxt, size
        if 3 * cur_size <= end_start - cur:
            size = 2 * cur_size
        else:
            cur_size = end_start - cur
        nxt = cur + cur_size
        out.append((cur, nxt - 1))
    out.append((end_start, warmup - 1))
    return out


class DualAveraging:
    """Nesterov's dual averaging on x = log(step size) with t0 = 10, kappa = 0.75, gamma = 0.05."""

    def __init__(self, prox_center: float = 0.0, t0: float = 10.0, kappa: float = 0.75, gamma: float = 0.05):
        self.prox_center, self.t0, self.kappa, self.gamma = prox_center, t0, kappa, gamma
        self.reset()

    def reset(self):
        self.t, self.g_avg, self.x_avg, self.x = 0, 0.0, 0.0, 0.0

    def step(self, g: float):
        self.t += 1
        self.g_avg = (1.0 - 1.0 / (self.t + self.t0)) * self.g_avg + g / (self.t + self.t0)
        self.x = self.prox_center - math.sqrt(self.t) / self.gamma * self.g_avg
        w = self.t ** (-self.kappa)
        self.x_avg = (1.0 - w) * self.x_avg + w * self.x
        return self.x, self.x_avg


class Welford:
    """Running diagonal variance; `variance()` is regularised as n/(n+5) var + 1e-3 * 5/(n+5)."""

    def __init__(self, dim: int):
        self.n, self.mean, self.m2 = 0, np.zeros(dim), np.zeros(dim)

    def update(self, x):
        self.n += 1
        pre = x - self.mean
        self.mean = self.mean + pre / self.n
        self.m2 = self.m2 + pre * (x - self.mean)

    def variance(self):
        n = self.n
        return (n / (n + 5.0)) * self.m2 / (n - 1) + 1e-3 * (5.0 / (n + 5.0))


def kinetic(r, minv, g=None) -> float:
    if g is not None and not np.all(np.isfinite(g)):
        return float("nan")
    return float(0.5 * np.sum(minv * r * r))


def leapfrog(z, r, g, step: float, minv, potential: Callable):
    """One velocity-Verlet step of signed size `step`; `potential(z) -> (U, grad U)`."""
    r = r - 0.5 * step * g
    z = z + step * minv * r
    pe, g = potential(z)
    r = r - 0.5 * step * g
    return z, r, g, pe


def _logaddexp(a, b):
    m = max(a, b)
    if m == -math.inf:
        return -math.inf
    return m + math.log(math.exp(a - m) + math.exp(b - m))


def _delta(pe, kin, h0):
    dh = pe + kin - h0
    return math.inf if math.isnan(dh) else dh


@dataclass
class _Tree:
    last: tuple                  # (z, r, g) of the last leaf in build order
    r_first: np.ndarray
    r_last: np.ndarray
    rsum: np.ndarray
    w: float
    prop: tuple                  # (z, g, pe)
    turning: bool
    diverging: bool
    sacc: float
    n: int


@dataclass
class Record:
    z: np.ndarray
    minv: np.ndarray
    depth: int
    n_leapfrog: int
    diverging: bool
    accept: float
    step_size: float
    margin: float = math.inf


@dataclass
class ChainResult:
    records: List[Record] = field(default_factory=list)
    samples: List[np.ndarray] = field(default_factory=list)


class _Chain:
    def __init__(self, z0, logp_grad: Callable, draws: Sequence, c: int, algo: str, warmup: int, num_samples: int,
                 step_size: float, adapt_step_size: bool, adapt_mass_matrix: bool, target_accept: float,
                 max_tree_depth: int, trajectory_length: float):
        self.z = np.asarray(z0, dtype=np.float64).copy()
        self.logp_grad, self.draws, self.c = logp_grad, draws, c
        self.algo, self.warmup, self.num_samples = algo, warmup, num_samples
        self.eps, self.adapt_step, self.adapt_mass = float(step_size), adapt_step_size, adapt_mass_matrix
        self.target, self.K, self.traj_len = target_accept, max_tree_depth, trajectory_length
        self.minv = np.ones_like(self.z)
        self.e = 0
        self.margin = math.inf
        self.da = DualAveraging()
        self.wf = Welford(self.z.size)
        self.windows = adaptation_schedule(warmup)
        self.win = 0

    # ---- potential and draws
    def potential(self, z):
        """U and grad U at the float32 point the kernel hands to the host; the analytic potential's value and
        gradient are rounded to float32 as the host's are."""
        lp, g = self.logp_grad(np.asarray(z, dtype=np.float32).astype(np.float64))
        self.e += 1
        return -float(np.float32(lp)), -np.asarray(g, dtype=np.float32).astype(np.float64)

    def normal(self):
        return np.asarray(self.draws[self.e - 1][0][:, self.c], dtype=np.float64)

    def uniform(self, k):
        return float(self.draws[self.e - 1][1][k, self.c])

    def note(self, m):
        self.margin = min(self.margin, abs(m))

    def draw_u(self, k, p):
        u = self.uniform(k)
        self.note(u - p)
        return u < p

    def momentum(self):
        r = self.normal() / np.sqrt(self.minv)
        return r, self.pe + kinetic(r, self.minv)

    def turning(self, rsum, ra, rb):
        rho = rsum - 0.5 * (ra + rb)
        ta, tb = self.minv * ra * rho, self.minv * rb * rho
        la, lb = float(ta.sum()), float(tb.sum())
        self.note(la / max(np.abs(ta).sum(), 1e-300))
        self.note(lb / max(np.abs(tb).sum(), 1e-300))
        return la <= 0.0 or lb <= 0.0

    # ---- step-size search
    def search(self):
        def trial(eps):
            r, h0 = self.momentum()
            _, r1, g1, pe1 = leapfrog(self.z, r, self.g, eps, self.minv, self.potential)
            dh = _delta(pe1, kinetic(r1, self.minv, g1), h0)
            self.note(-dh - SEARCH_LOG_ACCEPT)
            return 1 if SEARCH_LOG_ACCEPT < -dh else -1

        eps = self.eps
        d = trial(eps)
        trials = 0
        while True:
            eps = 2.0 * eps if d > 0 else 0.5 * eps
            trials += 1
            if trial(eps) != d or trials >= MAX_SEARCH_TRIALS:
                break
        self.eps = eps
        self.da = DualAveraging(prox_center=math.log(10.0 * eps))

    # ---- NUTS
    def leaf(self, z, r, g, step, h0):
        z, r, g, pe = leapfrog(z, r, g, step, self.minv, self.potential)
        dh = _delta(pe, kinetic(r, self.minv, g), h0)
        self.note(dh - MAX_DELTA_ENERGY)
        acc = math.exp(-dh) if dh > 0 else 1.0
        return _Tree((z, r, g), r, r, r.copy(), -dh, (z, g, pe), False, dh > MAX_DELTA_ENERGY, acc, 1)

    def build_tree(self, z, r, g, d, j, h0):
        if j == 0:
            return self.leaf(z, r, g, d * self.eps, h0)
        a = self.build_tree(z, r, g, d, j - 1, h0)
        if a.turning or a.diverging:
            return a
        b = self.build_tree(*a.last, d, j - 1, h0)
        sacc, n = a.sacc + b.sacc, a.n + b.n
        if b.turning or b.diverging:
            return _Tree(b.last, a.r_first, b.r_last, a.rsum, a.w, a.prop, b.turning, b.diverging, sacc, n)
        w = _logaddexp(a.w, b.w)
        prop = b.prop if self.draw_u(j, math.exp(b.w - w)) else a.prop     # uniform[1 + (j - 1)]
        rsum = a.rsum + b.rsum
        turning = self.turning(rsum, a.r_first, b.r_last)
        return _Tree(b.last, a.r_first, b.r_last, rsum, w, prop, turning, False, sacc, n)

    def nuts(self):
        r, h0 = self.momentum()
        left = right = (self.z, r, self.g)
        rsum, w_tree, depth, sacc, n, div = r.copy(), 0.0, 0, 0.0, 0, False
        while depth < self.K:
            d = 1 if self.draw_u(0, 0.5) else -1
            t = self.build_tree(*(right if d > 0 else left), d, depth, h0)
            sacc, n = sacc + t.sacc, n + t.n
            if d > 0:
                right = t.last
            else:
                left = t.last
            if t.diverging:
                div = True
                break
            if t.turning:
                break
            depth += 1
            if self.draw_u(self.K, math.exp(t.w - w_tree)):
                self.z, self.g, self.pe = t.prop
            rsum = rsum + t.rsum
            if self.turning(rsum, left[1], right[1]):
                break
            w_tree = _logaddexp(w_tree, t.w)
        return sacc / n, depth, n, div

    # ---- HMC
    def hmc(self):
        r, h0 = self.momentum()
        n_steps = int(max(1.0, min(1e9, math.floor(self.traj_len / self.eps))))
        z, g = self.z, self.g
        for i in range(n_steps):
            z, r, g, pe = leapfrog(z, r, g, self.eps, self.minv, self.potential)
            dh = _delta(pe, kinetic(r, self.minv, g), h0)
            self.note(dh - MAX_DELTA_ENERGY)
            if dh > MAX_DELTA_ENERGY:
                return 0.0, 0, i + 1, True
        acc = math.exp(-dh) if dh > 0 else 1.0
        if self.draw_u(self.K, acc):
            self.z, self.g, self.pe = z, g, pe
        return acc, 0, n_steps, False

    # ---- adaptation
    def adapt(self, t, acc):
        nw = len(self.windows)
        mass_phase = self.adapt_mass and 0 < self.win < nw - 1
        if self.adapt_step:
            x, _ = self.da.step(self.target - acc)
            self.eps = math.exp(x)
        if mass_phase:
            self.wf.update(self.z)
        if self.win >= nw or t != self.windows[self.win][1]:
            return
        self.win += 1
        if self.win == nw:
            if self.adapt_step:
                self.eps = math.exp(self.da.x_avg)
            return
        if not mass_phase:
            return
        if self.wf.n >= 2:
            self.minv = self.wf.variance()
        self.wf = Welford(self.z.size)
        if self.adapt_step:
            self.search()

    def run(self) -> ChainResult:
        out = ChainResult()
        self.pe, self.g = self.potential(self.z)
        if self.adapt_step:
            self.search()
        for t in range(self.warmup + self.num_samples):
            minv, eps = self.minv.copy(), self.eps
            acc, depth, n, div = self.nuts() if self.algo == "nuts" else self.hmc()
            out.records.append(Record(self.z.copy(), minv, depth, n, div, acc, eps, self.margin))
            self.margin = math.inf
            if t < self.warmup:
                self.adapt(t, acc)
            else:
                out.samples.append(self.z.copy())
        return out


def run_chain(z0, logp_grad: Callable, draws: Sequence, c: int, algo: str = "nuts", warmup: int = 200,
              num_samples: int = 100, step_size: float = 1.0, adapt_step_size: bool = True,
              adapt_mass_matrix: bool = True, target_accept: float = 0.8, max_tree_depth: int = 10,
              trajectory_length: float = 2 * math.pi) -> ChainResult:
    """Chain `c` of a lock-step run: `logp_grad(z) -> (log p, d log p / dz)` at one float64 point, `draws` as in
    the module docstring.  A search that follows transition t is charged to the record of transition t + 1."""
    return _Chain(z0, logp_grad, draws, c, algo, warmup, num_samples, step_size, adapt_step_size,
                  adapt_mass_matrix, target_accept, max_tree_depth, trajectory_length).run()


class NumpyDraws:
    """Draws for a CPU-only run: lock-step k's numbers come from `np.random.default_rng(seed)` in lock-step
    order, generated on demand."""

    def __init__(self, num_chains: int, dim: int, max_tree_depth: int, seed: int = 0):
        self.C, self.D, self.K = num_chains, dim, max_tree_depth
        self.rng = np.random.default_rng(seed)
        self.cache: List[Tuple[np.ndarray, np.ndarray]] = []

    def __getitem__(self, k):
        while len(self.cache) <= k:
            self.cache.append((self.rng.standard_normal((self.D, self.C)), self.rng.random((self.K + 1, self.C))))
        return self.cache[k]
