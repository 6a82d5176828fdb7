"""Gradient-based MCMC: the NUTS and HMC transition kernels behind `mcmc_method="nuts_pyro"` / `"hmc_pyro"`.

The reference hands these methods to pyro, whose MCMC loop launches work per leapfrog step, per chain and per
process.  Here all chains advance in lock-step: every lock-step is one potential-and-gradient evaluation of the
(C, D) points the chains asked for, then one launch of the per-chain state machine (csrc/hmc.cu), which takes one
leapfrog step per chain and runs the tree building, the accept decisions and the per-chain adaptation.  Groups
of `check_every` lock-steps are replayed from a CUDA graph, and the host reads the device "done" count once per
group, as `SliceSamplerVectorized` does.  The algorithm and its defaults (pyro's) are written down in DESIGN §3.6;
`oracle/hmc_port.py` restates it on the CPU and consumes the same random numbers.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
from typing import Callable, List, Optional, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib as L

ADAPT_START_BUFFER, ADAPT_INITIAL_WINDOW, ADAPT_END_BUFFER = 75, 25, 50


def adaptation_schedule(warmup_steps: int) -> List[Tuple[int, int]]:
    """Stan's warm-up windows as inclusive (start, end) transition indices: an initial buffer (step size only),
    doubling mass-matrix windows, the last one stretched to the terminal buffer, and a terminal buffer (step size
    only).  When 75 + 25 + 50 transitions do not fit, the buffers are 15 % and 10 % of the warm-up with one
    window between them; below 20 warm-up transitions there is one step-size-only window."""
    if warmup_steps < 20:
        return [(0, warmup_steps - 1)] if warmup_steps > 0 else []
    start, end, init = ADAPT_START_BUFFER, ADAPT_END_BUFFER, ADAPT_INITIAL_WINDOW
    if start + end + init > warmup_steps:
        start, end = int(0.15 * warmup_steps), int(0.1 * warmup_steps)
        init = warmup_steps - start - end
    windows = [(0, start - 1)]
    end_start = warmup_steps - end
    size, nxt = init, start
    while nxt < end_start:
        cur, cur_size = nxt, size
        if 3 * cur_size <= end_start - cur:
            size = 2 * cur_size
        else:
            cur_size = end_start - cur
        nxt = cur + cur_size
        windows.append((cur, nxt - 1))
    windows.append((end_start, warmup_steps - 1))
    return windows


@contextlib.contextmanager
def frozen_parameters(*objs):
    """Sets `requires_grad=False` on the parameters of every module held by `objs` (or by their attributes) for
    the duration of the block and restores the flags afterwards, so that the gradient of a potential with
    respect to theta does not also reduce the estimator's parameter partials."""
    params = []
    for o in objs:
        mods = [o] if isinstance(o, torch.nn.Module) else [v for v in vars(o).values()
                                                             if isinstance(v, torch.nn.Module)]
        for m in mods:
            params.extend(p for p in m.parameters() if p.requires_grad)
    for p in params:
        p.requires_grad_(False)
    try:
        yield
    finally:
        for p in params:
            p.requires_grad_(True)


class HMCSamplerVectorized:
    """NUTS (`method="nuts"`) or HMC (`method="hmc"`) over `num_chains` chains with pyro's defaults: initial step
    size 1, step size and diagonal mass matrix adapted per chain during `warmup_steps` transitions, target
    accept probability 0.8, NUTS with multinomial sampling and max_tree_depth 10, HMC with trajectory length 2 pi.

    `log_prob_fn` maps a (C, D) float32 tensor to log p (C,) and must be differentiable with autograd (the
    gradient is `torch.autograd.grad` of its sum).  `run(num_samples)` returns the post-warm-up positions,
    (chains, num_samples, D).  After a run, per chain: `step_size`, `inverse_mass_matrix`, `num_divergences`,
    `mean_accept_prob` and, for NUTS, `mean_tree_depth` (means and counts over the recorded transitions).
    `graph=True` replays groups of `check_every` lock-steps from a CUDA graph; the potential must then be pure
    device work.  `record_draws=True` (eager only) keeps every lock-step's random numbers, and `trace=True` keeps
    the per-transition record (position, inverse mass, tree depth, leapfrog steps, divergence, accept statistic,
    step size), both for checking the kernel against `oracle/hmc_port.py`."""

    def __init__(self, log_prob_fn: Callable, init_params: Union[np.ndarray, Tensor], num_chains: int = 1,
                 method: str = "nuts", warmup_steps: int = 200, step_size: float = 1.0,
                 adapt_step_size: bool = True, adapt_mass_matrix: bool = True, target_accept_prob: float = 0.8,
                 max_tree_depth: int = 10, trajectory_length: float = 2 * math.pi, device: str = "cuda",
                 check_every: int = 16, graph: bool = False, record_draws: bool = False, trace: bool = False):
        if method not in ("nuts", "hmc"):
            raise ValueError(f"method must be 'nuts' or 'hmc', got {method!r}")
        if not 1 <= max_tree_depth <= L.SBI_HMC_MAX_TREE_DEPTH:
            raise ValueError(f"max_tree_depth must be in [1, {L.SBI_HMC_MAX_TREE_DEPTH}], got {max_tree_depth}")
        self._log_prob_fn = log_prob_fn
        self.x = init_params
        self.num_chains = num_chains
        self.method = method
        self.warmup_steps = int(warmup_steps)
        self.initial_step_size = float(step_size)
        self.adapt_step_size, self.adapt_mass_matrix = bool(adapt_step_size), bool(adapt_mass_matrix)
        self.target_accept_prob = float(target_accept_prob)
        self.max_tree_depth = int(max_tree_depth)
        self.trajectory_length = float(trajectory_length)
        self._device = device
        self._check_every = check_every
        self._graph = bool(graph) and not record_draws
        self._record = record_draws
        self._trace = trace
        self._samples = None
        self.draws: List[Tuple[Tensor, Tensor]] = []
        self.num_potential_evals = 0
        self.num_lock_steps = 0

    def run(self, num_samples: int) -> np.ndarray:
        assert num_samples >= 0
        lib = L.load()
        dev = torch.device(self._device)
        z = torch.as_tensor(np.asarray(self.x.detach().cpu() if isinstance(self.x, Tensor) else self.x),
                            dtype=torch.float64).reshape(self.num_chains, -1).to(dev).contiguous()
        L.require_cuda(z, "init_params")
        Cn, D = z.shape
        K = self.max_tree_depth
        windows = adaptation_schedule(self.warmup_steps)
        if len(windows) > L.SBI_HMC_MAX_WINDOWS:
            raise ValueError(f"{self.warmup_steps} warm-up steps give {len(windows)} adaptation windows "
                             f"(at most {L.SBI_HMC_MAX_WINDOWS})")
        f64 = dict(dtype=torch.float64, device=dev)
        vec = torch.zeros(L.SBI_HMC_NV0 + 4 * K, D, Cn, **f64)
        istate = torch.zeros(L.SBI_HMC_NI, Cn, dtype=torch.int32, device=dev)
        fstate = torch.zeros(L.SBI_HMC_NF0 + 2 * K, Cn, **f64)
        normal = torch.zeros(D, Cn, **f64)
        uniform = torch.zeros(K + 1, Cn, **f64)
        logp = torch.zeros(Cn, dtype=torch.float32, device=dev)
        grad = torch.zeros(Cn, D, dtype=torch.float32, device=dev)
        params = torch.zeros(Cn, D, dtype=torch.float32, device=dev)
        samples = torch.empty(Cn, max(int(num_samples), 1), D, **f64)
        total = self.warmup_steps + int(num_samples)
        trace = torch.zeros(Cn, max(total, 1), 2 * D + L.SBI_HMC_TRACE_SCALARS, **f64) if self._trace else None
        n_done = torch.zeros(1, dtype=torch.int32, device=dev)
        win = (C.c_int32 * L.SBI_HMC_MAX_WINDOWS)(*[e for _, e in windows])
        s = L.HmcChains(Cn, D, L.SBI_HMC_HMC if self.method == "hmc" else L.SBI_HMC_NUTS, K, self.warmup_steps,
                        int(num_samples), int(self.adapt_step_size), int(self.adapt_mass_matrix), len(windows), win,
                        self.initial_step_size, self.target_accept_prob, self.trajectory_length,
                        z.data_ptr(), vec.data_ptr(), istate.data_ptr(), fstate.data_ptr(), normal.data_ptr(),
                        uniform.data_ptr(), logp.data_ptr(), grad.data_ptr(), params.data_ptr(),
                        samples.data_ptr(), None if trace is None else trace.data_ptr())
        L.check(lib.sbi_b200_hmc_init(C.byref(s), L.stream_ptr()), "hmc_init")
        self.draws = []

        def lock_step():
            with torch.enable_grad():
                p = params.detach().requires_grad_(True)
                lp = torch.as_tensor(self._log_prob_fn(p)).reshape(-1)
                g = torch.autograd.grad(lp.sum(), p, allow_unused=True)[0]
            logp.copy_(lp.detach())
            if g is None:
                grad.zero_()
            else:
                grad.copy_(g)
            normal.normal_()
            uniform.uniform_()
            if self._record:
                self.draws.append((normal.clone(), uniform.clone()))
            L.check(lib.sbi_b200_hmc_step(C.byref(s), L.ptr(n_done), L.stream_ptr()), "hmc_step")

        it = 0
        graph = None
        while True:
            if graph is not None:
                graph.replay()
                it += self._check_every
            else:
                lock_step()
                it += 1
            if it % self._check_every == 0:
                if int(n_done.item()) == Cn:
                    break
                if self._graph and graph is None:
                    side = torch.cuda.Stream(device=dev)
                    side.wait_stream(torch.cuda.current_stream(dev))
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=side):
                        for _ in range(self._check_every):
                            lock_step()
                    torch.cuda.current_stream(dev).wait_stream(side)
        self.num_lock_steps = it
        self.num_potential_evals = it * Cn
        n = max(int(num_samples), 1)
        self.step_size = fstate[2].cpu().numpy().copy()
        self.inverse_mass_matrix = vec[8].T.cpu().numpy().copy()
        self.num_divergences = istate[12].cpu().numpy().copy()
        self.mean_accept_prob = (fstate[8] / n).cpu().numpy()
        self.mean_tree_depth = (fstate[9] / n).cpu().numpy() if self.method == "nuts" else None
        self.trace = None if trace is None else trace[:, :total].cpu().numpy()
        out = samples[:, :int(num_samples)].cpu().numpy()
        self._samples = out
        self._final_x = z
        return out

    def get_samples(self, num_samples: Optional[int] = None, group_by_chain: bool = True) -> np.ndarray:
        if self._samples is None:
            raise ValueError("No samples found from MCMC run.")
        samples = self._samples if group_by_chain else self._samples.reshape(-1, self._samples.shape[2])
        if num_samples is None:
            return samples
        return samples[:, -num_samples:, :] if group_by_chain else samples[-num_samples:, :]
