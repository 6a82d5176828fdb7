"""Samplers that loop over the estimator kernels, mirroring the reference's sampler API.

* `SliceSamplerVectorized` -- same constructor / `run(num_samples) -> (chains, samples, dim)` as
  /root/reference/sbi/samplers/mcmc/slice_numpy.py:353-620, but the per-chain state machine is ONE
  kernel launch per lock-step (`sbi_b200_slice_step`) instead of a Python loop over chains with a
  host sync per chain: a lock-step costs the potential evaluation + one tiny kernel, and the host
  looks at the device only every `check_every` steps (termination test).
* `rejection_sample` -- /root/reference/sbi/samplers/rejection/rejection.py:18-227, incl. the
  `gradient_ascent` search for max(potential - log q) (sbiutils.py:1160-1285); the acceptance
  uniforms are drawn with the CPU generator and uploaded, exactly as the reference does (:178), so
  accepted-index sets are comparable.
* `importance_sample` / `sampling_importance_resampling` -- importance_sampling.py:11-37 and sir.py:13-71; the SIR
  selection and compaction is one kernel sequence (`sbi_b200_sir_select`).
* `resample_given_potential_fn` / `sir_init` -- init strategies of
  /root/reference/sbi/samplers/mcmc/init_strategy.py:37-114.
"""
from __future__ import annotations

import logging
import time
import warnings
from typing import Any, Callable, Optional, Tuple, Union
from warnings import warn

import numpy as np
import torch
from torch import Tensor
from torch.distributions import transforms as torch_tf
from torch.optim import Adam

from . import _lib as L


class SliceSamplerVectorized:
    def __init__(self, log_prob_fn: Callable, init_params: Union[np.ndarray, Tensor], num_chains: int = 1,
                 thin: int = 1, tuning: int = 50, verbose: bool = False,
                 init_width: Union[float, np.ndarray] = 0.01, max_width: float = float("inf"),
                 num_workers: int = 1, device: str = "cuda", seed: Optional[int] = None,
                 check_every: int = 16, graph: bool = False):
        self._log_prob_fn = log_prob_fn
        self.x = init_params
        self.num_chains = num_chains
        self.thin = 1 if thin is None else thin
        self.tuning = tuning
        self.verbose = verbose
        self.init_width = init_width
        self.max_width = max_width
        self._samples = None
        self._device = device
        self._seed = seed
        self._check_every = check_every
        # graph=True: `check_every` lock-steps [potential -> state machine] are captured once as a CUDA graph
        # and replayed (the potential must be pure device work without host synchronisation: the estimator
        # potentials of sbi_b200.potentials with a device-resident prior are; a numpy callback is not)
        self._graph = bool(graph)
        self.num_potential_evals = 0
        if num_workers > 1:
            warn("Parallelization of vectorized slice sampling not implement, running serially.", stacklevel=2)

    def run(self, num_samples: int) -> np.ndarray:
        assert num_samples >= 0
        dev = self._device
        x = torch.as_tensor(np.asarray(self.x.cpu() if isinstance(self.x, Tensor) else self.x),
                            dtype=torch.float64).reshape(self.num_chains, -1).to(dev).contiguous()
        Cn, D = x.shape
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if self._seed is None else int(self._seed)
        # initial bracket widths per dimension, a scalar broadcast (np.full(n_dims, init_width) in the reference)
        width = torch.as_tensor(np.asarray(self.init_width, dtype=np.float64)).to(dev).expand(Cn, D).contiguous()
        order = torch.empty(Cn, D, dtype=torch.int32, device=dev)
        istate = torch.zeros(Cn, 4, dtype=torch.int32, device=dev)
        fstate = torch.zeros(Cn, 8, dtype=torch.float64, device=dev)
        rng = torch.zeros(Cn, 64, dtype=torch.uint8, device=dev)
        samples = torch.empty(Cn, max(int(num_samples), 1), D, dtype=torch.float64, device=dev)
        params = torch.empty(Cn, D, dtype=torch.float32, device=dev)
        n_done = torch.zeros(1, dtype=torch.int32, device=dev)
        s = L.SliceChains(Cn, D, int(num_samples), int(self.tuning), float(min(self.max_width, 1e300)), seed,
                          x.data_ptr(), width.data_ptr(), order.data_ptr(), istate.data_ptr(), fstate.data_ptr(),
                          rng.data_ptr(), samples.data_ptr())
        # the chains' device state, readable while and after the sampler runs (final widths, state machine)
        self._chain_state = {"width": width, "order": order, "istate": istate, "fstate": fstate}
        L.call("slice_init", s, params)
        it = 0

        def lock_step():
            lp = self._log_prob_fn(params)
            lp = torch.as_tensor(lp, dtype=torch.float32).to(dev).reshape(-1).contiguous()
            L.call("slice_step", s, lp, params, n_done)

        graph = None
        while True:
            if graph is not None:
                graph.replay()
                it += self._check_every
                self.num_potential_evals += Cn * self._check_every
            else:
                lock_step()
                it += 1
                self.num_potential_evals += Cn
            if it % self._check_every == 0:
                if int(n_done.item()) == Cn:
                    break
                if self._graph and graph is None:
                    # the eager round above warmed everything up; capture the next rounds
                    side = torch.cuda.Stream(device=dev)
                    side.wait_stream(torch.cuda.current_stream(dev))
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=side):
                        for _ in range(self._check_every):
                            lock_step()
                    torch.cuda.current_stream(dev).wait_stream(side)
        self.num_lock_steps = it
        out = samples[:, :int(num_samples)].cpu().numpy()
        out = out[:, :: self.thin, :]
        self._samples = out
        self._final_x = x
        return out

    def get_samples(self, num_samples: Optional[int] = None, group_by_chain: bool = True) -> np.ndarray:
        if self._samples is None:
            raise ValueError("No samples found from MCMC run.")
        samples = self._samples if group_by_chain else self._samples.reshape(-1, self._samples.shape[2])
        if num_samples is None:
            return samples
        return samples[:, -num_samples:, :] if group_by_chain else samples[-num_samples:, :]


class SliceSampler:
    """Single-chain coordinate-wise slice sampler with the reference's interface
    (/root/reference/sbi/samplers/mcmc/slice_numpy.py:57-216: `SliceSampler(x, lp_f, max_width,
    init_width, thin, tuning)`, `.gen(n_samples)` -> (n_samples, dim) array, `.set_state(x)`).
    `lp_f` maps one parameter vector (1-D numpy array) to its log-probability, as in the
    reference.  The chain's state machine is the same device kernel as the vectorized sampler
    (one chain, lock-step with the host callback)."""

    def __init__(self, x, lp_f: Callable, max_width: float = float("inf"), init_width: Union[float, np.ndarray] = 0.01,
                 thin: Optional[int] = None, tuning: int = 50, verbose: bool = False, device: str = "cuda",
                 seed: Optional[int] = None):
        self.x = np.array(x, dtype=float).reshape(-1)
        self.n_dims = self.x.size
        self.lp_f = lp_f
        self.L = lp_f(self.x)
        self.thin = 1 if thin is None else thin
        self.max_width, self.init_width, self.tuning, self.verbose = max_width, init_width, tuning, verbose
        self._device, self._seed = device, seed
        self._tuned = False

    def set_state(self, x):
        self.x = np.array(x, dtype=float).reshape(-1)
        self.L = self.lp_f(self.x)

    def gen(self, n_samples: int, logger=None, show_info: bool = False, rng=None) -> np.ndarray:
        assert n_samples >= 0, "number of samples can't be negative"

        def batch_lp(params: Tensor) -> Tensor:
            return torch.tensor([float(self.lp_f(params[0].double().cpu().numpy()))], dtype=torch.float32)

        vec = SliceSamplerVectorized(batch_lp, self.x[None, :], num_chains=1, thin=self.thin,
                                     tuning=0 if self._tuned else self.tuning, init_width=self.init_width,
                                     max_width=self.max_width, device=self._device, seed=self._seed, check_every=1)
        out = vec.run(int(n_samples) * self.thin)[0]
        self._tuned = True
        if out.shape[0] > 0:
            self.x = out[-1].copy()
            self.L = self.lp_f(self.x)
        return out


# ------------------------------------------------------------------------------------------------
def gradient_ascent(potential_fn: Callable, inits: Tensor, theta_transform: Optional[torch_tf.Transform] = None,
                    num_iter: int = 1_000, num_to_optimize: int = 100, learning_rate: float = 0.01,
                    save_best_every: int = 10, show_progress_bars: bool = False,
                    interruption_note: str = "") -> Tuple[Tensor, Tensor]:
    """sbiutils.py:1160-1285: Adam ascent from the best `num_to_optimize` inits in transformed
    space; returns (argmax, max).  Gradients flow through the estimator kernels' VJP."""
    if theta_transform is None:
        theta_transform = torch_tf.IndependentTransform(torch_tf.identity_transform, reinterpreted_batch_ndims=1)
    init_probs = potential_fn(inits).detach()
    inits = inits.to(init_probs.device)
    sort_indices = torch.argsort(init_probs, dim=0)
    sorted_inits = inits[sort_indices]
    optimize_inits = sorted_inits[-num_to_optimize:]
    best_log_prob_iter = torch.max(init_probs)
    best_theta_iter = sorted_inits[-1]
    best_theta_overall = best_theta_iter.detach().clone()
    best_log_prob_overall = best_log_prob_iter.detach().clone()
    optimize_inits = theta_transform(optimize_inits).detach().clone()
    optimize_inits.requires_grad_(True)
    optimizer = Adam([optimize_inits], lr=learning_rate)
    iter_ = 0
    while iter_ < num_iter:
        optimizer.zero_grad()
        probs = potential_fn(theta_transform.inv(optimize_inits)).squeeze()
        loss = -probs.sum()
        loss.backward()
        optimizer.step()
        with torch.no_grad():
            if iter_ % save_best_every == 0 or iter_ == num_iter - 1:
                log_probs_of_optimized = potential_fn(theta_transform.inv(optimize_inits))
                best_theta_iter = optimize_inits[torch.argmax(log_probs_of_optimized)].unsqueeze(0)
                best_log_prob_iter = potential_fn(theta_transform.inv(best_theta_iter))
                if best_log_prob_iter > best_log_prob_overall:
                    best_theta_overall = best_theta_iter.detach().clone()
                    best_log_prob_overall = best_log_prob_iter.detach().clone()
        iter_ += 1
    return theta_transform.inv(best_theta_overall), best_log_prob_overall


def rejection_sample(potential_fn: Callable, proposal: Any, theta_transform: Optional[torch_tf.Transform] = None,
                     num_samples: int = 1, show_progress_bars: bool = False, warn_acceptance: float = 0.01,
                     max_sampling_batch_size: int = 10_000, num_samples_to_find_max: int = 10_000,
                     num_iter_to_find_max: int = 100, m: float = 1.2, max_sampling_time: Optional[float] = None,
                     return_partial_on_timeout: bool = False, device: str = "cuda",
                     return_indices: bool = False):
    """rejection.py:18-227.  `return_indices=True` additionally returns the global proposal index of
    every accepted draw (the accept-set contract of BASELINE configs[4])."""
    if theta_transform is None:
        theta_transform = torch_tf.IndependentTransform(torch_tf.identity_transform, reinterpreted_batch_ndims=1)
    samples_to_find_max = proposal.sample((num_samples_to_find_max,))

    def potential_over_proposal(theta):
        return potential_fn(theta) - proposal.log_prob(theta)

    _, max_log_ratio = gradient_ascent(
        potential_fn=potential_over_proposal, inits=samples_to_find_max, theta_transform=theta_transform,
        num_iter=num_iter_to_find_max, learning_rate=0.01,
        num_to_optimize=max(1, int(num_samples_to_find_max / 10)))
    if m < 1.0:
        warnings.warn("A value of m < 1.0 will lead to systematically wrong results.", stacklevel=2)
    log_m = torch.log(torch.as_tensor(m))

    def scaled_log_prob(theta):
        return proposal.log_prob(theta) + max_log_ratio + log_m

    with torch.no_grad():
        from . import _lib as L
        lib = L.load()
        num_sampled_total, num_remaining = 0, num_samples
        acceptance_rate = float("Nan")
        leakage_warning_raised = False
        sampling_batch_size = min(num_samples, max_sampling_batch_size)
        start_time = time.time()
        # accepted draws are appended on the device, in proposal order (csrc/compact.cu); the host reads the
        # running count once per batch (the reference's boolean indexing synchronises once per batch too)
        out = out_idx = count = None
        collected = 0
        while num_remaining > 0:
            if max_sampling_time is not None and (time.time() - start_time) > max_sampling_time:
                if return_partial_on_timeout and collected > 0:
                    warnings.warn(f"Timeout exceeded after collecting {collected}/{num_samples} samples. "
                                  "Returning partial results.", stacklevel=2)
                    return out[:collected].clone(), torch.as_tensor(acceptance_rate)
                raise RuntimeError("Sampling aborted early because rejection sampling exceeded max_sampling_time. "
                                   "This is likely due to extremely low acceptance.")
            candidates = proposal.sample((sampling_batch_size,)).reshape(sampling_batch_size, -1)
            log_target = potential_fn(candidates).reshape(-1).float().contiguous()
            dev = log_target.device
            candidates = candidates.to(dev).float().contiguous()
            log_scaled = scaled_log_prob(candidates).reshape(-1).float().contiguous()
            uniform_rand = torch.rand(log_target.shape).to(dev)
            if out is None:
                Dth = candidates.shape[1]
                out = torch.empty(num_samples, Dth, dtype=torch.float32, device=dev)
                out_idx = torch.empty(num_samples, dtype=torch.int64, device=dev) if return_indices else None
                count = torch.zeros(1, dtype=torch.int32, device=dev)
            scratch = torch.empty(int(lib.sbi_b200_reject_scratch_ints(sampling_batch_size)), dtype=torch.int32,
                                  device=dev)
            L.call("reject_compact", candidates, candidates.shape[1], log_target, log_scaled, uniform_rand,
                   sampling_batch_size, num_sampled_total, out, out_idx, num_samples, count, scratch)
            total = int(count.item())
            collected = min(total, num_samples)
            num_sampled_total += sampling_batch_size
            num_remaining = num_samples - total
            acceptance_rate = (num_samples - num_remaining) / num_sampled_total
            sampling_batch_size = min(max_sampling_batch_size,
                                      max(int(1.5 * num_remaining / max(acceptance_rate, 1e-12)), 100))
            if num_sampled_total > 1000 and acceptance_rate < warn_acceptance and not leakage_warning_raised:
                logging.warning(f"Only {acceptance_rate:.3%} proposal samples were accepted. It may take a long "
                                f"time to collect the remaining {num_remaining} samples.")
                leakage_warning_raised = True
        samples = out
        assert collected == num_samples, "Number of accepted samples must match required samples."
    if return_indices:
        return samples, torch.as_tensor(acceptance_rate), out_idx
    return samples, torch.as_tensor(acceptance_rate)


def _proposal_draws(proposal: Any, num_samples: int, show_progress_bars: bool) -> Tensor:
    try:   # multi-round proposals take a progress-bar argument, torch distributions do not
        return proposal.sample((num_samples,), show_progress_bar=show_progress_bars)
    except TypeError:
        return proposal.sample((num_samples,))


def importance_sample(potential_fn: Callable, proposal: Any, num_samples: int = 1,
                      show_progress_bars: bool = False) -> Tuple[Tensor, Tensor]:
    """importance_sampling.py:11-37: proposal draws and their log importance weights, potential - log q."""
    samples = _proposal_draws(proposal, num_samples, show_progress_bars)
    potential_logprobs = potential_fn(samples)
    proposal_logprobs = proposal.log_prob(samples)
    log_importance_weights = potential_logprobs - proposal_logprobs
    return samples, log_importance_weights


def sampling_importance_resampling(potential_fn: Callable, proposal: Any, num_samples: int = 1,
                                   num_candidate_samples: int = 32, max_sampling_batch_size: int = 10_000,
                                   show_progress_bars: bool = False, device: str = "cuda", **kwargs: Any) -> Tensor:
    """sir.py:13-71: every posterior sample is one categorical draw, by importance weight, among
    `num_candidate_samples` proposal draws.  The proposal, potential and uniform draws are the reference's own
    calls in its order, so a seed gives the reference's candidates and uniforms; the softmax, cumulative weights,
    decision and compaction are one kernel sequence (csrc/compact.cu) appending the selected rows to a device
    buffer, where the reference's boolean indexing synchronises through `nonzero`.  The host reads the running
    count once per batch."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"sampling_importance_resampling selects on a CUDA device, got device={device!r} "
                           "(no CPU fallback)")
    lib = L.load()
    K = int(num_candidate_samples)
    sampling_batch_size = min(num_samples, max_sampling_batch_size)
    num_remaining = num_samples
    out = count = None
    total = groups_done = 0
    with torch.no_grad():
        while num_remaining > 0:
            batch_size = min(sampling_batch_size, num_remaining)
            thetas = _proposal_draws(proposal, batch_size * K, show_progress_bars)
            log_target = potential_fn(thetas)
            log_proposal = proposal.log_prob(thetas)
            uniform_decision = torch.rand(batch_size, 1, device=device)
            cand = thetas.reshape(batch_size * K, -1).to(dev).float().contiguous()
            if out is None:
                out = torch.empty(num_samples, cand.shape[1], dtype=torch.float32, device=dev)
                count = torch.zeros(1, dtype=torch.int32, device=dev)
            scratch = torch.empty(int(lib.sbi_b200_sir_scratch_ints(batch_size)), dtype=torch.int32, device=dev)
            lt = log_target.reshape(-1).to(dev).float().contiguous()
            lq = log_proposal.reshape(-1).to(dev).float().contiguous()
            u = uniform_decision.reshape(-1).to(dev).float().contiguous()
            L.call("sir_select", cand, cand.shape[1], lt, lq, u, batch_size, K, groups_done, out, None, num_samples,
                   count, scratch)
            groups_done += batch_size
            total = int(count.item())
            num_remaining = num_samples - total
    return out[:total]


def resample_given_potential_fn(proposal: Any, potential_fn: Callable, transform: torch_tf.Transform,
                                num_candidate_samples: int = 10_000, num_batches: int = 1,
                                num_inits: int = 1, **kwargs: Any) -> Tensor:
    """init_strategy.py:67-114 for `num_inits` chains: like the reference, every chain draws its own
    batch of proposal candidates, weights them by the potential and resamples one; each batch is ONE
    potential-kernel launch (10 000 rows) instead of a Python-level evaluation per chain."""
    with torch.set_grad_enabled(False):
        outs = []
        for _ in range(num_inits):
            log_weights, cands = [], []
            for _ in range(num_batches):
                batch_draws = proposal.sample((num_candidate_samples,)).detach()
                cands.append(batch_draws)
                log_weights.append(potential_fn(batch_draws).detach())
            log_weights = torch.cat(log_weights)
            cands = torch.cat(cands)
            log_weights = log_weights - torch.logsumexp(log_weights, dim=0)
            probs = torch.exp(log_weights.view(-1))
            probs[torch.isnan(probs)] = 0.0
            probs[torch.isinf(probs)] = 0.0
            probs /= probs.sum()
            idxs = torch.multinomial(probs, 1, replacement=False)
            outs.append(transform(cands[idxs, :]))
        return torch.cat(outs)


def sir_init(proposal: Any, potential_fn: Callable, transform: torch_tf.Transform,
             num_candidate_samples: int = 10_000, num_inits: int = 1, **kwargs: Any) -> Tensor:
    """init_strategy.py:37-64 (sampling-importance-resampling with the proposal correction)."""
    with torch.set_grad_enabled(False):
        outs = []
        for _ in range(num_inits):
            cands = proposal.sample((num_candidate_samples,)).detach()
            logw = potential_fn(cands).detach() - proposal.log_prob(cands)
            probs = torch.softmax(logw.view(-1), 0)
            probs[torch.isnan(probs)] = 0.0
            idx = torch.multinomial(probs, 1, replacement=False)
            outs.append(transform(cands[idx, :]))
        return torch.cat(outs)


def init_batched(proposal: Any, potential_fn: Any, transform: torch_tf.Transform, x: Tensor, num_chains: int,
                 init_strategy: str, num_candidate_samples: int = 10_000, num_batches: int = 1,
                 max_rows: int = 4_000_000, **kwargs: Any) -> Tensor:
    """Initial states of `num_chains` chains for every observation in `x` (B, *event_shape), observation-major
    (chain c belongs to observation c // num_chains), as `_get_initial_params_batched` (mcmc_posterior.py:661-735)
    with `proposal`, `resample` or `sir` (init_strategy.py:37-114).  Like the reference, every (observation,
    chain) group draws its own candidates; unlike its loop over observations, the potential runs with
    `x_is_iid=False` over the candidates of many groups at once, in chunks of at most `max_rows` rows, and the
    categorical draw is one `torch.multinomial` over the chunk's groups.  Leaves `potential_fn` set to the last
    chunk's rows."""
    B = x.shape[0]
    G = B * num_chains
    if init_strategy == "proposal":
        return transform(proposal.sample((G,)))
    if init_strategy not in ("resample", "sir"):
        raise NotImplementedError(init_strategy)
    K = num_candidate_samples * (num_batches if init_strategy == "resample" else 1)
    per_chunk = max(1, max_rows // K)
    outs = []
    with torch.set_grad_enabled(False):
        for g0 in range(0, G, per_chunk):
            g = min(per_chunk, G - g0)
            obs = torch.arange(g0, g0 + g, device=x.device) // num_chains
            cands = proposal.sample((g * K,)).detach()
            potential_fn.set_x(x[obs].repeat_interleave(K, dim=0), x_is_iid=False)
            logw = potential_fn(cands).detach().reshape(g, K)
            if init_strategy == "resample":
                probs = torch.exp(logw - torch.logsumexp(logw, dim=1, keepdim=True))
                probs[torch.isnan(probs)] = 0.0
                probs[torch.isinf(probs)] = 0.0
                probs /= probs.sum(dim=1, keepdim=True)
            else:
                logw = logw - proposal.log_prob(cands).reshape(g, K)
                probs = torch.softmax(logw, dim=1)
                probs[torch.isnan(probs)] = 0.0
            idx = torch.multinomial(probs, 1, replacement=False).reshape(-1)
            outs.append(transform(cands.reshape(g, K, -1)[torch.arange(g, device=idx.device), idx]))
    return torch.cat(outs)
