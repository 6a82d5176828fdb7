"""Posteriors and the accept/reject loop on the device, mirroring the reference.

`DirectPosterior` mirrors /root/reference/sbi/inference/posteriors/direct_posterior.py
(sample :142-216, log_prob :308-386, leakage_correction :467-523); `accept_reject_sample`
mirrors /root/reference/sbi/samplers/rejection/rejection.py:230-457 (same adaptive batch-size
rule :406-409, same truncation to the first `num_samples` accepted draws, same acceptance
rate bookkeeping) and `within_support` /root/reference/sbi/utils/sbiutils.py:729-766.
`accept_reject_sample` is the one rejection loop of the direct and vector-field posteriors (one
observation or a batch of them) and of `restriction.RestrictedPrior`.  Proposals come out of the
inverse-flow kernel; support checks and the placement of accepted rows are torch device ops, with
one host read per round, as the loop's data-dependent trip count requires.
"""
from __future__ import annotations

import logging
import time
import warnings
from math import log
from typing import Union, Any, Callable, Optional, Tuple

import torch
from torch import Tensor

from .estimators import NSFEstimator


def within_support(distribution: Any, samples: Tensor) -> Tensor:
    """sbiutils.py:729-766."""
    try:
        check = distribution.support.check(samples)
        if check.shape == samples.shape:
            check = torch.all(check, dim=-1)
        return check
    except (NotImplementedError, AttributeError):
        return torch.isfinite(distribution.log_prob(samples))


class DeviceMultivariateNormal(torch.distributions.MultivariateNormal):
    """MultivariateNormal whose `log_prob` is one (rows, D) x (D, D) product with the inverse Cholesky factor.
    torch's implementation solves a triangular system with the rows as right-hand sides, which on CUDA takes
    a long time for the 10^6-row batches of the rejection / MCMC potentials; same value to fp32 rounding."""

    def __init__(self, loc, covariance_matrix=None, scale_tril=None, validate_args=None):
        super().__init__(loc, covariance_matrix=covariance_matrix, scale_tril=scale_tril, validate_args=validate_args)
        L_ = self._unbroadcasted_scale_tril
        eye = torch.eye(L_.shape[-1], dtype=L_.dtype, device=L_.device)
        self._linv_t = torch.linalg.solve_triangular(L_, eye, upper=False).transpose(-1, -2).contiguous()
        self._half_log_det = L_.diagonal(dim1=-2, dim2=-1).log().sum(-1)

    def log_prob(self, value):
        if self._validate_args:
            self._validate_sample(value)
        if self.loc.dim() != 1:
            return super().log_prob(value)
        z = (value - self.loc) @ self._linv_t
        return -0.5 * (z * z).sum(-1) - self._half_log_det - 0.5 * self.loc.shape[-1] * 1.8378770664093453


def prior_to_device(prior, device):
    """Move a torch.distributions prior to `device` (the reference requires the user to do
    this, inference_on_device_test.py; we do it for the common families)."""
    if prior is None:
        return None
    try:
        import torch.distributions as td
        if isinstance(prior, td.MultivariateNormal):
            return DeviceMultivariateNormal(prior.loc.to(device), covariance_matrix=prior.covariance_matrix.to(device),
                                            validate_args=False)
        if isinstance(prior, td.Independent):
            return td.Independent(prior_to_device(prior.base_dist, device), prior.reinterpreted_batch_ndims)
        if isinstance(prior, td.Uniform):
            return td.Uniform(prior.low.to(device), prior.high.to(device), validate_args=False)
        if isinstance(prior, td.Normal):
            return td.Normal(prior.loc.to(device), prior.scale.to(device), validate_args=False)
    except Exception:   # pragma: no cover
        pass
    if hasattr(prior, "to"):
        try:
            prior.to(device)
        except Exception:
            pass
    return prior


@torch.no_grad()
def accept_reject_sample(
    proposal: Callable, accept_reject_fn: Callable, num_samples: int, num_xos: int = 1,
    show_progress_bars: bool = False, warn_acceptance: float = 0.01,
    sample_for_correction_factor: bool = False, max_sampling_batch_size: int = 10_000,
    proposal_sampling_kwargs: Optional[dict] = None, alternative_method: Optional[str] = None,
    max_sampling_time: Optional[float] = None, return_partial_on_timeout: bool = False,
    device: Optional[Union[str, torch.device]] = None, **kwargs,
) -> Tuple[Tensor, Tensor]:
    """rejection.py:230-457: draw from `proposal`, keep what `accept_reject_fn` accepts, until `num_samples` per
    observation are collected.  Returns (samples (num_samples, num_xos, *event), acceptance rate per observation).

    `proposal(shape, **proposal_sampling_kwargs)` returns (batch, num_xos, D) draws, or (batch, D) for one
    observation; with `device`, they are moved there before `accept_reject_fn` sees them.  Every accepted row is
    written to its slot by a cumulative count per observation, so the samples are the first `num_samples` accepted
    draws of every observation in draw order; rejected rows and those past `num_samples` go to one spare slot.
    The float32 acceptance rates (accepted over drawn) are computed beside the accept decisions, or on the host when
    `device` is given (as the reference computes them for its host-side proposals; a CUDA division by the drawn
    count is not always the correctly rounded one).  One host read per round brings the counts and rates back:
    `num_samples` minus the smallest count is what remains, and the smallest rate drives the reference's
    batch-size rule and its low-acceptance warning.
    After `max_sampling_time`, with `return_partial_on_timeout`, the first rows every observation has filled."""
    if kwargs:
        logging.warning(f"Unused arguments passed to accept_reject_sample: {list(kwargs)}")
    proposal_sampling_kwargs = proposal_sampling_kwargs or {}
    num_remaining, drawn, batch = num_samples, 0, min(num_samples, max_sampling_batch_size)
    leakage_warning_raised = False
    start = time.time()
    while num_remaining > 0:
        if drawn and max_sampling_time is not None and (time.time() - start) > max_sampling_time:
            num_collected = num_samples - num_remaining
            if return_partial_on_timeout and num_collected > 0:
                warnings.warn(f"Timeout exceeded after collecting {num_collected}/{num_samples}"
                              " samples. Returning partial results.", stacklevel=2)
                return out[:num_collected], rate.to(out.device)
            raise RuntimeError(
                "Sampling aborted early because rejection sampling exceeded max_sampling_time. "
                "This is likely due to extremely low acceptance.")
        candidates = proposal(torch.Size((batch,)), **proposal_sampling_kwargs)
        if device is not None:
            candidates = candidates.to(device)
        keep = accept_reject_fn(candidates).reshape(batch, num_xos)
        cands = candidates.reshape(batch, num_xos, candidates.shape[-1])
        if not drawn:
            out = cands.new_empty((num_samples + 1, num_xos, cands.shape[-1]))     # row num_samples: the spare slot
            accepted = torch.zeros(num_xos, dtype=torch.int64, device=keep.device)
        count = torch.cumsum(keep, dim=0).add_(accepted)           # accepted so far, up to and including each row
        slot = torch.where(keep, count - 1, num_samples).clamp_(max=num_samples)
        out.scatter_(0, slot.unsqueeze(-1).expand_as(cands), cands)
        accepted = count[-1]
        drawn += batch
        counts = accepted if device is None else accepted.cpu()
        rate = counts.float() / drawn
        stats = torch.cat((counts.double(), rate.double())).tolist()     # the round's one host read
        num_remaining, min_rate = num_samples - int(min(stats[:num_xos])), min(stats[num_xos:])
        batch = min(max_sampling_batch_size, max(int(1.5 * num_remaining / max(min_rate, 1e-12)), 100))
        if drawn > (batch - 1) and min_rate < warn_acceptance and not leakage_warning_raised:
            if sample_for_correction_factor:
                logging.warning(
                    f"Drawing samples from posterior to estimate the normalizing constant for "
                    f"`log_prob()`. However, only {min_rate:.3%} posterior samples are "
                    f"within the prior support. It may take a long time to collect the remaining "
                    f"{num_remaining} samples.")
            else:
                msg = (f"Only {min_rate:.3%} proposal samples are accepted. It may take "
                       f"a long time to collect the remaining {num_remaining} samples.")
                if alternative_method is not None:
                    msg += f" Alternatively, consider switching to `{alternative_method}`."
                logging.warning(msg)
            leakage_warning_raised = True
    samples = out[:num_samples].reshape(num_samples, *candidates.shape[1:])
    return samples, rate.to(samples.device)


class DirectPosterior:
    """p(theta | x) represented by the trained estimator itself (NPE)."""

    def __init__(self, posterior_estimator: NSFEstimator, prior, max_sampling_batch_size: int = 10_000,
                 device: Optional[str] = None, x_shape=None, enable_transform: bool = True):
        self.posterior_estimator = posterior_estimator
        self._device = device or str(posterior_estimator.flat.device)
        self.posterior_estimator.to(self._device)
        self.prior = prior_to_device(prior, self._device)
        self.max_sampling_batch_size = max_sampling_batch_size
        self._leakage_density_correction_factor = None
        self.default_x = None

    def set_default_x(self, x: Tensor):
        self.default_x = x.to(self._device)
        self._leakage_density_correction_factor = None
        return self

    def _x_else_default_x(self, x):
        if x is not None:
            return torch.as_tensor(x, dtype=torch.float32).to(self._device)
        if self.default_x is None:
            raise ValueError("Context `x` needed when a default has not been set. "
                             "If you'd like to have a default, use the `.set_default_x()` method.")
        return self.default_x

    def _batch_x(self, x: Tensor) -> Tensor:
        cs = self.posterior_estimator.condition_shape
        if x.shape == cs:
            x = x.unsqueeze(0)
        return x.reshape(-1, *cs)

    def sample(self, sample_shape=torch.Size(), x: Optional[Tensor] = None,
               max_sampling_batch_size: int = 10_000, show_progress_bars: bool = False,
               reject_outside_prior: bool = True, max_sampling_time: Optional[float] = None,
               return_partial_on_timeout: bool = False) -> Tensor:
        num_samples = torch.Size(sample_shape).numel()
        x = self._batch_x(self._x_else_default_x(x))
        if x.shape[0] > 1:
            raise ValueError(".sample() supports only `batchsize == 1`. If you intend "
                             "to sample multiple observations, use `.sample_batched()`.")
        if max_sampling_batch_size is None:
            max_sampling_batch_size = self.max_sampling_batch_size
        if reject_outside_prior and self.prior is not None:
            samples = accept_reject_sample(
                proposal=self.posterior_estimator.sample,
                accept_reject_fn=lambda theta: within_support(self.prior, theta),
                num_samples=num_samples, show_progress_bars=show_progress_bars,
                max_sampling_batch_size=max_sampling_batch_size,
                proposal_sampling_kwargs={"condition": x},
                alternative_method="build_posterior(..., sample_with='mcmc')",
                max_sampling_time=max_sampling_time,
                return_partial_on_timeout=return_partial_on_timeout)[0]
        else:
            samples = self.posterior_estimator.sample(torch.Size([num_samples]), condition=x)
        return samples[:, 0].reshape(*torch.Size(sample_shape), -1)

    def log_prob(self, theta: Tensor, x: Optional[Tensor] = None, norm_posterior: bool = True,
                 track_gradients: bool = False, leakage_correction_params: Optional[dict] = None) -> Tensor:
        x = self._batch_x(self._x_else_default_x(x))
        if x.shape[0] > 1:
            raise ValueError(".log_prob() supports only `batchsize == 1`. If you intend "
                             "to evaluate given multiple observations, use `.log_prob_batched()`.")
        theta = torch.as_tensor(theta, dtype=torch.float32).to(self._device)
        if theta.dim() == 1:
            theta = theta.unsqueeze(0)
        self.posterior_estimator.eval()
        with torch.set_grad_enabled(track_gradients):
            unnorm = self.posterior_estimator.log_prob(theta.unsqueeze(1), condition=x).squeeze(dim=1)
            if self.prior is not None:
                inside = within_support(self.prior, theta)
                unnorm = torch.where(inside, unnorm,
                                     torch.tensor(float("-inf"), dtype=torch.float32, device=theta.device))
            log_factor = (log(self.leakage_correction(x=x, **(leakage_correction_params or {})))
                          if norm_posterior and self.prior is not None else 0)
            return unnorm - log_factor

    # ---- batched observations (direct_posterior.py:218-306, 388-465): the hot loop of SBC / TARP / coverage ----
    @torch.no_grad()
    def sample_batched(self, sample_shape, x: Tensor, max_sampling_batch_size: int = 10_000,
                       show_progress_bars: bool = False, reject_outside_prior: bool = True,
                       max_sampling_time: Optional[float] = None, return_partial_on_timeout: bool = False) -> Tensor:
        """Samples from p(theta | x_1), ..., p(theta | x_B): (*sample_shape, B, *input_shape).  Every round is ONE
        sampling-kernel launch over (draws x B) rows; acceptance (prior support) is resolved for all observations
        at once with a cumulative count per observation -- no per-observation host loop."""
        num_samples = torch.Size(sample_shape).numel()
        x = self._batch_x(torch.as_tensor(x, dtype=torch.float32).to(self._device))
        B = x.shape[0]
        est = self.posterior_estimator
        D = int(torch.Size(est.input_shape).numel())
        if B * num_samples > 2 ** 21:
            warnings.warn(f"Batched sampling generates {B} * {num_samples} = {B * num_samples} samples.", stacklevel=2)
        if max_sampling_batch_size is None:
            max_sampling_batch_size = self.max_sampling_batch_size
        if max_sampling_batch_size * B > 4_000_000:          # rows per launch (the reference caps at 100 000)
            max_sampling_batch_size = max(1, 4_000_000 // B)
        if not (reject_outside_prior and self.prior is not None):
            return est.sample(torch.Size([num_samples]), condition=x).reshape(*torch.Size(sample_shape), B, *est.input_shape)
        out, self._last_acceptance_rate = accept_reject_sample(
            proposal=lambda shape: est.sample(shape, condition=x).reshape(shape[0], B, D),
            accept_reject_fn=lambda theta: within_support(self.prior, theta.reshape(-1, D)),
            num_samples=num_samples, num_xos=B, max_sampling_batch_size=max_sampling_batch_size,
            alternative_method="build_posterior(..., sample_with='mcmc')", max_sampling_time=max_sampling_time,
            return_partial_on_timeout=return_partial_on_timeout)
        if out.shape[0] < num_samples:          # partial result after a timeout
            return out
        return out.reshape(*torch.Size(sample_shape), B, *est.input_shape)

    def log_prob_batched(self, theta: Tensor, x: Tensor, norm_posterior: bool = True, track_gradients: bool = False,
                         leakage_correction_params: Optional[dict] = None) -> Tensor:
        """log p(theta_b | x_b) for a batch of observations: theta (*sample_shape, B, *input_shape) or
        (B, *input_shape), x (B, *condition_shape) -> (len(theta), B); -inf outside the prior support."""
        est = self.posterior_estimator
        x = self._batch_x(torch.as_tensor(x, dtype=torch.float32).to(self._device))
        theta = torch.as_tensor(theta, dtype=torch.float32).to(self._device)
        ev = len(est.input_shape)
        if theta.dim() == ev:
            theta = theta.unsqueeze(0)
        th = theta.unsqueeze(0) if theta.dim() - ev == 1 else theta.reshape(-1, *theta.shape[-(ev + 1):])
        est.eval()
        with torch.set_grad_enabled(track_gradients):
            unnorm = est.log_prob(th, condition=x)                                  # (S, B)
            if self.prior is not None:
                inside = within_support(self.prior, th.reshape(-1, *est.input_shape)).reshape(unnorm.shape)
                unnorm = torch.where(inside, unnorm, torch.full_like(unnorm, float("-inf")))
            if norm_posterior and self.prior is not None:
                kw = dict(leakage_correction_params or {})
                self.sample_batched((kw.get("num_rejection_samples", 10_000),), x,
                                    max_sampling_batch_size=kw.get("rejection_sampling_batch_size", 10_000))
                unnorm = unnorm - torch.log(self._last_acceptance_rate).unsqueeze(0)
            return unnorm

    def map(self, x: Optional[Tensor] = None, num_iter: int = 1_000, num_to_optimize: int = 100,
            learning_rate: float = 0.01, init_method: Union[str, Tensor] = "posterior", num_init_samples: int = 1_000,
            save_best_every: int = 10, show_progress_bars: bool = False, force_update: bool = False) -> Tensor:
        """Maximum-a-posteriori estimate by gradient ascent on the posterior potential in unconstrained space
        (base_posterior.py `_calculate_map` -> sbiutils.gradient_ascent); gradients w.r.t. theta come from the
        fused VJP kernels."""
        from .potentials import posterior_estimator_based_potential
        from .samplers import gradient_ascent
        x = self._batch_x(self._x_else_default_x(x))
        if not force_update and getattr(self, "_map", None) is not None and getattr(self, "_map_x", None) is not None \
                and self._map_x.shape == x.shape and bool((self._map_x == x).all()):
            return self._map
        potential_fn, theta_transform = posterior_estimator_based_potential(self.posterior_estimator, self.prior, x_o=x)
        if isinstance(init_method, str):
            if init_method == "posterior":
                inits = self.sample((num_init_samples,), x=x)
            elif init_method == "proposal":
                inits = self.prior.sample((num_init_samples,))
            else:
                raise ValueError
        else:
            inits = torch.as_tensor(init_method, dtype=torch.float32).to(self._device)
        self._map = gradient_ascent(potential_fn=potential_fn, inits=inits, theta_transform=theta_transform,
                                    num_iter=num_iter, num_to_optimize=num_to_optimize, learning_rate=learning_rate,
                                    save_best_every=save_best_every, show_progress_bars=show_progress_bars)[0]
        self._map_x = x
        return self._map

    @torch.no_grad()
    def leakage_correction(self, x: Tensor, num_rejection_samples: int = 10_000,
                           force_update: bool = False, show_progress_bars: bool = False,
                           rejection_sampling_batch_size: int = 10_000) -> Tensor:
        def acceptance_at(xx):
            return accept_reject_sample(
                proposal=self.posterior_estimator.sample,
                accept_reject_fn=lambda theta: within_support(self.prior, theta),
                num_samples=num_rejection_samples, sample_for_correction_factor=True,
                max_sampling_batch_size=rejection_sampling_batch_size,
                proposal_sampling_kwargs={"condition": self._batch_x(xx)})[1]

        is_new_x = self.default_x is None or (x is not self.default_x and (x != self.default_x).any())
        if is_new_x:
            return acceptance_at(x)
        if self._leakage_density_correction_factor is None or force_update:
            self._leakage_density_correction_factor = acceptance_at(self.default_x)
        return self._leakage_density_correction_factor


_HMC_OPTIONS = ("step_size", "adapt_step_size", "adapt_mass_matrix", "target_accept_prob", "max_tree_depth",
                "trajectory_length")


# =================================================================================================
class MCMCPosterior:
    """Posterior sampled with the lock-step vectorized slice sampler or with the lock-step NUTS / HMC sampler
    (reference: /root/reference/sbi/inference/posteriors/mcmc_posterior.py: sample :237-367, _slice_np_mcmc
    :737-811, _pyro_mcmc :813-878, _get_initial_params :590-659).  Supported methods: `slice_np_vectorized`
    (`slice_np`), `nuts_pyro` and `hmc_pyro` (sbi_b200.hmc; pyro's defaults, run on the device)."""

    def __init__(self, potential_fn, proposal, theta_transform=None, method: str = "slice_np_vectorized",
                 thin: int = -1, warmup_steps: int = 200, num_chains: int = 20,
                 init_strategy: str = "resample", init_strategy_parameters: Optional[dict] = None,
                 num_workers: int = 1, device: Optional[str] = None, x_shape=None):
        if method not in ("slice_np_vectorized", "slice_np", "nuts_pyro", "hmc_pyro"):
            raise NotImplementedError("sbi_b200.MCMCPosterior implements method='slice_np_vectorized', "
                                      "'nuts_pyro' and 'hmc_pyro'")
        self.potential_fn = potential_fn
        self._device = device or potential_fn.device
        self.proposal = prior_to_device(proposal, self._device)
        self.theta_transform = theta_transform
        if self.theta_transform is None:
            import torch.distributions.transforms as tt
            self.theta_transform = tt.IndependentTransform(tt.identity_transform, reinterpreted_batch_ndims=1)
        self.method, self.warmup_steps, self.num_chains = method, warmup_steps, num_chains
        self.thin = 10 if thin == -1 else thin       # reference default (mcmc_posterior.py: thin=-1 -> 10)
        self._thin_arg = thin                        # the pyro methods read -1 as 1 (_process_thin_default)
        self.init_strategy = init_strategy
        self.init_strategy_parameters = init_strategy_parameters or {}
        self._mcmc_init_params = None
        self._posterior_sampler = None
        self.default_x = None

    def set_default_x(self, x):
        self.default_x = x
        return self

    def _get_initial_params(self, init_strategy: str, num_chains: int) -> Tensor:
        from .samplers import resample_given_potential_fn, sir_init
        if init_strategy == "proposal":
            return self.theta_transform(self.proposal.sample((num_chains,)))
        if init_strategy == "resample":
            return resample_given_potential_fn(self.proposal, self.potential_fn, self.theta_transform,
                                               num_inits=num_chains, **self.init_strategy_parameters)
        if init_strategy == "sir":
            return sir_init(self.proposal, self.potential_fn, self.theta_transform, num_inits=num_chains,
                            **self.init_strategy_parameters)
        if init_strategy == "latest_sample":
            if self._mcmc_init_params is None or self._mcmc_init_params.shape[0] != num_chains:
                raise ValueError("No or mismatching previous samples for init_strategy='latest_sample'")
            return self._mcmc_init_params
        raise NotImplementedError(init_strategy)

    @torch.no_grad()
    def sample(self, sample_shape=torch.Size(), x: Optional[Tensor] = None, method: Optional[str] = None,
               thin: Optional[int] = None, warmup_steps: Optional[int] = None, num_chains: Optional[int] = None,
               init_strategy: Optional[str] = None, show_progress_bars: bool = False, **kwargs) -> Tensor:
        from math import ceil
        from .potentials import transformed_potential
        from .samplers import SliceSamplerVectorized
        x = x if x is not None else self.default_x
        if x is None:
            raise ValueError("Context `x` needed when a default has not been set.")
        self.potential_fn.set_x(x, x_is_iid=True)
        method = self.method if method is None else method
        if method in ("nuts_pyro", "hmc_pyro"):
            return self._sample_gradient_based(sample_shape, method, thin, warmup_steps, num_chains, init_strategy,
                                               **kwargs)
        thin = self.thin if thin is None else thin
        warmup_steps = self.warmup_steps if warmup_steps is None else warmup_steps
        num_chains = self.num_chains if num_chains is None else num_chains
        init_strategy = self.init_strategy if init_strategy is None else init_strategy
        num_samples = torch.Size(sample_shape).numel()
        initial_params = self._get_initial_params(init_strategy, num_chains)
        dim = initial_params.shape[1]

        def log_prob_fn(params):
            return transformed_potential(params, self.potential_fn, self.theta_transform, self._device,
                                         track_gradients=False).flatten()

        sampler = SliceSamplerVectorized(log_prob_fn=log_prob_fn, init_params=initial_params.double().cpu().numpy(),
                                         num_chains=num_chains, thin=thin, verbose=show_progress_bars,
                                         device=self._device, graph=True)
        warmup_ = warmup_steps * thin
        num_samples_ = ceil((num_samples * thin) / num_chains)
        samples = sampler.run(warmup_ + num_samples_)          # (chains, n, dim), already thinned
        samples = samples[:, warmup_steps:, :]
        samples = torch.from_numpy(samples)
        self._posterior_sampler = sampler
        self._mcmc_init_params = samples[:, -1, :].reshape(num_chains, dim).float().to(self._device)
        samples = samples.reshape(-1, dim)[:num_samples].type(torch.float32).to(self._device)
        samples = self.theta_transform.inv(samples)
        return samples.reshape((*torch.Size(sample_shape), -1))

    def _sample_gradient_based(self, sample_shape, method: str, thin: Optional[int], warmup_steps: Optional[int],
                               num_chains: Optional[int], init_strategy: Optional[str], **kwargs) -> Tensor:
        """_pyro_mcmc (mcmc_posterior.py:813-878): `ceil(thin * n / num_chains)` transitions per chain after
        `warmup_steps` warm-up transitions (not multiplied by `thin`), flattened chain-major, then `[::thin][:n]`.
        The energy is minus the potential in unconstrained space, log|det J| included (`_prepare_potential` with
        `track_gradients=True`).  The sampler options among `kwargs` (`step_size`, `adapt_step_size`,
        `adapt_mass_matrix`, `target_accept_prob`, `max_tree_depth`, `trajectory_length`) go to
        `HMCSamplerVectorized`; the others are ignored, as on the slice path."""
        from math import ceil
        from .hmc import HMCSamplerVectorized, frozen_parameters
        from .potentials import transformed_potential
        thin = self._thin_arg if thin is None else thin
        thin = 1 if thin == -1 else thin
        warmup_steps = self.warmup_steps if warmup_steps is None else warmup_steps
        num_chains = self.num_chains if num_chains is None else num_chains
        init_strategy = self.init_strategy if init_strategy is None else init_strategy
        num_samples = torch.Size(sample_shape).numel()
        initial_params = self._get_initial_params(init_strategy, num_chains)
        dim = initial_params.shape[1]

        def log_prob_fn(params):
            return transformed_potential(params, self.potential_fn, self.theta_transform, self._device,
                                         track_gradients=True).flatten()

        sampler = HMCSamplerVectorized(log_prob_fn, initial_params.detach(), num_chains=num_chains,
                                       method="nuts" if method == "nuts_pyro" else "hmc", warmup_steps=warmup_steps,
                                       device=self._device, graph=True,
                                       **{k: v for k, v in kwargs.items() if k in _HMC_OPTIONS})
        with frozen_parameters(self.potential_fn):
            samples = sampler.run(ceil((thin * num_samples) / num_chains))     # (chains, n, dim)
        samples = torch.from_numpy(samples)
        self._posterior_sampler = sampler
        if samples.shape[1] > 0:
            self._mcmc_init_params = samples[:, -1, :].reshape(num_chains, dim).float().to(self._device)
        samples = samples.reshape(-1, dim)[::thin][:num_samples].type(torch.float32).to(self._device)
        samples = self.theta_transform.inv(samples)
        return samples.reshape((*torch.Size(sample_shape), -1))

    @torch.no_grad()
    def sample_batched(self, sample_shape, x: Tensor, method: Optional[str] = None, thin: Optional[int] = None,
                       warmup_steps: Optional[int] = None, num_chains: Optional[int] = None,
                       init_strategy: Optional[str] = None, init_strategy_parameters: Optional[dict] = None,
                       num_workers: Optional[int] = None, mp_context: Optional[str] = None,
                       show_progress_bars: bool = True) -> Tensor:
        """Samples from p(theta | x_1), ..., p(theta | x_B): (*sample_shape, B, *input_shape)
        (mcmc_posterior.py:369-515).  `num_chains` chains per observation, observation-major, all B·C of them in
        ONE vectorized slice sampler: every lock-step is one potential launch over B·C (theta_c, x_{c // C}) rows
        (`x_is_iid=False`)."""
        from math import ceil
        from .potentials import transformed_potential
        from .samplers import SliceSamplerVectorized, init_batched
        method = self.method if method is None else method
        thin = self.thin if thin is None else thin
        warmup_steps = self.warmup_steps if warmup_steps is None else warmup_steps
        num_chains = self.num_chains if num_chains is None else num_chains
        init_strategy = self.init_strategy if init_strategy is None else init_strategy
        init_strategy_parameters = dict(self.init_strategy_parameters if init_strategy_parameters is None
                                        else init_strategy_parameters)
        assert method == "slice_np_vectorized", "Batched sampling only supported for vectorized samplers!"
        num_requested = torch.Size(sample_shape).numel()
        if num_chains > num_requested:
            warnings.warn("The passed number of MCMC chains is larger than the number of requested samples: "
                          f"{num_chains} > {num_requested}, resetting it to {num_requested}.", stacklevel=2)
            num_chains = num_requested
        x = torch.as_tensor(x, dtype=torch.float32).to(self._device)
        if x.dim() == 1:
            x = x.unsqueeze(0)
        B = x.shape[0]
        chains = B * num_chains
        if chains > 100:
            warnings.warn("Note that for batched sampling, we use num_chains many chains for each x in the batch. "
                          f"With the given settings, this results in a large number of chains ({chains}), which can "
                          "be slow and memory-intensive for vectorized MCMC. Consider reducing the number of chains "
                          "or batch size.", stacklevel=2)
        init_strategy_parameters.pop("num_return_samples", None)
        if init_strategy == "latest_sample":
            if self._mcmc_init_params is None or self._mcmc_init_params.shape[0] != chains:
                raise ValueError(f"init_strategy='latest_sample' needs {chains} stored chain states (num_chains per "
                                 "observation, observation-major) from an earlier call")
            initial_params = self._mcmc_init_params
        else:
            initial_params = init_batched(self.proposal, self.potential_fn, self.theta_transform, x, num_chains,
                                          init_strategy, **init_strategy_parameters)
        self.potential_fn.set_x(x.repeat_interleave(num_chains, dim=0), x_is_iid=False)
        dim = initial_params.shape[1]

        def log_prob_fn(params):
            return transformed_potential(params, self.potential_fn, self.theta_transform, self._device,
                                         track_gradients=False).flatten()

        sampler = SliceSamplerVectorized(log_prob_fn=log_prob_fn, init_params=initial_params.double().cpu().numpy(),
                                         num_chains=chains, thin=thin, verbose=show_progress_bars,
                                         device=self._device, graph=True)
        num_samples_ = ceil((num_requested * B * thin) / chains)
        samples = sampler.run(warmup_steps * thin + num_samples_)        # (B·C, n, dim), already thinned
        samples = torch.from_numpy(samples[:, warmup_steps:, :])
        self._posterior_sampler = sampler
        self._mcmc_init_params = samples[:, -1, :].reshape(chains, dim).float().to(self._device)
        samples = self.theta_transform.inv(samples.type(torch.float32).to(self._device))
        # chain c belongs to observation c // num_chains: (B, C·n, dim) -> (C·n, B, dim), chain-major per observation
        samples = samples.reshape(B, -1, dim).permute(1, 0, 2)[:num_requested]
        return samples.reshape(*torch.Size(sample_shape), B, dim)

    def log_prob(self, theta: Tensor, x: Optional[Tensor] = None, track_gradients: bool = False) -> Tensor:
        """Unnormalised potential (mcmc_posterior.py:205-235)."""
        x = x if x is not None else self.default_x
        self.potential_fn.set_x(x)
        return self.potential_fn(torch.as_tensor(theta, dtype=torch.float32).to(self._device),
                                 track_gradients=track_gradients)


class RejectionPosterior:
    """/root/reference/sbi/inference/posteriors/rejection_posterior.py:131-226."""

    def __init__(self, potential_fn, proposal, theta_transform=None, max_sampling_batch_size: int = 10_000,
                 num_samples_to_find_max: int = 10_000, num_iter_to_find_max: int = 100, m: float = 1.2,
                 device: Optional[str] = None, x_shape=None):
        self.potential_fn = potential_fn
        self._device = device or potential_fn.device
        self.proposal = prior_to_device(proposal, self._device)
        self.theta_transform = theta_transform
        self.max_sampling_batch_size = max_sampling_batch_size
        self.num_samples_to_find_max = num_samples_to_find_max
        self.num_iter_to_find_max = num_iter_to_find_max
        self.m = m
        self.default_x = None

    def set_default_x(self, x):
        self.default_x = x
        return self

    def sample(self, sample_shape=torch.Size(), x: Optional[Tensor] = None,
               max_sampling_batch_size: Optional[int] = None, num_samples_to_find_max: Optional[int] = None,
               num_iter_to_find_max: Optional[int] = None, m: Optional[float] = None,
               show_progress_bars: bool = False, max_sampling_time: Optional[float] = None,
               return_partial_on_timeout: bool = False) -> Tensor:
        from .samplers import rejection_sample
        num_samples = torch.Size(sample_shape).numel()
        x = x if x is not None else self.default_x
        self.potential_fn.set_x(x)
        pot = lambda th: self.potential_fn(th, track_gradients=True)   # noqa: E731
        samples, _ = rejection_sample(
            pot, proposal=self.proposal, num_samples=num_samples,
            max_sampling_batch_size=max_sampling_batch_size or self.max_sampling_batch_size,
            num_samples_to_find_max=num_samples_to_find_max or self.num_samples_to_find_max,
            num_iter_to_find_max=num_iter_to_find_max or self.num_iter_to_find_max, m=m or self.m,
            max_sampling_time=max_sampling_time, return_partial_on_timeout=return_partial_on_timeout,
            device=self._device)
        return samples.reshape((*torch.Size(sample_shape), -1))

    def sample_batched(self, sample_shape, x: Tensor, max_sampling_batch_size: int = 10_000,
                       show_progress_bars: bool = True) -> Tensor:
        """rejection_posterior.py:228-239: not implemented, so batched callers fall back to one `sample` per x."""
        raise NotImplementedError(
            "Batched sampling is not implemented for RejectionPosterior. "
            "Alternatively you can use `sample` in a loop "
            "[posterior.sample(theta, x_o) for x_o in x]."
        )

    def log_prob(self, theta: Tensor, x: Optional[Tensor] = None, track_gradients: bool = False) -> Tensor:
        x = x if x is not None else self.default_x
        self.potential_fn.set_x(x)
        return self.potential_fn(torch.as_tensor(theta, dtype=torch.float32).to(self._device),
                                 track_gradients=track_gradients)


class ImportanceSamplingPosterior:
    """/root/reference/sbi/inference/posteriors/importance_posterior.py:18-380: samples by sampling-importance-
    resampling from `proposal` (`method="sir"`), or returns the proposal draws with their log importance weights
    (`method="importance"`); `log_prob` is the potential minus an importance-sampled log normalising constant.
    The SIR selection runs in csrc/compact.cu (`samplers.sampling_importance_resampling`)."""

    def __init__(self, potential_fn, proposal, theta_transform=None, method: str = "sir",
                 oversampling_factor: int = 32, max_sampling_batch_size: int = 10_000,
                 device: Optional[str] = None, x_shape=None):
        self.potential_fn = potential_fn
        self._device = device or potential_fn.device
        self.proposal = prior_to_device(proposal, self._device)
        self.theta_transform = theta_transform
        self.method = method
        self.oversampling_factor = oversampling_factor
        self.max_sampling_batch_size = max_sampling_batch_size
        self._normalization_constant = None
        self._map = None
        self.default_x = None

    def set_default_x(self, x: Tensor):
        self.default_x = self._batch_x(x)
        self._normalization_constant = None     # the cached estimate belongs to the old default x
        self._map = None
        return self

    def _batch_x(self, x) -> Tensor:
        x = torch.as_tensor(x, dtype=torch.float32).to(self._device)
        return x.unsqueeze(0) if x.dim() < 2 else x

    def _x_else_default_x(self, x):
        if x is not None:
            return self._batch_x(x)
        if self.default_x is None:
            raise ValueError("Context `x` needed when a default has not been set."
                             "If you'd like to have a default, use the `.set_default_x()` method.")
        return self.default_x

    def log_prob(self, theta: Tensor, x: Optional[Tensor] = None, track_gradients: bool = False,
                 normalization_constant_params: Optional[dict] = None) -> Tensor:
        """importance_posterior.py:109-149: potential(theta) - log Z(x)."""
        x = self._x_else_default_x(x)
        self.potential_fn.set_x(x)
        theta = torch.as_tensor(theta)
        if theta.dim() == 1:
            theta = theta.unsqueeze(0)
        with torch.set_grad_enabled(track_gradients):
            potential_values = self.potential_fn(theta.to(self._device), track_gradients=track_gradients)
            normalization_constant = self.estimate_normalization_constant(x, **(normalization_constant_params or {}))
            return (potential_values - torch.log(normalization_constant)).to(self._device)

    @torch.no_grad()
    def estimate_normalization_constant(self, x: Tensor, num_samples: int = 10_000,
                                        force_update: bool = False) -> Tensor:
        """importance_posterior.py:151-185: Z = mean(exp(log w)) over `num_samples` proposal draws; kept only at
        the default x (recomputed with `force_update`), computed unsaved at any other x."""
        from .samplers import importance_sample
        is_new_x = self.default_x is None or (x is not self.default_x and (x != self.default_x).any())
        if is_new_x:
            _, log_importance_weights = importance_sample(self.potential_fn, proposal=self.proposal,
                                                          num_samples=num_samples)
            return torch.mean(torch.exp(log_importance_weights))
        if self._normalization_constant is None or force_update:
            _, log_importance_weights = importance_sample(self.potential_fn, proposal=self.proposal,
                                                          num_samples=num_samples)
            self._normalization_constant = torch.mean(torch.exp(log_importance_weights))
        return self._normalization_constant.to(self._device)

    def sample(self, sample_shape=torch.Size(), x: Optional[Tensor] = None, method: Optional[str] = None,
               oversampling_factor: int = 32, max_sampling_batch_size: int = 10_000,
               show_progress_bars: bool = False) -> Union[Tensor, Tuple[Tensor, Tensor]]:
        """importance_posterior.py:187-228.  As in the reference, `sample`'s own defaults are passed on: the
        constructor's `oversampling_factor` / `max_sampling_batch_size` apply only when the caller passes None."""
        method = self.method if method is None else method
        self.potential_fn.set_x(self._x_else_default_x(x))
        if method == "sir":
            return self._sir_sample(sample_shape, oversampling_factor=oversampling_factor,
                                    max_sampling_batch_size=max_sampling_batch_size,
                                    show_progress_bars=show_progress_bars)
        elif method == "importance":
            return self._importance_sample(sample_shape)
        else:
            raise NameError

    def sample_batched(self, sample_shape, x: Tensor, max_sampling_batch_size: int = 10_000,
                       show_progress_bars: bool = True) -> Tensor:
        """importance_posterior.py:230-241: not implemented, so batched callers fall back to one `sample` per x."""
        raise NotImplementedError(
            "Batched sampling is not implemented for ImportanceSamplingPosterior. \
           Alternatively you can use `sample` in a loop \
           [posterior.sample(theta, x_o) for x_o in x]."
        )

    def _importance_sample(self, sample_shape=torch.Size(), show_progress_bars: bool = False) -> Tuple[Tensor, Tensor]:
        from .samplers import importance_sample
        num_samples = torch.Size(sample_shape).numel()
        samples, log_importance_weights = importance_sample(self.potential_fn, proposal=self.proposal,
                                                            num_samples=num_samples,
                                                            show_progress_bars=show_progress_bars)
        samples = samples.reshape((*sample_shape, -1)).to(self._device)
        return samples, log_importance_weights.to(self._device)

    def _sir_sample(self, sample_shape=torch.Size(), oversampling_factor: Optional[int] = 32,
                    max_sampling_batch_size: Optional[int] = 10_000, show_progress_bars: bool = False) -> Tensor:
        from .samplers import sampling_importance_resampling
        oversampling_factor = self.oversampling_factor if oversampling_factor is None else oversampling_factor
        max_sampling_batch_size = (self.max_sampling_batch_size if max_sampling_batch_size is None
                                   else max_sampling_batch_size)
        num_samples = torch.Size(sample_shape).numel()
        samples = sampling_importance_resampling(
            self.potential_fn, proposal=self.proposal, num_samples=num_samples,
            num_candidate_samples=oversampling_factor, show_progress_bars=show_progress_bars,
            max_sampling_batch_size=max_sampling_batch_size, device=self._device)
        return samples.reshape((*sample_shape, -1)).to(self._device)

    def map(self, x: Optional[Tensor] = None, num_iter: int = 1_000, num_to_optimize: int = 100,
            learning_rate: float = 0.01, init_method: Union[str, Tensor] = "proposal", num_init_samples: int = 1_000,
            save_best_every: int = 10, show_progress_bars: bool = False, force_update: bool = False) -> Tensor:
        """importance_posterior.py:315-380 -> base_posterior.py:216-323: gradient ascent on the potential from
        the best of `num_init_samples` starting points; gradients come from the estimator kernels' VJP."""
        from .samplers import gradient_ascent
        if x is not None:
            raise ValueError("Passing `x` directly to `.map()` has been deprecated."
                             "Use `.self_default_x()` to set `x`, and then run `.map()` ")
        if self.default_x is None:
            raise ValueError("Default `x` has not been set."
                             "To set the default, use the `.set_default_x()` method.")
        if self._map is None or force_update:
            self.potential_fn.set_x(self.default_x)
            if isinstance(init_method, str) and init_method == "posterior":
                inits = self.sample((num_init_samples,))
            elif isinstance(init_method, str) and init_method == "proposal":
                inits = self.proposal.sample((num_init_samples,))
            elif isinstance(init_method, Tensor):
                inits = init_method.to(self._device)
            else:
                raise ValueError
            self._map = gradient_ascent(potential_fn=self.potential_fn, inits=inits,
                                        theta_transform=self.theta_transform, num_iter=num_iter,
                                        num_to_optimize=num_to_optimize, learning_rate=learning_rate,
                                        save_best_every=save_best_every, show_progress_bars=show_progress_bars)[0]
        return self._map


class VectorFieldPosterior:
    """Posterior of a flow-matching estimator sampled by integrating its ODE or its reverse SDE
    (reference: /root/reference/sbi/inference/posteriors/vector_field_posterior.py: sample :155-329,
    sample_via_ode :436-465, _sample_via_diffusion :331-433 with the Euler-Maruyama predictor);
    draws outside the prior support are rejected like the reference (`reject_outside_prior=True`)."""

    def __init__(self, vector_field_estimator, prior, device: Optional[str] = None, max_sampling_batch_size: int = 10_000,
                 sample_with: str = "ode"):
        self.sample_with = sample_with
        self.vector_field_estimator = vector_field_estimator
        self._device = device or str(vector_field_estimator.flat.device)
        self.prior = prior_to_device(prior, self._device)
        self.max_sampling_batch_size = max_sampling_batch_size
        self.default_x = None
        self.num_function_evaluations = 0

    def set_default_x(self, x):
        self.default_x = x
        return self

    @torch.no_grad()
    def sample(self, sample_shape=torch.Size(), x: Optional[Tensor] = None, sample_with: Optional[str] = None,
               reject_outside_prior: bool = True, max_sampling_batch_size: Optional[int] = None,
               show_progress_bars: bool = False, **kwargs) -> Tensor:
        from .flowmatching import sample_ode, sample_sde
        sample_with = sample_with or self.sample_with
        if sample_with not in ("ode", "sde"):
            raise ValueError(f"Expected sample_with to be 'ode' or 'sde', but got {sample_with}.")
        steps, ts, eta = kwargs.get("steps", 500), kwargs.get("ts"), (kwargs.get("predictor_params") or {}).get("eta", 1.0)
        if kwargs.get("predictor", "euler_maruyama") != "euler_maruyama":
            raise NotImplementedError("predictor: only 'euler_maruyama' (the reference's only predictor)")
        if kwargs.get("guidance_method") is not None:
            raise NotImplementedError("guided sampling is not implemented")
        iid_method, iid_params = kwargs.get("iid_method"), kwargs.get("iid_params")
        corrector, corrector_params = kwargs.get("corrector"), kwargs.get("corrector_params")
        x = x if x is not None else self.default_x
        if x is None:
            raise ValueError("Context `x` needed when a default has not been set.")
        x = torch.as_tensor(x, dtype=torch.float32).to(self._device)
        num_samples = torch.Size(sample_shape).numel()
        est = self.vector_field_estimator
        if x.numel() > int(torch.Size(est.condition_shape).numel()) and sample_with == "ode":
            raise NotImplementedError("iid observations are sampled with sample_with='sde' and iid_method='fnpe'")

        def proposal(shape, **kw):
            n = torch.Size(shape).numel()
            if sample_with == "sde":
                s = sample_sde(est, n, x, steps=steps, ts=ts, eta=eta, corrector=corrector,
                               corrector_params=corrector_params, iid_method=iid_method, prior=self.prior,
                               iid_params=iid_params)
                self.num_function_evaluations += (steps if ts is None else ts.numel()) - 1
            else:
                s, nfe = sample_ode(est, n, x, return_nfe=True)
                self.num_function_evaluations += nfe
            return s.unsqueeze(1)

        if reject_outside_prior and self.prior is not None:
            samples = accept_reject_sample(
                proposal=proposal, accept_reject_fn=lambda th: within_support(self.prior, th.reshape(-1, th.shape[-1])),
                num_samples=num_samples,
                max_sampling_batch_size=max_sampling_batch_size or max(self.max_sampling_batch_size, num_samples))[0]
            samples = samples[:, 0]
        else:
            samples = proposal((num_samples,))[:, 0]
        return samples.reshape(*torch.Size(sample_shape), -1)

    @torch.no_grad()
    def sample_batched(self, sample_shape, x: Tensor, predictor: str = "euler_maruyama", corrector: Optional[str] = None,
                       predictor_params: Optional[dict] = None, corrector_params: Optional[dict] = None,
                       steps: int = 500, ts: Optional[Tensor] = None, max_sampling_batch_size: int = 10_000,
                       show_progress_bars: bool = True, reject_outside_prior: bool = True,
                       max_sampling_time: Optional[float] = None, return_partial_on_timeout: bool = False) -> Tensor:
        """Samples from p(theta | x_1), ..., p(theta | x_B): (*sample_shape, B, *input_shape)
        (vector_field_posterior.py:507-640).  Each round is ONE ODE solve or ONE SDE run over draws x B particles
        with one condition row per particle (each observation embedded once); draws outside the prior support
        are rejected per observation with a cumulative count, one host sync per round."""
        from .flowmatching import sample_ode, sample_sde
        est = self.vector_field_estimator
        if est.compose_enabled:
            raise NotImplementedError("compose_standardization does not yet support sample_batched (batched / "
                                      "multi-observation sampling). Use a single observation via sample(), or "
                                      "disable compose_standardization.")
        if predictor != "euler_maruyama":
            raise NotImplementedError("predictor: only 'euler_maruyama' (the reference's only predictor)")
        cs = est.condition_shape
        x = torch.as_tensor(x, dtype=torch.float32).to(self._device)
        if x.dim() == len(cs):
            x = x.unsqueeze(0)
        if x.dim() != len(cs) + 1 or x.shape[1:] != cs:
            raise NotImplementedError("Batched sampling for multiple `x` is not supported for iid conditions: "
                                      f"expected x of shape (B, *{tuple(cs)}), got {tuple(x.shape)}.")
        B = x.shape[0]
        D = int(torch.Size(est.input_shape).numel())
        num_samples = torch.Size(sample_shape).numel()
        if max_sampling_batch_size is None:
            max_sampling_batch_size = self.max_sampling_batch_size
        if max_sampling_batch_size * B > 100_000:
            capped = max(1, 100_000 // B)
            warnings.warn(f"Capping max_sampling_batch_size from {max_sampling_batch_size} to {capped} to avoid "
                          "excessive memory usage.", stacklevel=2)
            max_sampling_batch_size = capped
        eta = (predictor_params or {}).get("eta", 1.0)

        def proposal(shape) -> Tensor:
            n = shape[0]
            if self.sample_with == "sde":
                s = sample_sde(est, n, x, steps=steps, ts=ts, eta=eta, corrector=corrector,
                               corrector_params=corrector_params, batched=True)
                self.num_function_evaluations += (steps if ts is None else ts.numel()) - 1
            else:
                s, nfe = sample_ode(est, n, x, return_nfe=True, batched=True)
                self.num_function_evaluations += nfe
            return s

        if not (reject_outside_prior and self.prior is not None):
            return proposal((num_samples,)).reshape(*torch.Size(sample_shape), B, *est.input_shape)
        samples, _ = accept_reject_sample(
            proposal=proposal, accept_reject_fn=lambda theta: within_support(self.prior, theta.reshape(-1, D)),
            num_samples=num_samples, num_xos=B, max_sampling_batch_size=max_sampling_batch_size,
            max_sampling_time=max_sampling_time, return_partial_on_timeout=return_partial_on_timeout)
        if samples.shape[0] < num_samples:          # partial result after a timeout
            return samples
        return samples.reshape(*torch.Size(sample_shape), B, *est.input_shape)

    @torch.no_grad()
    def log_prob(self, theta: Tensor, x: Optional[Tensor] = None, track_gradients: bool = False,
                 ode_kwargs: Optional[dict] = None) -> Tensor:
        """log q(theta | x) via the probability-flow ODE with the exact trace (reference:
        vector_field_posterior.py:467-505 -> VectorFieldBasedPotential.__call__,
        vector_field_potential.py:145-212): -inf outside the prior support."""
        from .flowmatching import log_prob_ode
        if track_gradients:
            raise NotImplementedError("gradients of the neural-ODE log-probability are not implemented")
        x = x if x is not None else self.default_x
        if x is None:
            raise ValueError("Context `x` needed when a default has not been set.")
        x = torch.as_tensor(x, dtype=torch.float32).to(self._device)
        est = self.vector_field_estimator
        if x.reshape(-1).numel() != int(torch.Size(est.condition_shape).numel()):
            raise NotImplementedError("iid observations are not supported by the ODE log-probability here")
        th = torch.as_tensor(theta, dtype=torch.float32).to(self._device)
        th = th.reshape(-1, th.shape[-1])
        kw = dict(ode_kwargs or {})
        lp, nfe = log_prob_ode(est, th, x, atol=kw.get("atol", 1e-6), rtol=kw.get("rtol", 1e-5), return_nfe=True)
        self.num_function_evaluations += nfe
        if self.prior is not None:
            lp = torch.where(within_support(self.prior, th), lp, torch.full_like(lp, float("-inf")))
        return lp
