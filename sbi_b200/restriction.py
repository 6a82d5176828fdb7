"""Truncated sequential NPE (TSNPE, Deistler et al. 2022): the prior restricted to a posterior's high-density region.

`get_density_thresholder` and `RestrictedPrior` mirror the reference's sbi/utils/restriction_estimator.py:484-521
and :613-846.  The restricted prior's rejection sampling runs through `posteriors.accept_reject_sample`
(sbi/samplers/rejection/rejection.py:230-457) for one observation, draw for draw: the user's prior draws each batch
on its own generator, the draws move to the CUDA device, `accept_reject_fn` decides there and the accepted rows are
collected there in draw order.  The acceptance rate is computed on the host in the reference's float32 arithmetic,
wherever the prior draws.
"""
from __future__ import annotations

import sys
from typing import Any, Callable, Optional

import torch
from torch import Tensor
from torch.distributions import Distribution

from .posteriors import accept_reject_sample


def get_density_thresholder(dist: Any, quantile: float = 1e-4,
                            num_samples_to_estimate_support: int = 1_000_000) -> Callable:
    """A predicate that is True for theta inside the `1 - quantile` high-probability region of `dist`.

    The threshold is the `int(quantile * N)`-th smallest `dist.log_prob` of `N = num_samples_to_estimate_support`
    draws of `dist`; the predicate is `dist.log_prob(theta) > threshold` (strict, so NaN and -inf reject).
    `dist` needs `sample` and `log_prob`; for a `DirectPosterior` both run on the estimator kernels."""
    samples = dist.sample((num_samples_to_estimate_support,))
    log_probs = dist.log_prob(samples)
    sorted_log_probs, _ = torch.sort(log_probs)
    log_prob_threshold = sorted_log_probs[int(quantile * num_samples_to_estimate_support)]

    def density_thresholder(theta: Tensor) -> Tensor:
        return (dist.log_prob(theta) > log_prob_threshold).bool()

    return density_thresholder


def _compute_device(device: str) -> torch.device:
    """The CUDA device the sampling runs on: `device` itself when it is a CUDA device, else the current one."""
    if not torch.cuda.is_available():
        raise RuntimeError("RestrictedPrior samples on a CUDA (sm_90a) device and none is available "
                           "(no CPU fallback)")
    d = torch.device(device)
    return d if d.type == "cuda" and d.index is not None else torch.device("cuda", torch.cuda.current_device())


def _process_device(device: Optional[str]) -> str:
    """Where results live (torchutils.process_device): "cpu", or a CUDA device with its index."""
    if device is None:
        return "cpu"
    if device == "gpu":
        device = "cuda"
    d = torch.device(device)
    if d.type == "cuda" and d.index is None:
        d = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
    return str(d)


class RestrictedPrior(Distribution):
    """The prior restricted to the region where `accept_reject_fn` is True (restriction_estimator.py:613-846).

    Sampling runs on a CUDA device whatever `device` says; `device` only decides where samples are returned,
    as in the reference.  `sample_with="sir"` resamples draws of `posterior`, weighted by
    `accept_reject_fn(theta).float() - log q(theta)`."""

    def __init__(self, prior: Distribution, accept_reject_fn: Callable, posterior: Optional[Any] = None,
                 sample_with: str = "rejection", device: str = "cpu") -> None:
        super().__init__(validate_args=False)
        self._prior = prior
        self._accept_reject_fn = accept_reject_fn
        self._posterior = posterior     # only used for SIR
        self._sample_with = sample_with
        self._device = _process_device(device)
        self.acceptance_rate = None     # only defined for rejection sampling

    def sample(self, sample_shape=torch.Size(), sample_with: Optional[str] = None,
               max_sampling_batch_size: int = 10_000, oversampling_factor: int = 1024,
               save_acceptance_rate: bool = False, show_progress_bars: bool = False,
               print_rejected_frac: bool = True) -> Tensor:
        """Draws from the restricted prior, (*sample_shape, D).  With `rejection`, prior draws are accepted by
        `accept_reject_fn` in batches of at most `max_sampling_batch_size`; `save_acceptance_rate` keeps the
        acceptance rate for `log_prob`.  With `sir`, `oversampling_factor` is accepted but, as in the reference,
        does not reach the sampler: every sample is chosen among 32 posterior draws, and the selection uniforms
        are drawn on the CUDA device."""
        num_samples = torch.Size(sample_shape).numel()
        sample_with = self._sample_with if sample_with is None else sample_with
        dev = _compute_device(self._device)
        if sample_with == "rejection":
            if num_samples < 1:
                raise ValueError(f"num_samples must be positive, got {num_samples}")
            with torch.cuda.device(dev):
                samples, rate = accept_reject_sample(
                    lambda shape: self._prior.sample(shape).reshape(shape[0], -1).to(torch.float32),
                    lambda theta: self._accept_reject_fn(theta).to(device=dev, dtype=torch.bool),
                    num_samples, max_sampling_batch_size=max_sampling_batch_size,
                    alternative_method="sample_with='sir'", device=dev)
            acceptance_rate = rate.item()
            if save_acceptance_rate:
                self.acceptance_rate = torch.as_tensor(acceptance_rate)
            if print_rejected_frac:
                print(f"The `RestrictedPrior` rejected {(1.0 - acceptance_rate) * 100:.1f}% of prior samples. "
                      f"You will get a speed-up of {(1.0 / acceptance_rate - 1.0) * 100:.1f}%.")
        elif sample_with == "sir":
            assert self._posterior is not None, (
                "In order to use SIR sampling, you must provide a `posterior`: "
                "`RestrictionEstimator(..., posterior=posterior)`.")
            from .samplers import sampling_importance_resampling
            samples = sampling_importance_resampling(
                lambda theta: self._accept_reject_fn(theta).type(torch.float32), proposal=self._posterior,
                num_samples=num_samples, oversampling_factor=oversampling_factor,
                show_progress_bars=show_progress_bars, max_sampling_batch_size=max_sampling_batch_size,
                device=str(dev))
        else:
            raise ValueError("Only [rejection | sir] implemented as `method`")
        return samples.reshape((*torch.Size(sample_shape), -1)).to(self._device)

    def log_prob(self, theta: Tensor, norm_restricted_prior: bool = True, track_gradients: bool = False,
                 prior_acceptance_params: Optional[dict] = None) -> Tensor:
        """`prior.log_prob(theta)` where `accept_reject_fn` accepts, -inf elsewhere; minus log `prior_acceptance()`
        when `norm_restricted_prior` (its keyword arguments in `prior_acceptance_params`)."""
        theta = torch.as_tensor(theta)
        if theta.ndim == 1:
            theta = theta.unsqueeze(0)
        with torch.set_grad_enabled(track_gradients):
            prior_log_prob = self._prior.log_prob(theta)
            accepted = self._accept_reject_fn(theta).bool()
            masked_log_prob = torch.where(accepted, prior_log_prob, torch.tensor(float("-inf"), dtype=torch.float32))
            log_factor = (torch.log(self.prior_acceptance(**(prior_acceptance_params or {})))
                          if norm_restricted_prior else 0)
            return masked_log_prob - log_factor

    @torch.no_grad()
    def prior_acceptance(self, num_rejection_samples: int = 10_000, force_update: bool = False,
                         show_progress_bars: bool = False, rejection_sampling_batch_size: int = 10_000) -> Tensor:
        """Fraction of prior draws `accept_reject_fn` accepts, estimated once by rejection sampling and cached in
        `acceptance_rate` (re-estimated with `force_update`)."""
        if self.acceptance_rate is None or force_update:
            self.sample(sample_shape=torch.Size((num_rejection_samples,)), sample_with="rejection",
                        show_progress_bars=show_progress_bars, max_sampling_batch_size=rejection_sampling_batch_size,
                        save_acceptance_rate=True)
        return self.acceptance_rate

    @property
    def mean(self) -> Tensor:
        raise NotImplementedError("Mean is not implemented for RestrictedPrior.")

    @property
    def variance(self) -> Tensor:
        raise NotImplementedError("Variance is not implemented for RestrictedPrior.")

    @property
    def support(self):
        try:
            return self._prior.support
        except AttributeError as e:
            raise NotImplementedError("Support is not implemented for this RestrictedPrior.") from e


def is_restricted_prior(proposal: Any) -> bool:
    """Whether `proposal` is a `RestrictedPrior`: this module's, or the reference's when the caller's process has
    imported `sbi` (as `_refabc` binds to the reference's classes)."""
    if isinstance(proposal, RestrictedPrior):
        return True
    if "sbi" not in sys.modules:
        return False
    try:
        from sbi.utils.restriction_estimator import RestrictedPrior as RefRestrictedPrior
    except Exception:   # a partial / foreign `sbi` module
        return False
    return isinstance(proposal, RefRestrictedPrior)
