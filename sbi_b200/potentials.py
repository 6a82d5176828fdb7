"""Potential functions theta -> log p~(theta | x_o) built from a trained estimator and the prior.

Mirrors /root/reference/sbi/inference/potentials/: `posterior_estimator_based_potential`
(posterior_based_potential.py:20-191), `likelihood_estimator_based_potential`
(likelihood_based_potential.py:24-239), `ratio_estimator_based_potential`
(ratio_based_potential.py:18-160), `mcmc_transform` (sbiutils.py:867-984) and
`transformed_potential` (potentialutils.py:14-48).  Each potential evaluates a whole batch of
theta in one estimator-kernel launch; x_o is never re-expanded per call beyond a (n_iid, C) view.
"""
from __future__ import annotations

import warnings
from typing import Callable, Optional, Tuple

import torch
from torch import Tensor
from torch.distributions import biject_to, constraints
from torch.distributions import transforms as torch_tf

from .posteriors import prior_to_device, within_support


def mcmc_transform(prior, num_prior_samples_for_zscoring: int = 1000, enable_transform: bool = True,
                   device: str = "cuda", **kwargs) -> torch_tf.Transform:
    """sbiutils.py:867-984: bounded support -> biject_to(support); unbounded -> affine z-scoring
    with the prior's mean / std.  Returns the transform from constrained to unconstrained space."""
    if enable_transform:
        def mean_std_transform():
            try:
                mean, std = prior.mean.to(device), prior.stddev.to(device)
            except (NotImplementedError, AttributeError):
                th = prior.sample(torch.Size((num_prior_samples_for_zscoring,)))
                mean, std = th.mean(dim=0).to(device), th.std(dim=0).to(device)
            return torch_tf.AffineTransform(loc=mean, scale=std)

        try:
            _ = prior.support
            has_support = True
        except (NotImplementedError, AttributeError):
            warnings.warn("The passed prior has no support property, transform will be constructed from "
                          "mean and std.", stacklevel=2)
            has_support = False
        if has_support:
            constraint = getattr(prior.support, "base_constraint", prior.support)
            if getattr(prior.support, "is_discrete", False):
                transform = mean_std_transform()
            elif isinstance(constraint, constraints._Real):
                transform = mean_std_transform()
            else:
                transform = biject_to(prior.support)
        else:
            transform = mean_std_transform()
    else:
        transform = torch_tf.identity_transform
    if not isinstance(transform, torch_tf.IndependentTransform):
        transform = torch_tf.IndependentTransform(transform, reinterpreted_batch_ndims=1)
    return transform.inv


def transformed_potential(theta, potential_fn: Callable, theta_transform: torch_tf.Transform, device: str,
                          track_gradients: bool = False) -> Tensor:
    """potentialutils.py:14-48: potential in unconstrained space = potential(T^-1 u) - log|det J|."""
    u = torch.as_tensor(theta, dtype=torch.float32)
    if u.dim() == 1:
        u = u.unsqueeze(0)
    u = u.to(device)
    th = theta_transform.inv(u)
    log_abs_det = theta_transform.log_abs_det_jacobian(th, u)
    return potential_fn(th, track_gradients=track_gradients).to(device) - log_abs_det.to(device)


class BasePotential:
    """base_potential.py:15-104."""

    def __init__(self, prior, x_o: Optional[Tensor] = None, device: str = "cuda"):
        self.device = device
        self.prior = prior_to_device(prior, device)
        self._x_o = None
        self._x_is_iid = True
        if x_o is not None:
            self.set_x(x_o)

    def set_x(self, x_o: Optional[Tensor], x_is_iid: Optional[bool] = True):
        if x_o is not None:
            x_o = torch.as_tensor(x_o, dtype=torch.float32).to(self.device)
        self._x_o = x_o
        self._x_is_iid = x_is_iid

    @property
    def x_o(self) -> Tensor:
        if self._x_o is None:
            raise ValueError("No observed data is available. Use `potential_fn.set_x(x_o)`.")
        return self._x_o

    @x_o.setter
    def x_o(self, x_o):
        self.set_x(x_o)

    def return_x_o(self):
        return self._x_o


class PosteriorBasedPotential(BasePotential):
    """posterior_based_potential.py:65-191: log q(theta | x_o), -inf outside the prior support."""

    def __init__(self, posterior_estimator, prior, x_o=None, device="cuda"):
        super().__init__(prior, x_o, device)
        self.posterior_estimator = posterior_estimator
        self.posterior_estimator.eval()

    def __call__(self, theta: Tensor, track_gradients: bool = True) -> Tensor:
        theta = torch.as_tensor(theta, dtype=torch.float32).to(self.device)
        if theta.dim() == 1:
            theta = theta.unsqueeze(0)
        x = self.x_o.reshape(-1, *self.posterior_estimator.condition_shape)
        if x.shape[0] > 1:
            raise NotImplementedError("iid x is not supported by posterior-based potentials "
                                      "(posterior_based_potential.py:139-152).")
        with torch.set_grad_enabled(track_gradients):
            lp = self.posterior_estimator.log_prob(theta.unsqueeze(1), condition=x)[:, 0]
            inside = within_support(self.prior, theta)
            return torch.where(inside, lp, torch.full_like(lp, float("-inf")))    # (no host scalar: graph-capturable)


def _check_pairs(theta: Tensor, x: Tensor):
    """x_is_iid=False: row r of theta pairs with row r of x_o (likelihood_based_potential.py:117-124)."""
    if theta.shape[0] != x.shape[0]:
        raise AssertionError(f"Batch size mismatch: {theta.shape[0]} and {x.shape[0]}. When performing batched "
                             "sampling for multiple `x`, the batch size of `theta` must match the batch size of `x`.")


class LikelihoodBasedPotential(BasePotential):
    """likelihood_based_potential.py:59-130: sum_trials log q(x_o,i | theta) + log p(theta); with
    `x_is_iid=False`, log q(x_o,r | theta_r) + log p(theta_r) per row."""

    def __init__(self, likelihood_estimator, prior, x_o=None, device="cuda"):
        super().__init__(prior, x_o, device)
        self.likelihood_estimator = likelihood_estimator
        self.likelihood_estimator.eval()

    def __call__(self, theta: Tensor, track_gradients: bool = True) -> Tensor:
        theta = torch.as_tensor(theta, dtype=torch.float32).to(self.device)
        if theta.dim() == 1:
            theta = theta.unsqueeze(0)
        est = self.likelihood_estimator
        x = self.x_o.reshape(-1, *est.input_shape)          # (n_iid, Dx), or (R, Dx) paired with theta
        if not self._x_is_iid:
            _check_pairs(theta, x)
            with torch.set_grad_enabled(track_gradients):     # one launch, input and condition per row
                return est.log_prob(x.unsqueeze(0), condition=theta)[0] + self.prior.log_prob(theta)
        with torch.set_grad_enabled(track_gradients):
            # _log_likelihoods_over_trials (:186-239): x (n_iid, 1, Dx) broadcast against theta (R, D)
            ll = est.log_prob(x.unsqueeze(1).expand(-1, theta.shape[0], *est.input_shape), condition=theta).sum(0)
            return ll + self.prior.log_prob(theta)


class RatioBasedPotential(BasePotential):
    """ratio_based_potential.py:49-119: sum_trials log r(theta, x_o,i) + log p(theta); with `x_is_iid=False`,
    log r(theta_r, x_o,r) + log p(theta_r) per row.  The rows of x_o go through the x embedding net once per
    `set_x` (the reference re-embeds them on every call); iid trials are paired with theta by index in the
    kernel, never materialised as n x R rows."""

    def __init__(self, ratio_estimator, prior, x_o=None, device="cuda"):
        self.ratio_estimator = ratio_estimator
        self.ratio_estimator.eval()
        super().__init__(prior, x_o, device)

    def set_x(self, x_o: Optional[Tensor], x_is_iid: Optional[bool] = True):
        super().set_x(x_o, x_is_iid)
        self._x_rows = None
        if self._x_o is not None:
            est = self.ratio_estimator
            with torch.no_grad():
                self._x_rows = est.embed_x(self._x_o.reshape(-1, *est.x_shape))     # (n_iid, Dx) kernel rows

    def __call__(self, theta: Tensor, track_gradients: bool = True) -> Tensor:
        from .ratio import _RatioFn
        theta = torch.as_tensor(theta, dtype=torch.float32).to(self.device)
        if theta.dim() == 1:
            theta = theta.unsqueeze(0)
        est = self.ratio_estimator
        self.x_o      # raises without an observation
        x = self._x_rows
        with torch.set_grad_enabled(track_gradients):
            th = est.embed_theta(theta.reshape(-1, *est.theta_shape))
            if not self._x_is_iid:   # one pairs launch over the R (theta_r, x_r) rows
                _check_pairs(th, x)
                lr = _RatioFn.apply(est.net.flat, th, x, est, None, None, False)
            elif x.shape[0] == 1:   # one observation: x is shared by every pair, never repeated
                lr = _RatioFn.apply(est.net.flat, th, x, est, None, None, True)
            else:                 # _log_ratios_over_trials (:122-160): pair k = (theta[k % R], x[k // R])
                n, R = x.shape[0], th.shape[0]
                ti = torch.arange(R, device=th.device).repeat(n)
                xi = torch.arange(n, device=th.device).repeat_interleave(R)
                lr = _RatioFn.apply(est.net.flat, th, x, est, ti, xi, False, True).reshape(n, -1).sum(0)
            return lr + self.prior.log_prob(theta)


def posterior_estimator_based_potential(posterior_estimator, prior, x_o=None, enable_transform: bool = True):
    device = str(posterior_estimator.flat.device)
    prior = prior_to_device(prior, device)      # the unconstraining transform's constants live with the chains
    return (PosteriorBasedPotential(posterior_estimator, prior, x_o, device),
            mcmc_transform(prior, device=device, enable_transform=enable_transform))


def likelihood_estimator_based_potential(likelihood_estimator, prior, x_o=None, enable_transform: bool = True):
    device = str(likelihood_estimator.flat.device)
    prior = prior_to_device(prior, device)      # the unconstraining transform's constants live with the chains
    return (LikelihoodBasedPotential(likelihood_estimator, prior, x_o, device),
            mcmc_transform(prior, device=device, enable_transform=enable_transform))


def ratio_estimator_based_potential(ratio_estimator, prior, x_o=None, enable_transform: bool = True):
    device = str(ratio_estimator.flat.device)
    prior = prior_to_device(prior, device)      # the unconstraining transform's constants live with the chains
    return (RatioBasedPotential(ratio_estimator, prior, x_o, device),
            mcmc_transform(prior, device=device, enable_transform=enable_transform))
