"""Coverage diagnostics that hammer `posterior.sample` (SURVEY 8f-4): simulation-based calibration and TARP with
the reference's signatures and return values (/root/reference/sbi/diagnostics/sbc.py:23-188,
/root/reference/sbi/diagnostics/tarp.py:27-195).  The posterior draws for ALL observations come from one
batched sampling call (`sample_batched` of the direct, MCMC and vector-field posteriors), and the
rank statistics are single device reductions instead of the reference's Python loop with a host read per
(observation, dimension).  The downstream checks (`check_sbc`, `check_tarp`: KS / c2st tests on the returned
tensors) are the reference's own, unchanged."""
from __future__ import annotations

import warnings
from typing import Callable, List, Optional, Tuple, Union

import torch
from torch import Tensor

from .misspecification import calc_misspecification_mmd  # noqa: F401  (the MMD misspecification test)

_LC2ST_NAMES = ("LC2ST", "LC2ST_NF", "LC2STScores", "LC2STState")


def __getattr__(name):
    """The local test (`sbi_b200.lc2st`) on first use: it needs scikit-learn, SBC and TARP do not."""
    if name in _LC2ST_NAMES:
        from . import lc2st
        return getattr(lc2st, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")


def _clean(thetas: Tensor, xs: Tensor) -> Tuple[Tensor, Tensor]:
    """remove_nans_and_infs_in_x (utils/diagnostics_utils.py:101-120)."""
    xf = xs.reshape(xs.shape[0], -1)
    ok = torch.isfinite(xf).all(dim=1)
    if not bool(ok.all()):
        warnings.warn(f"Removed {int((~ok).sum())} entries with NaNs or infs in x.", stacklevel=3)
    return thetas[ok], xs[ok]


def _posterior_samples(xs: Tensor, posterior, num_posterior_samples: int, show_progress_bar: bool,
                       use_batched_sampling: bool = True) -> Tensor:
    """(num_posterior_samples, num_xs, dim): batched sampling when asked for and the posterior has it, else one
    call per x (utils/diagnostics_utils.py:19-98)."""
    if use_batched_sampling and hasattr(posterior, "sample_batched"):
        try:
            return posterior.sample_batched((num_posterior_samples,), x=xs, show_progress_bars=show_progress_bar)
        except (NotImplementedError, AssertionError):
            warnings.warn("Batched sampling not implemented for this posterior. Falling back to non-batched sampling.",
                          stacklevel=3)
    outs = [posterior.sample((num_posterior_samples,), x=x, show_progress_bars=False) for x in xs]
    return torch.stack(outs).permute(1, 0, 2)


def sbc_ranks(thetas: Tensor, xs: Tensor, posterior_samples: Tensor,
              reduce_fns: Union[str, Callable, List[Callable]] = "marginals") -> Tensor:
    """Ranks of the ground-truth parameters among the posterior draws (sbc.py:137-219).  "marginals": one
    comparison + reduction over the whole (draws, observations, dims) tensor."""
    thetas = thetas.to(posterior_samples.device)
    if isinstance(reduce_fns, str):
        assert reduce_fns == "marginals", "`reduce_fn` must either be the string `marginals` or a Callable or a List " \
                                          "of Callables."
        return (posterior_samples < thetas.unsqueeze(0)).sum(dim=0).to(torch.float32)
    fns = reduce_fns if isinstance(reduce_fns, list) else [reduce_fns]
    ranks = torch.zeros((thetas.shape[0], len(fns)), device=posterior_samples.device)
    for i, (true_theta, x_i) in enumerate(zip(thetas, xs)):
        for j, fn in enumerate(fns):
            ranks[i, j] = (fn(posterior_samples[:, i, :], x_i) < fn(true_theta.unsqueeze(0), x_i)).sum()
    return ranks


def run_sbc(thetas: Tensor, xs: Tensor, posterior, num_posterior_samples: int = 1000,
            reduce_fns: Union[str, Callable, List[Callable]] = "marginals", num_workers: int = 1,
            show_progress_bar: bool = False, use_batched_sampling: bool = True) -> Tuple[Tensor, Tensor]:
    """Simulation-based calibration / expected coverage (sbc.py:23-112): returns (ranks, dap_samples)."""
    thetas, xs = _clean(thetas, xs)
    n = thetas.shape[0]
    if n < 100:
        warnings.warn("Number of SBC samples should be on the order of 100s to give reliable results.", stacklevel=2)
    if num_posterior_samples < 100:
        warnings.warn("Number of posterior samples for ranking should be on the order of 100s to give reliable SBC "
                      "results.", stacklevel=2)
    if thetas.shape[0] != xs.shape[0]:
        raise ValueError("Unequal number of parameters and observations.")
    samples = _posterior_samples(xs, posterior, num_posterior_samples, show_progress_bar, use_batched_sampling)
    dap_samples = samples[0, :, :]
    assert dap_samples.shape == (n, thetas.shape[1]), "Wrong DAP shape."
    return sbc_ranks(thetas, xs, samples, reduce_fns), dap_samples


def l2(x: Tensor, y: Tensor, axis: int = -1) -> Tensor:
    """utils/metrics.py l2."""
    return torch.sqrt(torch.sum((x - y) ** 2, dim=axis))


def l1(x: Tensor, y: Tensor, axis: int = -1) -> Tensor:
    return torch.sum(torch.abs(x - y), dim=axis)


def get_tarp_references(thetas: Tensor) -> Tensor:
    """tarp.py:196-206."""
    lo, hi = thetas.min(dim=0).values, thetas.max(dim=0).values
    return torch.distributions.Uniform(low=lo, high=hi).sample(torch.Size([thetas.shape[0]]))


def tarp_coverage(posterior_samples: Tensor, thetas: Tensor, references: Tensor, distance: Callable = l2,
                  num_bins: Optional[int] = None, z_score_theta: bool = False) -> Tuple[Tensor, Tensor]:
    """tarp.py:106-193 (`_run_tarp`), device tensors throughout except the histogram (torch.histogram is CPU-only)."""
    num_posterior_samples, num_tarp_samples, _ = posterior_samples.shape
    dev = posterior_samples.device
    thetas, references = thetas.to(dev), references.to(dev)
    assert references.shape == thetas.shape, "references must have the same shape as thetas"
    if num_bins is None:
        num_bins = num_tarp_samples // 10
    if z_score_theta:
        lo = thetas.min(dim=0, keepdim=True).values
        hi = thetas.max(dim=0, keepdim=True).values
        posterior_samples = (posterior_samples - lo) / (hi - lo + 1e-10)
        thetas = (thetas - lo) / (hi - lo + 1e-10)
        references = (references - lo) / (hi - lo + 1e-10)
    sample_dists = distance(references, posterior_samples)
    theta_dists = distance(references, thetas)
    coverage_values = torch.sum(sample_dists < theta_dists, dim=0) / num_posterior_samples
    hist, alpha_grid = torch.histogram(coverage_values.cpu(), density=True, bins=num_bins)
    hist, alpha_grid = hist.to(dev), alpha_grid.to(dev)
    ecp = torch.cumsum(hist, dim=0) / hist.sum()
    ecp = torch.cat([torch.zeros((1,), device=dev), ecp])
    return ecp, alpha_grid


def run_tarp(thetas: Tensor, xs: Tensor, posterior, references: Optional[Tensor] = None,
             num_posterior_samples: int = 1000, num_workers: int = 1, show_progress_bar: bool = False,
             distance: Callable = l2, num_bins: Optional[int] = None, z_score_theta: bool = True,
             use_batched_sampling: bool = True) -> Tuple[Tensor, Tensor]:
    """TARP expected-coverage curve (tarp.py:27-103): returns (ecp, alpha)."""
    thetas, xs = _clean(thetas, xs)
    n, d = thetas.shape
    if n < 100:
        warnings.warn("Number of TARP samples should be on the order of 100s to give reliable results.", stacklevel=2)
    samples = _posterior_samples(xs, posterior, num_posterior_samples, show_progress_bar, use_batched_sampling)
    assert samples.shape == (num_posterior_samples, n, d), f"Wrong posterior samples shape for TARP: {samples.shape}"
    if references is None:
        references = get_tarp_references(thetas)
    return tarp_coverage(samples, thetas, references, distance, num_bins, z_score_theta)
