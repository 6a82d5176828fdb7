"""Host logic of batched sampling, with stand-in estimators on the CPU: the paired (`x_is_iid=False`) likelihood
potential, the batched MCMC inits (observation-major chain order, chunking), the argument checks of the
`sample_batched` methods, and the diagnostics' choice between batched and per-observation sampling."""
import warnings

import pytest
import torch
from torch.distributions import Independent, Normal

from sbi_b200 import diagnostics as dg
from sbi_b200.posteriors import MCMCPosterior, RejectionPosterior, VectorFieldPosterior
from sbi_b200.potentials import LikelihoodBasedPotential
from sbi_b200.samplers import init_batched


class _Gauss:
    """log q(x | theta) = sum -0.5 ((x - theta) / s)^2, (sample, batch) shaped like the flow estimators."""
    input_shape = torch.Size([1])

    def __init__(self, s):
        self.s = s

    def eval(self):
        return self

    def log_prob(self, input, condition):
        return (-0.5 * ((input - condition) / self.s) ** 2).sum(-1)


def _prior(D=1, sd=3.0):
    return Independent(Normal(torch.zeros(D), sd * torch.ones(D)), 1)


def test_paired_likelihood_potential():
    pot = LikelihoodBasedPotential(_Gauss(0.5), _prior(), device="cpu")
    g = torch.Generator().manual_seed(0)
    th, xs = torch.randn(7, 1, generator=g), torch.randn(7, 1, generator=g)
    pot.set_x(xs, x_is_iid=False)
    got = pot(th, track_gradients=False)
    want = []
    for r in range(7):
        pot.set_x(xs[r:r + 1])
        want.append(pot(th[r:r + 1], track_gradients=False))
    assert torch.equal(got, torch.cat(want))
    pot.set_x(xs)                                  # iid: every theta against all 7 trials
    assert torch.allclose(pot(th[:2]), torch.stack([(-2 * (xs - t) ** 2).sum() for t in th[:2]]) +
                          pot.prior.log_prob(th[:2]))
    pot.set_x(xs, x_is_iid=False)
    with pytest.raises(AssertionError, match="Batch size mismatch"):
        pot(th[:6])


@pytest.mark.parametrize("strategy", ["resample", "sir"])
def test_batched_inits_are_observation_major(strategy):
    pot = LikelihoodBasedPotential(_Gauss(0.05), _prior(), device="cpu")
    xo = torch.tensor([[-3.0], [0.0], [3.0]])
    ident = torch.distributions.transforms.identity_transform
    torch.manual_seed(0)
    # 250 rows per chunk at 100 candidates per chain: two chains per chunk, chunks straddle observations
    init = init_batched(pot.prior, pot, ident, xo, 4, strategy, num_candidate_samples=100, max_rows=250)
    assert init.shape == (12, 1)
    assert (init.reshape(3, 4) - xo).abs().max() < 0.5
    assert init_batched(pot.prior, pot, ident, xo, 4, "proposal").shape == (12, 1)


def test_sample_batched_argument_checks():
    pot = LikelihoodBasedPotential(_Gauss(0.5), _prior(), device="cpu")
    with pytest.raises(AssertionError, match="vectorized"):
        MCMCPosterior(pot, _prior(), method="slice_np", device="cpu").sample_batched((10,), torch.zeros(2, 1))
    with pytest.raises(NotImplementedError, match="Batched sampling is not implemented for RejectionPosterior"):
        RejectionPosterior(pot, _prior(), device="cpu").sample_batched((10,), torch.zeros(2, 1))
    from sbi_b200.flowmatching import build_vector_field_estimator
    est = build_vector_field_estimator(torch.randn(50, 2), torch.randn(50, 3), hidden_features=8, num_layers=2)
    post = VectorFieldPosterior(est, _prior(2), device="cpu")
    with pytest.raises(NotImplementedError, match="iid"):
        post.sample_batched((10,), torch.zeros(4, 5, 3))


class _Post:
    def __init__(self, batched_raises):
        self.batched_raises, self.calls = batched_raises, []

    def sample(self, shape, x, show_progress_bars=False):
        self.calls.append("sample")
        return x[:2].expand(*shape, 2).clone()

    def sample_batched(self, shape, x, show_progress_bars=False):
        self.calls.append("batched")
        if self.batched_raises:
            raise NotImplementedError
        return x[:, :2].expand(*shape, x.shape[0], 2).clone()


def test_diagnostics_honour_use_batched_sampling():
    xs = torch.randn(4, 3)
    p = _Post(False)
    a = dg._posterior_samples(xs, p, 5, False)
    b = dg._posterior_samples(xs, p, 5, False, use_batched_sampling=False)
    assert p.calls == ["batched"] + ["sample"] * 4 and torch.equal(a, b)
    p = _Post(True)
    with pytest.warns(UserWarning, match="Falling back"):
        c = dg._posterior_samples(xs, p, 5, False)
    assert torch.equal(a, c)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        dg._posterior_samples(xs, _Post(True), 5, False, use_batched_sampling=False)
