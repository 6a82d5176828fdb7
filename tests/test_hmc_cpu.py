"""NUTS / HMC without a GPU: the CPU port's pieces (leapfrog, dual averaging, regularised Welford, Stan's windows),
the port's NUTS and HMC on Gaussian targets, and `MCMCPosterior`'s handling of `nuts_pyro` / `hmc_pyro` with a
stand-in sampler (thinning, per-chain counts, chain-major flattening, the batched-sampling assertion, the pymc
names)."""
import math

import numpy as np
import pytest
import torch
from torch.distributions import Independent, Normal

from oracle import hmc_port as H
from sbi_b200 import hmc as device_hmc
from sbi_b200.posteriors import MCMCPosterior
from sbi_b200.potentials import LikelihoodBasedPotential


def test_leapfrog_matches_harmonic_oscillator_and_is_reversible():
    # U = q^2 / 2 with inverse mass m: q(t) = q0 cos(w t) + (m p0 / w) sin(w t), w = sqrt(m)
    m = np.array([2.0])
    pot = lambda q: (0.5 * float(q @ q), q.copy())       # noqa: E731
    q0, p0 = np.array([1.0]), np.array([0.5])
    h, n = 1e-3, 3000
    q, p, g = q0, p0, q0.copy()
    for _ in range(n):
        q, p, g, _ = H.leapfrog(q, p, g, h, m, pot)
    w, t = math.sqrt(2.0), h * n
    q_exact = q0 * math.cos(w * t) + m * p0 / w * math.sin(w * t)
    p_exact = p0 * math.cos(w * t) - q0 * w / m * math.sin(w * t)
    assert np.allclose(q, q_exact, atol=1e-5) and np.allclose(p, p_exact, atol=1e-5)
    # reversibility: n steps forward, flip the momentum, n steps forward again
    q, p, g = q0, p0, q0.copy()
    for _ in range(50):
        q, p, g, _ = H.leapfrog(q, p, g, 0.3, m, pot)
    p = -p
    for _ in range(50):
        q, p, g, _ = H.leapfrog(q, p, g, 0.3, m, pot)
    assert np.allclose(q, q0, atol=1e-12) and np.allclose(-p, p0, atol=1e-12)


def test_dual_averaging_hand_computed():
    # prox centre log(10 * 0.5); g_t = target - accept; by hand:
    # t=1: gbar = 0.3/11, x = log 5 - 1/0.05 * gbar = 1.06398..., xbar = x (weight 1)
    # t=2: gbar = (1 - 1/12) gbar + (-0.1)/12 = 1/60, x = log 5 - sqrt(2)/0.05/60, xbar = (1 - 2^-0.75) x1 + 2^-0.75 x2
    da = H.DualAveraging(prox_center=math.log(5.0))
    want = [(0.02727272727272727, 1.0639833669795549, 1.0639833669795549),
            (0.016666666666666663, 1.1380333916430687, 1.1080137750775436),
            (0.05384615384615385, -0.25584757264007507, 0.5096996160770366),
            (0.10714285714285715, -2.676276373280186, -0.6167129973089693)]
    for g, (gbar, x, xbar) in zip([0.3, -0.1, 0.5, 0.8], want):
        got_x, got_xbar = da.step(g)
        assert da.g_avg == pytest.approx(gbar, rel=1e-14)
        assert got_x == pytest.approx(x, rel=1e-13) and got_xbar == pytest.approx(xbar, rel=1e-13)


def test_regularised_welford_matches_numpy():
    rng = np.random.default_rng(3)
    x = rng.normal(size=(37, 4)) * np.array([0.01, 1.0, 5.0, 100.0]) + 3.0
    wf = H.Welford(4)
    for row in x:
        wf.update(row)
    n = x.shape[0]
    want = n / (n + 5.0) * x.var(axis=0, ddof=1) + 1e-3 * 5.0 / (n + 5.0)
    assert np.allclose(wf.mean, x.mean(0), rtol=1e-13)
    assert np.allclose(wf.variance(), want, rtol=1e-12)


@pytest.mark.parametrize("warmup, windows", [
    (200, [(0, 74), (75, 99), (100, 149), (150, 199)]),
    (100, [(0, 14), (15, 89), (90, 99)]),
    (30, [(0, 3), (4, 26), (27, 29)]),
    (19, [(0, 18)]),
    (1000, [(0, 74), (75, 99), (100, 149), (150, 249), (250, 449), (450, 949), (950, 999)]),
])
def test_window_boundaries(warmup, windows):
    assert device_hmc.adaptation_schedule(warmup) == windows
    assert H.adaptation_schedule(warmup) == windows


def _gauss(cov):
    prec = np.linalg.inv(cov)
    return lambda z: (-0.5 * float(z @ prec @ z), -prec @ z)


_CORR = np.array([[1.0, 0.9], [0.9, 1.0]]) * np.array([[1.0, 2.0], [2.0, 4.0]])   # sd 1 and 2, correlation 0.9
_SCALES = np.array([0.01, 0.1, 1.0, 3.0, 10.0])


@pytest.mark.parametrize("algo", ["nuts", "hmc"])
@pytest.mark.parametrize("cov", [_CORR, np.diag(_SCALES ** 2)], ids=["corr2d", "scaled5d"])
def test_port_samples_gaussians(algo, cov):
    D, C, warmup, n = cov.shape[0], 4, 300, 400
    draws = H.NumpyDraws(C, D, 10, seed=11)
    runs = [H.run_chain(np.full(D, 0.5) * np.sqrt(np.diag(cov)), _gauss(cov), draws, c, algo=algo, warmup=warmup,
                        num_samples=n) for c in range(C)]
    s = np.stack([np.array(r.samples) for r in runs])                 # (C, n, D)
    sd = np.sqrt(np.diag(cov))
    # Monte-Carlo error of the mean from batch means (batches of 50 transitions)
    bm = s.reshape(C, n // 50, 50, D).mean(2).reshape(-1, D)
    se = bm.std(0, ddof=1) / math.sqrt(bm.shape[0])
    assert np.all(np.abs(s.reshape(-1, D).mean(0)) < 5 * se + 0.02 * sd)
    assert np.allclose(s.reshape(-1, D).std(0) / sd, 1.0, atol=0.25)
    assert sum(rec.diverging for r in runs for rec in r.records[warmup:]) == 0
    minv = np.stack([r.records[-1].minv for r in runs])
    # the adapted inverse mass estimates the marginal variances (last window: 100 transitions) to within 4x
    assert np.all(minv / np.diag(cov) > 0.25) and np.all(minv / np.diag(cov) < 4.0)


# ---- MCMCPosterior host logic with a stand-in sampler -------------------------------------------------------
class _Gauss:
    input_shape = torch.Size([1])

    def eval(self):
        return self

    def log_prob(self, input, condition):
        return (-0.5 * (input - condition) ** 2).sum(-1)


def _posterior(method, **kw):
    prior = Independent(Normal(torch.zeros(1), torch.ones(1)), 1)
    pot = LikelihoodBasedPotential(_Gauss(), prior, device="cpu")
    return MCMCPosterior(pot, prior, method=method, device="cpu", init_strategy="proposal", **kw)


class _FakeSampler:
    """Records its arguments; sample i of chain c is (1000 c + i)."""
    calls = []

    def __init__(self, log_prob_fn, init_params, num_chains, method, warmup_steps, device, graph, **kw):
        self.num_chains, self.method, self.warmup_steps = num_chains, method, warmup_steps
        _FakeSampler.calls.append(self)

    def run(self, num_samples):
        self.num_samples = num_samples
        c = np.arange(self.num_chains)[:, None, None]
        i = np.arange(num_samples)[None, :, None]
        return (1000.0 * c + i).astype(np.float64)


@pytest.mark.parametrize("method", ["nuts_pyro", "hmc_pyro"])
def test_posterior_counts_thinning_and_flattening(monkeypatch, method):
    monkeypatch.setattr(device_hmc, "HMCSamplerVectorized", _FakeSampler)
    _FakeSampler.calls.clear()
    post = _posterior(method, num_chains=3, warmup_steps=7)
    out = post.sample((10,), x=torch.zeros(1, 1))                     # thin -1 -> 1
    smp = _FakeSampler.calls[-1]
    assert (smp.method, smp.warmup_steps, smp.num_chains) == (method[:-5], 7, 3)
    assert smp.num_samples == math.ceil(10 / 3)                       # warm-up not multiplied by thin
    flat = (1000.0 * np.arange(3)[:, None] + np.arange(4)[None, :]).reshape(-1)
    assert out.shape == (10, 1) and np.array_equal(out[:, 0].numpy(), flat[:10])
    assert post._mcmc_init_params[:, 0].tolist() == [3.0, 1003.0, 2003.0]
    out = post.sample((2, 5), x=torch.zeros(1, 1), thin=4)
    assert _FakeSampler.calls[-1].num_samples == math.ceil(4 * 10 / 3)
    flat = (1000.0 * np.arange(3)[:, None] + np.arange(14)[None, :]).reshape(-1)
    assert out.shape == (2, 5, 1) and np.array_equal(out.reshape(-1).numpy(), flat[::4][:10])
    assert post.thin == 10                                            # the slice path keeps its default


def test_posterior_method_names():
    post = _posterior("nuts_pyro")
    with pytest.raises(AssertionError, match="Batched sampling only supported for vectorized samplers!"):
        post.sample_batched((10,), torch.zeros(2, 1))
    for name in ("hmc_pymc", "nuts_pymc", "slice_pymc"):
        with pytest.raises(NotImplementedError):
            _posterior(name)


def test_frozen_parameters_restores_flags():
    net = torch.nn.Sequential(torch.nn.Linear(2, 2), torch.nn.Linear(2, 1))
    net[1].bias.requires_grad_(False)

    class Holder:
        def __init__(self):
            self.estimator = net

    with device_hmc.frozen_parameters(Holder()):
        assert not any(p.requires_grad for p in net.parameters())
    assert [p.requires_grad for p in net.parameters()] == [True, True, True, False]
