"""NUTS and HMC on the GPU (csrc/hmc.cu): the kernel against the CPU port on the same random numbers, graph replay
against eager lock-steps, the linear-Gaussian posterior through NLE and NRE, the `mlp` classifier's theta gradient
under the iid gather, and a bounded prior."""
import math

import numpy as np
import pytest
import torch
from torch.distributions import Independent, MultivariateNormal, Uniform

from oracle import hmc_port as H

pytestmark = pytest.mark.gpu

_CORR = torch.tensor([[1.0, 1.8], [1.8, 4.0]])            # sd 1 and 2, correlation 0.9


_CONST = {}     # per (dtype, device), built by the first (eager) lock-steps, before any graph capture


def _const(z):
    from sbi_b200.potentials import mcmc_transform
    key = (z.dtype, str(z.device))
    if key not in _CONST:
        lo = torch.full((2,), -3.0, dtype=z.dtype, device=z.device)
        hi = torch.full((2,), 3.0, dtype=z.dtype, device=z.device)
        box = Independent(Uniform(lo, hi, validate_args=False), 1)
        _CONST[key] = (torch.linalg.inv(_CORR.to(z.dtype)).to(z.device), mcmc_transform(box, device=str(z.device)))
    return _CONST[key]


def _gauss_logp(z):
    prec, _ = _const(z)
    return -0.5 * torch.einsum("ci,ij,cj->c", z, prec, z)


def _banana_logp(u):
    """Banana density on the box [-3, 3]^2, in the unconstrained coordinates of the box (log|det J| included)."""
    _, tf = _const(u)
    th = tf.inv(u)
    lp = -0.5 * (th[:, 0] ** 2 + (th[:, 1] - 0.5 * th[:, 0] ** 2 + 1.0) ** 2 / 0.25)
    return lp - tf.log_abs_det_jacobian(th, u)


def _port_logp_grad(fn):
    def f(z):
        t = torch.tensor(z, dtype=torch.float64).reshape(1, -1).requires_grad_(True)
        lp = fn(t).sum()
        (g,) = torch.autograd.grad(lp, t)
        return float(lp.detach()), g[0].numpy()
    return f


def _run(fn, algo, C, z0, warmup, n, **kw):
    """The analytic potentials are evaluated in float64 and rounded to float32, as the port rounds them, so that
    the kernel and the port see the same values up to float64 rounding."""
    from sbi_b200.hmc import HMCSamplerVectorized
    s = HMCSamplerVectorized(lambda p: fn(p.double()).float(), z0, num_chains=C, method=algo, warmup_steps=warmup,
                             device="cuda", **kw)
    out = s.run(n)
    return s, out


@pytest.mark.parametrize("algo", ["nuts", "hmc"])
@pytest.mark.parametrize("target", ["gauss", "banana"])
def test_kernel_matches_port_on_the_same_draws(cuda_lib, algo, target):
    fn = _gauss_logp if target == "gauss" else _banana_logp
    C, D, warmup, n = 16, 2, 40, 20        # warm-up windows [0, 5], [6, 35], [36, 39]: two searches, one mass update
    torch.manual_seed(5)
    z0 = 0.5 * torch.randn(C, D, dtype=torch.float64)
    # HMC's end point after int(2 pi / eps) steps, and with it the accept statistic and the next dual-averaging
    # step size, is very sensitive to eps: through that loop float64 rounding differences between the device and
    # the port grow by orders of magnitude over a few transitions.  So HMC is compared at a fixed step size with the
    # mass matrix adapted; dual averaging and the step-size search are compared by the NUTS cases.
    kw = dict(adapt_step_size=False, step_size=0.3) if algo == "hmc" else {}
    s, _ = _run(fn, algo, C, z0, warmup, n, record_draws=True, trace=True, **kw)
    draws = [(a.cpu().numpy(), b.cpu().numpy()) for a, b in s.draws]
    flips, checked = 0, 0
    for c in range(C):
        port = H.run_chain(z0[c].numpy(), _port_logp_grad(fn), draws, c, algo=algo, warmup=warmup, num_samples=n,
                           **kw)
        prev_margin = math.inf
        for t, rec in enumerate(port.records):
            tr = s.trace[c, t]
            same = (int(tr[2 * D]) == rec.depth and int(tr[2 * D + 1]) == rec.n_leapfrog
                    and bool(tr[2 * D + 2]) == rec.diverging
                    and np.allclose(tr[:D], rec.z, rtol=1e-4, atol=1e-4)
                    and np.allclose(tr[D:2 * D], rec.minv, rtol=1e-4)
                    and math.isclose(tr[2 * D + 4], rec.step_size, rel_tol=1e-4))
            if not same:
                # a decision flipped: allowed only when the port saw a margin within 1e-5 at or just before it
                assert min(rec.margin, prev_margin) < 1e-5, (c, t, tr.tolist(), rec)
                flips += 1
                break
            assert abs(tr[2 * D + 3] - rec.accept) < 1e-4, (c, t)
            prev_margin = rec.margin
            checked += 1
    print(f"{algo}/{target}: {checked} transitions equal, {flips} of {C} chains flipped a near-tie decision")
    assert flips <= C // 4
    assert checked >= 0.75 * C * (warmup + n)


def test_graph_replay_equals_eager_and_is_reproducible(cuda_lib):
    z0 = torch.zeros(64, 2, dtype=torch.float64)
    outs = []
    for graph in (False, True, True):
        torch.manual_seed(123)
        s, out = _run(_banana_logp, "nuts", 64, z0, 50, 40, graph=graph, check_every=8)
        outs.append((out, s.step_size, s.inverse_mass_matrix))
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert np.array_equal(a, b)


# ---- linear Gaussian through NLE and NRE -----------------------------------------------------------------------
_TRAINED = {}


def _trained(kind, D):
    if (kind, D) not in _TRAINED:
        from sbi_b200.inference import NLE, NRE_B
        torch.manual_seed(0)
        prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
        theta = prior.sample((6000 if D == 2 else 20000,))
        x = theta + math.sqrt(0.1) * torch.randn_like(theta)
        if kind == "nle":
            tr = NLE(prior, density_estimator="nsf", device="cuda")
            tr.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=60)
        else:
            tr = NRE_B(prior, classifier="resnet", device="cuda")
            tr.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
        _TRAINED[(kind, D)] = tr
    return _TRAINED[(kind, D)]


@pytest.mark.parametrize("D", [2, 10])
@pytest.mark.parametrize("kind", ["nle", "nre"])
@pytest.mark.parametrize("method", ["nuts_pyro", "hmc_pyro"])
@pytest.mark.parametrize("n_iid", [1, 5])
def test_linear_gaussian_posterior(cuda_lib, D, kind, method, n_iid):
    """Prior N(0, 0.1 I), x = theta + N(0, 0.1 I): the posterior is N(x_o / 2, 0.05 I) for one observation and
    N(5 mean(x_o) / 6, I / 60) for 5 iid trials."""
    tr = _trained(kind, D)
    g = torch.Generator().manual_seed(7)
    theta_o = 0.3 * torch.randn(1, D, generator=g)
    x_o = theta_o + math.sqrt(0.1) * torch.randn(n_iid, D, generator=g)
    mean = x_o.mean(0) * (0.5 if n_iid == 1 else 5.0 / 6.0)
    sd = math.sqrt(0.05 if n_iid == 1 else 1.0 / 60.0)
    torch.manual_seed(1)
    post = tr.build_posterior(mcmc_method=method, mcmc_parameters=dict(num_chains=100))
    s = post.sample((4000,), x=x_o).cpu()
    smp = post._posterior_sampler
    assert int(smp.num_divergences.sum()) == 0
    # the bars of the slice-sampler and rejection tests (NLE 0.05 / 0.2, NRE 0.06 / 0.25); at D = 10 the
    # estimators are trained on the same budget for five times the dimensions and their own error grows, so
    # the bars widen by half
    m_bar, s_bar = (0.05, 0.2) if kind == "nle" else (0.06, 0.25)
    if D == 10:
        m_bar, s_bar = 1.5 * m_bar, 1.5 * s_bar
    if D == 10 and n_iid == 5 and kind == "nle":
        # the flow's error in each trial's log-likelihood enters five times; NUTS and HMC both give a posterior sd
        # up to 1.5x the analytic one in one of the ten dimensions on this estimator
        s_bar = 0.6
    assert (s.mean(0) - mean).abs().max() < m_bar, (s.mean(0), mean)
    assert (s.std(0) / sd - 1).abs().max() < s_bar, s.std(0) / sd
    assert smp.step_size.shape == (100,) and smp.inverse_mass_matrix.shape == (100, D)
    assert np.all(smp.mean_accept_prob > 0.3)
    if method == "nuts_pyro":
        assert np.all(smp.mean_tree_depth >= 1)
    assert post._mcmc_init_params.shape == (100, D)
    again = post.sample((200,), x=x_o, init_strategy="latest_sample", warmup_steps=10)
    assert again.shape == (200, D) and torch.isfinite(again).all()


def test_mlp_ratio_gather_gradient_and_nuts(cuda_lib):
    from sbi_b200.potentials import ratio_estimator_based_potential
    from sbi_b200.ratio import build_mlp_classifier
    g = torch.Generator().manual_seed(0)
    Dt, Dx, R, n = 3, 4, 7, 5
    est = build_mlp_classifier(torch.randn(200, Dt, generator=g), torch.randn(200, Dx, generator=g)).cuda()
    th = torch.randn(R, Dt, generator=g).cuda().requires_grad_(True)
    x = torch.randn(n, Dx, generator=g).cuda()
    prior = Independent(Uniform(-4 * torch.ones(Dt), 4 * torch.ones(Dt)), 1)
    pot, tf = ratio_estimator_based_potential(est, prior, x_o=x)
    (g_gather,) = torch.autograd.grad(pot(th).sum(), th)
    # per-pair expression: pair k = (theta[k % R], x[k // R]), every pair its own row
    th2 = th.detach().clone().requires_grad_(True)
    lr = est(th2.repeat(n, 1), x.repeat_interleave(R, dim=0)).reshape(n, R).sum(0)
    (g_pairs,) = torch.autograd.grad((lr + pot.prior.log_prob(th2)).sum(), th2)
    assert torch.allclose(g_gather, g_pairs, rtol=1e-4, atol=1e-5)
    from sbi_b200.posteriors import MCMCPosterior
    post = MCMCPosterior(pot, prior, theta_transform=tf, method="nuts_pyro", num_chains=20, warmup_steps=50)
    s = post.sample((200,), x=x)
    assert s.shape == (200, Dt) and torch.isfinite(s).all()
    assert ((s > -4) & (s < 4)).all()
    assert est.net.flat.requires_grad                       # restored after sampling


class _GaussLik:
    """log q(x | theta) = sum -0.5 ((x - theta) / 0.5)^2 in torch ops (a stand-in likelihood)."""
    input_shape = torch.Size([2])

    def eval(self):
        return self

    def log_prob(self, input, condition):
        return (-0.5 * ((input - condition) / 0.5) ** 2).sum(-1)


def test_box_prior_matches_long_slice_run(cuda_lib):
    from sbi_b200.posteriors import MCMCPosterior
    from sbi_b200.potentials import LikelihoodBasedPotential, mcmc_transform
    prior = Independent(Uniform(-torch.ones(2), torch.ones(2)), 1)
    x_o = torch.tensor([[0.8, -0.3]])
    pot = LikelihoodBasedPotential(_GaussLik(), prior, device="cuda")
    tf = mcmc_transform(pot.prior, device="cuda")
    torch.manual_seed(2)
    nuts = MCMCPosterior(pot, prior, theta_transform=tf, method="nuts_pyro", num_chains=50).sample((5000,), x=x_o)
    assert ((nuts > -1) & (nuts < 1)).all()
    ref = MCMCPosterior(pot, prior, theta_transform=tf, method="slice_np_vectorized", num_chains=200,
                        thin=1).sample((40000,), x=x_o)
    nuts, ref = nuts.cpu().double(), ref.cpu().double()
    assert (nuts.mean(0) - ref.mean(0)).abs().max() < 0.03, (nuts.mean(0), ref.mean(0))
    assert (nuts.std(0) / ref.std(0) - 1).abs().max() < 0.08, (nuts.std(0), ref.std(0))
