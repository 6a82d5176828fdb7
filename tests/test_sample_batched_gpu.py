"""`sample_batched` of the MCMC and vector-field posteriors on the device: the paired (`x_is_iid=False`) NLE / NRE
potentials against per-observation evaluation, chain / observation order, accuracy against the analytic posterior of
a linear-Gaussian task, prior support, and SBC / TARP taking the batched path."""
import math
import warnings

import pytest
import torch
from torch.distributions import Independent, MultivariateNormal, Normal, Uniform

from tests.helpers import c2st

pytestmark = pytest.mark.gpu

D, SIG, PRIOR_SD = 2, 0.5, 3.0
SHRINK = PRIOR_SD ** 2 / (PRIOR_SD ** 2 + SIG ** 2)           # posterior mean = SHRINK * x
POST_SD = math.sqrt(SIG ** 2 * SHRINK)
MCMC = dict(num_chains=20, warmup_steps=100, thin=5)


@pytest.fixture(scope="module")
def task():
    """prior N(0, 9 I), x = theta + 0.5 eps  ->  posterior N(x * 9 / 9.25, 0.25 * 9 / 9.25 I): x_o = +-5 is inside
    the simulated data."""
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), PRIOR_SD ** 2 * torch.eye(D))
    theta = prior.sample((8000,))
    return prior, theta, theta + SIG * torch.randn_like(theta)


def _train(inf, theta, x, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est = inf.append_simulations(theta, x).train(**kw)
    return inf, est


@pytest.fixture(scope="module")
def nle_nsf(cuda_lib, task):
    from sbi_b200.inference import NLE
    prior, theta, x = task
    torch.manual_seed(1)                   # MCMC on the learnt likelihood reaches the tails: train it to convergence
    th = prior.sample((20_000,))
    return _train(NLE(prior, density_estimator="nsf", device="cuda"), th, th + SIG * torch.randn_like(th),
                  training_batch_size=500, max_num_epochs=200)


@pytest.fixture(scope="module")
def nre_resnet(cuda_lib, task):
    from sbi_b200.inference import NRE_B
    prior, theta, x = task
    return _train(NRE_B(prior, classifier="resnet", device="cuda"), theta, x, training_batch_size=500,
                  max_num_epochs=40)


@pytest.fixture(scope="module")
def fmpe(cuda_lib, task):
    from sbi_b200.inference import FMPE
    prior, theta, x = task
    return _train(FMPE(prior, device="cuda"), theta, x, training_batch_size=500, max_num_epochs=80)


@pytest.fixture(scope="module")
def npse_ve(cuda_lib, task):
    from sbi_b200.inference import NPSE
    prior, theta, x = task
    return _train(NPSE(prior, sde_type="ve", device="cuda"), theta, x, training_batch_size=500, learning_rate=2e-3,
                  max_num_epochs=150, stop_after_epochs=150)


def _estimator(request, task, kind, model):
    fixture = {("nle", "nsf"): "nle_nsf", ("nre", "resnet"): "nre_resnet"}.get((kind, model))
    if fixture is not None:
        return request.getfixturevalue(fixture)[1]
    from sbi_b200.inference import NLE, NRE_B
    prior, theta, x = task
    inf = NLE(prior, density_estimator=model, device="cuda") if kind == "nle" else \
        NRE_B(prior, classifier=model, device="cuda")
    return _train(inf, theta[:2000], x[:2000], training_batch_size=200, max_num_epochs=3)[1]


def _potential(kind, est):
    from sbi_b200.potentials import likelihood_estimator_based_potential, ratio_estimator_based_potential
    # element-wise prior: its log_prob is the same number for a row whatever the batch around it
    prior = Independent(Normal(torch.zeros(D), PRIOR_SD * torch.ones(D)), 1)
    make = likelihood_estimator_based_potential if kind == "nle" else ratio_estimator_based_potential
    return make(est, prior)[0]


def _per_observation(pot, theta, xs):
    out = []
    for r in range(theta.shape[0]):
        pot.set_x(xs[r:r + 1])
        out.append(pot(theta[r:r + 1], track_gradients=False).reshape(-1))
    return torch.cat(out)


def _pairs(n, seed):
    g = torch.Generator().manual_seed(seed)
    th = PRIOR_SD * torch.randn(n, D, generator=g)
    return th.cuda(), (th + SIG * torch.randn(n, D, generator=g)).cuda()


@pytest.mark.parametrize("kind,model", [("nle", "nsf"), ("nle", "maf"), ("nre", "resnet"), ("nre", "mlp")])
def test_paired_potential_equals_per_observation_potential(request, task, kind, model):
    est = _estimator(request, task, kind, model)
    pot = _potential(kind, est)
    th, xs = _pairs(64, 5)
    with torch.no_grad():
        pot.set_x(xs, x_is_iid=False)
        got = pot(th, track_gradients=False)
        assert got.shape == (64,) and torch.isfinite(got).all()
        assert torch.equal(got, _per_observation(pot, th, xs))          # both launches on the SIMT kernel
        # the iid path is unchanged: the sum over trials of the one-observation expression
        xi = xs[:5]
        pot.set_x(xi)
        got_iid = pot(th, track_gradients=False)
        if kind == "nle":
            want = est.log_prob(xi.unsqueeze(1).expand(-1, 64, D), condition=th).sum(0)
        else:
            want = est(th.repeat(5, 1), xi.repeat_interleave(64, dim=0)).reshape(5, -1).sum(0)
        assert torch.equal(got_iid, want + pot.prior.log_prob(th))
        pot.set_x(xs[:10], x_is_iid=False)
        with pytest.raises(AssertionError, match="Batch size mismatch"):
            pot(th[:9], track_gradients=False)


@pytest.mark.parametrize("kind,model,rows", [("nle", "nsf", 2048), ("nre", "resnet", 32768)])
def test_paired_potential_across_the_tensor_core_switch(request, task, kind, model, rows):
    """Batched rows on the wgmma kernel, single rows on the SIMT kernel."""
    est = _estimator(request, task, kind, model)
    assert est._tc_state(est._model(nbuf=2)) is not None
    pot = _potential(kind, est)
    th, xs = _pairs(rows, 6)
    with torch.no_grad():
        pot.set_x(xs, x_is_iid=False)
        got = pot(th, track_gradients=False)
        pick = torch.arange(0, rows, rows // 48, device="cuda")
        want = _per_observation(pot, th[pick], xs[pick])
    assert (got[pick] - want).abs().max() <= 2e-3 * max(1.0, want.abs().max().item())


def test_chains_stay_with_their_observation(nle_nsf):
    inf, _ = nle_nsf
    post = inf.build_posterior(mcmc_parameters=MCMC)
    xo = torch.tensor([[-5.0, -5.0], [0.0, 0.0], [5.0, 5.0]])
    s = post.sample_batched((600,), x=xo, show_progress_bars=False).cpu()
    assert s.shape == (600, 3, D)
    for b in range(3):
        assert (s[:, b].mean(0) - SHRINK * xo[b]).abs().max() < 0.2, (b, s[:, b].mean(0), s[:, b].std(0))
    # every init strategy, then the stored chain states of the last call
    for how in ("proposal", "sir", "resample"):
        s = post.sample_batched((40,), x=xo, init_strategy=how, warmup_steps=20, show_progress_bars=False)
        assert s.shape == (40, 3, D) and torch.isfinite(s).all()
    assert post._mcmc_init_params.shape == (3 * MCMC["num_chains"], D)
    s = post.sample_batched((40,), x=xo, init_strategy="latest_sample", warmup_steps=0, show_progress_bars=False)
    assert s.shape == (40, 3, D)
    with pytest.raises(ValueError, match="latest_sample"):
        post.sample_batched((40,), x=xo[:2], init_strategy="latest_sample", show_progress_bars=False)
    with pytest.warns(UserWarning, match="larger than the number of requested samples"):
        s = post.sample_batched((5,), x=xo[:2], num_chains=8, warmup_steps=10, show_progress_bars=False)
    assert s.shape == (5, 2, D)
    assert post._mcmc_init_params.shape == (2 * 5, D)


def _xs10():
    g = torch.Generator().manual_seed(11)
    th = PRIOR_SD * torch.randn(10, D, generator=g)
    return th + SIG * torch.randn(10, D, generator=g)


def _posterior(request, which):
    if which in ("nle", "nre"):
        inf = request.getfixturevalue("nle_nsf" if which == "nle" else "nre_resnet")[0]
        return inf.build_posterior(mcmc_parameters=MCMC)
    if which == "npse_sde":
        return request.getfixturevalue("npse_ve")[0].build_posterior(sample_with="sde")
    return request.getfixturevalue("fmpe")[0].build_posterior(sample_with=which.split("_")[1])


@pytest.mark.parametrize("which", ["nle", "nre", "fmpe_ode", "fmpe_sde", "npse_sde"])
def test_batched_posteriors_match_the_analytic_posterior(request, which):
    post = _posterior(request, which)
    xs = _xs10()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        s = post.sample_batched((1000,), x=xs, show_progress_bars=False).cpu()
    assert s.shape == (1000, 10, D) and torch.isfinite(s).all()
    err = (s.mean(0) - SHRINK * xs).abs().max().item()
    rel = (s.std(0) / POST_SD - 1).abs().max().item()
    print(which, "max mean err", err, "max std rel err", rel, "per observation:",
          (s.mean(0) - SHRINK * xs).abs().amax(1).tolist(), (s.std(0) / POST_SD - 1).abs().amax(1).tolist())
    if which in ("nle", "nre"):                        # against one `sample()` run per observation
        accs = [c2st(s[:, b], post.sample((1000,), x=xs[b:b + 1]).cpu()) for b in range(10)]
        print(which, "c2st batched vs per-observation", accs)
        assert max(accs) <= 0.6
    assert err < 0.16 and rel < 0.35                   # the tolerances of tests/test_score_gpu.py


@pytest.mark.parametrize("which", ["nle", "fmpe_ode"])
def test_sbc_and_tarp_sample_every_observation_in_one_call(request, task, which, recwarn):
    from scipy.stats import kstest
    from sbi_b200.diagnostics import run_sbc, run_tarp
    post = _posterior(request, which)
    prior = task[0]
    torch.manual_seed(7)
    N, S = 200, 200
    th = prior.sample((N,))
    xs = th + SIG * torch.randn_like(th)
    ranks, dap = run_sbc(th, xs, post, num_posterior_samples=S)
    assert ranks.shape == (N, D) and dap.shape == (N, D)
    for d in range(D):
        p = kstest(ranks[:, d].cpu().numpy(), "uniform", args=(0, S))[1]
        assert p > 0.01, (d, p)
    ecp, alpha = run_tarp(th, xs, post, num_posterior_samples=S)
    assert torch.isfinite(ecp).all() and ecp.shape == alpha.shape
    assert not [w for w in recwarn if "Falling back" in str(w.message)]


def test_batched_draws_lie_inside_a_box_prior(fmpe, nle_nsf):
    box = Independent(Uniform(-torch.ones(D), torch.ones(D)), 1)
    xo = torch.tensor([[-1.5, -1.5], [0.0, 0.0], [1.0, -0.5]])
    posts = [fmpe[0].build_posterior(prior=box, sample_with=how) for how in ("ode", "sde")]
    posts.append(nle_nsf[0].build_posterior(prior=box, mcmc_parameters=MCMC))
    for post in posts:
        s = post.sample_batched((400,), x=xo, show_progress_bars=False).cpu()
        assert s.shape == (400, 3, D)
        assert ((s > -1) & (s < 1)).all()
