"""TSNPE on the GPU: `RestrictedPrior` rejection and SIR sampling against torch restatements of the reference's
loops (rejection.py:230-457, sir.py:13-71) on the same seed and the same prior object, the density thresholder
against its defining expression, and the truncated sequential loop on the linear-Gaussian task against the analytic
posterior."""
import inspect
import math
import warnings

import pytest
import torch
from torch.distributions import Independent, MultivariateNormal, Uniform

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu
D = 3
MARGIN = 1e-5


def _posterior(prior, x_o, seed=0):
    from sbi_b200.posteriors import DirectPosterior
    flow, theta, x = oracle_nsf(D, D, n=2000, seed=seed)
    post = DirectPosterior(b200_from_oracle(flow, theta, x), prior)
    post.set_default_x(x_o)
    return post


def _box():
    return Independent(Uniform(-4 * torch.ones(D), 4 * torch.ones(D)), 1)


def _gauss():
    return MultivariateNormal(torch.zeros(D), 4.0 * torch.eye(D))


def _box_cuda():
    return Independent(Uniform(-4 * torch.ones(D, device="cuda"), 4 * torch.ones(D, device="cuda")), 1)


def _gauss_cuda():
    return MultivariateNormal(torch.zeros(D, device="cuda"), 4.0 * torch.eye(D, device="cuda"))


def _restated_accept_reject(prior, fn, num_samples, max_batch):
    """rejection.py:310-457 for one observation: proposal draws on the prior's own generator (on the prior's
    device), boolean indexing, the float32 acceptance bookkeeping on the CPU and the adaptive batch size."""
    accepted = []
    num_sampled_total = torch.zeros(1)
    num_samples_possible = 0
    num_remaining = num_samples
    batch = min(num_samples, max_batch)
    while num_remaining > 0:
        cand = prior.sample((batch,))
        are_accepted = fn(cand).reshape(batch, 1).cpu()
        accepted.append(cand.reshape(batch, 1, -1)[are_accepted[:, 0].to(cand.device), 0])
        num_accepted = are_accepted.sum(dim=0)
        num_sampled_total += num_accepted
        num_samples_possible += batch
        num_remaining -= num_accepted.min().item()
        rate = (num_sampled_total / num_samples_possible).min().item()
        batch = min(max_batch, max(int(1.5 * num_remaining / max(rate, 1e-12)), 100))
    return torch.cat(accepted)[:num_samples], rate


@pytest.mark.parametrize("make_prior", [_box, _gauss, _box_cuda, _gauss_cuda])
def test_rejection_sampling_equals_reference_loop(cuda_lib, make_prior, capsys, caplog):
    from sbi_b200.restriction import RestrictedPrior, get_density_thresholder
    prior = make_prior()
    x_o = torch.tensor([[0.4, -0.3, 0.2]])
    post = _posterior(prior, x_o)
    torch.manual_seed(0)
    thr = get_density_thresholder(post, quantile=0.5, num_samples_to_estimate_support=20_000)
    rp = RestrictedPrior(prior, thr, device="cuda")
    for n, max_batch in ((2000, 1000), (300, 10_000)):
        torch.manual_seed(5)
        with caplog.at_level("WARNING"):
            got = rp.sample((n,), max_sampling_batch_size=max_batch, save_acceptance_rate=True)
        torch.manual_seed(5)
        want, rate = _restated_accept_reject(prior, thr, n, max_batch)
        assert got.shape == (n, D) and got.device.type == "cuda"
        assert torch.equal(got.cpu(), want.cpu()), (n, max_batch)
        assert torch.equal(rp.acceptance_rate, torch.as_tensor(rate)) and 0 < rate < 0.5
        assert thr(got).all()
        printed = capsys.readouterr().out
        assert f"The `RestrictedPrior` rejected {(1.0 - rate) * 100:.1f}% of prior samples." in printed
        if rate < 0.01:
            assert "Alternatively, consider switching to `sample_with='sir'`." in caplog.text
    # sample_shape and the result device
    rp_cpu = RestrictedPrior(prior, thr)
    s = rp_cpu.sample((4, 5), print_rejected_frac=False)
    assert s.shape == (4, 5, D) and s.device.type == "cpu"
    # prior_acceptance: one rejection run of 10 000, cached
    torch.manual_seed(9)
    a = rp_cpu.prior_acceptance()
    torch.manual_seed(9)
    _, rate = _restated_accept_reject(prior, thr, 10_000, 10_000)
    assert torch.equal(a, torch.as_tensor(rate)) and rp_cpu.prior_acceptance() is a


def test_density_thresholder_equals_sorted_log_prob(cuda_lib):
    from sbi_b200.restriction import get_density_thresholder
    prior = _box()
    post = _posterior(prior, torch.tensor([[0.4, -0.3, 0.2]]))
    post.log_prob(torch.zeros(1, D))            # the leakage factor is estimated once and cached at default_x
    for q, N in ((1e-4, 1_000_000), (0.1, 50_000)):
        torch.manual_seed(3)
        thr = get_density_thresholder(post, quantile=q, num_samples_to_estimate_support=N)
        torch.manual_seed(3)
        s = post.sample((N,))
        want = torch.sort(post.log_prob(s))[0][int(q * N)]
        got = inspect.getclosurevars(thr).nonlocals["log_prob_threshold"]
        assert torch.equal(got, want), q
        theta = 3 * torch.rand(5000, D, device="cuda") - 1.5
        assert torch.equal(thr(theta), post.log_prob(theta) > want)


def test_sir_equals_reference_selection(cuda_lib):
    from sbi_b200.restriction import RestrictedPrior, get_density_thresholder
    prior = _box()
    post = _posterior(prior, torch.tensor([[0.4, -0.3, 0.2]]))
    torch.manual_seed(0)
    thr = get_density_thresholder(post, quantile=0.5, num_samples_to_estimate_support=20_000)
    rp = RestrictedPrior(prior, thr, posterior=post, sample_with="sir", device="cuda")
    n, K = 600, 32
    torch.manual_seed(4)
    got = rp.sample((n,), oversampling_factor=4)     # reaches SIR only through **kwargs: K stays 32
    torch.manual_seed(4)
    th = post.sample((n * K,))
    lw = (thr(th).float() - post.log_prob(th)).reshape(n, K)
    u = torch.rand(n, 1, device="cuda")
    w = torch.softmax(lw, -1).cumsum(-1)
    mask = torch.cumsum(w >= u, -1) == 1
    assert mask.any(-1).all()
    want = th.reshape(n, K, D)[mask]
    near = ((lw.double().softmax(-1).cumsum(-1) - u.double()).abs() <= MARGIN).any(-1)
    assert got.shape == want.shape
    differ = (got != want).any(-1)
    assert not (differ & ~near).any() and int(differ.sum()) <= 2
    with pytest.raises(AssertionError, match="you must provide a `posterior`"):
        RestrictedPrior(prior, thr, sample_with="sir").sample((5,))
    with pytest.raises(ValueError, match=r"Only \[rejection \| sir\]"):
        RestrictedPrior(prior, thr).sample((5,), sample_with="mcmc")


@pytest.mark.parametrize("sample_with", ["rejection", "sir"])
def test_tsnpe_linear_gaussian(cuda_lib, sample_with):
    """TSNPE (the reference's tsnpe_rejection / tsnpe_sir, tests/linearGaussian_snpe_test.py): round 1 from the
    prior, round 2 from the prior truncated to the round-1 posterior's 1 - 1e-4 region, both trained with the
    first-round loss; the final posterior matches the analytic one within the bars of the two-round NPE-C test
    (with `sir`, a wider std bar: see below)."""
    from sbi_b200.inference import NPE
    from sbi_b200.restriction import RestrictedPrior, get_density_thresholder
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    x_o = torch.tensor([[0.6, -0.4, 0.2]])
    sim = lambda th: th + math.sqrt(0.3) * torch.randn_like(th)   # noqa: E731
    inf = NPE(prior, density_estimator="nsf", device="cuda")
    proposal = prior
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for r in range(2):
            theta = proposal.sample((3000,)).cpu().reshape(-1, D)
            x = sim(theta)
            inf.append_simulations(theta, x, proposal=proposal).train(
                training_batch_size=200, max_num_epochs=40 if r == 0 else 25, force_first_round_loss=True)
            posterior = inf.build_posterior().set_default_x(x_o)
            if r == 0:
                accept_reject_fn = get_density_thresholder(posterior, quantile=1e-4)
                proposal = RestrictedPrior(prior, accept_reject_fn, posterior=posterior, sample_with=sample_with)
                round2_theta = None
            else:
                round2_theta = theta
    assert inf._data_round_index == [0, 0] and len(inf.summary["epochs_trained"]) == 2
    inside = accept_reject_fn(round2_theta)
    if sample_with == "rejection":
        assert inside.all()
    else:
        # the reference's SIR potential is accept_reject_fn(theta).float(): its target is exp({0, 1}), so a draw
        # outside the region keeps weight 1 / e of one inside; only tail draws of the posterior fall there
        assert inside.float().mean() > 0.98
    s = posterior.sample((5000,), x=x_o).cpu()
    assert (s.mean(0) - x_o[0] / 1.3).abs().max() < 0.08
    # with `sir` the round-2 draws follow exp({0, 1}) over theta rather than the prior, so the first-round loss
    # widens the posterior towards the likelihood's sqrt(0.3) (ratio 1.14 to the analytic std)
    std_bar = 0.2 if sample_with == "rejection" else 0.35
    assert (s.std(0) / math.sqrt(0.3 / 1.3) - 1).abs().max() < std_bar
