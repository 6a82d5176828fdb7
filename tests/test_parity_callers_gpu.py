"""Parity of the callers around the estimator kernels with the UNMODIFIED reference (imported through
oracle.ref_shim from the copy staged under oracle/_ref): potentials, mcmc_transform /
transformed_potential, the rejection accept set on fixed seeds (BASELINE north_star), gradient
ascent, leakage correction, and BASELINE configs[2] (two-moons NLE + vectorized slice sampling,
c2st against the reference's own posterior samples).

The reference side runs on the CPU in fp32 with estimators built by the reference's builders; the
sbi_b200 side loads the same state_dict and runs on the GPU."""
import math
import os
import warnings

import pytest
import torch
from torch.distributions import Independent, MultivariateNormal, Uniform

from oracle import ref_shim

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")]
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


def _perturb(net, seed=3, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in net.named_parameters():
            s = scale if ("entries" not in n and "diag" not in n) else 0.05
            p.add_(s * torch.randn(p.shape, generator=g))


def _priors(D):
    return {"box": Independent(Uniform(-2 * torch.ones(D), 2 * torch.ones(D)), 1),
            "mvn": MultivariateNormal(0.2 * torch.ones(D), 0.7 * torch.eye(D))}


def _data(D, C, n=800, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = 0.8 * torch.randn(n, D, generator=g)
    x = torch.cat([theta, theta], 1)[:, :C] + 0.5 * torch.randn(n, C, generator=g)
    return theta, x


# -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prior_kind", ["box", "mvn"])
def test_posterior_based_potential_and_transforms(cuda_lib, ref, prior_kind):
    """posterior_based_potential.py:109-191, sbiutils.py:867-984, potentialutils.py:14-48."""
    from sbi.inference.potentials.posterior_based_potential import posterior_estimator_based_potential as ref_pot
    from sbi.neural_nets import posterior_nn as ref_nn
    from sbi.utils.potentialutils import transformed_potential as ref_tp
    from sbi_b200.neural_nets import posterior_nn
    from sbi_b200.potentials import posterior_estimator_based_potential, transformed_potential
    D, C = 3, 4
    theta, x = _data(D, C)
    prior = _priors(D)[prior_kind]
    torch.manual_seed(1)
    r_est = ref_nn("nsf")(theta, x)
    _perturb(r_est)
    est = posterior_nn("nsf")(theta, x)
    est.load_state_dict(r_est.state_dict())
    est = est.cuda()
    x_o = x[5:6]
    rp, rt = ref_pot(r_est, prior, x_o=x_o)
    op, ot = posterior_estimator_based_potential(est, prior, x_o=x_o)
    th = torch.cat([theta[:300], 3.0 * torch.randn(100, D, generator=torch.Generator().manual_seed(2))])
    with torch.no_grad():
        a = rp(th, track_gradients=False)
        b = op(th.cuda(), track_gradients=False).cpu()
    assert torch.equal(torch.isinf(a), torch.isinf(b))           # identical support pattern
    fin = torch.isfinite(a)
    assert fin.sum() > 50 and (a[fin] - b[fin]).abs().max() <= 2e-3
    # the unconstraining transform and the potential in unconstrained space
    inside = th[fin][:200]
    u_ref = rt(inside)
    u_our = ot(inside.cuda()).cpu()
    assert torch.allclose(u_ref, u_our, rtol=1e-5, atol=1e-5)
    assert torch.allclose(rt.inv(u_ref), ot.inv(u_ref.cuda()).cpu(), rtol=1e-5, atol=1e-5)
    assert torch.allclose(rt.log_abs_det_jacobian(inside, u_ref),
                          ot.log_abs_det_jacobian(inside.cuda(), u_ref.cuda()).cpu(), rtol=1e-5, atol=1e-5)
    tp_ref = ref_tp(u_ref, rp, rt, "cpu", track_gradients=False)
    tp_our = transformed_potential(u_ref, op, ot, "cuda", track_gradients=False).cpu()
    assert (tp_ref - tp_our).abs().max() <= 2e-3


@pytest.mark.parametrize("n_iid", [1, 3])
def test_likelihood_and_ratio_potentials(cuda_lib, ref, n_iid):
    """likelihood_based_potential.py:97-130 + :186-239, ratio_based_potential.py:85-160 (iid trials)."""
    from sbi.inference.potentials.likelihood_based_potential import likelihood_estimator_based_potential as ref_lik
    from sbi.inference.potentials.ratio_based_potential import ratio_estimator_based_potential as ref_rat
    from sbi.neural_nets import classifier_nn as ref_cls
    from sbi.neural_nets import likelihood_nn as ref_lnn
    from sbi_b200.neural_nets import likelihood_nn
    from sbi_b200.potentials import likelihood_estimator_based_potential, ratio_estimator_based_potential
    from sbi_b200.ratio import classifier_nn
    D, C = 3, 4
    theta, x = _data(D, C)
    prior = _priors(D)["mvn"]
    x_o = x[7:7 + n_iid]
    th = theta[:400]
    torch.manual_seed(2)
    r_lik = ref_lnn("nsf")(theta, x)
    _perturb(r_lik)
    lik = likelihood_nn("nsf")(theta, x)
    lik.load_state_dict(r_lik.state_dict())
    rp, _ = ref_lik(r_lik, prior, x_o=x_o)
    op, _ = likelihood_estimator_based_potential(lik.cuda(), prior, x_o=x_o)
    with torch.no_grad():
        a, b = rp(th, track_gradients=False), op(th.cuda(), track_gradients=False).cpu()
    assert (a - b).abs().max() <= 2e-3 * n_iid, (a - b).abs().max()
    torch.manual_seed(3)
    r_rat = ref_cls("resnet")(theta, x)
    _perturb(r_rat)
    rat = classifier_nn("resnet")(theta, x)
    rat.load_state_dict(r_rat.state_dict())
    rp, _ = ref_rat(r_rat, prior, x_o=x_o)
    op, _ = ratio_estimator_based_potential(rat.cuda(), prior, x_o=x_o)
    with torch.no_grad():
        a, b = rp(th, track_gradients=False), op(th.cuda(), track_gradients=False).cpu()
    assert (a - b).abs().max() <= 1e-3 * n_iid, (a - b).abs().max()


# -------------------------------------------------------------------------------------------------
def test_rejection_accept_set_identity_1m_proposals(cuda_lib, ref):
    """BASELINE north_star: "identical accepted-index sets for rejection on fixed seeds"; cfg5 size
    (resnet classifier, D = 10, 1 000 000 prior proposals).  Candidates and the uniforms come from
    the CPU generator exactly as rejection.py:170-200 draws them; the reference side evaluates its
    own RatioBasedPotential (CPU fp32), ours the wgmma ratio kernel.  The accept decision is
    exp(potential - log q - log_bound) > u, so a draw can only differ when the two fp32 evaluations
    straddle u: every such flip is reported with its margin, and the margin must be rounding-sized."""
    from sbi.inference.potentials.ratio_based_potential import ratio_estimator_based_potential as ref_rat
    from sbi.neural_nets import classifier_nn as ref_cls
    from sbi_b200 import parallel
    from sbi_b200.potentials import ratio_estimator_based_potential
    from sbi_b200.ratio import classifier_nn
    D, N = 10, 1_000_000
    g = torch.Generator().manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = math.sqrt(0.1) * torch.randn(4000, D, generator=g)
    x = theta + math.sqrt(0.1) * torch.randn(4000, D, generator=g)
    torch.manual_seed(4)
    r_rat = ref_cls("resnet")(theta, x)
    _perturb(r_rat, scale=0.05)
    rat = classifier_nn("resnet")(theta, x)
    rat.load_state_dict(r_rat.state_dict())
    x_o = x[:1]
    rp, _ = ref_rat(r_rat, prior, x_o=x_o)
    op, _ = ratio_estimator_based_potential(rat.cuda(), prior, x_o=x_o)
    chol = torch.linalg.cholesky(prior.covariance_matrix)

    def proposal_sample(n, gen):
        return prior.loc + torch.randn(n, D, generator=gen) @ chol.T

    seed = 1234
    gg = torch.Generator().manual_seed(seed)
    cands = proposal_sample(N, gg)
    u = torch.rand(N, generator=gg)
    with torch.no_grad():
        lr_ref = torch.cat([rp(c, track_gradients=False) - prior.log_prob(c) for c in cands.split(1 << 17)])
    log_bound = float(lr_ref.max()) + math.log(1.2)          # max log ratio + log m (rejection.py:150-160)
    ratio_ref = torch.exp(lr_ref - log_bound)
    acc_ref = torch.nonzero(ratio_ref > u).reshape(-1)
    prior_gpu = MultivariateNormal(prior.loc.cuda(), prior.covariance_matrix.cuda())
    rows, idx = parallel.rejection_fixed_budget(
        lambda t: op(t, track_gradients=False), proposal_sample, prior_gpu.log_prob, log_bound, N, seed, device="cuda")
    idx = idx.cpu()
    assert rat.TC_MIN_ROWS <= N                                  # the tensor-core kernel evaluated them
    assert torch.equal(rows.cpu(), cands[idx])                   # rows travel with their global index
    a, b = set(acc_ref.tolist()), set(idx.tolist())
    flips = sorted(a ^ b)
    margins = [(i, float(ratio_ref[i] - u[i]) / max(float(u[i]), 1e-30)) for i in flips]
    print(f"rejection accept set: reference {len(a)} accepted, sm_90a {len(b)}, flips {len(flips)}: {margins[:20]}")
    assert len(a) > 1000
    # identical sets up to draws whose acceptance ratio equals u within fp32 rounding of the logit
    assert len(flips) <= max(3, int(2e-5 * N)), margins
    assert all(abs(m) < 1e-4 for _, m in margins), margins
    # determinism: the same call returns the same set, bit for bit
    rows2, idx2 = parallel.rejection_fixed_budget(
        lambda t: op(t, track_gradients=False), proposal_sample, prior_gpu.log_prob, log_bound, N, seed, device="cuda")
    assert torch.equal(idx2.cpu(), idx) and torch.equal(rows2, rows)


# -------------------------------------------------------------------------------------------------
def test_gradient_ascent_matches_reference(cuda_lib, ref):
    """sbiutils.py:1160-1285 on the posterior-based potential: same inits, same Adam -> same MAP."""
    from sbi.inference.potentials.posterior_based_potential import posterior_estimator_based_potential as ref_pot
    from sbi.neural_nets import posterior_nn as ref_nn
    from sbi.utils.sbiutils import gradient_ascent as ref_ga
    from sbi_b200.neural_nets import posterior_nn
    from sbi_b200.potentials import posterior_estimator_based_potential
    from sbi_b200.samplers import gradient_ascent
    D, C = 2, 3
    theta, x = _data(D, C)
    prior = _priors(D)["box"]
    torch.manual_seed(5)
    r_est = ref_nn("nsf")(theta, x)
    _perturb(r_est, scale=0.05)
    est = posterior_nn("nsf")(theta, x)
    est.load_state_dict(r_est.state_dict())
    x_o = x[3:4]
    rp, rt = ref_pot(r_est, prior, x_o=x_o)
    op, ot = posterior_estimator_based_potential(est.cuda(), prior, x_o=x_o)
    inits = prior.sample((300,))
    th_r, v_r = ref_ga(rp, inits, theta_transform=rt, num_iter=60, num_to_optimize=20, learning_rate=0.05,
                       show_progress_bars=False)
    th_o, v_o = gradient_ascent(op, inits.cuda(), theta_transform=ot, num_iter=60, num_to_optimize=20,
                                learning_rate=0.05)
    assert abs(float(v_r) - float(v_o)) < 5e-3, (v_r, v_o)
    assert (th_r.reshape(-1) - th_o.cpu().reshape(-1)).abs().max() < 2e-2, (th_r, th_o)


def test_leakage_correction_matches_reference(cuda_lib, ref):
    """direct_posterior.py:467-523: acceptance rate of posterior draws inside a prior box that cuts
    the posterior; ours vs the reference's DirectPosterior on the SAME weights (both Monte Carlo)."""
    from sbi.inference.posteriors import DirectPosterior as RefDirect
    from sbi.neural_nets import posterior_nn as ref_nn
    from sbi_b200.neural_nets import posterior_nn
    from sbi_b200.posteriors import DirectPosterior
    D, C = 2, 2
    theta, x = _data(D, C)
    prior = Independent(Uniform(-0.6 * torch.ones(D), 0.9 * torch.ones(D)), 1)
    torch.manual_seed(6)
    r_est = ref_nn("nsf")(theta, x)
    est = posterior_nn("nsf")(theta, x)
    est.load_state_dict(r_est.state_dict())
    x_o = x[9:10]
    n = 20_000
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a = float(RefDirect(r_est, prior).leakage_correction(x_o, num_rejection_samples=n, show_progress_bars=False))
        b = float(DirectPosterior(est.cuda(), prior, device="cuda").leakage_correction(x_o.cuda(), num_rejection_samples=n))
    sigma = math.sqrt(max(a * (1 - a), 1e-4) / n)
    print(f"leakage correction: reference {a:.4f}, sm_90a {b:.4f} (sigma {sigma:.4f})")
    assert 0.02 < a < 0.98 and abs(a - b) < 6 * sigma + 2e-3, (a, b)
    # and the normalised log-prob uses it: log q - log(acceptance)  (direct_posterior.py:370-386)
    th = theta[:50]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        post = DirectPosterior(est, prior, device="cuda")
        lp_n = post.log_prob(th.cuda(), x=x_o.cuda(), norm_posterior=True)
        lp_u = post.log_prob(th.cuda(), x=x_o.cuda(), norm_posterior=False)
    fin = torch.isfinite(lp_u)
    assert fin.any() and ((lp_n - lp_u)[fin] + math.log(b)).abs().max() < 0.05


# -------------------------------------------------------------------------------------------------
def test_cfg3_two_moons_nle_slice_c2st(cuda_lib):
    """BASELINE configs[2]: two-moons, likelihood_nn='nsf' on 50k simulations, slice_np_vectorized with
    1000 chains, c2st against the reference's posterior samples for observation 1
    (/root/reference/tests/mini_sbibm/files/two_moons/samples_1.pt, copied to tests/golden/two_moons)."""
    from sbi_b200.inference import NLE
    from tests.helpers import c2st, two_moons_simulator
    torch.manual_seed(0)
    prior = Independent(Uniform(-torch.ones(2), torch.ones(2)), 1)
    theta = prior.sample((50_000,))
    x = two_moons_simulator(theta)
    x_o = torch.load(os.path.join(GOLD, "two_moons", "x_o_1.pt")).reshape(1, 2).float()
    ref_samples = torch.load(os.path.join(GOLD, "two_moons", "samples_1.pt")).float()
    nle = NLE(prior, density_estimator="nsf", device="cuda")
    nle.append_simulations(theta, x).train(training_batch_size=1000, max_num_epochs=150)
    post = nle.build_posterior(mcmc_method="slice_np_vectorized",
                               mcmc_parameters=dict(num_chains=1000, warmup_steps=200, thin=1))
    s = post.sample((10_000,), x=x_o).cpu()
    assert s.shape == (10_000, 2) and torch.isfinite(s).all()
    score = c2st(ref_samples[:10_000], s)
    print(f"two-moons NLE-nsf / slice_np_vectorized: c2st = {score:.3f} ({nle.summary['epochs_trained'][-1]} epochs)")
    assert score < 0.65, score
