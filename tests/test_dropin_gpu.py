"""Drop-in at the estimator boundary: the UNMODIFIED reference trainers / posteriors
(`sbi.inference.NPE / NLE / NRE_B / FMPE`, from the copy staged under oracle/_ref) run end to end on
estimators built by sbi_b200's build functions -- the reference's DataLoader loop, Adam, clipping,
convergence check, `build_posterior`, `sample`, `log_prob`, with every estimator call going through
the sm_90a kernels.  Acceptance: the analytic linear-Gaussian posterior (as
tests/linearGaussian_snpe_test.py:53-152 does with c2st; here mean / std bars)."""
import math
import warnings

import pytest
import torch

from oracle import ref_shim

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")]


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


def _task(D=3, n=4000, device="cuda"):
    from torch.distributions import MultivariateNormal
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D, device=device), 0.1 * torch.eye(D, device=device))
    theta = prior.sample((n,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    x_o = torch.tensor([[0.3, -0.2, 0.1][:D]], device=device)
    return prior, theta, x, x_o


def _check(samples, x_o, tol_mean=0.06, tol_std=0.25):
    s = samples.cpu()
    assert (s.mean(0) - x_o.cpu()[0] / 2).abs().max() < tol_mean, s.mean(0)
    assert (s.std(0) / math.sqrt(0.05) - 1).abs().max() < tol_std, s.std(0)


def test_reference_npe_on_b200_nsf(cuda_lib, ref):
    from sbi.inference import NPE
    from sbi.inference.posteriors import DirectPosterior
    from sbi.neural_nets.estimators.base import ConditionalDensityEstimator
    from sbi_b200.estimators import FlowEstimator
    from sbi_b200.neural_nets import posterior_nn
    prior, theta, x, x_o = _task()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NPE(prior, density_estimator=posterior_nn("nsf"), device="cuda", show_progress_bars=False)
        est = inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
        assert isinstance(est, FlowEstimator) and isinstance(est, ConditionalDensityEstimator)
        assert est.flat.is_cuda
        post = inf.build_posterior()
        assert isinstance(post, DirectPosterior)
        s = post.sample((3000,), x=x_o, show_progress_bars=False)
        lp = post.log_prob(s[:200], x=x_o)
    assert torch.isfinite(lp).all()
    _check(s, x_o)
    # the log-probs are the analytic posterior's up to the fit error
    from torch.distributions import MultivariateNormal
    true = MultivariateNormal(x_o[0] / 2, 0.05 * torch.eye(3, device="cuda")).log_prob(s[:200])
    assert (lp - true).abs().mean() < 0.5


def test_reference_nle_mcmc_on_b200_nsf(cuda_lib, ref):
    from sbi.inference import NLE
    from sbi_b200.neural_nets import likelihood_nn
    prior, theta, x, x_o = _task(D=2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NLE(prior, density_estimator=likelihood_nn("nsf"), device="cuda", show_progress_bars=False)
        inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
        post = inf.build_posterior(sample_with="mcmc", mcmc_method="slice_np_vectorized",
                                   mcmc_parameters=dict(num_chains=50, warmup_steps=30, thin=2))
        s = post.sample((1000,), x=x_o, show_progress_bars=False)
    _check(s, x_o, tol_mean=0.08, tol_std=0.3)


def test_reference_nre_b_rejection_on_b200_resnet(cuda_lib, ref):
    from sbi.inference import NRE_B
    from sbi_b200.ratio import classifier_nn
    prior, theta, x, x_o = _task(D=2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NRE_B(prior, classifier=classifier_nn("resnet"), device="cuda", show_progress_bars=False)
        inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=30)
        post = inf.build_posterior(sample_with="rejection")
        s = post.sample((1000,), x=x_o, show_progress_bars=False)
    _check(s, x_o, tol_mean=0.08, tol_std=0.3)


def test_reference_fmpe_on_b200_mlp(cuda_lib, ref):
    """The reference's FMPE trainer (base_vf_inference.py:206-350) on the sm_90a flow-matching
    estimator.  The reference's VectorFieldPosterior needs zuko's ODE solver at construction (absent
    offline), so the trained estimator is sampled through sbi_b200's posterior (SDE and ODE)."""
    from sbi.inference import FMPE
    from sbi.neural_nets.estimators.base import ConditionalVectorFieldEstimator
    from sbi_b200.flowmatching import posterior_flow_nn
    from sbi_b200.posteriors import VectorFieldPosterior
    prior, theta, x, x_o = _task(D=2, n=6000)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = FMPE(prior, vf_estimator=posterior_flow_nn("mlp"), device="cuda", show_progress_bars=False)
        est = inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=60)
    assert isinstance(est, ConditionalVectorFieldEstimator) and est.flat.is_cuda
    tl = inf.summary["training_loss"]
    assert tl[-1] < tl[0]
    for how in ("sde", "ode"):
        s = VectorFieldPosterior(est, prior, device="cuda", sample_with=how).sample((1000,), x=x_o)
        _check(s, x_o, tol_mean=0.1, tol_std=0.35)
