"""The estimators bind to the UNMODIFIED reference's ABCs (trainers/base.py:690,985,999 gates) and
refuse CPU compute.  Runs wherever build() staged a copy of the reference
(oracle/_ref)."""
import pytest
import torch

from oracle import ref_shim

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


def _data(D=3, n=400):
    torch.manual_seed(0)
    theta = torch.randn(n, D)
    return theta, theta + 0.3 * torch.randn(n, D)


def test_estimators_are_virtual_subclasses_of_the_reference_abcs(ref):
    from sbi.neural_nets.estimators.base import (ConditionalDensityEstimator, ConditionalEstimator,
                                                 ConditionalVectorFieldEstimator)
    from sbi.neural_nets.ratio_estimators import RatioEstimator as RefRatio
    from sbi_b200.flowmatching import posterior_flow_nn
    from sbi_b200.neural_nets import likelihood_nn, posterior_nn
    from sbi_b200.ratio import classifier_nn
    theta, x = _data()
    for build in (posterior_nn("nsf"), posterior_nn("maf"), likelihood_nn("nsf")):
        est = build(theta, x)
        assert isinstance(est, ConditionalDensityEstimator) and isinstance(est, ConditionalEstimator)
    assert isinstance(classifier_nn("resnet")(theta, x), RefRatio)
    assert isinstance(classifier_nn("resnet")(theta, x), ConditionalEstimator)
    assert isinstance(posterior_flow_nn("mlp")(theta, x), ConditionalVectorFieldEstimator)


def test_reference_trainers_accept_the_build_functions(ref):
    """Constructor + append_simulations + the estimator gate of the reference (no compute)."""
    from sbi.inference import FMPE, NLE, NPE, NRE_B
    from torch.distributions import MultivariateNormal
    from sbi_b200.flowmatching import posterior_flow_nn
    from sbi_b200.neural_nets import likelihood_nn, posterior_nn
    from sbi_b200.ratio import classifier_nn
    theta, x = _data()
    prior = MultivariateNormal(torch.zeros(3), torch.eye(3))
    npe = NPE(prior, density_estimator=posterior_nn("nsf"), show_progress_bars=False).append_simulations(theta, x)
    NLE(prior, density_estimator=likelihood_nn("nsf"), show_progress_bars=False).append_simulations(theta, x)
    NRE_B(prior, classifier=classifier_nn("resnet"), show_progress_bars=False).append_simulations(theta, x)
    FMPE(prior, vf_estimator=posterior_flow_nn("mlp"), show_progress_bars=False).append_simulations(theta, x)
    est = posterior_nn("nsf")(theta, x)
    got, device = npe._resolve_estimator(est)     # trainers/base.py:690
    assert got is est and device == "cpu"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU error path")
def test_cpu_probe_without_a_device_raises(ref):
    from sbi_b200.neural_nets import posterior_nn
    theta, x = _data()
    est = posterior_nn("nsf")(theta, x)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        est.log_prob(theta[None, :2], condition=x[:2])
