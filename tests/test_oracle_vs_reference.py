"""Cross-check of oracle.sbi_port against the UNMODIFIED reference sbi (imported through
oracle.ref_shim).  Skipped where no copy of the reference was staged (oracle/_ref)."""
import warnings

import pytest
import torch

from oracle import ref_shim, sbi_port

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi (oracle/_ref)")


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


@pytest.mark.parametrize("D,C", [(10, 10), (3, 2), (2, 5)])
def test_build_nsf_matches_reference(ref, D, C):
    from sbi.neural_nets import likelihood_nn, posterior_nn
    theta, x = torch.randn(300, D), torch.randn(300, C)
    torch.manual_seed(5)
    a = posterior_nn("nsf")(theta, x)
    torch.manual_seed(5)
    b = sbi_port.build_nsf(theta, x)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    with torch.no_grad():
        assert torch.equal(a.log_prob(theta[:50], x[:50]), b.log_prob(theta[:50], x[:50]))
        assert torch.equal(a.loss(theta[:50], x[:50]), b.loss(theta[:50], x[:50]))
    # NLE swaps the roles (factory.py:316-318)
    torch.manual_seed(6)
    c = likelihood_nn("nsf")(theta, x) if C > 1 else None
    if c is not None:
        torch.manual_seed(6)
        d = sbi_port.build_nsf(x, theta)
        for k in c.state_dict():
            assert torch.equal(c.state_dict()[k], d.state_dict()[k]), k


def test_reference_npe_runs_end_to_end_on_the_port(ref):
    """The reference's own NPE.train / build_posterior / sample / log_prob execute unmodified."""
    from sbi.inference import NPE
    from sbi.neural_nets import posterior_nn
    from torch.distributions import MultivariateNormal
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(3), 0.1 * torch.eye(3))
    theta = prior.sample((600,))
    x = theta + (0.1 ** 0.5) * torch.randn_like(theta)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NPE(prior, density_estimator=posterior_nn("nsf"), show_progress_bars=False)
        inf.append_simulations(theta, x).train(training_batch_size=100, max_num_epochs=2)
        post = inf.build_posterior()
        s = post.sample((50,), x=x[:1], show_progress_bars=False)
        lp = post.log_prob(s, x=x[:1])
    assert s.shape == (50, 3) and torch.isfinite(lp).all()


@pytest.mark.parametrize("D,C", [(3, 2), (5, 4)])
def test_build_maf_matches_reference(ref, D, C):
    """posterior_nn("maf") of the unmodified reference (flow.py:115-209) vs the port: same state dict
    (incl. the random permutations drawn from the global generator) and identical log-probs."""
    from sbi.neural_nets import posterior_nn
    theta, x = torch.randn(300, D), torch.randn(300, C)
    torch.manual_seed(7)
    a = posterior_nn("maf")(theta, x)
    torch.manual_seed(7)
    b = sbi_port.build_maf(theta, x)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    with torch.no_grad():
        assert torch.equal(a.log_prob(theta[:40], x[:40]), b.log_prob(theta[:40], x[:40]))


def test_resnet_classifier_matches_reference(ref):
    """classifier_nn("resnet") (classifier.py:172-235) vs the port: same parameters from the same
    seed, identical logits; NRE-B loss of the port against the reference trainer's `_loss`."""
    from sbi.neural_nets import classifier_nn
    theta, x = torch.randn(400, 4), torch.randn(400, 6)
    torch.manual_seed(8)
    a = classifier_nn("resnet")(theta, x)
    torch.manual_seed(8)
    b = sbi_port.build_resnet_classifier(theta, x)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    with torch.no_grad():
        assert torch.equal(a(theta[:64], x[:64]), b(theta[:64], x[:64]))


def test_flow_matching_estimator_matches_reference(ref):
    """posterior_flow_nn("mlp") (factory.py:531-620, vector_field_nets.py:610-719,
    flowmatching_estimator.py:205-347) vs the port: same state dict, identical velocity field, and
    the same loss when t and theta_1 come from the same generator state."""
    from sbi.neural_nets import posterior_flow_nn
    theta, x = torch.randn(500, 5) * 0.7 + 0.2, torch.randn(500, 3)
    torch.manual_seed(9)
    a = posterior_flow_nn("mlp")(theta, x)
    torch.manual_seed(9)
    b = sbi_port.build_flow_matching_estimator(theta, x)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) == set(sb), set(sa) ^ set(sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    t = torch.rand(32)
    with torch.no_grad():
        va = a(theta[:32], x[:32], t)
        vb = b(theta[:32], x[:32], t)
        assert torch.allclose(va, vb, atol=1e-6, rtol=1e-5)
        torch.manual_seed(11)
        la = a.loss(theta[:64], x[:64])
        torch.manual_seed(11)
        lb = b.loss(theta[:64], x[:64])
        assert torch.allclose(la, lb, atol=1e-6, rtol=1e-5)


@pytest.mark.parametrize("model,D", [("made", 2), ("maf_rqs", 2), ("nsf", 1)])
def test_reference_builders_not_yet_on_the_gpu_run_on_the_port(ref, model, D):
    """The reference's `made` (MADE-MoG), `maf_rqs` and 1-D `nsf` (ContextSplineMap) builders — not
    built as kernels yet (DESIGN §8) — already run on the nflows port: finite log-probs, samples of
    the right shape, and a density that integrates to one at a fixed condition (trapezoid rule).
    This pins the port's MADEMoG / autoregressive-spline / 1-D coupling pieces for the next round."""
    from sbi.neural_nets import posterior_nn
    torch.manual_seed(0)
    C = 3
    theta, x = torch.randn(500, D) * 0.8 + 0.1, torch.randn(500, C)
    est = posterior_nn(model)(theta, x)
    with torch.no_grad():
        for p in est.parameters():
            p.add_(0.05 * torch.randn_like(p))
        lp = est.log_prob(theta[:8], x[:8])
        s = est.sample((5,), x[:2])
        assert lp.shape == (1, 8) and torch.isfinite(lp).all() and s.shape == (5, 2, D)
        if D == 1:
            g = torch.linspace(-12, 12, 20001)[:, None]
            dens = est.log_prob(g.unsqueeze(1), x[:1]).exp()[:, 0]
            integ = torch.trapz(dens, g[:, 0]).item()
        else:
            a = torch.linspace(-10, 10, 601)
            gx, gy = torch.meshgrid(a, a, indexing="ij")
            pts = torch.stack([gx.reshape(-1), gy.reshape(-1)], 1)
            dens = est.log_prob(pts.unsqueeze(1), x[:1]).exp()[:, 0].reshape(601, 601)
            integ = torch.trapz(torch.trapz(dens, a), a).item()
    assert abs(integ - 1.0) < 2e-3, integ
