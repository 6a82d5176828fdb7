"""Score estimators of sbi_b200/score.py (NPSE, SURVEY 8f-3) against the UNMODIFIED reference classes on the CPU
(through oracle.ref_shim).  Everything around the network is element-wise torch arithmetic that runs unchanged on
the device; the network call itself (the sm_90a kernel) is replaced by the reference's own `VectorFieldMLP` with
the same weights, so forward / loss / schedules / SDE coefficients must agree exactly, and the divergence algebra
of `ode_fn_and_divergence` is checked against an autograd trace.  (GPU side: tests/test_score_gpu.py.)"""
import warnings

import pytest
import torch

from oracle import ref_shim

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")

D, C = 3, 4


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


def _data(n=400, seed=0):
    g = torch.Generator().manual_seed(seed)
    theta = 0.8 * torch.randn(n, D, generator=g) + 0.3
    x = torch.cat([theta, theta], 1)[:, :C] + 0.5 * torch.randn(n, C, generator=g)
    return theta, x


def _pair(sde_type, seed=3, **kw):
    """(reference estimator, ours with the network call routed to the reference's network)."""
    from sbi.neural_nets import posterior_score_nn as ref_build
    from sbi_b200.score import posterior_score_nn
    theta, x = _data()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.manual_seed(seed)
        a = ref_build(sde_type=sde_type, hidden_features=32, num_layers=2, **kw)(theta, x)
        torch.manual_seed(seed)
        b = posterior_score_nn(sde_type=sde_type, hidden_features=32, num_layers=2, **kw)(theta, x)
    b._net_call = lambda enc, cond, tenc: a.net(enc, a._embedding_net(cond).expand(enc.shape[0], -1), tenc)
    return a, b, theta, x


@pytest.mark.parametrize("sde_type", ["ve", "vp", "subvp"])
def test_builder_state_matches_reference(ref, sde_type):
    a, b, _, _ = _pair(sde_type)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) == set(sb), set(sa) ^ set(sb)
    for k in sa:
        assert sa[k].shape == sb[k].shape and torch.equal(sa[k], sb[k]), k
    assert (a.t_min, a.t_max) == (b.t_min, b.t_max)
    assert type(a).__name__ == type(b).__name__
    b.load_state_dict(sa)                       # a reference checkpoint loads


@pytest.mark.parametrize("sde_type", ["ve", "vp", "subvp"])
def test_forward_loss_and_sde_terms_equal_reference(ref, sde_type):
    a, b, theta, x = _pair(sde_type)
    with torch.no_grad():                       # the builder zero-initialises the output layer: make it count
        a.net.output_layer.weight.normal_(0, 0.3)
    t = torch.rand(32) * (a.t_max - a.t_min) + a.t_min
    th = theta[:32]
    with torch.no_grad():
        for f in ("mean_t_fn", "std_fn", "approx_marginal_mean", "approx_marginal_std", "noise_schedule"):
            assert torch.equal(getattr(a, f)(t), getattr(b, f)(t)), f
        assert torch.equal(a.mean_fn(th, t), b.mean_fn(th, t))
        assert torch.equal(a.drift_fn(th, t).expand(32, D), b.drift_fn(th, t).expand(32, D))
        assert torch.equal(a.diffusion_fn(th, t), b.diffusion_fn(th, t))
        for w in ("identity", "max_likelihood", "variance"):
            a._set_weight_fn(w), b._set_weight_fn(w)
            wa, wb = a.weight_fn(t), b.weight_fn(t)
            assert wa == wb if isinstance(wa, int) else torch.equal(wa, wb)
        assert torch.equal(a(th, x[:32], t), b(th, x[:32], t))
        assert torch.equal(a(th.expand(5, 32, D), x[:1], t), b(th.expand(5, 32, D), x[:1], t))    # broadcast batch
        assert torch.equal(a.ode_fn(th, x[:32], t), b.ode_fn(th, x[:32], t))
        assert torch.equal(a.solve_schedule(17), b.solve_schedule(17))
        torch.manual_seed(5); ta = a.train_schedule(64)
        torch.manual_seed(5); tb = b.train_schedule(64)
        assert torch.equal(ta, tb)
        for cv in (True, False):
            torch.manual_seed(11); la = a.loss(theta[:64], x[:64], control_variate=cv)
            torch.manual_seed(11); lb = b.loss(theta[:64], x[:64], control_variate=cv)
            assert torch.allclose(la, lb, rtol=1e-6, atol=1e-6), (la - lb).abs().max()
        tt = torch.rand(64) * 0.9 + 0.05
        torch.manual_seed(12); la = a.loss(theta[:64], x[:64], times=tt)
        torch.manual_seed(12); lb = b.loss(theta[:64], x[:64], times=tt)
        assert torch.allclose(la, lb, rtol=1e-6, atol=1e-6)


def test_ve_schedules_equal_reference(ref):
    kw = dict(train_schedule="lognormal", solve_schedule="power_law", sigma_min=1e-3, sigma_max=20.0,
              lognormal_mean=-0.5, lognormal_std=1.5, power_law_exponent=5.0)
    a, b, _, _ = _pair("ve", **kw)
    torch.manual_seed(2); ta = a.train_schedule(500)
    torch.manual_seed(2); tb = b.train_schedule(500)
    assert torch.equal(ta, tb)
    assert torch.equal(a.solve_schedule(40), b.solve_schedule(40))
    assert torch.equal(a.solve_schedule(1), b.solve_schedule(1))
    from sbi_b200.score import posterior_score_nn
    theta, x = _data()
    for bad in (dict(sigma_min=-1.0), dict(sigma_min=2.0, sigma_max=1.0), dict(train_schedule="x"),
                dict(solve_schedule="x"), dict(train_schedule="lognormal", lognormal_std=0.0),
                dict(solve_schedule="power_law", power_law_exponent=0.0)):
        with pytest.raises(ValueError):
            posterior_score_nn(sde_type="ve", **bad)(theta, x)
    with pytest.raises(ValueError):
        posterior_score_nn(sde_type="nope")(theta, x)
    with pytest.warns(UserWarning, match="clamped"):
        posterior_score_nn(sde_type="ve", train_schedule="lognormal", lognormal_mean=5.0)(theta, x)


@pytest.mark.parametrize("sde_type", ["ve", "vp", "subvp"])
def test_ode_divergence_algebra_matches_autograd_trace(ref, sde_type):
    """ode_fn_and_divergence with the kernel's (net, diag J) replaced by autograd on the reference network equals
    the exact trace of the reference's ode_fn (what zuko's exact FreeFormJacobianTransform integrates)."""
    a, b, theta, x = _pair(sde_type)
    with torch.no_grad():
        a.net.output_layer.weight.normal_(0, 0.3)
    R = 16
    th, xo = theta[:R].clone(), x[:1]
    t = torch.rand(R) * (a.t_max - a.t_min) + a.t_min

    def raw_diag(enc, cond, tenc):
        out = a.net(enc, a._embedding_net(cond).expand(enc.shape[0], -1), tenc)
        diag = torch.zeros_like(enc)
        for r in range(enc.shape[0]):
            J = torch.autograd.functional.jacobian(
                lambda e: a.net(e[None], a._embedding_net(cond), tenc[r:r + 1])[0], enc[r])
            diag[r] = torch.diagonal(J)
        return out.detach(), diag

    b._raw_forward_diag = raw_diag
    rhs, div = b.ode_fn_and_divergence(th, xo, t)
    want_div = torch.zeros(R)
    for r in range(R):
        J = torch.autograd.functional.jacobian(lambda y: a.ode_fn(y[None], xo, t[r:r + 1])[0], th[r])
        want_div[r] = torch.trace(J)
    with torch.no_grad():
        want_rhs = a.ode_fn(th, xo, t)
    assert torch.allclose(rhs, want_rhs, rtol=1e-5, atol=1e-6)
    assert torch.allclose(div, want_div, rtol=1e-4, atol=1e-4), (div - want_div).abs().max()


def test_estimator_is_a_reference_vector_field_estimator(ref):
    from sbi.inference import NPSE
    from sbi.neural_nets.estimators.base import ConditionalVectorFieldEstimator
    from torch.distributions import MultivariateNormal
    from sbi_b200.score import posterior_score_nn
    theta, x = _data()
    est = posterior_score_nn(sde_type="vp")(theta, x)
    assert isinstance(est, ConditionalVectorFieldEstimator)
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    NPSE(prior, vf_estimator=posterior_score_nn(sde_type="vp"), show_progress_bars=False).append_simulations(theta, x)


@pytest.mark.parametrize("sde_type,corrector,cp", [("ve", None, None), ("vp", "langevin", dict(step_size=1e-3, num_steps=2)),
                                                   ("subvp", "gibbs", dict(num_steps=2)), ("vp", "gibbs", None)])
def test_sde_sampler_with_correctors_equals_reference_diffuser(ref, sde_type, corrector, cp, monkeypatch):
    """sample_sde's generic path (Euler-Maruyama predictor + Langevin / Gibbs corrector) against the reference's
    Diffuser.run on the reference estimator: same seed, same draws, same arithmetic."""
    from sbi.inference.potentials.vector_field_potential import vector_field_estimator_based_potential
    from sbi.samplers.score.diffuser import Diffuser
    from torch.distributions import MultivariateNormal
    from sbi_b200.flowmatching import sample_sde
    a, b, theta, x = _pair(sde_type)
    with torch.no_grad():
        a.net.output_layer.weight.normal_(0, 0.3)
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    x_o = x[:1]
    # (the potential also builds a zuko neural ODE for log_prob; zuko is absent here and not needed for sampling)
    monkeypatch.setattr("sbi.inference.potentials.vector_field_potential.build_neural_ode",
                        lambda *aa, **kk: (lambda *u, **v: None))
    pot, _ = vector_field_estimator_based_potential(a, prior, x_o)
    ts = a.solve_schedule(12)
    torch.manual_seed(7)
    with torch.no_grad():
        want = Diffuser(pot, predictor="euler_maruyama", corrector=corrector, corrector_params=cp).run(
            50, ts, show_progress_bars=False)
    torch.manual_seed(7)
    got = sample_sde(b, 50, x_o, ts=ts, corrector=corrector, corrector_params=cp)
    assert torch.allclose(got, want.reshape(50, D), rtol=1e-5, atol=1e-5), (got - want.reshape(50, D)).abs().max()


@pytest.mark.parametrize("sde_type,corrector", [("vp", None), ("ve", "langevin")])
def test_factorised_iid_score_sampler_equals_reference(ref, sde_type, corrector, monkeypatch):
    """Several iid observations, iid_method='fnpe' (vector_field_adaptor.py:725-813; narrowed base of
    diffuser.py:104-121): same samples as the reference's Diffuser on the reference estimator."""
    from sbi.inference.potentials.vector_field_potential import vector_field_estimator_based_potential
    from sbi.samplers.score.diffuser import Diffuser
    from torch.distributions import MultivariateNormal
    from sbi_b200.flowmatching import sample_sde
    a, b, theta, x = _pair(sde_type)
    with torch.no_grad():
        a.net.output_layer.weight.normal_(0, 0.3)
    prior = MultivariateNormal(torch.zeros(D), 2.0 * torch.eye(D))
    x_o = x[:5]
    monkeypatch.setattr("sbi.inference.potentials.vector_field_potential.build_neural_ode",
                        lambda *aa, **kk: (lambda *u, **v: None))
    pot, _ = vector_field_estimator_based_potential(a, prior, None)
    pot.set_x(x_o, x_is_iid=True, iid_method="fnpe")
    ts = a.solve_schedule(10)
    cp = dict(step_size=1e-3, num_steps=2) if corrector else None
    torch.manual_seed(3)
    want = Diffuser(pot, predictor="euler_maruyama", corrector=corrector, corrector_params=cp).run(
        40, ts, show_progress_bars=False)
    torch.manual_seed(3)
    got = sample_sde(b, 40, x_o, ts=ts, corrector=corrector, corrector_params=cp, iid_method="fnpe", prior=prior)
    assert got.shape == (40, D)
    assert torch.allclose(got, want.reshape(40, D), rtol=1e-4, atol=1e-4), (got - want.reshape(40, D)).abs().max()
    with pytest.raises(NotImplementedError):
        sample_sde(b, 4, x_o, ts=ts, iid_method="auto_gauss", prior=prior)
