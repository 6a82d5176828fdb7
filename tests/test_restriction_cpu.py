"""TSNPE's public pieces without a GPU: `get_density_thresholder`, `RestrictedPrior.log_prob` / `prior_acceptance`
/ `mean` / `variance` / `support` and the NPE round rule for `RestrictedPrior` proposals, against the UNMODIFIED
reference (through oracle.ref_shim) on pure-torch distributions from the same seed.  (Sampling runs on the device:
tests/test_restriction_gpu.py.)"""
import inspect
import warnings

import pytest
import torch
from torch.distributions import Independent, MultivariateNormal, Uniform

from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
D = 3


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


def _mvn():
    return MultivariateNormal(torch.tensor([0.3, -0.2, 0.1]), torch.diag(torch.tensor([0.5, 1.0, 2.0])),
                              validate_args=False)


def _box():
    return Independent(Uniform(-2 * torch.ones(D), 2 * torch.ones(D), validate_args=False), 1, validate_args=False)


def test_sampling_needs_a_cuda_device(monkeypatch):
    from sbi_b200.restriction import RestrictedPrior
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    prior = _box()
    rp = RestrictedPrior(prior, lambda t: prior.log_prob(t) > -10)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        rp.sample((5,))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        rp.prior_acceptance()


@needs_ref
def test_density_thresholder_bit_equal(ref):
    from sbi.utils import get_density_thresholder as ref_thr
    from sbi_b200.restriction import get_density_thresholder
    dist = _mvn()
    for q, n in ((1e-4, 200_000), (0.05, 30_000), (0.0, 1000)):
        torch.manual_seed(7)
        r = ref_thr(dist, quantile=q, num_samples_to_estimate_support=n)
        torch.manual_seed(7)
        o = get_density_thresholder(dist, quantile=q, num_samples_to_estimate_support=n)
        tr = inspect.getclosurevars(r).nonlocals["log_prob_threshold"]
        to = inspect.getclosurevars(o).nonlocals["log_prob_threshold"]
        assert torch.equal(tr, to), q
        theta = dist.sample((5000,)) * 1.5
        assert o(theta).dtype == torch.bool and torch.equal(r(theta), o(theta))
        assert 0 < int(o(theta).sum()) < 5000
    # strict comparison: the threshold itself, NaN and -inf reject
    box = _box()
    torch.manual_seed(3)
    o = get_density_thresholder(box, quantile=0.1, num_samples_to_estimate_support=100)
    assert not o(torch.tensor([[0.0, 0.0, 0.0]])).any()          # uniform: every log_prob equals the threshold
    torch.manual_seed(3)
    thr = get_density_thresholder(_mvn(), quantile=0.5, num_samples_to_estimate_support=100)
    assert not thr(torch.tensor([[float("nan"), 0.0, 0.0]])).any()
    assert not o(torch.tensor([[5.0, 0.0, 0.0]])).any()            # outside the box: log_prob is -inf


def _pair(ref, prior, fn, **kw):
    from sbi.utils import RestrictedPrior as RefRP
    from sbi_b200.restriction import RestrictedPrior
    return RefRP(prior, fn, **kw), RestrictedPrior(prior, fn, **kw)


@needs_ref
def test_attributes_equal(ref):
    prior, post = _mvn(), object()
    fn = lambda t: prior.log_prob(t) > -4.0   # noqa: E731
    r, o = _pair(ref, prior, fn, posterior=post, sample_with="sir")
    for a in ("_prior", "_accept_reject_fn", "_posterior", "_sample_with", "acceptance_rate", "_device"):
        assert getattr(r, a) is getattr(o, a) or getattr(r, a) == getattr(o, a), a
    assert o.batch_shape == r.batch_shape and o.event_shape == r.event_shape and not o._validate_args
    assert isinstance(o, torch.distributions.Distribution)


@needs_ref
@pytest.mark.parametrize("make_prior", [_mvn, _box])
def test_log_prob_bit_equal(ref, make_prior):
    prior = make_prior()
    fn = lambda t: prior.log_prob(t) > -4.5   # noqa: E731
    r, o = _pair(ref, prior, fn)
    r.acceptance_rate = o.acceptance_rate = torch.as_tensor(0.3712)
    theta = 1.4 * torch.randn(400, D)
    for norm in (True, False):
        a, b = r.log_prob(theta, norm_restricted_prior=norm), o.log_prob(theta, norm_restricted_prior=norm)
        assert torch.equal(a, b), norm
        outside = ~fn(theta)
        assert outside.any() and (~outside).any()
        assert torch.isneginf(b[outside]).all() and torch.isfinite(b[~outside]).all()
        want = prior.log_prob(theta[~outside]) - (torch.log(torch.as_tensor(0.3712)) if norm else 0)
        assert torch.equal(b[~outside], want)
    # one unbatched theta
    assert torch.equal(r.log_prob(theta[0]), o.log_prob(theta[0])) and o.log_prob(theta[0]).shape == (1,)
    # gradients only when asked for
    th = theta[:4].clone().requires_grad_(True)
    assert not o.log_prob(th).requires_grad
    assert o.log_prob(th, track_gradients=True).requires_grad == r.log_prob(th, track_gradients=True).requires_grad


@needs_ref
def test_prior_acceptance_cache_and_force_update(ref, monkeypatch):
    prior = _box()
    fn = lambda t: prior.log_prob(t) > -4.0   # noqa: E731
    r, o = _pair(ref, prior, fn)
    calls = {id(r): [], id(o): []}

    def fake_sample(obj):
        def sample(sample_shape=torch.Size(), **kw):
            calls[id(obj)].append((tuple(torch.Size(sample_shape)), kw))
            if kw.get("save_acceptance_rate"):
                obj.acceptance_rate = torch.as_tensor(0.25 + 0.125 * len(calls[id(obj)]))
            return torch.zeros(*sample_shape, D)
        return sample

    for obj in (r, o):
        monkeypatch.setattr(obj, "sample", fake_sample(obj))
    seq = [dict(), dict(), dict(num_rejection_samples=300, force_update=True, rejection_sampling_batch_size=77),
           dict(), dict(force_update=True, show_progress_bars=True)]
    for kw in seq:
        assert torch.equal(r.prior_acceptance(**kw), o.prior_acceptance(**kw)), kw
    assert calls[id(r)] == calls[id(o)] and len(calls[id(o)]) == 3
    # log_prob normalises with the cached rate and forwards prior_acceptance_params
    theta = torch.rand(20, D)
    kw = dict(prior_acceptance_params=dict(force_update=True, num_rejection_samples=50))
    assert torch.equal(r.log_prob(theta, **kw), o.log_prob(theta, **kw))
    assert calls[id(r)] == calls[id(o)] and len(calls[id(o)]) == 4


@needs_ref
def test_mean_variance_support(ref):
    prior = _box()
    r, o = _pair(ref, prior, lambda t: prior.log_prob(t) > -4.0)
    for attr in ("mean", "variance"):
        with pytest.raises(NotImplementedError) as a:
            getattr(r, attr)
        with pytest.raises(NotImplementedError) as b:
            getattr(o, attr)
        assert str(a.value) == str(b.value)
    assert repr(o.support) == repr(r.support) == repr(prior.support)

    class Bare:     # a prior object with sample / log_prob and no support
        def sample(self, shape):
            return torch.zeros(*shape, D)

        def log_prob(self, theta):
            return torch.zeros(theta.shape[0])

    r, o = _pair(ref, Bare(), lambda t: torch.ones(t.shape[0], dtype=torch.bool))
    with pytest.raises(NotImplementedError) as a:
        r.support
    with pytest.raises(NotImplementedError) as b:
        o.support
    assert str(a.value) == str(b.value)


@needs_ref
def test_npe_round_rule_for_restricted_priors(ref, monkeypatch):
    import sbi_b200.inference as inference
    from sbi.inference import NPE as RefNPE
    from sbi.utils import RestrictedPrior as RefRP
    from sbi_b200.restriction import RestrictedPrior
    monkeypatch.setattr(inference, "_process_device", lambda device: "cpu")   # append_simulations runs no kernel
    prior, other = _mvn(), _box()
    fn = lambda t: torch.ones(t.shape[0], dtype=torch.bool)   # noqa: E731
    theta = prior.sample((50,))
    x = theta + 0.1 * torch.randn_like(theta)
    x_nan = x.clone()
    x_nan[3, 0] = float("nan")

    def rounds(trainer, restricted_cls):
        msgs = []
        for p, xx in ((prior, x_nan), (other, x)):
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                trainer.append_simulations(theta, xx, proposal=restricted_cls(p, fn))
            msgs.append([str(m.message) for m in w if "RestrictedPrior" in str(m.message)])
        return list(trainer._data_round_index), msgs

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want, want_msgs = rounds(RefNPE(prior, show_progress_bars=False), RefRP)
    assert want == [0, 1]
    for cls in (RestrictedPrior, RefRP):         # this module's class, and the reference's once sbi is imported
        ours = inference.NPE(prior, density_estimator="nsf", device="cuda")
        got, msgs = rounds(ours, cls)
        assert got == want and msgs == want_msgs, cls
        assert len(msgs[0]) == 0 and len(msgs[1]) == 1
        # round 0 drops the invalid simulation: exclude_invalid_x defaults to True there
        assert ours._round_rows == [49, 50]
