"""The importance-sampling posterior without a GPU: argument errors of the SIR selection entry point, and the
host logic around it -- `importance_sample`, `method="importance"`, `log_prob` and the caching of the
normalising constant -- bit-equal to the UNMODIFIED reference (through oracle.ref_shim) on a pure-torch
potential and a box-uniform proposal, from the same seed."""
import pytest
import torch

from oracle import ref_shim

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
D = 3


def test_sir_select_argument_errors(lib):
    p = 256   # a non-null address: the checks run before any device call, nothing is dereferenced
    assert lib.sbi_b200_sir_scratch_ints(0) == 1 and lib.sbi_b200_sir_scratch_ints(-5) == 1
    assert lib.sbi_b200_sir_scratch_ints(1) == 2
    assert lib.sbi_b200_sir_scratch_ints(100) == 13 + 100          # block counts, then one index per group
    ok = dict(cand=p, D=2, lt=p, lq=p, u=p, groups=4, K=3, base=0, out=p, idx=None, cap=4, count=p, scratch=p)
    bad = [dict(cand=None), dict(lt=None), dict(lq=None), dict(u=None), dict(out=None), dict(count=None),
           dict(scratch=None), dict(D=0), dict(K=0), dict(K=-1), dict(groups=-1), dict(cap=-1)]
    for change in bad:
        a = {**ok, **change}
        rc = lib.sbi_b200_sir_select(a["cand"], a["D"], a["lt"], a["lq"], a["u"], a["groups"], a["K"], a["base"],
                                     a["out"], a["idx"], a["cap"], a["count"], a["scratch"], None)
        assert rc == -1, (change, rc)


def test_sir_needs_a_cuda_device():
    from sbi_b200.samplers import sampling_importance_resampling
    prior = torch.distributions.Independent(torch.distributions.Uniform(-torch.ones(D), torch.ones(D)), 1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        sampling_importance_resampling(lambda t: prior.log_prob(t), prior, num_samples=4, device="cpu")


# -------------------------------------------------------------------------------------------------
def _gauss(theta, x):
    return -((theta - x.reshape(1, -1)) ** 2).sum(-1) / (2 * 0.3 ** 2)


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    import sbi  # noqa: F401
    return sbi


def _pair(ref):
    """The same Gaussian potential behind the reference's and our posterior class, a box-uniform proposal."""
    from sbi.inference.posteriors.importance_posterior import ImportanceSamplingPosterior as RefISP
    from sbi.inference.potentials.base_potential import BasePotential as RefBase
    from sbi.utils import BoxUniform
    from sbi_b200.posteriors import ImportanceSamplingPosterior
    from sbi_b200.potentials import BasePotential

    class RefPot(RefBase):
        def __call__(self, theta, track_gradients=True):
            with torch.set_grad_enabled(track_gradients):
                return _gauss(theta, self.x_o)

    class OurPot(BasePotential):
        def __call__(self, theta, track_gradients=True):
            with torch.set_grad_enabled(track_gradients):
                return _gauss(theta, self.x_o)

    prior = BoxUniform(-torch.ones(D), torch.ones(D))
    r = RefISP(RefPot(None, device="cpu"), proposal=prior, device="cpu")
    o = ImportanceSamplingPosterior(OurPot(None, device="cpu"), proposal=prior, device="cpu")
    return r, o


@needs_ref
def test_importance_sample_bit_equal(ref):
    from sbi.samplers.importance.importance_sampling import importance_sample as ref_is
    from sbi.utils import BoxUniform
    from sbi_b200.samplers import importance_sample
    prior = BoxUniform(-torch.ones(D), torch.ones(D))
    x_o = torch.tensor([0.2, -0.4, 0.1])
    pot = lambda t: _gauss(t, x_o)   # noqa: E731
    torch.manual_seed(11)
    rs, rw = ref_is(pot, prior, num_samples=5000)
    torch.manual_seed(11)
    s, w = importance_sample(pot, prior, num_samples=5000)
    assert torch.equal(rs, s) and torch.equal(rw, w)


@needs_ref
def test_method_importance_bit_equal(ref):
    r, o = _pair(ref)
    x_o = torch.tensor([[0.2, -0.4, 0.1]])
    for post in (r, o):
        post.set_default_x(x_o)
    torch.manual_seed(5)
    rs, rw = r.sample((40, 25), method="importance")
    torch.manual_seed(5)
    s, w = o.sample((40, 25), method="importance")
    assert s.shape == (40, 25, D) and w.shape == (1000,)
    assert torch.equal(rs, s) and torch.equal(rw, w)
    # the constructor's method is the default
    r.method = o.method = "importance"
    torch.manual_seed(6)
    rs, rw = r.sample((300,))
    torch.manual_seed(6)
    s, w = o.sample((300,))
    assert torch.equal(rs, s) and torch.equal(rw, w)


@needs_ref
def test_log_prob_and_normalization_cache_bit_equal(ref):
    r, o = _pair(ref)
    x_o = torch.tensor([[0.2, -0.4, 0.1]])
    x_new = torch.tensor([[-0.5, 0.3, 0.0]])
    for post in (r, o):
        post.set_default_x(x_o)
    theta = 2 * torch.rand(64, D) - 1

    def both(**kw):
        torch.manual_seed(21)
        a = r.log_prob(theta, **kw)
        torch.manual_seed(21)
        b = o.log_prob(theta, **kw)
        assert torch.equal(a, b), kw
        return b

    first = both()                                             # default x: estimated and stored
    assert o._normalization_constant is not None
    z = o._normalization_constant.clone()
    assert torch.equal(both(), first)                          # stored value reused: no new draws
    assert torch.equal(o._normalization_constant, z)
    at_new = both(x=x_new)                                     # another x: estimated, not stored
    assert torch.equal(o._normalization_constant, z) and not torch.equal(at_new, first)
    same_values = x_o.clone()                                  # equal values count as the default x
    assert torch.equal(both(x=same_values), first)
    both(normalization_constant_params=dict(force_update=True, num_samples=3000))   # re-estimated and stored
    assert not torch.equal(o._normalization_constant, z)
    assert torch.equal(o._normalization_constant, r._normalization_constant)
    # Z = mean(exp(log w)) exactly as the reference computes it
    torch.manual_seed(3)
    zr = r.estimate_normalization_constant(x_new, num_samples=2000)
    torch.manual_seed(3)
    zo = o.estimate_normalization_constant(o._batch_x(x_new), num_samples=2000)
    assert torch.equal(zr, zo)


@needs_ref
def test_messages_and_default_rule(ref, monkeypatch):
    from sbi_b200 import samplers
    r, o = _pair(ref)
    o.set_default_x(torch.zeros(1, D))
    with pytest.raises(NameError):
        o.sample((10,), method="rejection")
    with pytest.raises(NotImplementedError) as ours:
        o.sample_batched((10,), x=torch.zeros(2, D))
    with pytest.raises(NotImplementedError) as theirs:
        r.sample_batched((10,), x=torch.zeros(2, D))
    assert str(ours.value) == str(theirs.value)
    with pytest.raises(ValueError, match="deprecated"):
        o.map(x=torch.zeros(1, D))

    seen = []

    def fake_sir(potential_fn, proposal, num_samples, num_candidate_samples, max_sampling_batch_size, **kw):
        seen.append((num_candidate_samples, max_sampling_batch_size))
        return torch.zeros(num_samples, D)

    monkeypatch.setattr(samplers, "sampling_importance_resampling", fake_sir)
    o.oversampling_factor, o.max_sampling_batch_size = 7, 123
    assert o.sample((5,)).shape == (5, D)                                    # sample()'s own defaults win
    o.sample((5,), oversampling_factor=None, max_sampling_batch_size=None)   # None: the constructor's values
    o.sample((5,), oversampling_factor=4, max_sampling_batch_size=9)
    assert seen == [(32, 10_000), (7, 123), (4, 9)]
