"""The importance-sampling posterior on the GPU: the SIR selection kernel (csrc/compact.cu) against the
reference's expression on identical tensors, SIR and the posterior class end to end against the UNMODIFIED
reference (through oracle.ref_shim), SIR samples and the normalised log_prob against the analytic posterior
of the linear-Gaussian task, and the trainers' `build_posterior(sample_with="importance")`.

The kernel's softmax and cumulative sum run in another order than torch's, so a decision may differ where u
lies within rounding of a cumulative weight: every such group is counted and must be a margin case, |u -
cumw_k| <= 1e-5 for some k of the fp64 cumulative weights."""
import math
import warnings

import pytest
import torch
from torch.distributions import Independent, MultivariateNormal, Uniform

from oracle import ref_shim

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
MARGIN = 1e-5


def _reference_mask(lt, lq, u, g, K):
    """sir.py:59-62 on the same tensors, plus the groups within MARGIN of a fp64 cumulative weight."""
    lw = (lt - lq).reshape(g, K)
    weights = lw.softmax(-1).cumsum(-1)
    mask = torch.cumsum(weights >= u.reshape(g, 1), -1) == 1
    pick = torch.where(mask.any(-1), mask.int().argmax(-1), torch.full((g,), -1, device=lw.device))
    cw64 = lw.double().softmax(-1).cumsum(-1)
    near = ((cw64 - u.double().reshape(g, 1)).abs() <= MARGIN).any(-1)
    return mask, pick, near


def _select(cand, lt, lq, u, g, K, base=0, cap=None, count0=0, out=None, out_idx=None):
    from sbi_b200 import _lib as L
    lib = L.load()
    D = cand.shape[1]
    cap = g + count0 if cap is None else cap
    if out is None:
        out = torch.full((cap, D), float("nan"), device="cuda")
        out_idx = torch.full((cap,), -1, dtype=torch.int64, device="cuda")
    count = torch.full((1,), count0, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(lib.sbi_b200_sir_scratch_ints(g)), dtype=torch.int32, device="cuda")
    L.check(lib.sbi_b200_sir_select(cand.data_ptr(), D, lt.data_ptr(), lq.data_ptr(), u.data_ptr(), g, K, base,
                                    out.data_ptr(), out_idx.data_ptr(), cap, count.data_ptr(), scratch.data_ptr(),
                                    L.stream_ptr()), "sir_select")
    return out, out_idx, int(count.item())


def _inputs(g, K, D, seed, specials):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    cand = torch.randn(g * K, D, device="cuda", generator=gen)
    lt = 2 * torch.randn(g * K, device="cuda", generator=gen)
    lq = torch.randn(g * K, device="cuda", generator=gen)
    u = torch.rand(g, device="cuda", generator=gen)
    if specials:
        lt[::7] = float("-inf")                                   # single -inf weights
        lt.view(g, K)[3::50] = float("-inf")                       # whole groups at -inf: no selection
        lt.view(g, K)[5::97, 0] = float("nan")                     # a NaN weight: softmax NaN, no selection
        u[11::40] = 1.5                                            # cumw_{K-1} < u: no selection
    return cand, lt, lq, u


def _check(cand, lt, lq, u, g, K, base, count0, out, out_idx, count, cap):
    """Our rows, indices and count against `thetas.reshape(g, K, -1)[mask]`; returns the margin-case count."""
    D = cand.shape[1]
    mask, pick, near = _reference_mask(lt, lq, u, g, K)
    n_new, n_stored = count - count0, min(count, cap) - count0
    rows, gi = out[count0:count0 + n_stored], out_idx[count0:count0 + n_stored] - base
    assert (gi[1:] > gi[:-1]).all() and (gi >= 0).all() and (gi < g).all()       # group order, no repeats
    cand3 = cand.reshape(g, K, D)
    match = (cand3[gi] == rows[:, None, :]).all(-1)
    assert (match.sum(-1) == 1).all()                                          # every row is one of its group's
    ours = torch.full((g,), -1, dtype=torch.int64, device="cuda")
    ours[gi] = match.int().argmax(-1).long()
    seen = g if n_stored == n_new else int(gi[-1]) + 1                       # past a cap cut only the stored part
    diff = (ours[:seen] != pick[:seen])
    margin = int(diff.sum())
    assert bool(near[:seen][diff].all()), "a decision differs outside the rounding margin"
    if margin == 0:
        want = cand3[mask]
        assert torch.equal(rows, want[:n_stored])
        assert torch.equal(gi, torch.nonzero(mask.any(-1)).reshape(-1)[:n_stored])
        if n_stored == n_new:
            assert n_new == want.shape[0]
    assert abs(n_new - int((pick >= 0).sum())) <= int(near.sum())
    assert bool(torch.isnan(out[min(count, cap):]).all())                      # nothing written past the rows
    return margin


@pytest.mark.parametrize("K", [1, 7, 32, 33, 1000])
@pytest.mark.parametrize("D", [1, 3, 10, 33])
def test_sir_select_matches_reference_expression(cuda_lib, K, D):
    g = max(64, 100_000 // K)
    cand, lt, lq, u = _inputs(g, K, D, seed=10 * K + D, specials=K > 1)
    out, out_idx, count = _select(cand, lt, lq, u, g, K)
    margin = _check(cand, lt, lq, u, g, K, 0, 0, out, out_idx, count, out.shape[0])
    print(f"K={K} D={D}: {g} groups, {count} selected, {margin} margin cases")
    assert count > 0.5 * g


def test_sir_select_many_groups_base_count_and_cap(cuda_lib):
    """More than 2^16 groups (tens of thousands of scanned block counts), a non-zero index base, rows appended
    behind ones already collected, and the capacity cut across a second batch."""
    K, D = 32, 5
    g1, g2 = 70_001, 40_003
    count0, base1 = 17, 1_000_000
    cap = count0 + 90_000
    out = torch.full((cap, D), float("nan"), device="cuda")
    out_idx = torch.full((cap,), -1, dtype=torch.int64, device="cuda")
    c1 = _inputs(g1, K, D, seed=1, specials=True)
    _, _, n1 = _select(*c1, g1, K, base=base1, cap=cap, count0=count0, out=out, out_idx=out_idx)
    m1 = _check(*c1, g1, K, base1, count0, out, out_idx, n1, cap)
    c2 = _inputs(g2, K, D, seed=2, specials=True)
    base2 = base1 + g1
    _, _, n2 = _select(*c2, g2, K, base=base2, cap=cap, count0=n1, out=out, out_idx=out_idx)
    assert n2 > cap                                                 # overflow is counted, not stored
    m2 = _check(*c2, g2, K, base2, n1, out, out_idx, n2, cap)
    print(f"two batches: {n1 - count0} + {n2 - n1} selected, cap {cap}, margin cases {m1} + {m2}")
    # zero groups: nothing launched, nothing counted
    _, _, n0 = _select(*c2, 0, K, cap=cap, count0=5, out=out, out_idx=out_idx)
    assert n0 == 5


# -------------------------------------------------------------------------------------------------
def _perturb(net, seed=3, scale=0.1):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in net.named_parameters():
            s = scale if ("entries" not in n and "diag" not in n) else 0.05
            p.add_(s * torch.randn(p.shape, generator=g))


def _potentials(kind, D=3):
    """Our potential from perturbed weights of a reference-built estimator, and the reference's own potential on
    the same weights (CPU); prior a box."""
    from sbi.inference.potentials.likelihood_based_potential import likelihood_estimator_based_potential as ref_lik
    from sbi.inference.potentials.ratio_based_potential import ratio_estimator_based_potential as ref_rat
    from sbi.neural_nets import classifier_nn as ref_cls
    from sbi.neural_nets import likelihood_nn as ref_lnn
    from sbi_b200.neural_nets import likelihood_nn
    from sbi_b200.potentials import likelihood_estimator_based_potential, ratio_estimator_based_potential
    from sbi_b200.ratio import classifier_nn
    gen = torch.Generator().manual_seed(0)
    theta = 0.8 * torch.randn(800, D, generator=gen)
    x = torch.cat([theta, theta], 1)[:, :4] + 0.5 * torch.randn(800, 4, generator=gen)
    prior = Independent(Uniform(-2 * torch.ones(D), 2 * torch.ones(D)), 1)
    x_o = x[7:8]
    torch.manual_seed(2)
    if kind == "nle_nsf":
        r_est = ref_lnn("nsf")(theta, x)
        _perturb(r_est)
        est = likelihood_nn("nsf")(theta, x)
        est.load_state_dict(r_est.state_dict())
        rp, _ = ref_lik(r_est, prior, x_o=x_o)
        op, _ = likelihood_estimator_based_potential(est.cuda(), prior, x_o=x_o)
    else:
        r_est = ref_cls("resnet")(theta, x)
        _perturb(r_est)
        est = classifier_nn("resnet")(theta, x)
        est.load_state_dict(r_est.state_dict())
        rp, _ = ref_rat(r_est, prior, x_o=x_o)
        op, _ = ratio_estimator_based_potential(est.cuda(), prior, x_o=x_o)
    return rp, op, prior, x_o, theta


def _ref_view(op):
    """Our potential behind the reference's BasePotential interface, so reference classes can drive it."""
    from sbi.inference.potentials.base_potential import BasePotential as RefBase

    class View(RefBase):
        def __init__(self):
            super().__init__(None, device="cuda")

        def set_x(self, x_o, x_is_iid=True):
            super().set_x(x_o, x_is_iid)
            if x_o is not None:
                op.set_x(x_o, x_is_iid)

        def __call__(self, theta, track_gradients=True):
            return op(theta, track_gradients=track_gradients)

    return View()


@needs_ref
@pytest.mark.parametrize("kind", ["nle_nsf", "nre_resnet"])
def test_sir_and_posterior_match_reference(cuda_lib, kind):
    assert ref_shim.install()
    from sbi.inference.posteriors.importance_posterior import ImportanceSamplingPosterior as RefISP
    from sbi.samplers.importance.sir import sampling_importance_resampling as ref_sir
    from sbi.utils import BoxUniform
    from sbi_b200.posteriors import ImportanceSamplingPosterior
    from sbi_b200.samplers import sampling_importance_resampling
    rp, op, prior, x_o, theta = _potentials(kind)
    # the two potentials agree to fp32 rounding on proposal draws
    th = prior.sample((2000,))
    with torch.no_grad():
        a, b = rp(th, track_gradients=False), op(th.cuda(), track_gradients=False).cpu()
    assert (a - b).abs().max() <= 2e-3, (a - b).abs().max()
    D = th.shape[1]
    box = BoxUniform(-2 * torch.ones(D, device="cuda"), 2 * torch.ones(D, device="cuda"))
    pot = lambda t: op(t, track_gradients=False)     # noqa: E731
    # SIR: same seed -> the reference's candidates and uniforms; rows equal, in order, over several batches
    N, B = 25_000, 4_000
    torch.manual_seed(7)
    want = ref_sir(pot, box, num_samples=N, num_candidate_samples=32, max_sampling_batch_size=B, device="cuda")
    torch.manual_seed(7)
    got = sampling_importance_resampling(pot, box, num_samples=N, num_candidate_samples=32,
                                         max_sampling_batch_size=B, device="cuda")
    assert got.shape == want.shape == (N, D)
    assert torch.equal(got, want)
    # the posterior classes: method="importance" and the normalised log_prob
    r = RefISP(_ref_view(op), proposal=box, device="cuda")
    o = ImportanceSamplingPosterior(op, proposal=box, device="cuda")
    for post in (r, o):
        post.set_default_x(x_o.cuda())
    torch.manual_seed(8)
    rs, rw = r.sample((5000,), method="importance")
    torch.manual_seed(8)
    s, w = o.sample((5000,), method="importance")
    assert torch.equal(rs, s) and torch.equal(rw, w)
    torch.manual_seed(9)
    rl = r.log_prob(theta[:300].cuda())
    torch.manual_seed(9)
    ol = o.log_prob(theta[:300].cuda())
    assert torch.allclose(rl, ol, rtol=1e-6, atol=1e-5)
    torch.manual_seed(10)
    s1 = r.sample((3000,), max_sampling_batch_size=1000)
    torch.manual_seed(10)
    s2 = o.sample((3000,), max_sampling_batch_size=1000)
    assert torch.equal(s1, s2)


# -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def linear_gaussian():
    """x = theta + N(0, 0.1 I), prior N(0, 0.1 I): posterior N(x_o / 2, 0.05 I)."""
    from sbi_b200.inference import NLE, NPE, NRE_B, NRE_C
    D = 2
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((6000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        nle = NLE(prior, density_estimator="nsf", device="cuda")
        nle.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=60)
        nre = NRE_B(prior, classifier="resnet", device="cuda")
        nre.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
        nrec = NRE_C(prior, classifier="resnet", device="cuda")
        nrec.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=5)
        npe = NPE(prior, density_estimator="nsf", device="cuda")
        npe.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=5)
    return dict(NLE=nle, NRE_B=nre, NRE_C=nrec, NPE=npe, theta=theta, x=x)


@pytest.mark.parametrize("which,mean_tol,std_tol", [("NLE", 0.05, 0.2), ("NRE_B", 0.06, 0.25)])
def test_sir_recovers_analytic_posterior_and_log_prob_normalises(cuda_lib, linear_gaussian, which, mean_tol,
                                                                 std_tol):
    x_o = torch.tensor([[0.3, -0.2]])
    post = linear_gaussian[which].build_posterior(sample_with="importance")
    s = post.sample((20_000,), x=x_o).cpu()
    assert s.shape == (20_000, 2) and torch.isfinite(s).all()
    mean_err = (s.mean(0) - x_o[0] / 2).abs().max().item()
    std_err = (s.std(0) / math.sqrt(0.05) - 1).abs().max().item()
    print(f"{which} SIR: mean error {mean_err:.3f}, std ratio error {std_err:.3f}")
    assert mean_err < mean_tol and std_err < std_tol
    # exp(log_prob) integrates to ~1: a 161^2 grid over +-5.5 posterior std around the analytic mean
    post.set_default_x(x_o)
    h = 2.4 / 160
    ax = torch.linspace(-1.2, 1.2, 161)
    grid = torch.stack(torch.meshgrid(ax + 0.15, ax - 0.1, indexing="ij"), -1).reshape(-1, 2)
    lp = post.log_prob(grid.cuda(), normalization_constant_params=dict(num_samples=200_000)).cpu()
    integral = float(torch.exp(lp.double()).sum() * h * h)
    print(f"{which}: integral of exp(log_prob) = {integral:.4f}")
    assert abs(integral - 1) < 0.05, integral


@pytest.mark.parametrize("which", ["NLE", "NRE_B", "NRE_C", "NPE"])
def test_build_posterior_importance_wiring(cuda_lib, linear_gaussian, which):
    from sbi_b200 import diagnostics
    from sbi_b200.posteriors import ImportanceSamplingPosterior
    trainer = linear_gaussian[which]
    params = dict(method="sir", oversampling_factor=16, max_sampling_batch_size=700)
    post = trainer.build_posterior(sample_with="importance", importance_sampling_parameters=params)
    assert isinstance(post, ImportanceSamplingPosterior)
    assert (post.method, post.oversampling_factor, post.max_sampling_batch_size) == ("sir", 16, 700)
    x_o = torch.tensor([[0.3, -0.2]])
    s = post.sample((1500,), x=x_o, oversampling_factor=None, max_sampling_batch_size=None)
    assert s.shape == (1500, 2) and torch.isfinite(s).all()
    s, lw = post.sample((10, 20), x=x_o, method="importance")
    assert s.shape == (10, 20, 2) and lw.shape == (200,)
    post.set_default_x(x_o)
    m = post.map(num_iter=150, num_init_samples=200, num_to_optimize=10)
    assert m.shape == (1, 2) and torch.isfinite(m).all()
    print(f"{which} MAP {m.cpu().tolist()} (analytic {(x_o[0] / 2).tolist()})")
    if which in ("NLE", "NRE_B"):          # the two trained to convergence above
        assert (m.cpu()[0] - x_o[0] / 2).abs().max() < 0.15
    with pytest.warns(UserWarning, match="Falling back to non-batched sampling"):
        ranks, dap = diagnostics.run_sbc(linear_gaussian["theta"][:6], linear_gaussian["x"][:6], post,
                                         num_posterior_samples=100)
    assert ranks.shape == (6, 2) and dap.shape == (6, 2)
    assert ((ranks >= 0) & (ranks <= 100)).all()
