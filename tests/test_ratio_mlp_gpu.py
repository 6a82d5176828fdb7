"""The `mlp` and `linear` NRE classifiers (csrc/ratio_mlp.cu) on the GPU: logits and gradients against the
reference fixture and the reference's fp64 autograd, determinism, NRE losses, training and posteriors."""
import math
import os
import warnings

import pytest
import torch
from torch import nn

from oracle import ref_shim, sbi_port

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")

HERE = os.path.dirname(os.path.abspath(__file__))
MODELS = {"mlp": ("mlp", {}), "mlp_identity": ("mlp", dict(norm_layer=nn.Identity)), "linear": ("linear", {})}


def _ours(name, theta, x, H=50):
    from sbi_b200.ratio import classifier_nn
    model, kw = MODELS[name]
    if model == "mlp":
        kw = dict(kw, hidden_features=H)
    return classifier_nn(model, **kw)(theta, x)


def _grad_err(got, r32, r64):
    """max |error| / max |fp64|, and the same for torch's own fp32 autograd (ReLU kinks: a pre-activation
    within fp32 noise of 0 flips its mask)."""
    sc = max(r64.abs().max().item(), 1e-30)
    return (got - r64).abs().max().item() / sc, (r32 - r64).abs().max().item() / sc


def _assert_grad(got, r32, r64):
    err, err32 = _grad_err(got.cpu().double(), r32.cpu().double(), r64.cpu().double())
    assert err <= max(2e-3, 4 * err32), (err, err32)


@pytest.mark.parametrize("name", list(MODELS))
def test_logits_and_gradients_match_fixture(cuda_lib, name):
    gold = torch.load(os.path.join(HERE, "golden", "ratio_mlp_d4x6.pt"), weights_only=False)
    g = gold[name]
    est = _ours(name, gold["theta"], gold["x"])
    est.load_state_dict(g["state_dict"])
    est = est.cuda()
    th = gold["th"].cuda().requires_grad_(True)
    out = est(th, gold["xx"].cuda())
    assert (out.detach().cpu() - g["logits"]).abs().max() <= 1e-3
    shared = est.logits_raw(gold["th"].cuda(), gold["xx"][:1].cuda(), x_shared=True)
    assert (shared.cpu() - g["logits_shared"]).abs().max() <= 1e-3
    (out * gold["w"].cuda()).sum().backward()
    want = est.layout.pack({k: v for k, v in g["grad_params"].items() if k.startswith("net.")}).double()
    sc = want.abs().max()
    assert ((est.flat.grad.cpu().double() - want).abs().max() / sc) <= 2e-3
    sc = g["grad_theta"].abs().max()
    assert ((th.grad.cpu().double() - g["grad_theta"]).abs().max() / sc) <= 2e-3


def _ref_pair(name, Dt, Dx, H, seed=0, perturb=0.1):
    """(reference classifier, our estimator on cuda) with the same perturbed parameters."""
    assert ref_shim.install()
    from sbi.neural_nets import classifier_nn as ref_classifier_nn
    g = torch.Generator().manual_seed(seed)
    theta, x = torch.randn(600, Dt, generator=g) + 0.5, 2 * torch.randn(600, Dx, generator=g)
    model, kw = MODELS[name]
    if model == "mlp":
        kw = dict(kw, hidden_features=H)
    torch.manual_seed(seed)
    ref = ref_classifier_nn(model, **kw)(theta, x)
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(perturb * torch.randn(p.shape, generator=g))
    est = _ours(name, theta, x, H)
    est.load_state_dict(ref.state_dict(), strict=True)
    return ref, est.cuda()


def _ref_grads(ref, est, th, xx, w, dtype):
    r = ref.to(dtype)
    r.zero_grad()
    t = th.detach().to(dtype).clone().requires_grad_(True)
    o = r(t, xx.to(dtype))
    (o * w.to(dtype)).sum().backward()
    gp = est.layout.pack({k: p.grad for k, p in r.named_parameters() if k.startswith("net.")}).double()
    return o.detach().double(), gp, t.grad.double()


@needs_ref
@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("Dt,Dx,H,R", [(4, 6, 50, 300), (10, 10, 50, 4000), (1, 1, 50, 33), (2, 3, 30, 20000),
                                       (5, 100, 128, 2048)])
def test_logits_and_gradients_match_reference(cuda_lib, name, Dt, Dx, H, R):
    from sbi_b200.ratio import _RatioFn
    ref, est = _ref_pair(name, Dt, Dx, H)
    g0 = torch.Generator().manual_seed(1)
    th, xx, w = torch.randn(R, Dt, generator=g0), torch.randn(R, Dx, generator=g0), torch.randn(R, generator=g0)
    o32, gp32, gt32 = _ref_grads(ref, est, th, xx, w, torch.float32)
    o64, gp64, gt64 = _ref_grads(ref, est, th, xx, w, torch.float64)
    # pairs given directly
    tc = th.cuda().requires_grad_(True)
    est.zero_grad()
    out = est(tc, xx.cuda())
    (out * w.cuda()).sum().backward()
    assert (out.detach().cpu().double() - o64).abs().max() <= 1e-3
    _assert_grad(est.flat.grad, gp32, gp64)
    _assert_grad(tc.grad, gt32, gt64)
    # pairs through index gathers (the NRE trainers' contrastive pairs)
    gi = torch.Generator().manual_seed(2)
    ti, xi = torch.randint(0, R, (R,), generator=gi), torch.randint(0, R, (R,), generator=gi)
    o32i, gp32i, _ = _ref_grads(ref, est, th[ti], xx[xi], w, torch.float32)
    o64i, gp64i, _ = _ref_grads(ref, est, th[ti], xx[xi], w, torch.float64)
    est.zero_grad()
    out = _RatioFn.apply(est.net.flat, th.cuda(), xx.cuda(), est, ti.cuda(), xi.cuda(), False)
    (out * w.cuda()).sum().backward()
    assert (out.detach().cpu().double() - o64i).abs().max() <= 1e-3
    _assert_grad(est.flat.grad, gp32i, gp64i)
    # one shared x (the potential at a fixed observation)
    with torch.no_grad():
        o64s = ref.double()(th.double(), xx[:1].double().expand(R, -1))
    shared = est.logits_raw(th.cuda(), xx[:1].cuda(), x_shared=True)
    assert (shared.cpu().double() - o64s).abs().max() <= 1e-3


@needs_ref
def test_degenerate_layernorm_matches_reference(cuda_lib):
    """Zero first-layer weights: every row's pre-activations are the bias, constant across features after
    the bias is made constant, so the variance is exactly zero and LayerNorm divides by sqrt(eps)."""
    ref, est = _ref_pair("mlp", 3, 4, 50)
    with torch.no_grad():
        ref.net[0].weight.zero_()
        ref.net[0].bias.fill_(0.3)
    est.load_state_dict(ref.state_dict())
    g0 = torch.Generator().manual_seed(3)
    R = 500
    th, xx, w = torch.randn(R, 3, generator=g0), torch.randn(R, 4, generator=g0), torch.randn(R, generator=g0)
    o32, gp32, gt32 = _ref_grads(ref, est, th, xx, w, torch.float32)
    o64, gp64, gt64 = _ref_grads(ref, est, th, xx, w, torch.float64)
    tc = th.cuda().requires_grad_(True)
    est.zero_grad()
    out = est(tc, xx.cuda())
    (out * w.cuda()).sum().backward()
    assert torch.isfinite(out).all()
    assert (out.detach().cpu().double() - o64).abs().max() <= 1e-3
    _assert_grad(est.flat.grad, gp32, gp64)
    _assert_grad(tc.grad, gt32, gt64)


@pytest.mark.parametrize("name", ["mlp", "linear"])
def test_vjp_is_deterministic(cuda_lib, name):
    g0 = torch.Generator().manual_seed(4)
    theta, x = torch.randn(3000, 5, generator=g0), torch.randn(3000, 7, generator=g0)
    est = _ours(name, theta, x).cuda()
    w = torch.randn(3000, generator=g0).cuda()
    grads = []
    for _ in range(2):
        est.zero_grad()
        tc = theta.cuda().requires_grad_(True)
        (est(tc, x.cuda()) * w).sum().backward()
        grads.append((est.flat.grad.clone(), tc.grad.clone()))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


@needs_ref
@pytest.mark.parametrize("name", ["mlp", "linear"])
def test_nre_b_loss_matches_reference(cuda_lib, name):
    from sbi_b200.inference import NRE_B
    ref, est = _ref_pair(name, 3, 3, 50)
    g = torch.Generator().manual_seed(0)
    theta, x = torch.randn(600, 3, generator=g) + 0.5, 2 * torch.randn(600, 3, generator=g)
    tr = NRE_B(classifier=name)
    tr.append_simulations(theta, x)
    tr._x2d = tr._x.reshape(theta.shape[0], -1)
    B, A = 64, 10
    choices = NRE_B._contrastive_choices(B, A - 1, "cuda")
    loss_ref = sbi_port.nre_b_loss(ref.float(), theta[:B], x[:B], A, choices=choices.cpu())
    loss = tr._loss_on(est, torch.arange(B).cuda(), A, choices=choices)
    assert abs(loss.item() - loss_ref.item()) < 1e-4


def _task(D=2, n=6000):
    from torch.distributions import MultivariateNormal
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((n,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    return prior, theta, x


def _check(s, mean, var, tol_mean=0.06, tol_std=0.25):
    s = s.cpu()
    assert (s.mean(0) - mean).abs().max() < tol_mean, s.mean(0)
    assert (s.std(0) / math.sqrt(var) - 1).abs().max() < tol_std, s.std(0)


def test_nre_b_mlp_rejection_and_mcmc_linear_gaussian(cuda_lib):
    """NRE-B with `mlp` recovers the analytic posterior N(x_o/2, 0.05 I) by rejection and slice MCMC, and
    N(sum x_o,i / (n+1), 0.1/(n+1) I) for n iid observations (linearGaussian_snre_test.py:55-136)."""
    from sbi_b200.inference import NRE_B
    prior, theta, x = _task()
    x_o = torch.tensor([[0.3, -0.2]])
    nre = NRE_B(prior, classifier="mlp", device="cuda")
    nre.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
    post = nre.build_posterior(sample_with="rejection")
    _check(post.sample((2000,), x=x_o), x_o[0] / 2, 0.05)
    post = nre.build_posterior(mcmc_parameters=dict(num_chains=200, warmup_steps=50, thin=2))
    _check(post.sample((2000,), x=x_o), x_o[0] / 2, 0.05)
    x_iid = torch.tensor([[0.3, -0.2], [0.1, 0.0], [0.4, -0.3]])
    _check(post.sample((2000,), x=x_iid), x_iid.sum(0) / 4, 0.1 / 4, tol_mean=0.08, tol_std=0.35)


def test_nre_c_mlp_rejection_linear_gaussian(cuda_lib):
    from sbi_b200.inference import NRE_C
    prior, theta, x = _task()
    x_o = torch.tensor([[0.3, -0.2]])
    nre = NRE_C(prior, classifier="mlp", device="cuda")
    nre.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
    _check(nre.build_posterior(sample_with="rejection").sample((2000,), x=x_o), x_o[0] / 2, 0.05)


def test_nre_a_mlp_slice_mcmc_runs(cuda_lib):
    """The reference's on-device case NRE_A + `mlp` + slice MCMC (inference_on_device_test.py:89-90)."""
    from sbi_b200.inference import NRE_A
    prior, theta, x = _task(n=2000)
    nre = NRE_A(prior, classifier="mlp", device="cuda")
    nre.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=5)
    post = nre.build_posterior(sample_with="mcmc", mcmc_method="slice_np_vectorized",
                               mcmc_parameters=dict(num_chains=20, warmup_steps=10, thin=1))
    s = post.sample((100,), x=torch.tensor([[0.3, -0.2]]))
    assert s.shape == (100, 2) and torch.isfinite(s).all()


@pytest.mark.parametrize("cls", ["NRE_B", "BNRE"])
def test_linear_classifier_trains(cuda_lib, cls):
    import sbi_b200.inference as inf
    prior, theta, x = _task(n=3000)
    nre = getattr(inf, cls)(prior, classifier="linear", device="cuda")
    nre.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=10)
    tl = nre._summary["training_loss"]
    assert all(math.isfinite(v) for v in tl) and tl[-1] < tl[0]


@needs_ref
def test_reference_nre_b_trains_b200_mlp(cuda_lib):
    """Drop-in: the unmodified reference NRE_B trains the sm_90a `mlp` and samples by rejection."""
    assert ref_shim.install()
    from sbi.inference import NRE_B
    from sbi_b200.ratio import RatioEstimator, classifier_nn
    prior, theta, x = _task()
    prior = type(prior)(prior.loc.cuda(), prior.covariance_matrix.cuda())
    x_o = torch.tensor([[0.3, -0.2]], device="cuda")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NRE_B(prior, classifier=classifier_nn("mlp"), device="cuda", show_progress_bars=False)
        est = inf.append_simulations(theta.cuda(), x.cuda()).train(training_batch_size=500, max_num_epochs=30)
        assert isinstance(est, RatioEstimator) and est.flat.is_cuda
        s = inf.build_posterior(sample_with="rejection").sample((1000,), x=x_o, show_progress_bars=False)
    _check(s, x_o[0].cpu() / 2, 0.05, tol_mean=0.08, tol_std=0.3)
