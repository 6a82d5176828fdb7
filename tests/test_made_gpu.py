"""sbi's `made` estimator (MADE with a mixture-of-Gaussians head, flow.py:37-112) on the NSF kernels with the
MoG head: the reference fixture (log_prob), sampling against the moments / quantiles of 20 000 reference
samples and against the reference net sampled in fp64 on the same normal and uniform draws, gradients against the
reference's fp64 autograd, and an NPE training run."""
import math
import os
import warnings

import pytest
import torch

from oracle import ref_shim

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _load():
    from sbi_b200.neural_nets import build_made
    g = torch.load(os.path.join(GOLD, "made_d3c2.pt"))
    est = build_made(g["theta"], g["x"])
    est.load_state_dict(g["state_dict"])
    return g, est.cuda()


def test_made_log_prob_reproduces_reference_fixture(cuda_lib):
    g, est = _load()
    with torch.no_grad():
        lp = est.log_prob(g["inp"].cuda(), g["cond"].cuda())[0].cpu()
        lps = est.log_prob(g["inp"].unsqueeze(1).cuda(), g["cond"][:1].cuda())[:, 0].cpu()
        big = est.log_prob(g["inp"].repeat(200, 1).unsqueeze(1).cuda(), g["cond"][:1].cuda())[:, 0].cpu()
    assert (lp - g["log_prob"]).abs().max() <= 2e-3
    assert (lps - g["log_prob_shared"]).abs().max() <= 2e-3
    assert (big.reshape(200, -1) - g["log_prob_shared"]).abs().max() <= 2e-3      # 12 800 rows: many tiles


def test_made_sampling_matches_reference_sample_statistics(cuda_lib):
    g, est = _load()
    torch.manual_seed(0)
    s = est.sample((100_000,), g["cond"][:1].cuda())[:, 0].cpu()
    assert s.shape == (100_000, 3) and torch.isfinite(s).all()
    se = g["sample_std"] / math.sqrt(20000)
    assert ((s.mean(0) - g["sample_mean"]).abs() < 6 * se + 1e-3).all()
    assert (s.std(0) / g["sample_std"] - 1).abs().max() < 0.05
    q = torch.quantile(s, torch.tensor([0.1, 0.5, 0.9]), dim=0)
    assert (q - g["sample_q"]).abs().max() < 0.06 * g["sample_std"].max()
    # the samples are draws of the density log_prob evaluates: E_q[log q] ~ entropy consistency with a second
    # batch (a wrong sampler shifts the average log-density)
    with torch.no_grad():
        a = est.log_prob(s[:20000].unsqueeze(1).cuda(), g["cond"][:1].cuda()).mean().item()
        b = est.log_prob(s[20000:40000].unsqueeze(1).cuda(), g["cond"][:1].cuda()).mean().item()
    assert abs(a - b) < 0.05


@pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
def test_made_gradients_match_reference_autograd(cuda_lib):
    assert ref_shim.install()
    from sbi.neural_nets import posterior_nn as ref_posterior_nn
    g, est = _load()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = ref_posterior_nn("made")(g["theta"], g["x"])
    ref.load_state_dict(g["state_dict"])
    ref = ref.double()
    R = 100
    inp, cond = g["theta"][:R] * 1.4, g["x"][:R]
    w = torch.randn(R, dtype=torch.float64)
    a, c = inp.double().requires_grad_(True), cond.double().requires_grad_(True)
    lp64 = ref.log_prob(a, c)[0]
    (lp64 * w).sum().backward()
    want = est.layout.pack({k: p.grad for k, p in ref.named_parameters()}).double()
    ai, ci = inp.cuda().requires_grad_(True), cond.cuda().requires_grad_(True)
    lp = est.log_prob(ai, ci)[0]
    (lp * w.float().cuda()).sum().backward()
    assert (lp.detach().cpu().double() - lp64.detach()).abs().max() <= 2e-3
    mask = est.net._mask.cpu().bool()
    got = est.flat.grad.cpu().double() * mask
    want = want * mask
    sc = want.abs().max()
    assert (got - want).abs().max() <= 2e-3 * sc, ((got - want).abs().max() / sc).item()
    assert (ai.grad.cpu().double() - a.grad).abs().max() <= 2e-3 * a.grad.abs().max()
    assert (ci.grad.cpu().double() - c.grad).abs().max() <= 2e-3 * c.grad.abs().max()


def test_npe_with_made_fits_linear_gaussian(cuda_lib):
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPE
    D = 3
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    theta = prior.sample((6000,))
    x = theta + math.sqrt(0.3) * torch.randn_like(theta)
    inf = NPE(prior, density_estimator="made", device="cuda")
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=40)
    x_o = torch.tensor([[0.6, -0.4, 0.2]])
    s = inf.build_posterior().sample((4000,), x=x_o).cpu()
    assert (s.mean(0) - x_o[0] / 1.3).abs().max() < 0.08
    assert (s.std(0) / math.sqrt(0.3 / 1.3) - 1).abs().max() < 0.2


def _ref_made(theta, x, state_dict=None, perturb=0.0, seed=0):
    """The reference's `made` net in float64: the fixture's weights, or its own init moved by `perturb`."""
    assert ref_shim.install()
    from sbi.neural_nets import posterior_nn as ref_posterior_nn
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = ref_posterior_nn("made")(theta, x)
    if state_dict is not None:
        ref.load_state_dict(state_dict)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(perturb * torch.randn(p.shape, generator=g))
    return ref.double()


def made_sample_with_draws(ref, cond, noise, unif):
    """MixtureOfGaussiansMADE.sample (oracle/nflows_port/nn/nde/made.py:61-80) on given draws, in the precision of
    `ref`: one conditioner pass per feature, the wrapper's dummy feature 0 included; the component is the first m
    with u * sum(w) < cumsum(w)_m (else M - 1), w = exp(logit - max logit); the feature is mean + (softplus(s) +
    eps) * n; then the z-scoring is undone.  Also returns, per row, the smallest distance of u * sum(w) to an
    inner CDF boundary relative to sum(w) over the features (where float32 may pick the neighbouring
    component)."""
    dt = next(ref.parameters()).dtype
    net = ref.net
    made = net._distribution._made
    R, F = noise.shape
    M = made.num_mixture_components
    noise, unif = noise.to(dt), unif.to(dt)
    with torch.no_grad():
        ctx = net._embedding_net(cond.to(dt)).expand(R, -1)
        z = torch.zeros(R, F, dtype=dt)
        margin = torch.full((R,), math.inf, dtype=torch.float64)
        for f in range(F):
            out = made(z, ctx).reshape(R, F, M, 3)[:, f]
            logits, means, ustd = out[..., 0], out[..., 1], out[..., 2]
            w = torch.exp(logits - logits.max(dim=1, keepdim=True).values)
            tot, cum = w.sum(1), w.cumsum(1)
            target = unif[:, f] * tot
            below = target[:, None] < cum
            pick = torch.where(below.any(1), below.int().argmax(1), torch.full_like(tot, M - 1, dtype=torch.long))
            if M > 1:
                dist = ((target[:, None] - cum[:, :M - 1]).abs() / tot[:, None]).min(1).values
                margin = torch.minimum(margin, dist.double())
            mu = means.gather(1, pick[:, None])[:, 0]
            sd = torch.nn.functional.softplus(ustd.gather(1, pick[:, None])[:, 0]) + made.epsilon
            z[:, f] = mu + sd * noise[:, f]
        x = net._transform.inverse(z[:, 1:])[0]
    return x, margin


@pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
@pytest.mark.parametrize("model,shared", [("fixture", True), ("fixture", False), ("d8c5", False)])
def test_made_sampling_matches_reference_on_the_same_draws(cuda_lib, model, shared):
    """sbi_b200_made_sample with given normal draws and component-selecting uniforms against the reference net
    sampled on the same draws in float64.  64 rows per SM plus 7, so that CTAs loop over tiles and the last tile
    is ragged; rows with u = 0 and u = 1 - 2^-24 for every feature.  Rows whose u * sum(w) lies within 1e-5 of a
    CDF boundary (relative to sum(w)), where float32 may legitimately pick the neighbouring component, are left
    out and must be fewer than 1%; on the rest the bar is max(2e-3, 2 x torch-fp32's error)."""
    import ctypes as C
    from sbi_b200 import _lib as L
    from sbi_b200.neural_nets import build_made
    if model == "fixture":
        g, est = _load()
        ref = _ref_made(g["theta"], g["x"], g["state_dict"])
        conds = g["cond"]
    else:
        gen = torch.Generator().manual_seed(5)
        theta = 0.8 * torch.randn(500, 8, generator=gen) + 0.2
        x = 1.5 * torch.randn(500, 5, generator=gen) - 0.3
        ref = _ref_made(theta, x, perturb=0.05, seed=3)
        est = build_made(theta, x)
        est.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
        est = est.cuda()
        conds = x[:64]
    lib = L.load()
    F = est.layout.D
    R = 64 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    gen = torch.Generator().manual_seed(11)
    noise = torch.randn(R, F, generator=gen)
    unif = torch.rand(R, F, generator=gen)
    unif[:8] = 0.0
    unif[8:16] = 1.0 - 2.0 ** -24
    cond = conds[:1] if shared else conds[torch.randint(0, conds.shape[0], (R,), generator=gen)]
    ctx = est._embed(cond.cuda()).contiguous().float()
    noise_d, unif_d = noise.cuda(), unif.cuda()
    out = torch.full((R, F), float("nan"), device="cuda")
    rows = L.Rows(noise_d.data_ptr(), ctx.data_ptr(), None, R, 1 if shared else 0)
    L.check(lib.sbi_b200_made_sample(C.byref(est._model(nbuf=2)), C.byref(rows), unif_d.data_ptr(), out.data_ptr(),
                                     L.stream_ptr()), "made_sample")
    got = out.cpu()[:, 1:].double()
    want, margin = made_sample_with_draws(ref, cond, noise, unif)
    want32, _ = made_sample_with_draws(ref.float(), cond, noise, unif)
    keep = margin > 1e-5
    assert (~keep).sum().item() < 0.01 * R, (~keep).sum().item()
    assert keep[:16].all(), "edge rows fell on a CDF boundary"
    assert torch.isfinite(got).all()
    scale = max(1.0, want[keep].abs().max().item())
    err = (got - want)[keep].abs().max().item() / scale
    err32 = (want32.double() - want)[keep].abs().max().item() / scale
    print(f"made sample {model} shared={shared} R={R}: kernel err {err:.3e}  torch-fp32 err {err32:.3e}  "
          f"({(~keep).sum().item()} rows near a CDF boundary left out)")
    assert err <= max(2e-3, 2 * err32), (err, err32)
