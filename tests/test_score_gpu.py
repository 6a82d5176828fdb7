"""Score estimators (NPSE, SURVEY 8f-3) on the device: the bare-network mode of the flow-matching kernels
(forward, parameter gradient for a given output gradient, diagonal of the input Jacobian) against the CPU
oracle's VectorFieldMLP in float64, and end-to-end NPSE fits on a linear-Gaussian task whose posterior is known.
The arithmetic around the network is pinned against the unmodified reference in tests/test_score_cpu.py."""
import math

import pytest
import torch

from oracle import sbi_port

pytestmark = pytest.mark.gpu


def _pair(sde_type, D=4, C=5, seed=0, perturb=0.15):
    """(estimator on the device, the same estimator on the CPU in float64 with the oracle's network behind it)."""
    from sbi_b200.score import build_score_estimator
    g = torch.Generator().manual_seed(seed)
    theta, x = 0.7 * torch.randn(500, D, generator=g) + 0.4, 1.5 * torch.randn(500, C, generator=g) - 0.3
    torch.manual_seed(seed)
    port = sbi_port.build_flow_matching_estimator(theta, x, hidden_features=48, num_layers=3)
    with torch.no_grad():
        for p in port.parameters():
            p.add_(perturb * torch.randn(p.shape, generator=g))
    sub = {k[len("net."):]: v for k, v in port.state_dict().items() if k.startswith("net.")}
    est = build_score_estimator(theta, x, sde_type=sde_type, hidden_features=48, num_layers=3)
    est.net.load_state_dict(sub)
    chk = build_score_estimator(theta, x, sde_type=sde_type, hidden_features=48, num_layers=3).double()
    port = port.double()
    chk._net_call = lambda enc, cond, tenc: port.net(enc, port._embedding_net(cond).expand(enc.shape[0], -1), tenc)
    return est.cuda(), chk, port, theta, x


@pytest.mark.parametrize("sde_type", ["ve", "vp", "subvp"])
@pytest.mark.parametrize("R", [7, 300])
def test_score_forward_and_parameter_gradient_match_oracle(cuda_lib, sde_type, R):
    est, chk, port, theta, x = _pair(sde_type)
    g = torch.Generator().manual_seed(1)
    inp = torch.randn(R, 4, generator=g)
    cond = x[:R] if R <= x.shape[0] else torch.randn(R, 5, generator=g)
    t = torch.rand(R, generator=g) * (est.t_max - est.t_min) + est.t_min
    w = torch.randn(R, 4, generator=g)
    port.zero_grad()
    want = chk(inp.double(), cond.double(), t.double())
    (want * w.double()).sum().backward()
    want_g = est.layout.pack({k: p.grad for k, p in port.named_parameters() if k.startswith("net.")}).double()
    est.net.flat.grad = None
    got = est(inp.cuda(), cond.cuda(), t.cuda())
    (got * w.cuda()).sum().backward()
    scale = max(1.0, want.abs().max().item())
    assert (got.detach().cpu().double() - want.detach()).abs().max() <= 2e-3 * scale
    got_g = est.net.flat.grad.cpu().double() * est.net._mask.cpu().double()
    want_g = want_g * est.net._mask.cpu().double()
    assert (got_g - want_g).abs().max() <= 2e-3 * max(1.0, want_g.abs().max().item())
    # shared condition, shared time: the sampler's call pattern
    with torch.no_grad():
        a = est(inp.cuda(), cond[:1].cuda(), torch.tensor(0.4, device="cuda")).cpu().double()
        b = chk(inp.double(), cond[:1].double(), torch.tensor(0.4, dtype=torch.float64))
    assert (a - b).abs().max() <= 2e-3 * max(1.0, b.abs().max().item())


@pytest.mark.parametrize("sde_type", ["ve", "vp"])
def test_loss_gradient_matches_oracle(cuda_lib, sde_type, monkeypatch):
    """The full denoising-score-matching loss (control variate on) with the same times and noise on both sides."""
    est, chk, port, theta, x = _pair(sde_type)
    R = 128
    g = torch.Generator().manual_seed(4)
    times = torch.rand(R, generator=g) * (est.t_max - est.t_min) + est.t_min
    eps = torch.randn(R, 4, generator=g)
    real = torch.randn_like
    monkeypatch.setattr(torch, "randn_like", lambda t, **k: eps.to(t))
    port.zero_grad()
    want = chk.loss(theta[:R].double(), x[:R].double(), times=times.double())
    want.mean().backward()
    want_g = est.layout.pack({k: p.grad for k, p in port.named_parameters() if k.startswith("net.")}).double()
    est.net.flat.grad = None
    got = est.loss(theta[:R].cuda(), x[:R].cuda(), times=times.cuda())
    got.mean().backward()
    monkeypatch.setattr(torch, "randn_like", real)
    assert torch.allclose(got.detach().cpu().double(), want.detach(), rtol=5e-3, atol=5e-3 * want.abs().max().item())
    m = est.net._mask.cpu().double()
    got_g = est.net.flat.grad.cpu().double() * m
    assert (got_g - want_g * m).abs().max() <= 5e-3 * max(1.0, (want_g * m).abs().max().item())


@pytest.mark.parametrize("sde_type", ["ve", "subvp"])
def test_network_jacobian_diagonal_and_ode_divergence(cuda_lib, sde_type):
    est, chk, port, theta, x = _pair(sde_type)
    R = 33
    g = torch.Generator().manual_seed(2)
    enc = torch.randn(R, 4, generator=g)
    tenc = torch.rand(R, generator=g) + 0.05
    out, diag = est._raw_forward_diag(enc.cuda(), x[:1].cuda().contiguous(), tenc.cuda())
    c1 = port._embedding_net(x[:1].double())
    want = torch.zeros(R, 4, dtype=torch.float64)
    for r in range(R):
        J = torch.autograd.functional.jacobian(lambda e: port.net(e[None], c1, tenc[r:r + 1].double())[0], enc[r].double())
        want[r] = torch.diagonal(J)
    with torch.no_grad():
        want_out = port.net(enc.double(), c1.expand(R, -1), tenc.double())
    assert (out.cpu().double() - want_out).abs().max() <= 2e-3 * max(1.0, want_out.abs().max().item())
    assert (diag.cpu().double() - want).abs().max() <= 2e-3 * max(1.0, want.abs().max().item())
    # the probability-flow ODE's right-hand side and exact divergence
    th = theta[:R]
    t = torch.rand(R, generator=g) * 0.8 + 0.1
    rhs, div = est.ode_fn_and_divergence(th.cuda(), x[:1].cuda(), t.cuda())
    want_div = torch.zeros(R, dtype=torch.float64)
    for r in range(R):
        J = torch.autograd.functional.jacobian(
            lambda y: chk.ode_fn(y[None], x[:1].double(), t[r:r + 1].double())[0], th[r].double())
        want_div[r] = torch.trace(J)
    with torch.no_grad():
        want_rhs = chk.ode_fn(th.double(), x[:1].double(), t.double())
    assert (rhs.cpu().double() - want_rhs).abs().max() <= 3e-3 * max(1.0, want_rhs.abs().max().item())
    assert (div.cpu().double() - want_div).abs().max() <= 3e-3 * max(1.0, want_div.abs().max().item())


@pytest.mark.parametrize("sde_type", ["ve", "vp"])
def test_npse_fits_linear_gaussian(cuda_lib, sde_type):
    """prior N(0, I), x = theta + 0.5 eps  ->  posterior N(x / 1.25, 0.2 I)."""
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPSE
    D, sig = 2, 0.5
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    theta = prior.sample((6000,))
    x = theta + sig * torch.randn_like(theta)
    inf = NPSE(prior, sde_type=sde_type, device="cuda")
    inf.append_simulations(theta, x)
    with pytest.warns(UserWarning, match="Maximum number of epochs"):
        est = inf.train(training_batch_size=500, learning_rate=2e-3, max_num_epochs=150, stop_after_epochs=150)
    assert inf.summary["epochs_trained"][-1] >= 100
    tl = inf.summary["training_loss"]
    assert all(math.isfinite(v) for v in tl) and tl[-1] < tl[0]
    x_o = torch.tensor([0.8, -0.6])
    mu, sd = x_o / (1 + sig ** 2), math.sqrt(sig ** 2 / (1 + sig ** 2))
    post = inf.build_posterior().set_default_x(x_o)
    for how in ("sde", "ode"):
        s = post.sample((4000,), sample_with=how).cpu()
        assert s.shape == (4000, D) and torch.isfinite(s).all()
        print(sde_type, how, "mean", s.mean(0).tolist(), "std", s.std(0).tolist(), "want", mu.tolist(), sd)
        assert (s.mean(0) - mu).abs().max() < 0.16      # measured 0.06 .. 0.10 after 150 epochs (profiles/r02_score_gpu.log)
        assert (s.std(0) / sd - 1).abs().max() < 0.35   # measured 0.00 .. 0.13
    th = mu + sd * torch.randn(200, D)
    lp = post.log_prob(th).cpu()
    want = MultivariateNormal(mu, sd ** 2 * torch.eye(D)).log_prob(th)
    print(sde_type, "log_prob mean abs err", (lp - want).abs().mean().item())
    assert torch.isfinite(lp).all()
    assert (lp - want).abs().mean() < 0.5
    # the device-controlled ODE solve agrees with the host-controlled loop on the same start draws
    from sbi_b200.flowmatching import sample_ode
    torch.manual_seed(3); a = sample_ode(est, 256, x_o.cuda())
    torch.manual_seed(3); b = sample_ode(est, 256, x_o.cuda(), device_control=False)
    assert (a - b).abs().max() < 5e-3
