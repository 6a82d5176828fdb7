"""NRE classifier kernels, potentials and samplers on the GPU against the oracle / analytic targets."""
import math

import numpy as np
import pytest
import torch

from oracle import sbi_port

pytestmark = pytest.mark.gpu


def _ratio_pair(Dt=4, Dx=6, seed=0, perturb=0.1):
    from sbi_b200.ratio import build_resnet_classifier
    g = torch.Generator().manual_seed(seed)
    theta, x = torch.randn(600, Dt, generator=g) + 0.5, 2 * torch.randn(600, Dx, generator=g)
    torch.manual_seed(seed)
    ref = sbi_port.build_resnet_classifier(theta, x)
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(perturb * torch.randn(p.shape, generator=g))
    est = build_resnet_classifier(theta, x)
    est.load_state_dict(ref.state_dict())
    return ref, est.cuda(), theta, x


@pytest.mark.parametrize("Dt,Dx,R", [(4, 6, 300), (10, 10, 4000), (1, 1, 33), (2, 3, 20000)])
def test_ratio_logits_and_grads_match_oracle(cuda_lib, Dt, Dx, R):
    ref, est, theta, x = _ratio_pair(Dt, Dx)
    g0 = torch.Generator().manual_seed(1)
    th, xx = torch.randn(R, Dt, generator=g0), torch.randn(R, Dx, generator=g0)
    w = torch.randn(R, generator=g0)
    def oracle(dtype):
        r = ref.to(dtype)
        r.zero_grad()
        t = th.detach().to(dtype).clone().requires_grad_(True)
        o = r(t, xx.to(dtype))
        (o * w.to(dtype)).sum().backward()
        gp = est.layout.pack({k: p.grad for k, p in r.named_parameters() if k.startswith("net.")}).double()
        return o.detach().double(), gp, t.grad.double()

    o32, gp32, gt32 = oracle(torch.float32)
    o64, gp64, gt64 = oracle(torch.float64)
    tc = th.cuda().requires_grad_(True)
    est.zero_grad()
    out = est(tc, xx.cuda())
    (out * w.cuda()).sum().backward()
    assert (out.detach().cpu().double() - o64).abs().max() <= 1e-3
    # ReLU kinks: a pre-activation within fp32 noise of 0 flips its mask, so gradients are compared with
    # the larger of 2e-3 and 4x the error torch's own fp32 autograd makes against fp64
    for got, r32, r64 in ((est.flat.grad.cpu().double(), gp32, gp64), (tc.grad.cpu().double(), gt32, gt64)):
        sc = r64.abs().max().item()
        err, err32 = (got - r64).abs().max().item() / sc, (r32 - r64).abs().max().item() / sc
        assert err <= max(2e-3, 4 * err32), (err, err32)


def test_nre_b_loss_matches_oracle(cuda_lib):
    from sbi_b200.inference import NRE_B
    ref, est, theta, x = _ratio_pair(3, 3)
    tr = NRE_B(classifier="resnet")
    tr.append_simulations(theta, x)
    tr._x2d = tr._x.reshape(theta.shape[0], -1)
    B, A = 64, 10
    idx = torch.arange(B)
    choices = NRE_B._contrastive_choices(B, A - 1, "cuda")
    c = choices.cpu()
    assert ((c != torch.arange(B)[:, None]).all() and (c >= 0).all() and (c < B).all())
    assert all(len(set(r.tolist())) == A - 1 for r in c)
    loss_ref = sbi_port.nre_b_loss(ref.float(), theta[:B], x[:B], A, choices=c)
    loss = tr._loss_on(est, idx.cuda(), A, choices=choices)
    assert abs(loss.item() - loss_ref.item()) < 1e-4


def test_slice_sampler_gaussian_target(cuda_lib):
    """tests/mcmc_test.py:22-125 analogue: vectorized slice sampling of a correlated 2-D Gaussian."""
    from sbi_b200.samplers import SliceSamplerVectorized
    mean = torch.tensor([1.0, -2.0], device="cuda")
    cov = torch.tensor([[1.0, 0.6], [0.6, 2.0]], device="cuda")
    prec = torch.linalg.inv(cov)

    def logp(p):
        d = p.double() - mean.double()
        return (-0.5 * torch.einsum("ci,ij,cj->c", d, prec.double(), d)).float()

    C = 200
    s = SliceSamplerVectorized(logp, np.zeros((C, 2)), num_chains=C, thin=1, tuning=50, seed=3)
    out = s.run(150)
    assert out.shape == (C, 150, 2)
    flat = torch.from_numpy(out[:, 50:, :].reshape(-1, 2))
    assert (flat.mean(0) - mean.cpu().double()).abs().max() < 0.1
    assert (torch.cov(flat.T) - cov.cpu().double()).abs().max() < 0.2
    # reproducible under a fixed seed
    out2 = SliceSamplerVectorized(logp, np.zeros((C, 2)), num_chains=C, thin=1, tuning=50, seed=3).run(150)
    assert np.array_equal(out, out2)


def test_nle_mcmc_and_nre_rejection_linear_gaussian(cuda_lib):
    """NLE + slice MCMC and NRE-B + rejection on the linear-Gaussian task recover the analytic
    posterior N(x_o/2, 0.05 I) (tests/linearGaussian_snle_test.py:74-131, linearGaussian_snre_test.py:75-136)."""
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NLE, NRE_B
    D = 2
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((6000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    x_o = torch.tensor([[0.3, -0.2]])
    nle = NLE(prior, density_estimator="nsf", device="cuda")
    nle.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=60)
    post = nle.build_posterior(mcmc_parameters=dict(num_chains=200, warmup_steps=50, thin=2))
    s = post.sample((4000,), x=x_o).cpu()
    assert (s.mean(0) - x_o[0] / 2).abs().max() < 0.05
    assert (s.std(0) / math.sqrt(0.05) - 1).abs().max() < 0.2

    nre = NRE_B(prior, classifier="resnet", device="cuda")
    nre.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=40)
    post = nre.build_posterior(sample_with="rejection")
    s = post.sample((2000,), x=x_o).cpu()
    assert (s.mean(0) - x_o[0] / 2).abs().max() < 0.06
    assert (s.std(0) / math.sqrt(0.05) - 1).abs().max() < 0.25


@pytest.mark.parametrize("Dt,Dx,R,shared", [(10, 10, 5000, False), (10, 10, 129, True), (4, 6, 2048, False),
                                            (1, 1, 33, False), (2, 3, 20000, True)])
def test_ratio_tensor_core_matches_simt_and_oracle(cuda_lib, monkeypatch, Dt, Dx, R, shared):
    """Logits through the wgmma kernel (csrc/ratio_tc.cu, 3xTF32) vs the SIMT kernel (<= 2e-4) and
    the fp64 oracle (<= 1e-3, the bar of the SIMT test); pairs given directly, by index, or with a
    shared x."""
    ref, est, theta, x = _ratio_pair(Dt, Dx)
    g0 = torch.Generator().manual_seed(2)
    th = torch.randn(R, Dt, generator=g0)
    xx = torch.randn(1 if shared else R, Dx, generator=g0)
    with torch.no_grad():
        o64 = ref.double()(th.double(), xx.double().expand(R, -1) if shared else xx.double()).double()
    thc, xc = th.cuda(), xx.cuda()
    monkeypatch.setenv("SBI_B200_TC", "0")
    simt = est.logits_raw(thc, xc, x_shared=shared)
    monkeypatch.setenv("SBI_B200_TC", "1")
    tc = est.logits_raw(thc, xc, x_shared=shared)
    assert est._tc_state(est._model(nbuf=2)) is not None
    assert torch.isfinite(tc).all()
    assert (tc - simt).abs().max() <= 2e-4
    assert (tc.cpu().double() - o64.reshape(-1)).abs().max() <= 1e-3
    if not shared:
        ti = torch.randperm(R, device="cuda")[: R // 2]
        xi = torch.randperm(R, device="cuda")[: R // 2]
        a = est.logits_raw(thc, xc, ti, xi)
        monkeypatch.setenv("SBI_B200_TC", "0")
        b = est.logits_raw(thc, xc, ti, xi)
        assert (a - b).abs().max() <= 2e-4


def test_single_chain_slice_sampler_interface(cuda_lib):
    """`SliceSampler(x, lp_f).gen(n)` (slice_numpy.py:57-216): numpy in / numpy out, one chain;
    1-D standard-normal-ish target N(1, 0.5^2) x N(-2, 2^2)."""
    from sbi_b200.samplers import SliceSampler
    mu, sd = np.array([1.0, -2.0]), np.array([0.5, 2.0])
    calls = []

    def lp_f(p):
        assert isinstance(p, np.ndarray) and p.shape == (2,)
        calls.append(1)
        return float(-0.5 * (((p - mu) / sd) ** 2).sum())

    smp = SliceSampler(np.zeros(2), lp_f, tuning=50, thin=2, seed=7)
    out = smp.gen(1500)
    assert out.shape == (1500, 2) and np.isfinite(out).all()
    assert np.abs(out[200:].mean(0) - mu).max() < 0.35
    assert np.abs(out[200:].std(0) / sd - 1).max() < 0.3
    assert np.allclose(smp.x, out[-1])
    assert len(calls) > 1500


def test_reject_compact_kernel_equals_boolean_indexing(cuda_lib):
    """csrc/compact.cu: accepted rows, their order and their global indices equal `candidates[keep]` /
    `nonzero(keep)` of the reference expression (rejection.py:178-181), across two appended batches and with
    the capacity cut."""
    from sbi_b200 import _lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(0)
    D, cap = 10, 400_000
    out = torch.full((cap, D), float("nan"), device="cuda")
    out_idx = torch.full((cap,), -1, dtype=torch.int64, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    want_rows, want_idx, base = [], [], 0
    for n in (1_000_037, 300_001):
        cand = torch.randn(n, D, generator=g).cuda()
        lt = torch.randn(n, generator=g).cuda()
        ls = (torch.randn(n, generator=g) + 1.0).cuda()
        lt[::1000] = float("nan")
        u = torch.rand(n, generator=g).cuda()
        scratch = torch.empty(int(lib.sbi_b200_reject_scratch_ints(n)), dtype=torch.int32, device="cuda")
        L.check(lib.sbi_b200_reject_compact(cand.data_ptr(), D, lt.data_ptr(), ls.data_ptr(), u.data_ptr(), n, base,
                                            out.data_ptr(), out_idx.data_ptr(), cap, count.data_ptr(),
                                            scratch.data_ptr(), L.stream_ptr()), "reject_compact")
        keep = torch.exp(lt - ls) > u
        want_rows.append(cand[keep])
        want_idx.append(torch.nonzero(keep).reshape(-1) + base)
        base += n
    want_rows, want_idx = torch.cat(want_rows), torch.cat(want_idx)
    assert int(count.item()) == want_rows.shape[0] > cap          # overflow is counted, not stored
    assert torch.equal(out, want_rows[:cap]) and torch.equal(out_idx, want_idx[:cap])
