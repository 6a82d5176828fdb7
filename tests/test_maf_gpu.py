"""Parity of the sm_90a MAF kernels (BASELINE configs[0]: posterior_nn='maf', dim 3) against the
CPU oracle, through the C ABI.  Tolerances as in test_nsf_gpu.py."""
import math

import pytest
import torch

from tests.helpers import b200_maf_from_oracle, oracle_maf

pytestmark = pytest.mark.gpu
LOGP_TOL, GRAD_TOL = 2e-3, 2e-3


@pytest.mark.parametrize("D,C,R", [(3, 2, 200), (3, 3, 1000), (10, 10, 257), (2, 1, 31), (6, 4, 20000)])
def test_maf_logprob_matches_oracle(cuda_lib, D, C, R):
    flow, theta, x = oracle_maf(D, C, n=max(R, 500))
    est = b200_maf_from_oracle(flow, theta, x)
    inp, cond = theta[:R] * 1.5, x[:R]
    with torch.no_grad():
        ref64 = flow.double().log_prob(inp.double(), cond.double())[0]
        ref32 = flow.float().log_prob(inp, cond)[0]
        got = est.log_prob(inp.cuda(), cond.cuda())[0].cpu()
        ref_sh = flow.double().log_prob(inp[:50].double().unsqueeze(1), cond[:1].double())[:, 0]
        got_sh = est.log_prob(inp[:50].cuda().unsqueeze(1), cond[:1].cuda())[:, 0].cpu()
    err = (got.double() - ref64).abs().max().item()
    print(f"maf D={D} C={C} R={R}: kernel err {err:.3e} torch-fp32 err {(ref32.double() - ref64).abs().max().item():.3e}")
    assert err <= LOGP_TOL and (got_sh.double() - ref_sh).abs().max() <= LOGP_TOL


def test_maf_sigmoid_scale_variant(cuda_lib):
    flow, theta, x = oracle_maf(4, 3, scale_fn="sigmoid")
    est = b200_maf_from_oracle(flow, theta, x, scale_fn="sigmoid")
    with torch.no_grad():
        ref = flow.double().log_prob(theta[:300].double(), x[:300].double())[0]
        got = est.log_prob(theta[:300].cuda(), x[:300].cuda())[0].cpu()
    oracle_maf(2, 2, n=10)   # restore the default scale fn for later tests
    assert (got.double() - ref).abs().max() <= LOGP_TOL


def _grads(flow, est, inp, cond, g, dtype):
    flow = flow.to(dtype)
    flow.zero_grad()
    i = inp.to(dtype).detach().requires_grad_(True)
    c = cond.to(dtype).detach().requires_grad_(True)
    (flow.log_prob(i, c)[0] * g.to(dtype)).sum().backward()
    sd = {k: p.grad for k, p in flow.named_parameters()}
    return est.layout.pack(sd).double(), i.grad.double(), c.grad.double()


@pytest.mark.parametrize("D,C,R", [(3, 2, 200), (10, 10, 300), (2, 1, 31), (3, 3, 4096)])
def test_maf_vjp_matches_oracle_autograd(cuda_lib, D, C, R):
    flow, theta, x = oracle_maf(D, C, n=max(R, 500))
    est = b200_maf_from_oracle(flow, theta, x)
    inp, cond = theta[:R] * 1.3, x[:R]
    g = torch.randn(R, dtype=torch.float64)
    ref32 = _grads(flow, est, inp, cond, g, torch.float32)
    ref64 = _grads(flow, est, inp, cond, g, torch.float64)
    inp_c = inp.float().cuda().requires_grad_(True)
    cond_c = cond.float().cuda().requires_grad_(True)
    est.zero_grad()
    (est.log_prob(inp_c, cond_c)[0] * g.float().cuda()).sum().backward()
    got = (est.flat.grad.cpu().double(), inp_c.grad.cpu().double(), cond_c.grad.cpu().double())
    mask = est.net._mask.cpu().bool()
    # the kernels compute dense weight gradients; masked-out entries are frozen by the Adam mask and
    # must be ignored here exactly like nflows' `weight * mask` zeroes them
    for name, a, r32, r64 in zip(("param", "input", "cond"), got, ref32, ref64):
        if name == "param":
            a = a * mask
        scale = r64.abs().max().item()
        err = (a - r64).abs().max().item() / scale
        err32 = (r32 - r64).abs().max().item() / scale
        print(f"maf D={D} R={R} {name}-grad rel err {err:.3e} (torch-fp32 {err32:.3e})")
        assert err <= max(GRAD_TOL, 4 * err32), name


@pytest.mark.parametrize("D,C,R,B", [(3, 2, 500, 1), (10, 10, 100, 3), (2, 1, 20000, 1)])
def test_maf_inverse_matches_oracle(cuda_lib, D, C, R, B):
    flow, theta, x = oracle_maf(D, C)
    est = b200_maf_from_oracle(flow, theta, x)
    noise = torch.randn(B * R, D, generator=torch.Generator().manual_seed(5))
    cond = x[:B]
    with torch.no_grad():
        ctx = flow.net._embedding_net(cond.double()).repeat_interleave(R, dim=0)
        ref, ld_ref = flow.double().net._transform.inverse(noise.double(), context=ctx)
        got, ld = est.inverse_flow(noise.cuda(), cond.cuda(), R)
    err = (got.cpu().double() - ref).abs().max().item()
    eld = (ld.cpu().double() - ld_ref).abs().max().item()
    print(f"maf inverse D={D}: x err {err:.3e} logabsdet err {eld:.3e}")
    assert err <= 2e-3 and eld <= 5e-3


def test_npe_maf_linear_gaussian_cfg0(cuda_lib):
    """BASELINE configs[0] shape (tests/linearGaussian_snpe_test.py:312-372): theta-dim 3, x-dim 2,
    maf; here trained on the device-resident path and checked against the analytic posterior."""
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPE
    torch.manual_seed(0)
    D = 3
    prior = MultivariateNormal(torch.zeros(D), torch.eye(D))
    theta = prior.sample((4000,))
    # x = first two coordinates of theta, shifted, plus noise (likelihood cov 0.3 I)
    x = theta[:, :2] - 1.0 + math.sqrt(0.3) * torch.randn(4000, 2)
    inf = NPE(prior, density_estimator="maf", device="cuda")
    inf.append_simulations(theta, x).train(training_batch_size=200, max_num_epochs=150)
    post = inf.build_posterior()
    x_o = torch.zeros(1, 2)
    s = post.sample((4000,), x=x_o).cpu()
    # analytic: for the observed coords, posterior var = 0.3/1.3, mean = (x_o + 1) / 1.3; third coord = prior
    m = (x_o[0] + 1.0) / 1.3
    assert (s[:, :2].mean(0) - m).abs().max() < 0.1
    assert (s[:, :2].std(0) / math.sqrt(0.3 / 1.3) - 1).abs().max() < 0.2
    assert abs(s[:, 2].mean()) < 0.1 and abs(s[:, 2].std() - 1) < 0.15
