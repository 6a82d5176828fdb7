"""Tensor-core training step (csrc/nsf_tc.cu forward with activation save + csrc/nsf_vjp_tc.cu backward;
wgmma for every conditioner linear: forward, input gradient and weight gradient) against the fp64
oracle autograd, against the SIMT VJP kernel, and as a training step."""
import ctypes as C
import math
import os

import pytest
import torch

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu
GRAD_TOL = 2e-3


def _oracle_param_grads(flow, est, inp, cond, g, dtype):
    flow = flow.to(dtype)
    flow.zero_grad()
    lp = flow.log_prob(inp.to(dtype), cond.to(dtype))[0]
    (lp * g.to(dtype)).sum().backward()
    return est.layout.pack({k: p.grad for k, p in flow.named_parameters()}).double(), lp.detach().double()


def _grads(est, inp, cond, g, tc: bool):
    """(flat parameter gradient, log-probs, loss statistics) through est.vjp + reduce_partials."""
    from sbi_b200 import _lib as L
    lib = L.load()
    os.environ["SBI_B200_VJP_TC"] = "1" if tc else "0"
    est._cache.pop("tc_train", None)
    R = inp.shape[0]
    P = est.layout.n_params
    n_part = est.vjp_parts(R)
    gpart = torch.full((n_part, P), float("nan"), device="cuda")       # every entry must be written
    lp = torch.empty(R, device="cuda")
    acc = torch.zeros(2, device="cuda")
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    est.vjp(m, rows, R, g, 0.0, lp, gpart, None, None, acc)
    grad = torch.empty(P, device="cuda")
    L.check(lib.sbi_b200_reduce_partials(L.ptr(gpart), n_part, P, L.ptr(grad), L.stream_ptr()), "reduce")
    torch.cuda.synchronize()
    os.environ.pop("SBI_B200_VJP_TC", None)
    return grad.cpu().double(), lp.cpu().double(), acc.cpu(), n_part


@pytest.mark.parametrize("D,C,R", [(10, 10, 128), (10, 10, 300), (10, 10, 4096), (3, 2, 77), (2, 2, 1000),
                                   (5, 7, 640), (10, 10, 20000)])
def test_vjp_tc_matches_oracle_and_simt(cuda_lib, D, C, R):
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500))
    est = b200_from_oracle(flow, theta, x)
    inp, cond = (theta[:R] * 1.3).float().cuda().contiguous(), x[:R].float().cuda().contiguous()
    g = torch.randn(R, dtype=torch.float64)
    gc = g.float().cuda()
    got, lp, acc, n_part = _grads(est, inp, cond, gc, tc=True)
    simt, lp_s, acc_s, _ = _grads(est, inp, cond, gc, tc=False)
    assert n_part == min((R + 127) // 128, torch.cuda.get_device_properties(0).multi_processor_count)
    assert torch.isfinite(got).all()
    mask = est.net._mask.cpu().bool()
    assert (got[~mask] == 0).all(), "padding entries must receive zero gradient"
    ref64, lp64 = _oracle_param_grads(flow, est, inp.cpu(), cond.cpu(), g, torch.float64)
    ref32, _ = _oracle_param_grads(flow, est, inp.cpu(), cond.cpu(), g, torch.float32)
    scale = ref64.abs().max().item()
    err = (got - ref64).abs().max().item() / scale
    err_s = (simt - ref64).abs().max().item() / scale
    err32 = (ref32 - ref64).abs().max().item() / scale
    print(f"D={D} C={C} R={R}: tensor-core grad rel err {err:.3e} (SIMT kernel {err_s:.3e}, torch-fp32 {err32:.3e}); "
          f"logp err {(lp - lp64).abs().max().item():.3e}")
    assert (lp - lp64).abs().max() <= 2e-3
    assert err <= max(GRAD_TOL, 4 * err32)
    # loss statistics: sum of -log q, no non-finite rows
    assert abs(acc[0].item() + lp64.sum().item()) <= 2e-3 * R and acc[1].item() == 0
    assert abs(acc[0].item() - acc_s[0].item()) <= 1e-3 * R


def test_vjp_tc_kernels_are_the_ones_that_run(cuda_lib):
    """Default dispatch: from 256 rows (two tiles) the trainer's VJP is the tensor-core pair."""
    flow, theta, x = oracle_nsf(10, 10, n=5000)
    est = b200_from_oracle(flow, theta, x)
    os.environ.pop("SBI_B200_VJP_TC", None)
    assert est._vjp_uses_tc(4096, True) and not est._vjp_uses_tc(4096, False) and not est._vjp_uses_tc(100, True)
    # autograd with input gradients falls back to the SIMT kernel and still works
    inp = theta[:2048].cuda().requires_grad_(True)
    (est.log_prob(inp, x[:2048].cuda())[0]).sum().backward()
    assert inp.grad is not None and torch.isfinite(est.flat.grad).all()
    # parameter-only autograd at 2048 rows goes through the tensor-core path
    est.zero_grad()
    a = est.flat.grad
    est.log_prob(theta[:2048].cuda(), x[:2048].cuda())[0].sum().backward()
    g_tc = est.flat.grad.clone()
    os.environ["SBI_B200_VJP_TC"] = "0"
    est._cache.pop("tc_train", None)
    est.zero_grad()
    est.log_prob(theta[:2048].cuda(), x[:2048].cuda())[0].sum().backward()
    os.environ.pop("SBI_B200_VJP_TC", None)
    sc = est.flat.grad.abs().max()
    assert (g_tc - est.flat.grad).abs().max() <= 2e-3 * sc


def test_training_with_the_tensor_core_step_fits_the_posterior(cuda_lib):
    """NPE on the linear-Gaussian task with batch 2048 (tensor-core step inside the epoch graph)."""
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPE
    D = 3
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((40_000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    inf = NPE(prior, density_estimator="nsf", device="cuda")
    est = inf.append_simulations(theta, x).train(training_batch_size=2048, max_num_epochs=40)
    assert est._vjp_uses_tc(2048, True)
    vl = inf.summary["validation_loss"]
    assert vl[-1] < vl[0] - 0.5
    x_o = torch.tensor([[0.3, -0.2, 0.1]])
    s = inf.build_posterior().sample((4000,), x=x_o).cpu()
    assert (s.mean(0) - x_o[0] / 2).abs().max() < 0.05
    assert (s.std(0) / math.sqrt(0.05) - 1).abs().max() < 0.2
