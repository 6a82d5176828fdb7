"""Training-path parity on the GPU: the fused step vs the oracle step (the optimiser kernels alone are in
test_optim_gpu.py), and an end-to-end NPE fit against the analytic posterior."""
import ctypes as C
import math

import pytest
import torch
from torch.nn.utils.clip_grad import clip_grad_norm_

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu


def test_fused_train_step_with_scratch_matches_oracle_step(cuda_lib):
    """One full optimisation step (loss -> backward with an activation scratch -> clip -> Adam) against the
    oracle."""
    from sbi_b200 import _lib as L
    flow, theta, x = oracle_nsf(10, 10, n=2000)
    est = b200_from_oracle(flow, theta, x)
    B = 512
    lay = est.layout
    P = lay.n_params
    opt = torch.optim.Adam(list(flow.parameters()), lr=5e-4)
    grad = torch.zeros(P, device="cuda")
    state = torch.zeros(2 * P, device="cuda")
    step = torch.zeros(2, dtype=torch.int32, device="cuda")
    loss_acc = torch.zeros(2, device="cuda")
    n_part = cuda_lib.sbi_b200_nsf_vjp_parts(B)
    gpart = est._gpart(n_part)
    save = torch.empty(cuda_lib.sbi_b200_nsf_vjp_save_bytes(C.byref(est._model(nbuf=3)), B) // 4, device="cuda")
    th_d, x_d = theta.cuda(), x.cuda()
    for it in range(3):
        idx = torch.randperm(2000)[:B]
        opt.zero_grad()
        losses = flow.loss(theta[idx], x[idx])
        losses.mean().backward()
        clip_grad_norm_(flow.parameters(), max_norm=5.0)
        gref = lay.pack({k: p.grad for k, p in flow.named_parameters()})
        opt.step()
        m = est._model(nbuf=3)
        idx_d = idx.cuda()
        rows = L.Rows(th_d.data_ptr(), x_d.data_ptr(), idx_d.data_ptr(), B, 0)
        loss_acc.zero_()
        L.check(cuda_lib.sbi_b200_nsf_vjp(C.byref(m), C.byref(rows), None, -1.0 / B, None, L.ptr(gpart), None,
                                          None, L.ptr(loss_acc), L.ptr(save), save.numel() * 4, L.stream_ptr()), "vjp")
        L.check(cuda_lib.sbi_b200_reduce_partials(L.ptr(gpart), n_part, P, L.ptr(grad), L.stream_ptr()), "red")
        # unclipped gradient parity (the oracle's was clipped in place: compare direction + norm)
        g = grad.cpu()
        cos = torch.dot(g, gref) / (g.norm() * gref.norm())
        assert cos > 1 - 1e-5
        L.check(cuda_lib.sbi_b200_adam_clip_step(L.ptr(est.flat.data), L.ptr(grad), L.ptr(state), L.ptr(step),
                                                 L.ptr(est.net._mask), P, 5e-4, 0.9, 0.999, 1e-8, 5.0, 1.0,
                                                 L.stream_ptr()), "adam")
        assert abs(loss_acc[0].item() / B - losses.mean().item()) < 2e-3
        assert loss_acc[1].item() == 0
    ref_flat = lay.pack(flow.state_dict())
    diff = (est.flat.detach().cpu() - ref_flat).abs()
    # Adam normalises the step to ~lr per entry: an entry whose gradient is fp32-noise can move
    # by up to 2*lr in the opposite direction; everything else must agree closely.
    assert diff.max() <= 3 * 2 * 5e-4 + 1e-6
    assert (diff > 5e-5).float().mean() < 0.02


def test_train_step_host_entry_matches_device_step(cuda_lib):
    """Host-buffer C-ABI step == device-resident step on the same batch: the workspace has no activation
    scratch, so the host step recomputes where the device step spills, bit-identically."""
    from sbi_b200 import _lib as L
    flow, theta, x = oracle_nsf(10, 10, n=1000)
    outs = []
    for mode in ("device", "host"):
        est = b200_from_oracle(flow, theta, x)
        lay = est.layout
        P, B = lay.n_params, 300
        grad = torch.zeros(P, device="cuda"); state = torch.zeros(2 * P, device="cuda")
        step = torch.zeros(2, dtype=torch.int32, device="cuda"); loss_acc = torch.zeros(2, device="cuda")
        n_part = cuda_lib.sbi_b200_nsf_vjp_parts(B)
        gpart = est._gpart(n_part)
        m = est._model(nbuf=3)
        if mode == "device":
            th_d, x_d = theta[:B].cuda(), x[:B].cuda()
            rows = L.Rows(th_d.data_ptr(), x_d.data_ptr(), None, B, 0)
            save = torch.empty(cuda_lib.sbi_b200_nsf_vjp_save_bytes(C.byref(m), B) // 4, device="cuda")
            L.check(cuda_lib.sbi_b200_nsf_vjp(C.byref(m), C.byref(rows), None, -1.0 / B, None, L.ptr(gpart),
                                              None, None, L.ptr(loss_acc), L.ptr(save), save.numel() * 4,
                                              L.stream_ptr()), "vjp")
            L.check(cuda_lib.sbi_b200_reduce_partials(L.ptr(gpart), n_part, P, L.ptr(grad), L.stream_ptr()), "r")
            L.check(cuda_lib.sbi_b200_adam_clip_step(L.ptr(est.flat.data), L.ptr(grad), L.ptr(state), L.ptr(step),
                                                     L.ptr(est.net._mask), P, 5e-4, 0.9, 0.999, 1e-8, 5.0, 1.0,
                                                     L.stream_ptr()), "adam")
            loss = loss_acc.cpu()
        else:
            ws = L.TrainWs()
            st_in = torch.empty(B, 10, device="cuda"); st_c = torch.empty(B, 10, device="cuda")
            st_lp = torch.empty(B, device="cuda")
            ws.d_input, ws.d_cond, ws.d_logp = st_in.data_ptr(), st_c.data_ptr(), st_lp.data_ptr()
            ws.d_gpart, ws.d_grad, ws.d_state = gpart.data_ptr(), grad.data_ptr(), state.data_ptr()
            ws.d_step, ws.d_mask, ws.d_loss_acc = step.data_ptr(), est.net._mask.data_ptr(), loss_acc.data_ptr()
            ws.cap_rows = B
            h_th, h_x = theta[:B].contiguous().pin_memory(), x[:B].contiguous().pin_memory()
            h_loss = torch.zeros(2).pin_memory()
            L.check(cuda_lib.sbi_b200_nsf_train_step_host(C.byref(m), C.byref(ws), h_th.data_ptr(), h_x.data_ptr(),
                                                          B, 5e-4, 0.9, 0.999, 1e-8, 5.0, h_loss.data_ptr(),
                                                          L.stream_ptr()), "host step")
            loss = h_loss.clone()
            h_lp = torch.empty(B).pin_memory()
            L.check(cuda_lib.sbi_b200_nsf_logprob_host(C.byref(m), C.byref(ws), h_th.data_ptr(), h_x.data_ptr(), B, 0,
                                                       h_lp.data_ptr(), L.stream_ptr()), "host logprob")
            assert torch.isfinite(h_lp).all()
        outs.append((est.flat.detach().cpu().clone(), loss))
    assert torch.equal(outs[0][0], outs[1][0])
    # the loss sum is accumulated with float atomics across CTAs: order-dependent last bits
    assert torch.allclose(outs[0][1], outs[1][1], rtol=1e-5)


def test_pipelined_host_steps_equal_blocking_steps(cuda_lib):
    """sbi_b200_nsf_train_step_host_async (result one step late) == the blocking host step."""
    from sbi_b200 import _lib as L
    flow, theta, x = oracle_nsf(6, 4, n=2000)
    B, nsteps = 256, 5
    finals, losses = [], []
    for mode in ("blocking", "pipelined"):
        est = b200_from_oracle(flow, theta, x)
        P = est.layout.n_params
        grad = torch.zeros(P, device="cuda"); state = torch.zeros(2 * P, device="cuda")
        step = torch.zeros(2, dtype=torch.int32, device="cuda"); loss_acc = torch.zeros(2, device="cuda")
        gpart = est._gpart(cuda_lib.sbi_b200_nsf_vjp_parts(B))
        ws = L.TrainWs()
        st_in = torch.empty(B, 6, device="cuda"); st_c = torch.empty(B, 4, device="cuda"); st_lp = torch.empty(B, device="cuda")
        ws.d_input, ws.d_cond, ws.d_logp = st_in.data_ptr(), st_c.data_ptr(), st_lp.data_ptr()
        ws.d_gpart, ws.d_grad, ws.d_state = gpart.data_ptr(), grad.data_ptr(), state.data_ptr()
        ws.d_step, ws.d_mask, ws.d_loss_acc = step.data_ptr(), est.net._mask.data_ptr(), loss_acc.data_ptr()
        ws.cap_rows = B
        bufs = [(torch.empty(B, 6).pin_memory(), torch.empty(B, 4).pin_memory()) for _ in range(2)]
        out = torch.zeros(2).pin_memory()
        pipe = cuda_lib.sbi_b200_pipe_create()
        ls = []
        for i in range(nsteps):
            a, b = bufs[i & 1]
            a.copy_(theta[i * B:(i + 1) * B]); b.copy_(x[i * B:(i + 1) * B])
            m = est._model(nbuf=3)
            if mode == "blocking":
                L.check(cuda_lib.sbi_b200_nsf_train_step_host(C.byref(m), C.byref(ws), a.data_ptr(), b.data_ptr(), B,
                                                              5e-4, 0.9, 0.999, 1e-8, 5.0, out.data_ptr(), L.stream_ptr()), "s")
                ls.append(out[0].item())
            else:
                L.check(cuda_lib.sbi_b200_nsf_train_step_host_async(C.byref(m), C.byref(ws), pipe, a.data_ptr(), b.data_ptr(),
                                                                    B, 5e-4, 0.9, 0.999, 1e-8, 5.0, out.data_ptr(),
                                                                    L.stream_ptr()), "a")
                if i > 0:
                    ls.append(out[0].item())
                else:
                    assert math.isnan(out[0].item())
        if mode == "pipelined":
            L.check(cuda_lib.sbi_b200_pipe_drain(pipe, out.data_ptr()), "drain")
            ls.append(out[0].item())
        cuda_lib.sbi_b200_pipe_destroy(pipe)
        finals.append(est.flat.detach().cpu().clone())
        losses.append(ls)
    assert torch.equal(finals[0], finals[1])
    assert losses[0] == pytest.approx(losses[1], rel=1e-5)


def test_npe_fit_linear_gaussian(cuda_lib):
    """NPE + nsf on the linear-Gaussian task recovers the analytic posterior
    (reference acceptance test: tests/linearGaussian_snpe_test.py:53-152, c2st/KL checks)."""
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPE
    from sbi_b200.neural_nets import posterior_nn
    D = 3
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    theta = prior.sample((6000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)
    inf = NPE(prior, density_estimator=posterior_nn("nsf"), device="cuda")
    est = inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=60)
    s = inf.summary
    assert s["validation_loss"][-1] < s["validation_loss"][0] - 0.3
    post = inf.build_posterior()
    x_o = torch.tensor([[0.3, -0.2, 0.1]])
    samples = post.sample((4000,), x=x_o).cpu()
    # analytic posterior: N(x_o/2, 0.05 I)
    assert (samples.mean(0) - x_o[0] / 2).abs().max() < 0.04
    assert (samples.std(0) / math.sqrt(0.05) - 1).abs().max() < 0.2
    lp = post.log_prob(samples[:500].cuda(), x=x_o).cpu()
    true = MultivariateNormal(x_o[0] / 2, 0.05 * torch.eye(D)).log_prob(samples[:500])
    assert (lp - true).mean().abs() < 0.25


def test_calibration_kernel_weights_the_loss(cuda_lib):
    """npe_base.py:373-378, :563-575: loss_r = calibration_kernel(x_r) * (-log q_r).  A constant kernel of
    2 doubles the logged losses of the same run; a Gaussian kernel around x_o trains and stays finite."""
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NPE
    D = 3
    prior = MultivariateNormal(torch.zeros(D), 0.1 * torch.eye(D))
    torch.manual_seed(0)
    theta = prior.sample((6000,))
    x = theta + math.sqrt(0.1) * torch.randn_like(theta)

    def run(kernel):
        torch.manual_seed(1)
        inf = NPE(prior, density_estimator="nsf", device="cuda")
        inf.append_simulations(theta, x).train(training_batch_size=500, max_num_epochs=3, calibration_kernel=kernel)
        return inf.summary

    base = run(None)
    twice = run(lambda xx: 2.0 * torch.ones(xx.shape[0], device=xx.device))
    assert abs(twice["training_loss"][0] - 2 * base["training_loss"][0]) < 1e-3 * abs(base["training_loss"][0])
    assert abs(twice["validation_loss"][0] - 2 * base["validation_loss"][0]) < 2e-2 * abs(base["validation_loss"][0])
    x_o = torch.tensor([0.3, -0.2, 0.1])
    local = run(lambda xx: torch.exp(-((xx - x_o.to(xx.device)) ** 2).sum(-1) / 0.5))
    assert all(math.isfinite(v) for v in local["training_loss"] + local["validation_loss"])
    assert local["validation_loss"][-1] < local["validation_loss"][0]
