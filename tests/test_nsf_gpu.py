"""Parity of the sm_90a NSF kernels against the CPU oracle (through the C ABI).

Tolerances (fp32 kernels vs. the fp64 oracle; the fp32 oracle's own error against fp64 is
printed next to it):  |dlogp| <= 2e-3 absolute on log-probs of magnitude O(10..50),
samples |dx| <= 2e-3, parameter gradients <= 2e-3 relative to the gradient's max-norm.
"""
import pytest
import torch

from tests.helpers import b200_from_oracle, nsf_vjp_raw, oracle_nsf

pytestmark = pytest.mark.gpu

LOGP_TOL = 2e-3
GRAD_TOL = 2e-3


def _flat_grad_from_oracle(est, flow):
    sd = {k: p.grad for k, p in flow.named_parameters()}
    return est.layout.pack(sd)


@pytest.mark.parametrize("D,C,R", [(10, 10, 257), (2, 2, 64), (3, 2, 1000), (10, 10, 20000), (5, 7, 33)])
def test_logprob_matches_oracle(cuda_lib, D, C, R):
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500))
    est = b200_from_oracle(flow, theta, x)
    inp, cond = theta[:R] * 1.5, x[:R]        # some rows leave [-3,3] -> linear tails
    with torch.no_grad():
        ref64 = flow.double().log_prob(inp.double(), cond.double())[0]
        ref32 = flow.float().log_prob(inp, cond)[0]
        got = est.log_prob(inp.cuda(), cond.cuda())[0].cpu()
    err = (got.double() - ref64).abs().max().item()
    err32 = (ref32.double() - ref64).abs().max().item()
    print(f"D={D} C={C} R={R}: kernel err {err:.3e}  torch-fp32 err {err32:.3e}")
    assert torch.isfinite(got).all()
    assert err <= LOGP_TOL


def test_logprob_shared_condition_and_noise(cuda_lib):
    flow, theta, x = oracle_nsf(10, 10)
    est = b200_from_oracle(flow, theta, x)
    xo = x[:1]
    with torch.no_grad():
        ref = flow.double().log_prob(theta[:300].double().unsqueeze(1), xo.double())[:, 0]
        got = est.log_prob(theta[:300].cuda().unsqueeze(1), xo.cuda())[:, 0].cpu()
        z_ref = flow.inverse_transform(theta[:300].double(), xo.double())   # raw condition, like the reference
        z = est.inverse_transform(theta[:300].cuda(), xo.cuda()).cpu()
    assert (got.double() - ref).abs().max() <= LOGP_TOL
    assert (z.double() - z_ref).abs().max() <= 1e-3


def _oracle_grads(flow, est, inp, cond, g, dtype):
    flow = flow.to(dtype)
    flow.zero_grad()
    i = inp.to(dtype).detach().requires_grad_(True)
    c = cond.to(dtype).detach().requires_grad_(True)
    lp = flow.log_prob(i, c)[0]
    (lp * g.to(dtype)).sum().backward()
    return _flat_grad_from_oracle(est, flow).double(), i.grad.double(), c.grad.double()


@pytest.mark.parametrize("D,C,R", [(10, 10, 256), (3, 2, 77), (2, 2, 31), (10, 10, 4096)])
def test_vjp_matches_oracle_autograd(cuda_lib, D, C, R):
    """Gradients wrt parameters, inputs and conditions vs the fp64 oracle autograd.  The bar is
    GRAD_TOL of the gradient's max-norm, or 4x the error torch's own fp32 autograd makes against
    fp64 on the same problem, whichever is larger (a few rows sit on steep spline segments
    where fp32 itself loses digits)."""
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500))
    est = b200_from_oracle(flow, theta, x)
    inp, cond = theta[:R] * 1.3, x[:R]
    g = torch.randn(R, dtype=torch.float64)
    ref32 = _oracle_grads(flow, est, inp, cond, g, torch.float32)
    ref64 = _oracle_grads(flow, est, inp, cond, g, torch.float64)

    inp_c = inp.float().cuda().requires_grad_(True)
    cond_c = cond.float().cuda().requires_grad_(True)
    est.zero_grad()
    lpc = est.log_prob(inp_c, cond_c)[0]
    (lpc * g.float().cuda()).sum().backward()
    got = (est.flat.grad.cpu().double(), inp_c.grad.cpu().double(), cond_c.grad.cpu().double())
    mask = est.net._mask.cpu().bool()
    assert (got[0][~mask] == 0).all(), "padding entries must receive zero gradient"
    for name, a, r32, r64 in zip(("param", "input", "cond"), got, ref32, ref64):
        scale = r64.abs().max().item()
        err = (a - r64).abs().max().item() / scale
        err32 = (r32 - r64).abs().max().item() / scale
        print(f"D={D} R={R} {name}-grad: kernel rel err {err:.3e}  torch-fp32 rel err {err32:.3e}")
        assert err <= max(GRAD_TOL, 4 * err32), name


@pytest.mark.parametrize("D,C,R,B", [(10, 10, 1000, 1), (3, 2, 50, 4), (2, 2, 20000, 1)])
def test_inverse_matches_oracle(cuda_lib, D, C, R, B):
    flow, theta, x = oracle_nsf(D, C)
    est = b200_from_oracle(flow, theta, x)
    g = torch.Generator().manual_seed(5)
    noise = torch.randn(B * R, D, generator=g)
    cond = x[:B]
    with torch.no_grad():
        emb = flow.net._embedding_net(cond.double())
        ctx = emb.repeat_interleave(R, dim=0)
        ref, ld_ref = flow.double().net._transform.inverse(noise.double(), context=ctx)
        got, ld = est.inverse_flow(noise.cuda(), cond.cuda(), R)
    err = (got.cpu().double() - ref).abs().max().item()
    eld = (ld.cpu().double() - ld_ref).abs().max().item()
    print(f"inverse D={D}: x err {err:.3e}  logabsdet err {eld:.3e}")
    assert err <= 2e-3 and eld <= 5e-3


def test_sample_shapes_and_roundtrip(cuda_lib):
    flow, theta, x = oracle_nsf(10, 10)
    est = b200_from_oracle(flow, theta, x)
    cond = x[:3].cuda()
    s = est.sample((7, 2), cond)
    assert s.shape == (7, 2, 3, 10)
    # shapes for several conditions follow the reference (nflows_flow.py:130-151, which reshapes
    # nflows' (B, n, D) without transposing); value round trip is checked for one condition
    s3, lp3 = est.sample_and_log_prob(torch.Size((50,)), cond)
    assert s3.shape == (50, 3, 10) and lp3.shape == (50, 3)
    s2, lp2 = est.sample_and_log_prob(torch.Size((500,)), cond[:1])
    lp = est.log_prob(s2, cond[:1])
    assert (lp - lp2).abs().max() <= 5e-3
    # samples of sample() belong to their condition: log_prob under the right condition is finite
    assert torch.isfinite(est.log_prob(s.reshape(14, 3, 10), cond)).all()


def _seeded_batch(R, seed=0, D=10, C=10):
    """An estimator and R of its rows on the GPU, with a seeded upstream gradient per row."""
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500), seed=seed)
    est = b200_from_oracle(flow, theta, x)
    w = torch.randn(R, generator=torch.Generator().manual_seed(9))
    return est, theta[:R].float().cuda().contiguous(), x[:R].float().cuda().contiguous(), w.cuda()


def _scratch(est, R):
    import ctypes as C
    from sbi_b200 import _lib as L
    nbytes = L.load().sbi_b200_nsf_vjp_save_bytes(C.byref(est._model(nbuf=3)), R)
    assert nbytes > 0 and nbytes % 4 == 0
    return torch.empty(nbytes // 4, device="cuda")


def test_vjp_activation_spill_equals_recompute(cuda_lib):
    """The VJP kernel's activation spill (conditioner intermediates written to the caller's scratch in the forward
    sweep, read back in the backward sweep) gives bit-identical partial gradients, input and condition gradients
    and log-probs to the recompute path (no scratch)."""
    R = 4096
    est, inp, cond, w = _seeded_batch(R)
    spill = nsf_vjp_raw(est, inp, cond, w, _scratch(est, R))
    recompute = nsf_vjp_raw(est, inp, cond, w, None)
    assert spill[0] == 0 and recompute[0] == 0
    for name, a, b in zip(("gpart", "ginput", "gcond", "logp"), spill[1:], recompute[1:]):
        assert torch.isfinite(a).all() and torch.equal(a, b), name
    assert spill[1].abs().max() > 0


def test_vjp_undersized_scratch_is_rejected(cuda_lib):
    """A scratch one float smaller than sbi_b200_nsf_vjp_save_bytes: SBI_EINVAL, and nothing is written."""
    R = 1000
    est, inp, cond, w = _seeded_batch(R)
    save = _scratch(est, R)
    rc, *outs = nsf_vjp_raw(est, inp, cond, w, save[:-1], fill=float("nan"))
    torch.cuda.synchronize()
    assert rc == -1                      # SBI_EINVAL
    for name, t in zip(("gpart", "ginput", "gcond", "logp"), outs):
        assert torch.isnan(t).all(), name
    rc, *outs = nsf_vjp_raw(est, inp, cond, w, save, fill=float("nan"))
    assert rc == 0 and torch.isfinite(outs[1]).all()


def _vjp_outputs(est, inp, cond):
    R = inp.shape[0]
    return (torch.zeros(est.vjp_parts(R, False), est.layout.n_params, device="cuda"), torch.empty_like(inp),
            torch.empty_like(cond), torch.empty(R, device="cuda"))


def _est_vjp(est, inp, cond, w, outs):
    from sbi_b200 import _lib as L
    R = inp.shape[0]
    gpart, ginp, gcond, logp = outs
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    est.vjp(est._model(nbuf=3), rows, R, w, 0.0, logp, gpart, ginp, gcond)


def test_vjp_first_call_captured_in_a_graph_spills(cuda_lib):
    """A fresh estimator whose first SIMT VJP is captured in a CUDA graph allocates its activation scratch during
    the capture; the replay equals an eager call bit for bit."""
    import ctypes as C
    R = 300
    est, inp, cond, w = _seeded_batch(R)
    assert nsf_vjp_raw(est, inp, cond, w, _scratch(est, R))[0] == 0    # kernel attributes set outside the capture
    assert "vjp_save" not in est._cache
    captured, eager = _vjp_outputs(est, inp, cond), _vjp_outputs(est, inp, cond)
    graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(graph, stream=side):
        _est_vjp(est, inp, cond, w, captured)
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    _est_vjp(est, inp, cond, w, eager)
    torch.cuda.synchronize()
    nbytes = cuda_lib.sbi_b200_nsf_vjp_save_bytes(C.byref(est._model(nbuf=3)), R)
    assert est._cache["vjp_save"].numel() * 4 >= nbytes > 0
    for name, a, b in zip(("gpart", "ginput", "gcond", "logp"), captured, eager):
        assert torch.isfinite(a).all() and torch.equal(a, b), name


def test_vjp_of_two_estimators_on_two_streams(cuda_lib):
    """Two estimators run their SIMT VJPs at the same time on two streams, each grid small enough that both fit
    the GPU at once: each gives the gradients it gives alone (every estimator owns its activation scratch)."""
    R = 32 * (torch.cuda.get_device_properties(0).multi_processor_count // 2 - 4)
    runs = [_seeded_batch(R, seed=s) for s in (0, 1)]
    alone = []
    for est, inp, cond, w in runs:
        alone.append(_vjp_outputs(est, inp, cond))
        _est_vjp(est, inp, cond, w, alone[-1])
    together = [_vjp_outputs(est, inp, cond) for est, inp, cond, w in runs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    for s, (est, inp, cond, w), outs in zip(streams, runs, together):
        with torch.cuda.stream(s):
            _est_vjp(est, inp, cond, w, outs)
    torch.cuda.synchronize()
    for i, (a_outs, t_outs) in enumerate(zip(alone, together)):
        for name, a, b in zip(("gpart", "ginput", "gcond", "logp"), a_outs, t_outs):
            assert torch.equal(a, b), (i, name)
