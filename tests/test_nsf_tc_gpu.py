"""Parity of the tensor-core (wgmma, 3xTF32) NSF log_prob kernel, through the C ABI.

Bars: against the fp64 oracle the same LOGP_TOL as the SIMT kernel (2e-3 absolute on
log-probs of magnitude O(10..50)); against the SIMT fp32 kernel 5e-4 (the 3xTF32 split keeps
~21 mantissa bits per product; every op outside the linears is the same code).
"""
import pytest
import torch

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu

LOGP_TOL = 2e-3
VS_SIMT_TOL = 5e-4


def _both(est, inp, cond, monkeypatch):
    monkeypatch.setenv("SBI_B200_TC", "0")
    with torch.no_grad():
        simt = est.log_prob(inp, cond).clone()
    monkeypatch.setenv("SBI_B200_TC", "1")
    with torch.no_grad():
        tc = est.log_prob(inp, cond).clone()
    return simt, tc


def _tc_available(est):
    import ctypes as C
    from sbi_b200 import _lib as L
    m = est._model(nbuf=2)
    return est._tc_state(m) is not None


@pytest.mark.parametrize("D,C,R", [(10, 10, 128), (10, 10, 257), (10, 10, 20000), (2, 2, 1000),
                                   (3, 2, 77), (5, 7, 4097)])
def test_tc_logprob_matches_oracle(cuda_lib, monkeypatch, D, C, R):
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500))
    est = b200_from_oracle(flow, theta, x)
    assert _tc_available(est)
    inp, cond = theta[:R] * 1.5, x[:R]
    with torch.no_grad():
        ref64 = flow.double().log_prob(inp.double(), cond.double())[0]
    simt, tc = _both(est, inp.cuda(), cond.cuda(), monkeypatch)
    simt, tc = simt[0].cpu(), tc[0].cpu()
    err = (tc.double() - ref64).abs().max().item()
    err_simt = (simt.double() - ref64).abs().max().item()
    d = (tc - simt).abs().max().item()
    print(f"D={D} C={C} R={R}: tc err {err:.3e}  simt err {err_simt:.3e}  |tc-simt| {d:.3e}")
    assert torch.isfinite(tc).all()
    assert err <= LOGP_TOL
    assert d <= VS_SIMT_TOL


def test_tc_shared_condition_noise_and_index(cuda_lib, monkeypatch):
    flow, theta, x = oracle_nsf(10, 10)
    est = b200_from_oracle(flow, theta, x)
    xo = x[:1].cuda()
    th = theta[:1500].cuda()
    simt, tc = _both(est, th.unsqueeze(1), xo, monkeypatch)
    assert (simt - tc).abs().max() <= VS_SIMT_TOL
    # base-space point (inverse_transform) through both kernels
    monkeypatch.setenv("SBI_B200_TC", "0")
    z0 = est.inverse_transform(th, xo)
    monkeypatch.setenv("SBI_B200_TC", "1")
    z1 = est.inverse_transform(th, xo)
    assert (z0 - z1).abs().max() <= VS_SIMT_TOL
    # gathered rows (device-resident data set + index)
    idx = torch.randperm(1500, device="cuda")[:700]
    cond = x[:1500].cuda()
    m = est._model(nbuf=2)
    monkeypatch.setenv("SBI_B200_TC", "0")
    a, _ = est._logprob_raw(th, cond, False, index=idx, n_rows=700)
    monkeypatch.setenv("SBI_B200_TC", "1")
    b, _ = est._logprob_raw(th, cond, False, index=idx, n_rows=700)
    assert (a - b).abs().max() <= VS_SIMT_TOL


def test_tc_full_size_properties(cuda_lib, monkeypatch):
    """BASELINE-size batch (2^20 rows at one x_o): finite, matches the SIMT kernel, and is
    invariant to row order (each row is independent of its tile neighbours)."""
    flow, theta, x = oracle_nsf(10, 10)
    est = b200_from_oracle(flow, theta, x)
    g = torch.Generator(device="cuda").manual_seed(3)
    R = 1 << 20
    th = torch.randn(R, 10, device="cuda", generator=g) * 0.9 + 0.3
    xo = x[:1].cuda()
    simt, tc = _both(est, th.unsqueeze(1), xo, monkeypatch)
    assert torch.isfinite(tc).all()
    assert (simt - tc).abs().max() <= VS_SIMT_TOL
    perm = torch.randperm(R, device="cuda", generator=g)
    with torch.no_grad():
        tcp = est.log_prob(th[perm].unsqueeze(1), xo)
    assert torch.equal(tcp[:, 0], tc[perm, 0])


def test_tc_tracks_parameter_updates(cuda_lib, monkeypatch):
    """The packed operands follow in-place parameter changes made behind torch's back."""
    flow, theta, x = oracle_nsf(10, 10)
    est = b200_from_oracle(flow, theta, x)
    inp, cond = theta[:512].cuda(), x[:512].cuda()
    _, tc0 = _both(est, inp, cond, monkeypatch)
    with torch.no_grad():
        est.flat.data.mul_(1.01)
    simt1, tc1 = _both(est, inp, cond, monkeypatch)
    assert (tc1 - tc0).abs().max() > 1e-3
    assert (tc1 - simt1).abs().max() <= VS_SIMT_TOL


def test_tc_unsupported_model_uses_simt(cuda_lib, monkeypatch):
    flow, theta, x = oracle_nsf(4, 3, hidden_features=32)
    est = b200_from_oracle(flow, theta, x, hidden_features=32)
    assert not _tc_available(est)
    monkeypatch.setenv("SBI_B200_TC", "1")
    with torch.no_grad():
        ref = flow.double().log_prob(theta[:200].double(), x[:200].double())[0]
        got = est.log_prob(theta[:200].cuda(), x[:200].cuda())[0].cpu()
    assert (got.double() - ref).abs().max() <= LOGP_TOL


@pytest.mark.parametrize("D,C,R,shared", [(10, 10, 1000, True), (10, 10, 4097, False), (3, 2, 300, False),
                                          (2, 2, 129, True)])
def test_tc_sampling_matches_simt_and_oracle(cuda_lib, monkeypatch, D, C, R, shared):
    """x = T^{-1}(noise | cond) through the tensor-core kernel: same samples as the SIMT kernel
    (|dx| <= 5e-4) and as the fp64 oracle (|dx| <= 2e-3, the bar of test_nsf_gpu), and
    log_prob(sample) consistent with the returned log|det|."""
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500))
    est = b200_from_oracle(flow, theta, x)
    g = torch.Generator().manual_seed(5)
    noise = torch.randn(R, D, generator=g)
    cond = x[:1] if shared else x[:R]
    monkeypatch.setenv("SBI_B200_TC", "0")
    xs, ls = est.inverse_flow(noise.cuda(), cond.cuda())
    monkeypatch.setenv("SBI_B200_TC", "1")
    xt, lt = est.inverse_flow(noise.cuda(), cond.cuda())
    assert torch.isfinite(xt).all()
    assert (xs - xt).abs().max() <= VS_SIMT_TOL
    assert (ls - lt).abs().max() <= VS_SIMT_TOL
    with torch.no_grad():
        flow.double()
        emb = flow.net._embedding_net(cond.double())
        ctx = emb.expand(R, -1) if shared else emb
        ref, _ = flow.net._transform.inverse(noise.double(), context=ctx)
    assert (xt.cpu().double() - ref).abs().max() <= 2e-3
    # density of the samples through the tensor-core log_prob kernel:
    #   log q(x) = log N(noise) - log|det dx/dnoise|
    import math
    with torch.no_grad():
        lp = est.log_prob(xt.unsqueeze(1), cond.cuda())[:, 0] if shared else est.log_prob(xt, cond.cuda())[0]
    base = -0.5 * (noise ** 2).sum(1) - 0.5 * D * math.log(2 * math.pi)
    assert (lp.cpu() - (base - lt.cpu())).abs().max() <= 5e-3
