"""Weight gradients of the tensor-core training step in their own kernel (nsf_dw_tc_kernel, csrc/nsf_vjp_tc.cu):
the backward sweep writes every linear's output gradient to the dY region of the activation scratch and the
weight-gradient kernel multiplies it by the saved activations.  Batches of several chunks (more rows than one
tile per SM) with a ragged last tile, with and without the condition gradient, against the SIMT VJP kernel;
repeat calls bit-identical; a scratch without the dY region rejected."""
import ctypes as C

import pytest
import torch

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu


def _rows_past_one_chunk():
    # one chunk is one 128-row tile per SM; the second chunk ends on a 104-row tile
    return 128 * torch.cuda.get_device_properties(0).multi_processor_count + 1000


def _setup(R):
    from sbi_b200 import _lib as L
    flow, theta, x = oracle_nsf(10, 10, n=R)
    est = b200_from_oracle(flow, theta, x)
    g = torch.Generator().manual_seed(7)
    inp, cond = theta[:R].float().cuda().contiguous(), x[:R].float().cuda().contiguous()
    w = torch.randn(R, generator=g).cuda()
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    return est, rows, w, (inp, cond)


def _run(est, rows, R, w, cond_tc, with_cond):
    """(reduced parameter gradient, condition gradient or None) of sum_r w_r log q_r."""
    from sbi_b200 import _lib as L
    lib = L.load()
    n_part = est.vjp_parts(R, cond_tc or not with_cond)
    # the tensor-core pair writes every entry of its slabs: start them from NaN
    fill = float("nan") if est._vjp_uses_tc(R, True) and (cond_tc or not with_cond) else 0.0
    gp = torch.full((n_part, est.layout.n_params), fill, device="cuda")
    gc = torch.zeros(R, 10, device="cuda") if with_cond else None
    est.vjp(est._model(nbuf=3), rows, R, w, 0.0, None, gp, None, gc, None, cond_tc=cond_tc)
    grad = torch.empty(est.layout.n_params, device="cuda")
    L.check(lib.sbi_b200_reduce_partials(L.ptr(gp), n_part, est.layout.n_params, L.ptr(grad), L.stream_ptr()),
            "reduce")
    torch.cuda.synchronize()
    return grad, gc


def test_split_weight_gradients_match_simt_over_several_chunks(cuda_lib, monkeypatch):
    R = _rows_past_one_chunk()
    est, rows, w, _keep = _setup(R)
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    assert est.vjp_cond_uses_tc(R)
    g1, _ = _run(est, rows, R, w, False, False)
    g2, _ = _run(est, rows, R, w, False, False)
    gc1, c1 = _run(est, rows, R, w, True, True)
    gc2, c2 = _run(est, rows, R, w, True, True)
    assert torch.isfinite(g1).all() and torch.isfinite(c1).all()
    assert torch.equal(g1, g2) and torch.equal(gc1, gc2) and torch.equal(c1, c2)
    assert torch.equal(g1, gc1), "the condition gradient must not change the parameter gradients"

    monkeypatch.setenv("SBI_B200_VJP_TC", "0")
    est._cache.pop("tc_train", None)
    gs, _ = _run(est, rows, R, w, False, False)
    _, cs = _run(est, rows, R, w, False, True)
    sc, scc = gs.abs().max().item(), cs.abs().max().item()
    err, err_c = (g1 - gs).abs().max().item() / sc, (c1 - cs).abs().max().item() / scc
    print(f"R={R}: parameter gradient vs SIMT {err:.2e}, condition gradient vs SIMT {err_c:.2e}")
    assert err <= 2e-3 and err_c <= 2e-3


def test_scratch_without_the_dy_region_is_rejected(cuda_lib, monkeypatch):
    from sbi_b200 import _lib as L
    R = 4096
    est, rows, w, _keep = _setup(R)
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    m = est._model(nbuf=3)
    tcs = est._tc_train_state(m)
    assert tcs is not None
    parts = cuda_lib.sbi_b200_nsf_vjp_tc_parts(R)
    # per tile: T layer slabs of NB blocks of 4 [128][64] arrays, hf, the spline parameters, zin, v; then zt, lp
    layer = 4 * m.NB * 64 * 128 + 64 * 128 + m.TRmax * 32 * 128 + 2 * 16 * 128
    old_bytes = 4 * parts * (m.T * layer + 16 * 128 + 128)
    new_bytes = cuda_lib.sbi_b200_nsf_vjp_tc_save_bytes(C.byref(m), R)
    assert new_bytes == old_bytes + 4 * parts * m.T * (64 * ((m.TRmax + 1) // 2) + 192 * m.NB + 64) * 128
    save = torch.empty(new_bytes // 4, device="cuda")
    gp = torch.empty(parts, est.layout.n_params, device="cuda")
    lp = torch.empty(R, device="cuda")

    def call(nbytes):
        return cuda_lib.sbi_b200_nsf_vjp_tc(C.byref(m), C.byref(tcs[0]), C.byref(tcs[1]), C.byref(rows), L.ptr(w),
                                            0.0, L.ptr(lp), L.ptr(gp), None, L.ptr(save), nbytes, L.stream_ptr())

    assert call(old_bytes) == -1            # SBI_EINVAL
    assert call(new_bytes) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(gp).all()
