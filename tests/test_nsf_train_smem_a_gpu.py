"""Tensor-core NSF training step with its MMA A operands in shared memory (csrc/tc_common.cuh): the forward
sweep with activation save and the backward sweep reproduce, bit for bit, the gradients of the version that
read A from the accumulator store (fixture tests/golden/nsf_train_tc_d3c2.npz, written by that version with
`python tests/test_nsf_train_smem_a_gpu.py --write PATH`), and the training path is taken exactly when both
kernels' shared-memory layouts fit one SM."""
import ctypes as ct
import os
import sys

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, os.getcwd())
from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nsf_train_tc_d3c2.npz")
SIZES = (512, 17896)          # one partial chunk, and two chunks of one tile per SM (the second accumulates)
MAX_SMEM = 227 * 1024


def _model():
    flow, theta, x = oracle_nsf(3, 2, n=max(SIZES), num_blocks=1)
    return b200_from_oracle(flow, theta, x, num_blocks=1), theta, x


def _step(est, theta, x, R, with_cond):
    """Flat parameter gradient, log-probs and loss statistics (and with `with_cond` the condition gradient)
    of sum_r g_r log q_r over the first R rows, through one tensor-core training step."""
    from sbi_b200 import _lib as L
    lib = L.load()
    assert est._vjp_uses_tc(R, True) and (not with_cond or est.vjp_cond_uses_tc(R))
    inp, cond = (theta[:R] * 1.3).float().cuda().contiguous(), x[:R].float().cuda().contiguous()
    g = torch.randn(R, generator=torch.Generator().manual_seed(R)).cuda()
    P, n_part = est.layout.n_params, est.vjp_parts(R)
    gpart = torch.full((n_part, P), float("nan"), device="cuda")
    lp = torch.empty(R, device="cuda")
    acc = torch.zeros(2, device="cuda")
    gcond = torch.full((R, x.shape[1]), float("nan"), device="cuda") if with_cond else None
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    est.vjp(m, rows, R, g, 0.0, lp, gpart, None, gcond, acc, cond_tc=with_cond)
    grad = torch.empty(P, device="cuda")
    L.check(lib.sbi_b200_reduce_partials(L.ptr(gpart), n_part, P, L.ptr(grad), L.stream_ptr()), "reduce")
    torch.cuda.synchronize()
    out = {"grad": grad.cpu().numpy(), "logp": lp.cpu().numpy(), "loss_acc": acc.cpu().numpy()}
    if with_cond:
        out["gcond"] = gcond.cpu().numpy()
    return out


def _all_steps():
    est, theta, x = _model()
    return {f"{k}_{R}_{'cond' if wc else 'param'}": v
            for R in SIZES for wc in (False, True) for k, v in _step(est, theta, x, R, wc).items()}


def test_train_step_matches_fixture(cuda_lib, monkeypatch):
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    want = np.load(FIXTURE)
    got = _all_steps()
    assert sorted(got) == sorted(want.files)
    again = _all_steps()
    for k, v in got.items():
        assert np.isfinite(v).all(), k
        if k.startswith("loss_acc"):
            # the loss statistics are summed with float atomics in whatever order the warps finish
            np.testing.assert_allclose(v, want[k], rtol=1e-5, err_msg=k)
            continue
        d = np.abs(v.astype(np.float64) - want[k]).max()
        assert np.array_equal(v, want[k]), f"{k}: max |new - fixture| {d:.3e}"
        assert np.array_equal(v, again[k]), f"{k}: repeated call differs"


def _smem_bytes(est):
    """(forward with save, backward sweep, weight-gradient kernel) dynamic shared memory, restated from
    tc_smem_layout(..., a_smem = true) (nsf_tc.cu), bwd_smem_layout and dw_smem_bytes (nsf_vjp_tc.cu); None
    when the host plans decline the model."""
    m = est._model(nbuf=3)
    pf, pb = est.layout.tc_plan(), est.layout.tc_bwd_plan()
    if pf is None or pb is None:
        return None
    cf, cb = pf["stage_cap"], pb["stage_cap"]
    rows, lu, a_region = 128, 2 * 16 * 16 + 2 * 16, 2 * 64 * 128
    up = lambda f: (f + 31) & ~31
    fl = m.Dp * rows + m.Cp * rows + rows + lu + m.T * (64 + m.NB * 192 + m.TRmax * 32)
    fwd = (up(fl) + a_region + 3 * cf) * 4 + 3 * 8
    fl = up(up(16 * rows + rows + lu) + 3 * 16 * rows)
    bwd = (fl + a_region + 2 * cb) * 4 + 2 * 8
    ldmax = max(m.Hp, m.Cp + m.IDp, m.Cp)
    dw = (2 * 32 * 65 * 4 + 64 * ldmax + 64) * 4
    return fwd, bwd, dw


def _eval_tc_ok(est):
    from sbi_b200 import _lib as L
    plan = est.layout.tc_plan()
    tc = L.NsfTc(plan["n_words"], plan["stage_cap"], None, None, None)
    return bool(L.load().sbi_b200_nsf_tc_supported(ct.byref(est._model(nbuf=2)), ct.byref(tc)))


# the edges of the wgmma envelope of test_kernel_envelope_gpu.py (largest T = 5, NB, D and C), and the bench model
@pytest.mark.parametrize("D,C,NB", [(10, 10, 2), (2, 14, 1), (2, 14, 3), (16, 12, 1), (16, 13, 1), (2, 14, 4)],
                         ids=["bench", "HC64", "HC64_NB3", "D16_C12", "D16_C13", "NB4"])
def test_training_path_taken_when_layouts_fit(cuda_lib, monkeypatch, D, C, NB):
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    flow, theta, x = oracle_nsf(D, C, n=600, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    sizes = _smem_bytes(est)
    fits = sizes is not None and _eval_tc_ok(est) and max(sizes) <= MAX_SMEM
    print(f"D={D} C={C} NB={NB}: (forward-save, backward, dW) shared memory {sizes} B, eval kernel fits "
          f"{sizes is not None and _eval_tc_ok(est)} -> training pair {fits}")
    assert est._vjp_uses_tc(512, True) == fits
    if not fits:
        # the SIMT VJP runs instead, with the partial-gradient slabs of its own grid
        assert est.vjp_parts(512) == est._entry("vjp_parts")(512)


if __name__ == "__main__" and "--write" in sys.argv:
    path = sys.argv[sys.argv.index("--write") + 1]
    os.environ["SBI_B200_VJP_TC"] = "1"
    res = _all_steps()
    np.savez_compressed(path, **res)
    print("wrote", path, {k: v.shape for k, v in res.items()})
