"""Tensor-core NSF training step at the bench shape (D = C = 10, two blocks, 4096 rows: half tiles), whose MMA
stages keep their accumulators in shared memory and several K-steps in flight (csrc/tc_common.cuh): the reduced
parameter gradient, the log-probs and the condition gradient reproduce, bit for bit, the fixture
tests/golden/nsf_train_tc_d10c10_4096.npz, written by the version that kept the accumulators in the global store
and waited for every K-step (`python tests/test_nsf_train_stage_gpu.py --write PATH`).  At the edges of the wgmma
envelope the training path is taken as before, and a half-tile batch reproduces the leading tiles of a
whole-tile batch."""
import os
import sys

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, os.getcwd())
from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nsf_train_tc_d10c10_4096.npz")
R_BENCH = 4096


def _step(est, inp, cond, g, with_cond):
    """Per-tile partial gradients, log-probs and (with `with_cond`) condition gradient of sum_r g_r log q_r
    through one tensor-core training step."""
    from sbi_b200 import _lib as L
    R = inp.shape[0]
    assert est._vjp_uses_tc(R, True)
    gpart = torch.full((est.vjp_parts(R), est.layout.n_params), float("nan"), device="cuda")
    lp = torch.full((R,), float("nan"), device="cuda")
    acc = torch.zeros(2, device="cuda")
    gcond = torch.full((R, cond.shape[1]), float("nan"), device="cuda") if with_cond else None
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    est.vjp(m, rows, R, g, 0.0, lp, gpart, None, gcond, acc, cond_tc=with_cond)
    torch.cuda.synchronize()
    return gpart, lp, gcond


def bench_shape_steps():
    """{name: array} of the bench-shape training step, without and with the condition gradient: the gradient
    reduced over the tiles (sbi_b200_reduce_partials), the log-probs and the condition gradient."""
    from sbi_b200 import _lib as L
    os.environ["SBI_B200_VJP_TC"] = "1"
    flow, theta, x = oracle_nsf(10, 10, n=R_BENCH, seed=21, num_blocks=2)
    est = b200_from_oracle(flow, theta, x, num_blocks=2)
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    g = torch.randn(R_BENCH, generator=torch.Generator().manual_seed(22)).cuda()
    out = {}
    for wc in (False, True):
        gpart, lp, gcond = _step(est, inp, cond, g, wc)
        grad = torch.empty(est.layout.n_params, device="cuda")
        L.check(L.load().sbi_b200_reduce_partials(L.ptr(gpart), gpart.shape[0], gpart.shape[1], L.ptr(grad),
                                                  L.stream_ptr()), "reduce")
        torch.cuda.synchronize()
        tag = "cond" if wc else "param"
        out[f"grad_{tag}"] = grad.cpu().numpy()
        out[f"logp_{tag}"] = lp.cpu().numpy()
        if wc:
            out["gcond"] = gcond.cpu().numpy()
    return out


def fixture_arrays(steps):
    """The fixture's arrays: both variants share the gradient and the log-probs (the test checks each)."""
    return {"grad": steps["grad_param"], "logp": steps["logp_param"], "gcond": steps["gcond"]}


def test_bench_shape_step_matches_fixture(cuda_lib, monkeypatch):
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    want = np.load(FIXTURE)
    got = bench_shape_steps()
    for k, v in got.items():
        ref = want[k.split("_")[0]]
        assert np.isfinite(v).all(), k
        d = np.abs(v.astype(np.float64) - ref).max()
        assert np.array_equal(v, ref), f"{k}: max |new - fixture| {d:.3e}"


# edges of the wgmma envelope (test_kernel_envelope_gpu.py), with whether the training pair takes them, as before
# the accumulators moved into shared memory
@pytest.mark.parametrize("D,C,NB,takes", [(16, 12, 1, True), (2, 14, 3, True)], ids=["D16_C12", "HC64_NB3"])
def test_envelope_edge(cuda_lib, monkeypatch, D, C, NB, takes):
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    flow, theta, x = oracle_nsf(D, C, n=600, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    assert est._vjp_uses_tc(512, True) == takes
    if not takes:
        return
    # one chunk of one tile per SM runs on whole tiles; 4 tiles run on half tiles
    R = 128 * torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator().manual_seed(D + C + NB)
    inp = (0.7 * torch.randn(R, D, generator=g) + 0.3).cuda()
    cond = (1.3 * torch.randn(R, C, generator=g) - 0.2).cuda()
    gout = torch.randn(R, generator=g).cuda()
    whole = _step(est, inp, cond, gout, True)
    n = 512
    half = _step(est, inp[:n].contiguous(), cond[:n].contiguous(), gout[:n].contiguous(), True)
    for name, w, h in zip(("partial gradients", "log-probs", "condition gradient"), whole, half):
        w = w[:h.shape[0]]
        assert torch.isfinite(h).all(), name
        assert torch.equal(w, h), f"{name}: max |half - whole| {(w - h).abs().max().item():.3e}"


if __name__ == "__main__" and "--write" in sys.argv:
    path = sys.argv[sys.argv.index("--write") + 1]
    res = fixture_arrays(bench_shape_steps())
    np.savez_compressed(path, **res)
    print("wrote", path, {k: v.shape for k, v in res.items()})
