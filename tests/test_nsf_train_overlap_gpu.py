"""Weight-gradient kernel of the tensor-core NSF training step overlapped with the backward sweep
(csrc/nsf_vjp_tc.cu): each weight-gradient CTA waits on a ready counter in the activation scratch, which the
forward sweep zeroes and the backward sweep counts up.  One training step (forward, backward, weight gradients),
captured in a CUDA graph and replayed several times on the same rows and parameters, must give bit-identical
partial-gradient slabs, log-probs and condition gradients to an eager call after every replay -- that is, the
counters start from zero on every replay."""
import numpy as np
import pytest
import torch

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu
REPLAYS = 3


def _outputs(est, R, C):
    P, n_part = est.layout.n_params, est.vjp_parts(R)
    return (torch.empty((n_part, P), device="cuda"), torch.empty(R, device="cuda"), torch.zeros(2, device="cuda"),
            torch.empty((R, C), device="cuda"))


def _poison(gpart, lp, gcond):
    for t in (gpart, lp, gcond):
        t.fill_(float("nan"))


# 4096 and a ragged 4000 rows take half tiles; 17896 rows are a whole-tile chunk and a half-tile chunk that
# accumulates; D = 5 alternates layers of 3 and 2 spline features, so the second final-layer unit of every other
# layer has nothing to do
@pytest.mark.parametrize("with_cond", [False, True], ids=["param", "cond"])
@pytest.mark.parametrize("D,R", [(10, 4096), (10, 4000), (10, 17896), (5, 4096)],
                         ids=["4096", "4000", "17896", "D5_4096"])
def test_graph_replays_match_eager(cuda_lib, monkeypatch, D, R, with_cond):
    from sbi_b200 import _lib as L
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    flow, theta, x = oracle_nsf(D, 4, n=R, num_blocks=2)
    est = b200_from_oracle(flow, theta, x, num_blocks=2)
    assert est._vjp_uses_tc(R, True) and (not with_cond or est.vjp_cond_uses_tc(R))
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    g = torch.randn(R, generator=torch.Generator().manual_seed(R)).cuda()
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)

    def step(out):
        gpart, lp, acc, gcond = out
        est.vjp(m, rows, R, g, 0.0, lp, gpart, None, gcond if with_cond else None, acc, cond_tc=with_cond)

    eager = _outputs(est, R, x.shape[1])
    _poison(eager[0], eager[1], eager[3])
    step(eager)
    torch.cuda.synchronize()
    want = [t.cpu().numpy() for t in (eager[0], eager[1], eager[3])]
    assert np.isfinite(want[0]).all() and np.isfinite(want[1]).all()
    if with_cond:
        assert np.isfinite(want[2]).all()

    static = _outputs(est, R, x.shape[1])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step(static)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step(static)
    for rep in range(REPLAYS):
        _poison(static[0], static[1], static[3])
        graph.replay()
        torch.cuda.synchronize()
        got = [t.cpu().numpy() for t in (static[0], static[1], static[3])]
        for name, a, b in zip(("partial gradients", "log-probs", "condition gradients"), got, want):
            if name == "condition gradients" and not with_cond:
                continue
            assert np.array_equal(a, b), f"replay {rep}: {name} differ from the eager call"
