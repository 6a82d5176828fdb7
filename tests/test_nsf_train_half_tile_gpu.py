"""Half tiles of the tensor-core NSF training step (csrc/nsf_tc.cu, csrc/nsf_vjp_tc.cu): a chunk of n 128-row
tiles runs its forward and backward sweeps on two 64-row CTAs per tile when 2n <= SMs, else on one CTA per
tile.  The same seeded rows, run once as a batch that takes half tiles and once as the leading tiles of a
batch that takes whole tiles, must give bit-identical per-row log-probs, per-row condition gradients and
partial-gradient slabs of every tile the two batches share."""
import numpy as np
import pytest
import torch

from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _step(est, inp, cond, g, R, with_cond):
    """(log-probs, partial-gradient slabs, condition gradients or None) of one tensor-core training step over
    the first R rows."""
    from sbi_b200 import _lib as L
    assert est._vjp_uses_tc(R, True) and (not with_cond or est.vjp_cond_uses_tc(R))
    P, n_part = est.layout.n_params, est.vjp_parts(R)
    gpart = torch.full((n_part, P), float("nan"), device="cuda")
    lp = torch.full((R,), float("nan"), device="cuda")
    acc = torch.zeros(2, device="cuda")
    gcond = torch.full((R, cond.shape[1]), float("nan"), device="cuda") if with_cond else None
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    est.vjp(est._model(nbuf=3), rows, R, g[:R].contiguous(), 0.0, lp, gpart, None, gcond, acc, cond_tc=with_cond)
    torch.cuda.synchronize()
    return lp.cpu().numpy(), gpart.cpu().numpy(), None if gcond is None else gcond.cpu().numpy()


@pytest.mark.parametrize("with_cond", [False, True], ids=["param", "cond"])
@pytest.mark.parametrize("case", ["4096", "4000", "2n=SMs"])
def test_half_tiles_match_whole_tiles(cuda_lib, monkeypatch, case, with_cond):
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    sms = _sms()
    # whole tiles: a chunk of sms // 2 + 1 tiles (2n = SMs + 2 on an even SM count, at least 67 tiles on 132)
    r_full = (sms // 2 + 1) * 128
    r_half = {"4096": 4096, "4000": 4000, "2n=SMs": (sms // 2) * 128}[case]
    assert 2 * ((r_half + 127) // 128) <= sms < 2 * (r_full // 128)
    flow, theta, x = oracle_nsf(10, 10, n=r_full, num_blocks=2)
    est = b200_from_oracle(flow, theta, x, num_blocks=2)
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    g = torch.randn(r_full, generator=torch.Generator().manual_seed(7)).cuda()
    lp_h, part_h, gc_h = _step(est, inp, cond, g, r_half, with_cond)
    lp_f, part_f, gc_f = _step(est, inp, cond, g, r_full, with_cond)
    assert np.isfinite(lp_h).all() and np.isfinite(part_h).all()
    assert np.array_equal(lp_h, lp_f[:r_half])
    if with_cond:
        assert np.isfinite(gc_h).all()
        assert np.array_equal(gc_h, gc_f[:r_half])
    # a ragged last tile has fewer live rows in the half-tile batch: compare the complete tiles
    shared = r_half // 128
    for t in range(shared):
        d = np.abs(part_h[t].astype(np.float64) - part_f[t]).max()
        assert np.array_equal(part_h[t], part_f[t]), f"tile {t}: max |half - whole| {d:.3e}"
