"""The tensor-core NSF training step: the forward sweep that saves activations (csrc/nsf_tc.cu), the backward sweep
and the weight-gradient kernel (csrc/nsf_vjp_tc.cu), each step run by `tests.helpers.vjp_step`.

Frozen outputs: three fixtures under tests/golden/ hold the step bit for bit.  `python tests/test_nsf_train_tc_gpu.py
--write DIR` rewrites all three from the current build, for a change that moves them on purpose."""
import ctypes as C
import hashlib
import math
import os
import sys

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, os.getcwd())
from tests.helpers import b200_from_oracle, oracle_nsf, use_vjp_path, vjp_step

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GRAD_TOL = 2e-3


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(got, want), f"{what}: max |got - want| {np.abs(got.astype(np.float64) - want).max():.3e}"


# ------------------------------------------------------------------------------------------------ frozen outputs
def _d3c2_arrays(mp):
    """nsf_train_tc_d3c2.npz: D = 3, C = 2, one block; 512 rows (one partial chunk) and 17896 rows (a chunk of one
    tile per SM, then a second chunk that accumulates), without and with the condition gradient."""
    flow, theta, x = oracle_nsf(3, 2, n=17896, num_blocks=1)
    est = b200_from_oracle(flow, theta, x, num_blocks=1)
    use_vjp_path(mp, est, True)
    out = {}
    for R in (512, 17896):
        for wc in (False, True):
            inp, cond = (theta[:R] * 1.3).float().cuda().contiguous(), x[:R].float().cuda().contiguous()
            s = vjp_step(est, inp, cond, torch.randn(R, generator=torch.Generator().manual_seed(R)).cuda(),
                         with_cond=wc)
            tag = f"{R}_{'cond' if wc else 'param'}"
            out.update({f"grad_{tag}": s.grad.numpy(), f"logp_{tag}": s.logp.numpy(),
                        f"loss_acc_{tag}": s.loss_acc.numpy()})
            if wc:
                out[f"gcond_{tag}"] = s.gcond.numpy()
    return out


def _bench_arrays(mp):
    """The bench-shape step (D = C = 10, two blocks, 4096 rows: half tiles) without (`_param`) and with (`_cond`)
    the condition gradient.  nsf_train_tc_d10c10_4096.npz holds one `grad` and one `logp` for both."""
    flow, theta, x = oracle_nsf(10, 10, n=4096, seed=21, num_blocks=2)
    est = b200_from_oracle(flow, theta, x, num_blocks=2)
    use_vjp_path(mp, est, True)
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    g = torch.randn(4096, generator=torch.Generator().manual_seed(22)).cuda()
    p, c = (vjp_step(est, inp, cond, g, with_cond=wc) for wc in (False, True))
    return {"grad_param": p.grad, "logp_param": p.logp, "grad_cond": c.grad, "logp_cond": c.logp, "gcond": c.gcond}


LU_MODELS = {"D2_NB3": (2, 14, 3), "D16_C12": (16, 12, 1), "bench": (10, 10, 2)}
LU_BATCHES = ("half", "two_chunks")


def _lu_index(est):
    """Indices of every LULinear entry of the packed parameters, padding entries included."""
    from sbi_b200 import _lib as L
    D, idx = est.layout.D, []
    for t in est.layout.layer_tab:
        if t[L.L_HAS_LU]:
            for slot, n in ((L.L_LU_LOWER, D * (D - 1) // 2), (L.L_LU_UPPER, D * (D - 1) // 2),
                            (L.L_LU_DIAG, D), (L.L_LU_BIAS, D)):
                idx.append(int(t[slot]) + np.arange((n + 3) & ~3))
    return np.concatenate(idx)


def _lu_arrays(mp, model, batch, with_cond=False, graph=False):
    """nsf_train_tc_lu_grad.npz entries of one model and batch: the LULinear entries of the reduced gradient
    (`grad_lu`) and of slabs 0 and 1 (`lu`), and the SHA-256 of the whole reduced gradient's bytes (`grad_sha256`;
    the full gradients would make the fixture megabytes)."""
    D, C, NB = LU_MODELS[model]
    # half tiles: 32 tiles; two chunks: one tile per SM, then 8 ragged tiles (half tiles, accumulating)
    R = 4096 if batch == "half" else 128 * _sms() + 997
    flow, theta, x = oracle_nsf(D, C, n=R, seed=31 + D + NB, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    use_vjp_path(mp, est, True)
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    # per-row weights on half tiles, one weight for every row on the two-chunk batch (the trainer's case)
    g = torch.randn(R, generator=torch.Generator().manual_seed(R)).cuda() if batch == "half" else None
    s = vjp_step(est, inp, cond, g, g_const=-1.0 / R, with_cond=with_cond, graph=graph)
    lu, grad = _lu_index(est), s.grad.numpy()
    return {f"{model}_{batch}_grad_lu": grad[lu], f"{model}_{batch}_lu": s.gpart[:2].numpy()[:, lu],
            f"{model}_{batch}_grad_sha256": np.frombuffer(hashlib.sha256(grad.tobytes()).digest(), np.uint8)}


def test_d3c2_step_matches_fixture(cuda_lib, monkeypatch):
    want = np.load(os.path.join(GOLDEN, "nsf_train_tc_d3c2.npz"))
    got, again = _d3c2_arrays(monkeypatch), _d3c2_arrays(monkeypatch)
    assert sorted(got) == sorted(want.files)
    for k, v in got.items():
        assert np.isfinite(v).all(), k
        if k.startswith("loss_acc"):
            # the loss statistics are summed with float atomics in whatever order the warps finish
            np.testing.assert_allclose(v, want[k], rtol=1e-5, err_msg=k)
            continue
        _same(v, want[k], k)
        _same(v, again[k], f"{k} (repeated call)")


def test_bench_shape_step_matches_fixture(cuda_lib, monkeypatch):
    want = np.load(os.path.join(GOLDEN, "nsf_train_tc_d10c10_4096.npz"))
    got = _bench_arrays(monkeypatch)
    assert {k.split("_")[0] for k in got} == set(want.files)
    for k, v in got.items():
        assert torch.isfinite(v).all(), k
        _same(v, want[k.split("_")[0]], k)


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("with_cond", [False, True], ids=["param", "cond"])
@pytest.mark.parametrize("batch", LU_BATCHES)
@pytest.mark.parametrize("model", list(LU_MODELS))
def test_lu_gradients_match_fixture(cuda_lib, monkeypatch, model, batch, with_cond, graph):
    want = np.load(os.path.join(GOLDEN, "nsf_train_tc_lu_grad.npz"))
    got = _lu_arrays(monkeypatch, model, batch, with_cond, graph)
    names = {k[len(f"{model}_{batch}_"):] for k in got}
    assert set(want.files) == {f"{mo}_{b}_{n}" for mo in LU_MODELS for b in LU_BATCHES for n in names}
    for k, v in got.items():
        assert np.isfinite(v).all(), k
        _same(v, want[k], k)


# ------------------------------------------------------------------------------------------------ accuracy
def _oracle_param_grads(flow, est, inp, cond, g, dtype):
    flow = flow.to(dtype)
    flow.zero_grad()
    lp = flow.log_prob(inp.to(dtype), cond.to(dtype))[0]
    (lp * g.to(dtype)).sum().backward()
    return est.layout.pack({k: p.grad for k, p in flow.named_parameters()}).double(), lp.detach().double()


@pytest.mark.parametrize("D,C,R", [(10, 10, 128), (10, 10, 300), (10, 10, 4096), (3, 2, 77), (2, 2, 1000),
                                   (5, 7, 640), (10, 10, 20000)])
def test_vjp_tc_matches_oracle_and_simt(cuda_lib, monkeypatch, D, C, R):
    flow, theta, x = oracle_nsf(D, C, n=max(R, 500))
    est = b200_from_oracle(flow, theta, x)
    inp, cond = (theta[:R] * 1.3).float().cuda().contiguous(), x[:R].float().cuda().contiguous()
    g = torch.randn(R, dtype=torch.float64)
    use_vjp_path(monkeypatch, est, True)
    tc = vjp_step(est, inp, cond, g.float().cuda())
    use_vjp_path(monkeypatch, est, False)
    simt = vjp_step(est, inp, cond, g.float().cuda(), tc=False)
    got, lp, acc = tc.grad.double(), tc.logp.double(), tc.loss_acc
    assert tc.gpart.shape[0] == min((R + 127) // 128, _sms())
    assert torch.isfinite(got).all()
    mask = est.net._mask.cpu().bool()
    assert (got[~mask] == 0).all(), "padding entries must receive zero gradient"
    ref64, lp64 = _oracle_param_grads(flow, est, inp.cpu(), cond.cpu(), g, torch.float64)
    ref32, _ = _oracle_param_grads(flow, est, inp.cpu(), cond.cpu(), g, torch.float32)
    scale = ref64.abs().max().item()
    err = (got - ref64).abs().max().item() / scale
    err_s = (simt.grad.double() - ref64).abs().max().item() / scale
    err32 = (ref32 - ref64).abs().max().item() / scale
    print(f"D={D} C={C} R={R}: tensor-core grad rel err {err:.3e} (SIMT kernel {err_s:.3e}, torch-fp32 {err32:.3e}); "
          f"logp err {(lp - lp64).abs().max().item():.3e}")
    assert (lp - lp64).abs().max() <= 2e-3
    assert err <= max(GRAD_TOL, 4 * err32)
    # loss statistics: sum of -log q, no non-finite rows
    assert abs(acc[0].item() + lp64.sum().item()) <= 2e-3 * R and acc[1].item() == 0
    assert abs(acc[0].item() - simt.loss_acc[0].item()) <= 1e-3 * R


def _seeded_batch(R):
    """D = C = 10 estimator, its first R rows and seeded row weights."""
    flow, theta, x = oracle_nsf(10, 10, n=R)
    est = b200_from_oracle(flow, theta, x)
    g = torch.Generator().manual_seed(7)
    inp, cond = theta[:R].float().cuda().contiguous(), x[:R].float().cuda().contiguous()
    return est, inp, cond, torch.randn(R, generator=g).cuda()


def test_split_weight_gradients_match_simt_over_several_chunks(cuda_lib, monkeypatch):
    """The weight-gradient kernel over batches of several chunks (more rows than one tile per SM) with a ragged
    last tile: repeat calls bit-identical, the condition gradient leaves the parameter gradients alone, and both
    agree with the SIMT VJP kernel."""
    # one chunk is one 128-row tile per SM; the second chunk ends on a 104-row tile
    R = 128 * _sms() + 1000
    est, inp, cond, w = _seeded_batch(R)
    use_vjp_path(monkeypatch, est, True)
    p1, p2, c1, c2 = (vjp_step(est, inp, cond, w, with_cond=wc) for wc in (False, False, True, True))
    assert torch.isfinite(p1.grad).all() and torch.isfinite(c1.gcond).all()
    assert torch.equal(p1.grad, p2.grad) and torch.equal(c1.grad, c2.grad) and torch.equal(c1.gcond, c2.gcond)
    assert torch.equal(p1.grad, c1.grad), "the condition gradient must not change the parameter gradients"

    use_vjp_path(monkeypatch, est, False)
    gs = vjp_step(est, inp, cond, w, tc=False).grad
    cs = vjp_step(est, inp, cond, w, with_cond=True, tc=False).gcond
    sc, scc = gs.abs().max().item(), cs.abs().max().item()
    err, err_c = (p1.grad - gs).abs().max().item() / sc, (c1.gcond - cs).abs().max().item() / scc
    print(f"R={R}: parameter gradient vs SIMT {err:.2e}, condition gradient vs SIMT {err_c:.2e}")
    assert err <= 2e-3 and err_c <= 2e-3


# ------------------------------------------------------------------------------------------------ tile layouts and replays
HALF_EDGES = {"D16_C12": (16, 12, 1), "HC64_NB3": (2, 14, 3)}
HALF_CASES = [(c, wc) for c in ("4096", "4000", "2n=SMs") for wc in (False, True)] + [(e, True) for e in HALF_EDGES]


@pytest.mark.parametrize("case,with_cond", HALF_CASES, ids=[f"{c}-{'cond' if wc else 'param'}" for c, wc in HALF_CASES])
def test_half_tiles_match_whole_tiles(cuda_lib, monkeypatch, case, with_cond):
    """A chunk of n tiles runs each sweep on two 64-row CTAs per tile when 2n <= SMs, else on one CTA per tile.  The
    same rows, run as a batch that takes half tiles and as the leading rows of one that takes whole tiles, give
    bit-identical log-probs, condition gradients and partial-gradient slabs of every complete tile."""
    sms, edge = _sms(), HALF_EDGES.get(case)
    D, C, NB = edge or (10, 10, 2)
    # whole tiles: one chunk of one tile per SM at the envelope edges; else a chunk of sms // 2 + 1 tiles
    # (2n = SMs + 2 on an even SM count, at least 67 tiles on 132)
    r_full = 128 * sms if edge else (sms // 2 + 1) * 128
    flow, theta, x = oracle_nsf(D, C, n=600 if edge else r_full, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    use_vjp_path(monkeypatch, est, True)
    if edge:
        r_half, gen = 512, torch.Generator().manual_seed(D + C + NB)
        inp = (0.7 * torch.randn(r_full, D, generator=gen) + 0.3).cuda()
        cond = (1.3 * torch.randn(r_full, C, generator=gen) - 0.2).cuda()
        g = torch.randn(r_full, generator=gen).cuda()
    else:
        r_half = {"4096": 4096, "4000": 4000, "2n=SMs": (sms // 2) * 128}[case]
        inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
        g = torch.randn(r_full, generator=torch.Generator().manual_seed(7)).cuda()
    assert 2 * ((r_half + 127) // 128) <= sms < 2 * (r_full // 128)
    half = vjp_step(est, inp[:r_half], cond[:r_half], g[:r_half], with_cond=with_cond)
    whole = vjp_step(est, inp, cond, g, with_cond=with_cond)
    assert torch.isfinite(half.logp).all() and torch.isfinite(half.gpart).all()
    _same(half.logp, whole.logp[:r_half], "log-probs")
    if with_cond:
        assert torch.isfinite(half.gcond).all()
        _same(half.gcond, whole.gcond[:r_half], "condition gradients")
    # a ragged last tile has fewer live rows in the half-tile batch: compare the complete tiles
    for t in range(r_half // 128):
        _same(half.gpart[t], whole.gpart[t], f"tile {t}")


# 4096 and a ragged 4000 rows take half tiles; 17896 rows are a whole-tile chunk and a half-tile chunk that
# accumulates; D = 5 alternates layers of 3 and 2 spline features, so the second final-layer unit of every other
# layer has nothing to do
@pytest.mark.parametrize("with_cond", [False, True], ids=["param", "cond"])
@pytest.mark.parametrize("D,R", [(10, 4096), (10, 4000), (10, 17896), (5, 4096)],
                         ids=["4096", "4000", "17896", "D5_4096"])
def test_graph_replays_match_eager(cuda_lib, monkeypatch, D, R, with_cond):
    """Each weight-gradient CTA waits on a ready counter in the activation scratch, which the forward sweep zeroes
    and the backward sweep counts up.  Three replays of one captured step give the eager call's outputs bit for
    bit, so the counters start from zero on every replay."""
    flow, theta, x = oracle_nsf(D, 4, n=R, num_blocks=2)
    est = b200_from_oracle(flow, theta, x, num_blocks=2)
    use_vjp_path(monkeypatch, est, True)
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    g = torch.randn(R, generator=torch.Generator().manual_seed(R)).cuda()
    eager = vjp_step(est, inp, cond, g, with_cond=with_cond)
    replay = vjp_step(est, inp, cond, g, with_cond=with_cond, graph=3)
    for name in ("gpart", "logp", "gcond") if with_cond else ("gpart", "logp"):
        assert torch.isfinite(getattr(eager, name)).all(), name
        _same(getattr(replay, name), getattr(eager, name), f"{name} of the replays vs the eager call")


# ------------------------------------------------------------------------------------------------ envelope
def _smem_bytes(est):
    """Dynamic shared memory in bytes: the evaluation kernel, then (forward with activation save on whole and half
    tiles, backward sweep on whole and half tiles, weight-gradient kernel), restated from tc_smem_layout (nsf_tc.cu),
    bwd_smem_layout and dw_smem_bytes (nsf_vjp_tc.cu)."""
    m = est._model(nbuf=3)
    cf, cb = est.layout.tc_plan()["stage_cap"], est.layout.tc_bwd_plan()["stage_cap"]
    up = lambda f: (f + 31) & ~31
    lu = 2 * 16 * 16 + 2 * 16                   # LU factors, bias and diagonal
    a = lambda rpc: 2 * 64 * rpc                # A_hi | A_lo
    acc = lambda rpc: 128 * 68 if rpc < 128 else 0      # half tiles: the D | G accumulator columns

    def fwd(rpc, save):                         # 3 ring slots; half tiles keep 16 log|det| rows per row
        fl = up((m.Dp + m.Cp + 1 + (16 if rpc < 128 else 0)) * rpc + lu + m.T * (64 + 192 * m.NB + 32 * m.TRmax))
        return (fl + (a(rpc) + acc(rpc) if save else 0) + 3 * cf) * 4 + 3 * 8

    def bwd(rpc):                               # dz (16 rows) and the row weights; 2 ring slots
        return (up(17 * rpc + lu) + a(rpc) + acc(rpc) + 2 * cb) * 4 + 2 * 8

    dw = (2 * 32 * 65 * 4 + 64 * max(m.Hp, m.Cp + m.IDp, m.Cp) + 64) * 4
    return fwd(128, False), (fwd(128, True), fwd(64, True), bwd(128), bwd(64), dw)


# the edges of the wgmma envelope of test_kernel_envelope_gpu.py (largest T = 5, NB, D and C), and the bench model
@pytest.mark.parametrize("D,C,NB,takes", [(10, 10, 2, True), (2, 14, 1, True), (2, 14, 3, True), (16, 12, 1, True),
                                          (16, 13, 1, False), (2, 14, 4, False)],
                         ids=["bench", "HC64", "HC64_NB3", "D16_C12", "D16_C13", "NB4"])
def test_training_path_taken_when_layouts_fit(cuda_lib, monkeypatch, D, C, NB, takes):
    """The training pair runs when the evaluation kernel fits 112 KB (two CTAs per SM) and the five training
    layouts each fit the 227 KB one CTA may opt into."""
    flow, theta, x = oracle_nsf(D, C, n=600, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    use_vjp_path(monkeypatch, est, True)
    ev, sizes = _smem_bytes(est)
    fits = ev <= 112 * 1024 and max(sizes) <= 227 * 1024
    print(f"D={D} C={C} NB={NB}: evaluation {ev} B; (forward-save whole / half, backward whole / half, dW) {sizes} B "
          f"-> training pair {fits}")
    assert fits == takes and est._vjp_uses_tc(512, True) == takes
    if (D, C, NB) == (10, 10, 2):
        assert sizes[:4] == (178_712, 178_456, 141_968, 139_664), "update DESIGN.md §3.2 with the layouts"
    if not takes:
        # the SIMT VJP runs instead, with the partial-gradient slabs of its own grid
        assert est.vjp_parts(512) == est._entry("vjp_parts")(512)


# ------------------------------------------------------------------------------------------------ scratch contract
def test_scratch_without_the_dy_region_is_rejected(cuda_lib, monkeypatch):
    """The activation scratch has a dY region per tile and layer; a scratch sized without it gets SBI_EINVAL."""
    from sbi_b200 import _lib as L
    R = 4096
    est, inp, cond, w = _seeded_batch(R)
    use_vjp_path(monkeypatch, est, True)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
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


# ------------------------------------------------------------------------------------------------ dispatch and end-to-end fit
def test_vjp_tc_kernels_are_the_ones_that_run(cuda_lib, monkeypatch):
    """Default dispatch: from 256 rows (two tiles) the trainer's VJP is the tensor-core pair."""
    flow, theta, x = oracle_nsf(10, 10, n=5000)
    est = b200_from_oracle(flow, theta, x)
    monkeypatch.delenv("SBI_B200_VJP_TC", raising=False)
    assert est._vjp_uses_tc(4096, True) and not est._vjp_uses_tc(4096, False) and not est._vjp_uses_tc(100, True)
    # autograd with input gradients falls back to the SIMT kernel and still works
    inp = theta[:2048].cuda().requires_grad_(True)
    (est.log_prob(inp, x[:2048].cuda())[0]).sum().backward()
    assert inp.grad is not None and torch.isfinite(est.flat.grad).all()
    # parameter-only autograd at 2048 rows goes through the tensor-core path
    est.zero_grad()
    est.log_prob(theta[:2048].cuda(), x[:2048].cuda())[0].sum().backward()
    g_tc = est.flat.grad.clone()
    use_vjp_path(monkeypatch, est, False)
    est.zero_grad()
    est.log_prob(theta[:2048].cuda(), x[:2048].cuda())[0].sum().backward()
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


if __name__ == "__main__" and "--write" in sys.argv:
    out_dir = sys.argv[sys.argv.index("--write") + 1]
    with pytest.MonkeyPatch.context() as mp:
        bench = _bench_arrays(mp)
        files = {"nsf_train_tc_d3c2.npz": _d3c2_arrays(mp),
                 "nsf_train_tc_d10c10_4096.npz": {"grad": bench["grad_param"].numpy(),
                                                  "logp": bench["logp_param"].numpy(), "gcond": bench["gcond"].numpy()},
                 "nsf_train_tc_lu_grad.npz": {k: v for mo in LU_MODELS for b in LU_BATCHES
                                              for k, v in _lu_arrays(mp, mo, b).items()}}
    for name, arrays in files.items():
        np.savez_compressed(os.path.join(out_dir, name), **arrays)
        print("wrote", name, {k: v.shape for k, v in arrays.items()})
