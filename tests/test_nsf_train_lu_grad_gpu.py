"""LULinear parameter gradients of the tensor-core NSF training step (csrc/nsf_vjp_tc.cu): the weight-gradient
kernel computes them, one unit per (tile, layer), from the backward's dz and the saved LULinear input.  The LULinear
entries of the reduced parameter gradient and of the first two tiles' partial-gradient slabs reproduce, bit for bit,
the fixture tests/golden/nsf_train_tc_lu_grad.npz, written by the version whose backward sweep reduced them over
the tile's rows itself (`python tests/test_nsf_train_lu_grad_gpu.py --write PATH`); the whole reduced gradient
reproduces the SHA-256 of its bytes stored there (the full gradients would make the fixture megabytes).  Models: D = 2 (one
lower / upper entry, three padding entries each) with H + C = 64 and three blocks, the D = 16 / C = 12 edge of the
envelope, and the bench model; batches: 4096 rows (one chunk on half tiles) and
one chunk of whole tiles plus a ragged second chunk that accumulates into the first chunk's slabs.  Each is run
with and without the condition gradient, eagerly and as one CUDA-graph replay."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    sys.path.insert(0, os.getcwd())
from tests.helpers import b200_from_oracle, oracle_nsf

pytestmark = pytest.mark.gpu
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nsf_train_tc_lu_grad.npz")
MODELS = {"D2_NB3": (2, 14, 3), "D16_C12": (16, 12, 1), "bench": (10, 10, 2)}
BATCHES = ("half", "two_chunks")


def _rows(batch):
    # half tiles: 32 tiles; two chunks: one tile per SM, then 8 ragged tiles (half tiles, accumulating)
    return 4096 if batch == "half" else 128 * torch.cuda.get_device_properties(0).multi_processor_count + 997


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


def _setup(model, batch):
    D, C, NB = MODELS[model]
    R = _rows(batch)
    flow, theta, x = oracle_nsf(D, C, n=R, seed=31 + D + NB, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    inp, cond = (theta * 1.3).float().cuda().contiguous(), x.float().cuda().contiguous()
    # per-row weights on half tiles, one weight for every row on the two-chunk batch (the trainer's case)
    g = torch.randn(R, generator=torch.Generator().manual_seed(R)).cuda() if batch == "half" else None
    return est, inp, cond, g, R


def _run(est, inp, cond, g, R, with_cond, graph):
    """{name: array} of one training step, launched eagerly or as the replay of a captured CUDA graph: the LULinear
    entries of the reduced gradient (`grad_lu`) and of slabs 0 and 1 (`lu`), the SHA-256 of the whole reduced
    gradient's bytes (`grad_sha256`)."""
    from sbi_b200 import _lib as L
    assert est._vjp_uses_tc(R, True)
    gpart = torch.full((est.vjp_parts(R), est.layout.n_params), float("nan"), device="cuda")
    lp = torch.empty(R, device="cuda")
    acc = torch.zeros(2, device="cuda")
    gcond = torch.empty((R, cond.shape[1]), device="cuda") if with_cond else None
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    step = lambda: est.vjp(m, rows, R, g, -1.0 / R, lp, gpart, None, gcond, acc, cond_tc=with_cond)
    step()                                  # eager (and allocates the activation scratch before any capture)
    if graph:
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            step()
        gpart.fill_(float("nan"))
        gr.replay()
    torch.cuda.synchronize()
    grad = torch.empty(est.layout.n_params, device="cuda")
    L.check(L.load().sbi_b200_reduce_partials(L.ptr(gpart), gpart.shape[0], gpart.shape[1], L.ptr(grad),
                                              L.stream_ptr()), "reduce")
    torch.cuda.synchronize()
    lu = _lu_index(est)
    grad = grad.cpu().numpy()
    return {"grad_lu": grad[lu], "lu": gpart[:2].cpu().numpy()[:, lu],
            "grad_sha256": np.frombuffer(hashlib.sha256(grad.tobytes()).digest(), np.uint8)}


def fixture_arrays():
    os.environ["SBI_B200_VJP_TC"] = "1"
    out = {}
    for model in MODELS:
        for batch in BATCHES:
            est, inp, cond, g, R = _setup(model, batch)
            for name, v in _run(est, inp, cond, g, R, False, False).items():
                out[f"{model}_{batch}_{name}"] = v
    return out


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("with_cond", [False, True], ids=["param", "cond"])
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("model", list(MODELS))
def test_lu_gradients_match_fixture(cuda_lib, monkeypatch, model, batch, with_cond, graph):
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    want = np.load(FIXTURE)
    est, inp, cond, g, R = _setup(model, batch)
    got = _run(est, inp, cond, g, R, with_cond, graph)
    for name in ("grad_lu", "lu"):
        ref = want[f"{model}_{batch}_{name}"]
        assert np.isfinite(got[name]).all(), name
        d = np.abs(got[name].astype(np.float64) - ref).max()
        assert np.array_equal(got[name], ref), f"{name}: max |new - fixture| {d:.3e}"
    assert np.array_equal(got["grad_sha256"], want[f"{model}_{batch}_grad_sha256"]), \
        "the reduced gradient differs from the fixture's outside its LULinear entries"


if __name__ == "__main__" and "--write" in sys.argv:
    path = sys.argv[sys.argv.index("--write") + 1]
    res = fixture_arrays()
    np.savez_compressed(path, **res)
    print("wrote", path, {k: v.shape for k, v in res.items()})
