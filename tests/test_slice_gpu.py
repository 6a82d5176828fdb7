"""The vectorized slice sampler's kernel (csrc/slice.cu) draw for draw against the unmodified reference sampler.

Slice sampling leaves its target invariant for any bracket width and any order of the dimensions, so sample
moments cannot tell a wrong width adaptation, a missing reshuffle, draws taken in the wrong order or a wrong
step-out cap from the reference's algorithm.  These tests run the reference's own `SliceSamplerVectorized`
(sbi/samplers/mcmc/slice_numpy.py) on the kernel's random stream (tests/helpers.py `PhiloxDraws`) and require
every chain to ask for the same points, in the same order, and to end with the same samples and widths.

A chain's trajectory depends only on its own draws and its own potential values, so the reference runs each
chain on its own (`num_chains=1`): its k-th potential call is the kernel's k-th lock-step for that chain.  The
targets evaluate bit-identically on the host and on the device (float32 input, float64 `+ - *` in a fixed order,
float32 result), and the kernel's bracket arithmetic is numpy's to the bit, so equality is exact.  The one
remaining difference is the last ulp of the device `log` in the slice height `logu`: it can flip a comparison
only when a float32 potential value lies within one float64 ulp of `logu`, about 2^-29 per comparison."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests.helpers import PhiloxDraws

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")

SLICE_LOWER, SLICE_DONE = 1, 4


# ------------------------------------------------------------------------------------------------ targets
def _where(mask, val, xp):
    return np.where(mask, val, -np.inf) if xp is np else val.masked_fill(~mask, -math.inf)


_PREC = np.linalg.inv(np.array([[1.0, 0.6], [0.6, 2.0]]))
_GA, _GB, _GC = 0.5 * float(_PREC[0, 0]), float(_PREC[0, 1]), 0.5 * float(_PREC[1, 1])
_BOX = ((0.25, 1.5), (-2.5, -1.0))


def _gauss(x, xp):
    """Correlated 2-D Gaussian, mean (1, -2), covariance [[1, .6], [.6, 2]]."""
    d0, d1 = x[:, 0] - 1.0, x[:, 1] + 2.0
    return -(_GA * d0 * d0 + _GB * d0 * d1 + _GC * d1 * d1)


def _box(x, xp):
    """The Gaussian restricted to a box around its mean: brackets step out past the support into -inf."""
    (a0, b0), (a1, b1) = _BOX
    inside = (x[:, 0] >= a0) & (x[:, 0] <= b0) & (x[:, 1] >= a1) & (x[:, 1] <= b1)
    return _where(inside, _gauss(x, xp), xp)


def _quartic(x, xp):
    """Double well -(x_i^2 - 1)^2 per coordinate plus a nearest-neighbour coupling 0.3 x_i x_(i+1)."""
    s = 0.0 * x[:, 0]
    for i in range(x.shape[1]):
        t = x[:, i] * x[:, i] - 1.0
        s = s - t * t
    for i in range(x.shape[1] - 1):
        s = s + 0.3 * x[:, i] * x[:, i + 1]
    return s


TARGETS = {"gauss": _gauss, "box": _box, "quartic": _quartic}


def device_potential(target):
    """log p on the sampler's float32 (C, D) CUDA `params`: device work only, so CUDA graphs can capture it."""
    f = TARGETS[target]
    return lambda p: f(p.double(), torch).float()


def host_potential(target):
    """The same log p on the reference's float64 rows, cast to float32 first as the reference's potentials do."""
    f = TARGETS[target]
    return lambda p: f(np.asarray(p).astype(np.float32).astype(np.float64), np).astype(np.float32)


def initial_points(target, C_, D, seed=0):
    rs = np.random.RandomState(seed)
    if target == "box":
        lo, hi = np.array([b[0] for b in _BOX]), np.array([b[1] for b in _BOX])
        return lo + (hi - lo) * rs.uniform(0.05, 0.95, size=(C_, D))
    if target == "gauss":
        return np.array([1.0, -2.0]) + 0.7 * rs.randn(C_, D)
    return rs.randn(C_, D)


# ------------------------------------------------------------------------------------------------ runners
_REF_STATE_KEYS = ("state", "i", "t", "cxi", "wi", "lx", "ux", "xi", "logu")


def run_reference(target, x0, seed, num_samples, **kw):
    """The reference sampler, one chain at a time, each on its chain's Philox stream.  Per chain: the float32
    rows it evaluated, its state before every evaluation, its samples and its final widths."""
    assert ref_shim.install()
    from sbi.samplers.mcmc.slice_numpy import SliceSamplerVectorized as RefSampler
    lp = host_potential(target)
    chains = []
    for c in range(x0.shape[0]):
        rows, snaps = [], []
        ref = RefSampler(None, x0[c:c + 1].copy(), num_chains=1, verbose=False, **kw)

        def log_prob_fn(p, ref=ref, rows=rows, snaps=snaps):
            rows.append(np.asarray(p, dtype=np.float64)[0].astype(np.float32))
            snaps.append({k: ref.state[0].get(k) for k in _REF_STATE_KEYS})
            return lp(p)

        ref._log_prob_fn = log_prob_fn
        ref.rng = PhiloxDraws(seed, c)
        out = ref.run(num_samples)
        chains.append({"rows": np.stack(rows), "snaps": snaps, "samples": out[0],
                       "width": np.array(ref.state[0]["width"], dtype=np.float64)})
    return chains


def run_kernel(target, x0, seed, num_samples, **kw):
    """SliceSamplerVectorized, eager, one lock-step per host check.  Records the (C, D) float32 rows of every
    lock-step and the chains' state machine before it (and after the last one)."""
    from sbi_b200.samplers import SliceSamplerVectorized
    lp = device_potential(target)
    rows, istate, fstate = [], [], []

    def log_prob_fn(p):
        st = sampler._chain_state
        rows.append(p.cpu().numpy().copy())
        istate.append(st["istate"].cpu().numpy().copy())
        fstate.append(st["fstate"].cpu().numpy().copy())
        return lp(p)

    sampler = SliceSamplerVectorized(log_prob_fn, x0, num_chains=x0.shape[0], seed=seed, check_every=1, **kw)
    out = sampler.run(num_samples)
    istate.append(sampler._chain_state["istate"].cpu().numpy().copy())
    return {"rows": np.stack(rows), "istate": np.stack(istate), "fstate": np.stack(fstate), "samples": out,
            "width": sampler._chain_state["width"].cpu().numpy(), "num_lock_steps": sampler.num_lock_steps}


def _steps_to_done(istate, c):
    done = np.nonzero(istate[:, c, 0] == SLICE_DONE)[0]
    return int(done[0]) if done.size else None


def _divergence_report(c, k, ref, ker):
    """The first diverging chain and lock-step, with the state machine on both sides."""
    nr = len(ref["rows"])
    lines = [f"chain {c} diverges at lock-step {k} (reference: {nr} lock-steps to DONE, kernel: "
             f"{_steps_to_done(ker['istate'], c)})"]
    if k < nr:
        lines.append(f"  reference evaluates {ref['rows'][k].tolist()} in state {ref['snaps'][k]}")
    if k < len(ker["rows"]):
        ist, fst = ker["istate"][k, c], ker["fstate"][k, c]
        lines.append(f"  kernel    evaluates {ker['rows'][k, c].tolist()} in state (state, i, t) = "
                     f"{ist[:3].tolist()}, (cxi, wi, lx, ux, xi, logu) = {fst[:6].tolist()}")
    return "\n".join(lines)


def assert_chains_match(ker, ref_chains):
    for c, ref in enumerate(ref_chains):
        nr = len(ref["rows"])
        krows = ker["rows"][:nr, c]
        same = (krows == ref["rows"]) | (np.isnan(krows) & np.isnan(ref["rows"]))
        bad = np.nonzero(~same.all(axis=1))[0]
        k = int(bad[0]) if bad.size else nr
        ok = (k == nr and _steps_to_done(ker["istate"], c) == nr
              and np.array_equal(ker["samples"][c], ref["samples"]) and np.array_equal(ker["width"][c], ref["width"]))
        if not ok:
            msg = _divergence_report(c, k, ref, ker)
            if k == nr:
                msg += (f"\n  same points; samples equal: {np.array_equal(ker['samples'][c], ref['samples'])}, "
                        f"widths kernel {ker['width'][c].tolist()} vs reference {ref['width'].tolist()}")
            pytest.fail(msg)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("seed", [0, 7, 2 ** 40 + 3])
def test_draw_source_is_the_kernels_stream(cuda_lib, seed):
    """After init and one lock-step, the kernel's state gives away its first D + 1 draws: the dimension order
    (the first D - 1 words), the slice height logu = lp + log(1 - r) (the next word) and the lower bracket end
    lx = cxi - wi * r (the word after).  They must be the host stream's words, exactly; 300 chains span three
    128-thread blocks, and the last seed has a non-zero high key word."""
    from sbi_b200 import _lib as L
    lib = L.load()
    Cn, D, w0 = 300, 5, 0.01
    g = torch.Generator().manual_seed(seed % 1000)
    x = torch.randn(Cn, D, generator=g, dtype=torch.float64).cuda()
    width = torch.full((Cn, D), w0, dtype=torch.float64, device="cuda")
    order = torch.empty(Cn, D, dtype=torch.int32, device="cuda")
    istate = torch.zeros(Cn, 4, dtype=torch.int32, device="cuda")
    fstate = torch.zeros(Cn, 8, dtype=torch.float64, device="cuda")
    rng = torch.zeros(Cn, 64, dtype=torch.uint8, device="cuda")
    samples = torch.empty(Cn, 1, D, dtype=torch.float64, device="cuda")
    params = torch.empty(Cn, D, dtype=torch.float32, device="cuda")
    n_done = torch.zeros(1, dtype=torch.int32, device="cuda")
    lp = (-3.0 * torch.rand(Cn, generator=g)).float().cuda()
    s = L.SliceChains(Cn, D, 1, 0, 1e300, seed, x.data_ptr(), width.data_ptr(), order.data_ptr(),
                      istate.data_ptr(), fstate.data_ptr(), rng.data_ptr(), samples.data_ptr())
    L.check(lib.sbi_b200_slice_init(C.byref(s), L.ptr(params), L.stream_ptr()), "slice_init")
    L.check(lib.sbi_b200_slice_step(C.byref(s), L.ptr(lp), L.ptr(params), L.ptr(n_done), L.stream_ptr()),
            "slice_step")
    order, fstate, istate = order.cpu().numpy(), fstate.cpu().numpy(), istate.cpu().numpy()
    x, lp = x.cpu().numpy(), lp.cpu().numpy().astype(np.float64)
    assert (istate[:, 0] == SLICE_LOWER).all()
    for c in range(Cn):
        d = PhiloxDraws(seed, c)
        want = list(range(D))
        d.shuffle(want)
        assert order[c].tolist() == want, (c, order[c].tolist(), want)
        w_logu, w_lx = d.word(), d.word()
        cxi = x[c, want[0]]
        assert fstate[c, 0] == cxi and fstate[c, 1] == w0
        got_logu = round(math.exp(fstate[c, 5] - lp[c]) * 2.0 ** 32) - 1       # log(1 - r) = log(u)
        got_lx = round((1.0 - (cxi - fstate[c, 2]) / w0) * 2.0 ** 32) - 1      # r = 1 - u
        assert (got_logu, got_lx) == (w_logu, w_lx), (c, got_logu, w_logu, got_lx, w_lx)
        r = 1.0 - (w_lx * 2.0 ** -32 + 2.0 ** -32)
        assert fstate[c, 2] == cxi - w0 * r and fstate[c, 3] == fstate[c, 2] + w0   # no FMA: numpy's bits


_CASES = {
    # id: target, D, chains, kwargs, num_samples
    "gauss-tuned": ("gauss", 2, 130, dict(tuning=10, init_width=0.01), 40),
    "gauss-1chain-thin3": ("gauss", 2, 1, dict(tuning=0, init_width=0.5, thin=3), 40),
    "box-perdim-width": ("box", 2, 130, dict(tuning=0, init_width=np.array([1.0, 0.3])), 40),
    "box-capped-nosamples": ("box", 2, 1, dict(tuning=10, init_width=2.0, max_width=1.5), 0),
    "box-tuning-only": ("box", 2, 130, dict(tuning=10, init_width=0.05), 0),
    "quartic5-perdim-width": ("quartic", 5, 130, dict(tuning=10, thin=3,
                                                      init_width=np.array([0.05, 0.1, 0.2, 0.4, 0.8])), 40),
    "quartic5-capped": ("quartic", 5, 130, dict(tuning=0, init_width=0.01, max_width=0.05), 40),
    "quartic5-1chain-capped": ("quartic", 5, 1, dict(tuning=10, init_width=np.array([0.3, 0.3, 1.0, 1.0, 2.0]),
                                                     max_width=0.3), 40),
    "quartic1-tuned": ("quartic", 1, 130, dict(tuning=10, init_width=0.1), 40),
    "quartic1-nothing": ("quartic", 1, 1, dict(tuning=0, init_width=0.1), 0),
}


@needs_ref
@pytest.mark.parametrize("case", list(_CASES))
def test_lock_steps_match_reference(cuda_lib, case):
    """Every chain asks for the reference's points in the reference's order, needs as many lock-steps to DONE,
    and ends with the reference's samples (float64) and bracket widths."""
    target, D, Cn, kw, num_samples = _CASES[case]
    seed = 1234 + len(case)
    x0 = initial_points(target, Cn, D)
    ker = run_kernel(target, x0, seed, num_samples, **kw)
    ref = run_reference(target, x0, seed, num_samples, **kw)
    assert ker["samples"].shape == (Cn, len(range(0, num_samples, kw.get("thin", 1))), D)
    assert_chains_match(ker, ref)


@needs_ref
def test_step_out_cap_is_strict(cuda_lib):
    """The lower bracket end steps out only while it is less than `max_width` below the current point, as in the
    reference.  The draws are known ahead, so `max_width` is set to exactly the distance of the first lower end:
    the chain, sitting at the mode of the double well, must then go straight to the upper end."""
    seed, w0, x0 = 21, 0.01, np.array([[1.0]])
    d = PhiloxDraws(seed, 0)
    log_u = math.log(d.word() * 2.0 ** -32 + 2.0 ** -32)
    lx = 1.0 - w0 * d.rand()
    kw = dict(tuning=0, init_width=w0, max_width=1.0 - lx)
    assert host_potential("quartic")(np.array([[lx]]))[0] >= 0.0 + log_u, "the first lower end must be in the slice"
    ker = run_kernel("quartic", x0, seed, 5, **kw)
    ref = run_reference("quartic", x0, seed, 5, **kw)
    assert [s["state"] for s in ref[0]["snaps"][:3]] == ["BEGIN", "LOWER", "UPPER"]
    assert_chains_match(ker, ref)


_GRAPH_CASE = ("quartic", 3, 130, dict(tuning=5, init_width=np.array([0.1, 0.5, 1.0]), thin=2), 24)
_graph_ref = {}


@needs_ref
@pytest.mark.parametrize("check_every", [1, 16])
def test_graph_replay_equals_eager_equals_reference(cuda_lib, check_every):
    """The production path: `check_every` lock-steps captured once as a CUDA graph and replayed, with a potential
    that never synchronises with the host.  Samples are bit-identical to the eager run and to the reference, and
    the host stops at the first check after the slowest chain's last lock-step."""
    from sbi_b200.samplers import SliceSamplerVectorized
    target, D, Cn, kw, num_samples = _GRAPH_CASE
    seed, x0 = 99, initial_points(target, Cn, D, seed=1)
    runs = {}
    for graph in (False, True):
        s = SliceSamplerVectorized(device_potential(target), x0, num_chains=Cn, seed=seed, check_every=check_every,
                                   graph=graph, **kw)
        assert s._graph == graph
        runs[graph] = (s.run(num_samples), s.num_lock_steps)
    if not _graph_ref:
        _graph_ref["chains"] = run_reference(target, x0, seed, num_samples, **kw)
    ref = _graph_ref["chains"]
    ref_steps = max(len(r["rows"]) for r in ref)
    assert np.array_equal(runs[True][0], runs[False][0])
    for c, r in enumerate(ref):
        assert np.array_equal(runs[True][0][c], r["samples"]), f"chain {c}"
    want_steps = math.ceil(ref_steps / check_every) * check_every
    assert runs[True][1] == runs[False][1] == want_steps
