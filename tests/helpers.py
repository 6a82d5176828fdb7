"""Shared helpers for the parity tests (oracle side = oracle/, CUDA side = sbi_b200)."""
from collections import namedtuple

import torch

from oracle import sbi_port


def oracle_nsf(D=10, C=10, n=2000, seed=0, perturb=0.1, lu_perturb=0.1, **kw):
    """Oracle NSF (reference builder restated) with weights moved off their init so that
    every code path (GLU, LU off-diagonals, all spline bins) is exercised."""
    g = torch.Generator().manual_seed(seed)
    theta = 0.7 * torch.randn(n, D, generator=g) + 0.3
    x = 1.3 * torch.randn(n, C, generator=g) - 0.2
    torch.manual_seed(seed)
    flow = sbi_port.build_nsf(theta, x, **kw)
    with torch.no_grad():
        for name, p in flow.named_parameters():
            s = lu_perturb if ("entries" in name or "diag" in name) else perturb
            p.add_(s * torch.randn(p.shape, generator=g))
    return flow, theta, x


def b200_from_oracle(flow, theta, x, device="cuda", **kw):
    from sbi_b200.neural_nets import build_nsf
    est = build_nsf(theta, x, **kw)
    est.load_state_dict(flow.state_dict())
    return est.to(device)


def nsf_vjp_raw(est, inp, cond, g, save, fill=0.0):
    """sbi_b200_nsf_vjp of sum_r g_r log q(inp_r | cond_r) on the current stream, with `save` (a CUDA tensor, or
    None) as the activation scratch: (return code, per-CTA partials, input gradient, condition gradient,
    log-probs), the four outputs allocated and filled with `fill` before the call."""
    import ctypes as C
    from sbi_b200 import _lib as L
    lib = L.load()
    R = inp.shape[0]
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)
    gpart = torch.full((lib.sbi_b200_nsf_vjp_parts(R), est.layout.n_params), fill, device=inp.device)
    ginp, gcond = torch.full_like(inp, fill), torch.full_like(cond, fill)
    logp = torch.full((R,), fill, device=inp.device)
    rc = lib.sbi_b200_nsf_vjp(C.byref(m), C.byref(rows), L.ptr(g), 0.0, L.ptr(logp), L.ptr(gpart), L.ptr(ginp),
                              L.ptr(gcond), None, L.ptr(save), 0 if save is None else save.numel() * 4,
                              torch.cuda.current_stream().cuda_stream)
    return rc, gpart, ginp, gcond, logp


VjpStep = namedtuple("VjpStep", "gpart grad logp loss_acc gcond")


def use_vjp_path(monkeypatch, est, tc):
    """Run the training VJP of `est` on the tensor-core pair (`tc`) or on the SIMT kernel for the rest of the test
    (SBI_B200_VJP_TC through `monkeypatch`), and drop the estimator's cached verdict."""
    monkeypatch.setenv("SBI_B200_VJP_TC", "1" if tc else "0")
    est._cache.pop("tc_train", None)


def vjp_step(est, inp, cond, g, *, g_const=0.0, with_cond=False, tc=True, graph=False):
    """One training step of sum_r g_r log q(inp_r | cond_r) (g_const for every row when `g` is None) through
    est.vjp, on the tensor-core pair when `tc`, else on the SIMT kernel (asserted either way); with `with_cond`
    also the condition gradient.  Outputs start as NaN on the tensor-core pair, which writes every entry, and as
    zero on the SIMT kernel.  Eager, or with `graph` captured once in a CUDA graph (after a warm-up on a side
    stream) and replayed `int(graph)` times from fresh outputs, every replay bit-identical to the first.
    Returns CPU copies: VjpStep(partial-gradient slabs, their sum, log-probs, loss statistics, condition gradient
    or None)."""
    from sbi_b200 import _lib as L
    R = inp.shape[0]
    assert est._vjp_uses_tc(R, True) == tc
    P, n_part = est.layout.n_params, est.vjp_parts(R)
    fill = float("nan") if tc else 0.0
    gpart = torch.full((n_part, P), fill, device="cuda")
    lp = torch.full((R,), fill, device="cuda")
    acc = torch.zeros(2, device="cuda")
    gcond = torch.full((R, cond.shape[1]), fill, device="cuda") if with_cond else None
    m = est._model(nbuf=3)
    rows = L.Rows(inp.data_ptr(), cond.data_ptr(), None, R, 0)

    def step():
        est.vjp(m, rows, R, g, g_const, lp, gpart, None, gcond, acc, cond_tc=with_cond)

    def result():
        grad = L.reduce_partials(gpart, n_part, P)
        return VjpStep(gpart.cpu(), grad.cpu(), lp.cpu(), acc.cpu(), None if gcond is None else gcond.cpu())

    if not graph:
        step()
        return result()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    cuda_graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(cuda_graph):
        step()
    outs = []
    for _ in range(int(graph)):
        for t in (gpart, lp, gcond):
            if t is not None:
                t.fill_(fill)
        acc.zero_()
        cuda_graph.replay()
        outs.append(result())
    for rep, out in enumerate(outs[1:], 1):
        for name in ("gpart", "logp", "gcond"):
            a, b = getattr(out, name), getattr(outs[0], name)
            assert a is None or torch.equal(a, b), f"replay {rep}: {name} differ from the first replay"
    return outs[0]


def oracle_maf(D=3, C=2, n=2000, seed=0, perturb=0.1, scale_fn="softplus", rqs=False, **kw):
    """Oracle MAF, or with `rqs` MAF-RQS (spline element-wise maps), with perturbed weights."""
    from oracle.nflows_port.transforms import autoregressive as _ar
    _ar.MAF_SCALE_FN = scale_fn
    g = torch.Generator().manual_seed(seed)
    theta = 0.7 * torch.randn(n, D, generator=g) + 0.3
    x = 1.3 * torch.randn(n, C, generator=g) - 0.2
    torch.manual_seed(seed)
    flow = (sbi_port.build_maf_rqs if rqs else sbi_port.build_maf)(theta, x, **kw)
    with torch.no_grad():
        for name, p in flow.named_parameters():
            p.add_(perturb * torch.randn(p.shape, generator=g))
    return flow, theta, x


def b200_maf_from_oracle(flow, theta, x, device="cuda", scale_fn="softplus", rqs=False, **kw):
    from sbi_b200.neural_nets import build_maf, build_maf_rqs
    if rqs:
        est = build_maf_rqs(theta, x, **kw)
    else:
        est = build_maf(theta, x, maf_scale_softplus=(scale_fn == "softplus"), **kw)
    est.load_state_dict(flow.state_dict())
    return est.to(device)


_M32 = 0xFFFFFFFF
_PHILOX_M0, _PHILOX_M1 = 0xD2511F53, 0xCD9E8D57      # round multipliers
_PHILOX_W0, _PHILOX_W1 = 0x9E3779B9, 0xBB67AE85      # key schedule (Weyl) increments


def philox4x32_10(ctr, key):
    """Random123's Philox4x32-10 block function as cuRAND computes it (curand_philox4x32_x.h): ten rounds of
    two 32x32->64 multiplies on the 4-word counter, the 2-word key bumped by the Weyl constants between rounds.
    Returns the four output words."""
    c0, c1, c2, c3 = (int(w) & _M32 for w in ctr)
    k0, k1 = (int(w) & _M32 for w in key)
    for rnd in range(10):
        if rnd:
            k0, k1 = (k0 + _PHILOX_W0) & _M32, (k1 + _PHILOX_W1) & _M32
        p0, p1 = _PHILOX_M0 * c0, _PHILOX_M1 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & _M32, (p0 >> 32) ^ c3 ^ k1, p0 & _M32
    return c0, c1, c2, c3


class PhiloxDraws:
    """The random stream of one slice-sampler chain (csrc/slice.cu), restated on the host.

    Chain `c` of a run with seed `s` draws from `curand_init(s, subsequence=c, offset=0)` on Philox4x32-10: the key
    is the seed's low and high 32-bit words, the counter starts at (0, 0, low, high) of the subsequence, and
    `curand()` hands out the four words of each block in order before the counter's low 64 bits step by one.
    `curand_uniform_double` takes ONE word x and returns x * 2^-32 + 2^-32 in (0, 1].

    On top of that, the kernel's own conventions, so that the object stands in for `np.random` inside the
    reference sampler: `rand()` is `1 - uniform` in [0, 1) (`rand01`) and `shuffle(list)` is the kernel's
    Fisher-Yates (`shuffle_order`).  Every value is exact in float64."""

    def __init__(self, seed: int, subsequence: int = 0):
        self.key = (seed & _M32, (seed >> 32) & _M32)
        self.ctr = [0, 0, subsequence & _M32, (subsequence >> 32) & _M32]
        self._block = philox4x32_10(self.ctr, self.key)
        self._next = 0
        self.n_words = 0          # words handed out so far

    def word(self) -> int:
        """curand(): the next 32-bit word."""
        if self._next == 4:
            lo = ((self.ctr[1] << 32) | self.ctr[0]) + 1
            self.ctr[0], self.ctr[1] = lo & _M32, (lo >> 32) & _M32
            if lo >> 64:              # carry into the high half of the counter
                hi = (((self.ctr[3] << 32) | self.ctr[2]) + 1) & ((1 << 64) - 1)
                self.ctr[2], self.ctr[3] = hi & _M32, hi >> 32
            self._block = philox4x32_10(self.ctr, self.key)
            self._next = 0
        w = self._block[self._next]
        self._next += 1
        self.n_words += 1
        return w

    def rand(self) -> float:
        return 1.0 - (self.word() * 2.0 ** -32 + 2.0 ** -32)

    def shuffle(self, order: list) -> None:
        for i in range(len(order) - 1, 0, -1):
            j = min(int(self.rand() * (i + 1)), i)
            order[i], order[j] = order[j], order[i]


def two_moons_simulator(parameters, r_loc=0.1, r_scale=0.01, base_offset=0.25):
    """The two-moons simulator of the reference's mini benchmark, restated
    (/root/reference/tests/mini_sbibm/two_moons.py:15-78): a noisy half circle shifted by
    (-|z0|, z1), z = parameters rotated by -45 degrees."""
    import math
    n = parameters.shape[0]
    a = (torch.rand(n, 1) - 0.5) * math.pi
    r = r_loc + r_scale * torch.randn(n, 1)
    p = torch.cat((torch.cos(a) * r + base_offset, torch.sin(a) * r), dim=1)
    c, s = math.cos(-math.pi / 4.0), math.sin(-math.pi / 4.0)
    z0 = (c * parameters[:, 0] - s * parameters[:, 1]).reshape(-1, 1)
    z1 = (s * parameters[:, 0] + c * parameters[:, 1]).reshape(-1, 1)
    return p + torch.cat((-torch.abs(z0), z1), dim=1)


def c2st(X, Y, seed=1, n_folds=5):
    """Classifier two-sample test accuracy as the reference computes it by default
    (/root/reference/sbi/utils/metrics.py:56-190): both sets z-scored with X's statistics, a
    RandomForestClassifier (100 trees... sklearn defaults) scored by 5-fold shuffled cross-validation."""
    import numpy as np
    from sklearn.ensemble import RandomForestClassifier
    from sklearn.model_selection import KFold, cross_val_score
    X, Y = X.double(), Y.double()
    mean, std = X.mean(0), X.std(0)
    std[std == 0] = 1.0
    X, Y = (X - mean) / std, (Y - mean) / std
    data = np.concatenate((X.numpy(), Y.numpy()))
    target = np.concatenate((np.zeros(X.shape[0]), np.ones(Y.shape[0])))
    clf = RandomForestClassifier(random_state=seed, n_jobs=-1)
    shuffle = KFold(n_splits=n_folds, shuffle=True, random_state=seed)
    return float(cross_val_score(clf, data, target, cv=shuffle, scoring="accuracy").mean())
