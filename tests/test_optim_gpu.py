"""The optimizer kernels of csrc/optim.cu against plain references, at the lengths, masks, step counts and
non-finite inputs where they can go wrong:

- `reduce_partials[_norm]` against a float32 emulation of its documented summation order (bit for bit), and
  its masked sum(g^2) partials against a float64 sum;
- `adam_clip_step[_norm]` against `clip_grad_norm_` + `torch.optim.Adam` in float32 on the CPU, with the
  norm taken three ways (in the step, from the reduction's partials, from the peer exchange's partials),
  under CUDA-graph replay, and with NaN / inf gradients;
- `nll_stats` against a float64 sum and an exact count of the non-finite entries.

The reference Adam runs with the float32 values of lr, betas and eps, which are what the C entry point
receives.  With the Python doubles (0.9, 0.999) torch would weight g^2 by float(0.001) where the kernel uses
1 - float(0.999) (1.3e-5 apart), and its bias corrections would differ from the kernel's by up to ~4e-6
relative at step 1000; those are differences of hyperparameter representation, not of the step."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                 # float32 unit roundoff
LR, BETA1, BETA2, EPS = (float(np.float32(v)) for v in (5e-4, 0.9, 0.999, 1e-8))
N_STEPS = 6


def _L():
    from sbi_b200 import _lib as L
    return L


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sync_check(rc, what):
    _L().check(rc, what)
    torch.cuda.synchronize()


def _mask(n, gen, zeros=0.3):
    return (torch.rand(n, generator=gen) >= zeros).to(torch.uint8)


def _assert_same(a, b, what):
    """Equal entry for entry, NaN equal to NaN, finite entries bit for bit."""
    a, b = a.detach().cpu(), b.detach().cpu()
    assert torch.equal(torch.isnan(a), torch.isnan(b)), what
    fin = ~torch.isnan(a)
    assert torch.equal(a[fin].view(torch.int32), b[fin].view(torch.int32)), what


# ---------------------------------------------------------------------------------------------------------
# gradient reduction

def _reduce_emulated(gpart):
    """grad = ((g0 + g1) + g2) + g3 in float32, group q adding partials q, q + 4, ... in order."""
    gp = gpart.numpy()
    groups = []
    for q in range(4):
        a = np.zeros(gp.shape[1], np.float32)
        for p in range(q, gp.shape[0], 4):
            a = a + gp[p]
        groups.append(a)
    return torch.from_numpy(((groups[0] + groups[1]) + groups[2]) + groups[3])


@pytest.mark.parametrize("n", [4, 256, 260, 100_000])
@pytest.mark.parametrize("n_part", [1, 2, 3, 4, 5, 8, 33, 264])
def test_reduce_partials_matches_fixed_order_sum(cuda_lib, n, n_part):
    L = _L()
    gen = torch.Generator().manual_seed(n * 1000 + n_part)
    gpart = torch.randn(n_part, n, generator=gen) * torch.exp(torch.randn(n_part, 1, generator=gen))
    mask = _mask(n, gen)
    mask[0] = 0
    gpart[:, mask == 0] = float("nan")     # must not reach the masked sum(g^2)
    want = _reduce_emulated(gpart)
    nb = cuda_lib.sbi_b200_sumsq_blocks(n)
    assert nb == math.ceil(n / 256)
    gp_d, mask_d = gpart.cuda(), mask.cuda()

    def run(with_norm, m):
        grad = torch.full((n,), 7.0, device="cuda")
        if not with_norm:
            _sync_check(cuda_lib.sbi_b200_reduce_partials(L.ptr(gp_d), n_part, n, L.ptr(grad), L.stream_ptr()), "r")
            return grad.cpu(), None
        ss = torch.full((nb,), 7.0, device="cuda")
        _sync_check(cuda_lib.sbi_b200_reduce_partials_norm(L.ptr(gp_d), n_part, n, L.ptr(grad), L.ptr(m),
                                                           L.ptr(ss), L.stream_ptr()), "rn")
        return grad.cpu(), ss.cpu()

    g0, _ = run(False, None)
    _assert_same(g0, want, "reduce_partials")
    for m in (None, mask_d):
        g, ss = run(True, m)
        _assert_same(g, want, "reduce_partials_norm grad")
        g2, ss2 = run(True, m)
        _assert_same(g2, g, "rerun grad")
        _assert_same(ss2, ss, "rerun sumsq")
        if m is None:
            assert torch.isnan(ss).any()       # the unmasked norm sees the NaN entries
            continue
        assert torch.isfinite(ss).all(), "a masked NaN leaked into the sum(g^2) partials"
        keep = mask.bool()
        sq = want.double()[keep] ** 2
        ref = sq.sum().item()
        # each partial: a product and 3 fused multiply-adds per thread, then an 8-level tree over 256 threads
        # (positive terms: within gamma_12 < 13u)
        assert abs(ss.double().sum().item() - ref) <= 13 * U * ref, (ss.double().sum().item(), ref)
        # per block as well: block b covers entries [256 b, 256 b + 256)
        per = torch.zeros(nb, dtype=torch.float64).index_add_(
            0, torch.arange(n)[keep] // 256, sq)
        assert torch.all((ss.double() - per).abs() <= 13 * U * per)
    # no mask: finite inputs give a finite norm equal to the float64 sum of squares
    fin = torch.randn(n_part, n, generator=gen).cuda()
    grad = torch.empty(n, device="cuda")
    ss = torch.empty(nb, device="cuda")
    _sync_check(cuda_lib.sbi_b200_reduce_partials_norm(L.ptr(fin), n_part, n, L.ptr(grad), None, L.ptr(ss),
                                                       L.stream_ptr()), "rn")
    ref = (_reduce_emulated(fin.cpu()).double() ** 2).sum().item()
    assert abs(ss.double().sum().item() - ref) <= 13 * U * ref


# ---------------------------------------------------------------------------------------------------------
# clip + Adam

def _gradients(n, mask, gen, steps=N_STEPS):
    """`steps` gradients whose unmasked norm alternates 20 and 0.5 (clipped / unclipped at max_norm 5).  The
    scalar tail (n % 4 entries) carries large entries, so a tail left out of the norm shows; masked entries are
    NaN, +inf or huge, so a masked entry let into the norm or the update shows."""
    keep = torch.ones(n, dtype=torch.bool) if mask is None else mask.bool()
    out = []
    for k in range(steps):
        g = torch.randn(n, generator=gen)
        tail = n % 4
        if tail:
            g[n - tail:] *= 30.0
        nrm = g[keep].double().norm().item()
        g = (g * ((20.0 if k % 2 == 0 else 0.5) / max(nrm, 1e-30))).float()
        if mask is not None:
            bad = torch.tensor([float("nan"), float("inf"), -1e30])[torch.arange(n) % 3]
            g = torch.where(keep, g, bad)
        out.append(g)
    return out


def _clip_(g, max_norm):
    """clip_grad_norm_(max_norm) in place, with the total norm taken in float64 (torch's float32 CPU norm
    is off by ~1e-5 relative at 1e6 entries, more than the kernel's float32 sum).  torch.clamp(max=1)
    keeps a NaN coefficient NaN."""
    if max_norm > 0:
        total = torch.linalg.vector_norm(g.double())
        g.mul_(torch.clamp(max_norm / (total + 1e-6), max=1.0).float())


class _Reference:
    """torch Adam in float32 on the CPU over the unmasked entries, with an elementwise first-order bound on
    how far the kernel may sit from it.

    Per step both sides round the clip coefficient (the kernel: float32 sum of squares, sqrt, + 1e-6, divide;
    the reference: one cast) and the product g * clip; `eps_g` bounds the resulting relative gap in the
    clipped gradient.  The moments carry it forward, each side adding its own roundings (lerp: 2 of
    (1 - beta1)(|g| + |m|) and |m_new|; second moment: 2 on the kernel's side and 3 on torch's, all of v_new):
        dm_k = beta1 dm_{k-1} + (1 - beta1) (eps_g |g_k| + 2u (|g_k| + |m_{k-1}|)) + 2u |m_k|
        dv_k = beta2 dv_{k-1} + (1 - beta2) 2 eps_g g_k^2 + 5u v_k
    The update step_size m / (sqrt(v) / bc2 + eps) then moves by at most
        step_size (dm + |m| dv / 2v) / denom + 14u |update|     (8 roundings on the kernel's side, 6 on torch's)
    and the parameters, which both sides round once more per step, by the sum over steps of that plus
    ulp(|p|)."""

    def __init__(self, p0, m0, v0, t0, n_sum):
        self.p = torch.nn.Parameter(p0.clone())
        self.opt = torch.optim.Adam([self.p], lr=LR, betas=(BETA1, BETA2), eps=EPS)
        if t0:
            self.opt.state[self.p] = {"step": torch.tensor(float(t0)), "exp_avg": m0.clone(),
                                      "exp_avg_sq": v0.clone()}
        self.t = t0
        # the float32 sum of squares: <= ceil(n / 1024) terms per chain, 2 combines, an 8-level tree
        sigma = (math.ceil(n_sum / 1024) + 10) * U
        self.eps_g = sigma / 2 + 6 * U
        z = torch.zeros_like(p0, dtype=torch.float64)
        self.dm, self.dv, self.dp = z.clone(), z.clone(), z.clone()
        self.m_prev = m0.double()

    def step(self, g, max_norm):
        eps_g = self.eps_g if max_norm > 0 else 0.0      # unclipped: the same float32 gradient on both sides
        g = g.clone()
        _clip_(g, max_norm)
        self.p.grad = g
        self.opt.step()
        self.t += 1
        st = self.opt.state[self.p]
        m_prev = self.m_prev
        m, v, gd = st["exp_avg"].double(), st["exp_avg_sq"].double(), g.double()
        self.m_prev = m
        self.dm = (BETA1 * self.dm + (1 - BETA1) * (eps_g * gd.abs() + 2 * U * (gd.abs() + m_prev.abs()))
                   + 2 * U * m.abs())
        self.dv = BETA2 * self.dv + (1 - BETA2) * 2 * eps_g * gd * gd + 5 * U * v
        bc1, bc2s = 1 - BETA1 ** self.t, math.sqrt(1 - BETA2 ** self.t)
        denom = v.sqrt() / bc2s + EPS
        upd = LR / bc1 * m / denom
        rel_v = torch.where(v > 0, self.dv / (2 * v), torch.zeros_like(v))
        ulp = torch.from_numpy(np.spacing(self.p.detach().abs().numpy())).double()
        self.dp = self.dp + LR / bc1 * (self.dm + m.abs() * rel_v) / denom + 14 * U * upd.abs() + ulp

    def worst(self, p, m, v):
        """max over entries of |kernel - reference| / bound, for params, m and v; NaN must sit where the
        reference has NaN."""
        st = self.opt.state[self.p]
        pr = self.p.detach()
        out = []
        for got, ref, bound in ((p, pr, self.dp), (m, st["exp_avg"], self.dm), (v, st["exp_avg_sq"], self.dv)):
            nan = torch.isnan(ref)
            assert torch.equal(torch.isnan(got), nan), "NaN pattern differs from torch"
            err = (got.double() - ref.double()).abs()[~nan]
            ratio = torch.where(err == 0, torch.zeros_like(err), err / bound[~nan])
            out.append(ratio.max().item() if ratio.numel() else 0.0)
        return out


class _Kernel:
    def __init__(self, lib, p0, m0, v0, t0, mask):
        self.lib = lib
        self.n = p0.numel()
        self.p = p0.cuda()
        self.state = torch.cat([m0, v0]).cuda()
        self.step = torch.tensor([t0, 0], dtype=torch.int32, device="cuda")
        self.mask = None if mask is None else mask.cuda()

    def adam(self, grad, max_norm, sumsq=None):
        L = _L()
        if sumsq is None:
            rc = self.lib.sbi_b200_adam_clip_step(L.ptr(self.p), L.ptr(grad), L.ptr(self.state), L.ptr(self.step),
                                                  L.ptr(self.mask), self.n, LR, BETA1, BETA2, EPS, max_norm, 1.0,
                                                  L.stream_ptr())
        else:
            rc = self.lib.sbi_b200_adam_clip_step_norm(L.ptr(self.p), L.ptr(grad), L.ptr(self.state),
                                                       L.ptr(self.step), L.ptr(self.mask), self.n, LR, BETA1,
                                                       BETA2, EPS, max_norm, 1.0, L.ptr(sumsq), sumsq.numel(),
                                                       L.stream_ptr())
        L.check(rc, "adam_clip_step")

    def tensors(self):
        return self.p.cpu(), self.state[:self.n].cpu(), self.state[self.n:].cpu()


def _start(n, t0, gen):
    p0 = torch.randn(n, generator=gen) * 0.05       # small, so that ulp(|p|) hides little of the update
    if t0 == 1:
        return p0, torch.zeros(n), torch.zeros(n)
    # a state as after many steps: |m| below sqrt(v), both on the scale of the gradients
    v0 = (torch.rand(n, generator=gen) * 2 + 0.1) * (10.0 / n)
    m0 = torch.randn(n, generator=gen) * v0.sqrt() * 0.5
    return p0, m0, v0


_LENGTHS = [1, 3, 5, 1023, 1025, 10_000, 132 * 1024 + 3, 1_000_003]


@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "mask"])
@pytest.mark.parametrize("t0", [1, 1000, 100_000])
@pytest.mark.parametrize("max_norm", [5.0, 0.0])
@pytest.mark.parametrize("n", _LENGTHS)
def test_adam_clip_step_matches_torch(cuda_lib, n, max_norm, t0, masked):
    """`sbi_b200_adam_clip_step` (norm taken in the step) over six clipped / unclipped gradients against
    clip_grad_norm_ + torch Adam; masked entries of params, m and v keep their bits; d_step counts."""
    gen = torch.Generator().manual_seed(n + int(max_norm) + t0 + masked)
    mask = None
    if masked:
        mask = _mask(n, gen)
        mask[0] = 1                              # at least one trainable entry
    keep = torch.ones(n, dtype=torch.bool) if mask is None else mask.bool()
    p0, m0, v0 = _start(n, t0, gen)
    grads = _gradients(n, mask, gen)
    k = _Kernel(cuda_lib, p0, m0, v0, t0, mask)
    ref = _Reference(p0[keep], m0[keep], v0[keep], t0, n)
    worst = [0.0, 0.0, 0.0]
    for it, g in enumerate(grads):
        k.adam(g.cuda(), max_norm)
        ref.step(g[keep], max_norm)
        assert k.step.cpu().tolist() == [t0 + it + 1, 0], (it, k.step.cpu().tolist())
        p, m, v = k.tensors()
        w = ref.worst(p[keep], m[keep], v[keep])
        worst = [max(a, b) for a, b in zip(worst, w)]
        assert max(w) <= 1.0, (it, w)
        if masked:
            for got, was in ((p, p0), (m, m0), (v, v0)):
                assert torch.equal(got[~keep].view(torch.int32), was[~keep].view(torch.int32)), it
    print(f"n={n} max_norm={max_norm} t0={t0} mask={masked} grid={min(math.ceil(n / 1024), _num_sms())}: "
          f"worst |err|/bound params {worst[0]:.3f}  m {worst[1]:.3f}  v {worst[2]:.3f}")


@pytest.mark.parametrize("n", [10_000, 1_000_000])
@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "mask"])
def test_norm_sources_agree(cuda_lib, n, masked):
    """One gradient, reduced from three per-CTA partials, and its clip norm taken three ways: in the Adam
    step, from the reduction's sum(g^2) partials, and from the peer exchange's partials (one rank, so no
    peer to wait for).  The norms differ only in float32 summation order, so the parameters agree within the
    torch reference's bound with both norms in error."""
    L = _L()
    lib = cuda_lib
    gen = torch.Generator().manual_seed(n + masked)
    mask = _mask(n, gen) if masked else None
    mask_d = None if mask is None else mask.cuda()
    p0, m0, v0 = _start(n, 1000, gen)
    peer = lib.sbi_b200_peer_alloc(n)
    assert peer
    try:
        ptrs = (C.c_void_p * 1)(peer)
        runs = [_Kernel(lib, p0, m0, v0, 1000, mask) for _ in range(3)]
        grad = torch.empty(n, device="cuda")
        grad_peer = torch.empty(n, device="cuda")
        ss = torch.empty(lib.sbi_b200_sumsq_blocks(n), device="cuda")
        ss_peer = torch.empty(lib.sbi_b200_peer_blocks(n), device="cuda")
        keep = torch.ones(n, dtype=torch.bool) if mask is None else mask.bool()
        env = _Reference(p0[keep], m0[keep], v0[keep], 1000, n)
        env.eps_g *= 2                           # two float32 norms, each within eps_g of the exact one
        for it in range(N_STEPS):
            gpart = (torch.randn(3, n, generator=gen) * (4.0 if it % 2 == 0 else 1e-3)).cuda()
            L.check(lib.sbi_b200_reduce_partials_norm(L.ptr(gpart), 3, n, L.ptr(grad), L.ptr(mask_d), L.ptr(ss),
                                                      L.stream_ptr()), "reduce")
            L.check(lib.sbi_b200_peer_sum(L.ptr(grad), ptrs, 1, 0, n, L.ptr(grad_peer), L.ptr(mask_d),
                                          L.ptr(ss_peer), None, L.stream_ptr()), "peer_sum")
            runs[0].adam(grad, 5.0)
            runs[1].adam(grad, 5.0, ss)
            runs[2].adam(grad_peer, 5.0, ss_peer)
            torch.cuda.synchronize()
            _assert_same(grad_peer, grad, "one-rank peer sum")
            env.step(grad.cpu()[keep], 5.0)
        p = [r.p.cpu()[keep] for r in runs]
        bound = env.dp
        for other in p[1:]:
            err = (other.double() - p[0].double()).abs()
            print(f"n={n} mask={masked}: worst |err|/bound between norm sources {(err / bound).max().item():.3f}")
            assert torch.all(err <= bound), (err / bound).max().item()
        for r in runs:
            assert r.step.cpu().tolist() == [1000 + N_STEPS, 0]
    finally:
        torch.cuda.synchronize()
        lib.sbi_b200_peer_free(C.c_void_p(peer))


def test_graph_replay_matches_eager(cuda_lib):
    """reduce_partials_norm + adam_clip_step_norm captured once and replayed 7 times, with fresh partials
    copied into the captured input each time, gives the bits of 7 eager launches, and the step counter
    advances once per replay."""
    L = _L()
    lib = cuda_lib
    n, n_part = 10_000, 5
    gen = torch.Generator().manual_seed(7)
    mask = _mask(n, gen).cuda()
    p0 = torch.randn(n, generator=gen)
    parts = [torch.randn(n_part, n, generator=gen) * (3.0 if i % 2 == 0 else 0.01) for i in range(7)]
    nb = lib.sbi_b200_sumsq_blocks(n)

    def setup():
        return (p0.clone().cuda(), torch.zeros(2 * n, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda"),
                torch.zeros(n_part, n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(nb, device="cuda"))

    def launch(p, state, step, gpart, grad, ss):
        L.check(lib.sbi_b200_reduce_partials_norm(L.ptr(gpart), n_part, n, L.ptr(grad), L.ptr(mask), L.ptr(ss),
                                                  L.stream_ptr()), "reduce")
        L.check(lib.sbi_b200_adam_clip_step_norm(L.ptr(p), L.ptr(grad), L.ptr(state), L.ptr(step), L.ptr(mask), n,
                                                 LR, BETA1, BETA2, EPS, 5.0, 1.0, L.ptr(ss), nb, L.stream_ptr()),
                "adam")

    eager = setup()
    for gp in parts:
        eager[3].copy_(gp)
        launch(*eager)
    torch.cuda.synchronize()
    assert eager[2].cpu().tolist() == [7, 0]

    static = setup()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch(*static)
    torch.cuda.synchronize()
    assert static[2].cpu().tolist() == [0, 0], "capture must not run the step"
    for gp in parts:
        static[3].copy_(gp)
        graph.replay()
    torch.cuda.synchronize()
    assert static[2].cpu().tolist() == [7, 0]
    for a, b, what in ((static[0], eager[0], "params"), (static[1], eager[1], "state"), (static[4], eager[4], "grad")):
        _assert_same(a, b, what)


@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "mask"])
@pytest.mark.parametrize("n", [5, 1025, 132 * 1024 + 3])
def test_unmasked_nan_gradient_makes_every_parameter_nan(cuda_lib, n, masked):
    """One NaN in the trainable gradient makes clip_grad_norm_'s coefficient NaN, so torch turns every
    gradient, moment and parameter NaN; the kernel must do the same (masked entries keep their bits)."""
    gen = torch.Generator().manual_seed(n + masked)
    mask = _mask(n, gen) if masked else None
    keep = torch.ones(n, dtype=torch.bool) if mask is None else mask.bool()
    keep[n // 2] = True
    if mask is not None:
        mask[n // 2] = 1
    p0, m0, v0 = _start(n, 1000, gen)
    g = _gradients(n, mask, gen, steps=1)[0]
    g[n // 2] = float("nan")
    ref = _Reference(p0[keep], m0[keep], v0[keep], 1000, n)
    ref.step(g[keep], 5.0)
    assert torch.isnan(ref.p.detach()).all()     # torch: every trainable parameter
    k = _Kernel(cuda_lib, p0, m0, v0, 1000, mask)
    k.adam(g.cuda(), 5.0)
    p, m, v = k.tensors()
    for got, was, what in ((p, p0, "params"), (m, m0, "m"), (v, v0, "v")):
        assert torch.isnan(got[keep]).all(), f"{what}: {int((~torch.isnan(got[keep])).sum())} finite entries"
        assert torch.equal(got[~keep].view(torch.int32), was[~keep].view(torch.int32)), what
    assert k.step.cpu().tolist() == [1001, 0]


@pytest.mark.parametrize("bad", ["nan_unclipped", "inf"])
@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "mask"])
@pytest.mark.parametrize("n", [5, 1025, 132 * 1024 + 3])
def test_nonfinite_gradient_matches_torch_entrywise(cuda_lib, n, masked, bad):
    """A +inf with clipping (coefficient 0: NaN in that entry alone, the others take a zero-gradient step), and
    a NaN without clipping (NaN in that entry alone): entry for entry as torch, NaN equal to NaN."""
    gen = torch.Generator().manual_seed(n + masked + len(bad))
    mask = _mask(n, gen) if masked else None
    keep = torch.ones(n, dtype=torch.bool) if mask is None else mask.bool()
    j = n - 1                                   # in the scalar tail when n % 4 != 0
    keep[j] = True
    if mask is not None:
        mask[j] = 1
    max_norm = 5.0 if bad == "inf" else 0.0
    p0, m0, v0 = _start(n, 1000, gen)
    k = _Kernel(cuda_lib, p0, m0, v0, 1000, mask)
    ref = _Reference(p0[keep], m0[keep], v0[keep], 1000, n)
    g = _gradients(n, mask, gen, steps=1)[0]
    g[j] = float("inf") if bad == "inf" else float("nan")
    k.adam(g.cuda(), max_norm)
    ref.step(g[keep], max_norm)
    assert int(torch.isnan(ref.p.detach()).sum()) == 1        # torch: NaN in that entry alone
    p, m, v = k.tensors()
    w = ref.worst(p[keep], m[keep], v[keep])
    assert max(w) <= 1.0, w
    if mask is not None:
        for got, was in ((p, p0), (m, m0), (v, v0)):
            assert torch.equal(got[~keep].view(torch.int32), was[~keep].view(torch.int32))


# ---------------------------------------------------------------------------------------------------------
# validation statistics

@pytest.mark.parametrize("n", [0, 1, 31, 32, 1023, 1024, 1025, 1_000_000])
def test_nll_stats(cuda_lib, n):
    """-sum of the finite log-probs and the exact count of the non-finite ones."""
    L = _L()
    gen = torch.Generator().manual_seed(n)
    lp = torch.randn(max(n, 1), generator=gen) * 3 - 2
    if n:
        idx = torch.randperm(n, generator=gen)[:min(n, max(3, n // 50))]
        lp[idx] = torch.tensor([float("nan"), float("inf"), -float("inf")])[torch.arange(idx.numel()) % 3]
    lp_d = lp.cuda()
    out = torch.full((2,), 123.0, device="cuda")
    _sync_check(cuda_lib.sbi_b200_nll_stats(L.ptr(lp_d), n, L.ptr(out), L.stream_ptr()), "nll_stats")
    s, bad = out.cpu().tolist()
    x = lp[:n].double()
    fin = torch.isfinite(x)
    assert bad == float((~fin).sum().item())
    want = -x[fin].sum().item()
    assert abs(s - want) <= 1e-6 * x[fin].abs().sum().item(), (s, want)
    if n == 0:
        assert [s, bad] == [0.0, 0.0]


# ---------------------------------------------------------------------------------------------------------
# argument errors that need a device pointer to reach (a null pointer is caught first; test_abi_cpu.py)

def test_argument_errors_with_device_pointers(cuda_lib):
    L = _L()
    lib = cuda_lib
    s = L.stream_ptr()
    gp = torch.ones(3, 8, device="cuda")
    grad = torch.full((8,), 7.0, device="cuda")
    ss = torch.full((2,), 7.0, device="cuda")
    assert lib.sbi_b200_reduce_partials_norm(L.ptr(gp), 3, 6, L.ptr(grad), None, L.ptr(ss), s) == -1   # n % 4
    assert lib.sbi_b200_reduce_partials_norm(L.ptr(gp), 3, 2, L.ptr(grad), None, L.ptr(ss), s) == -1   # n < 4
    assert lib.sbi_b200_reduce_partials_norm(L.ptr(gp), 0, 8, L.ptr(grad), None, L.ptr(ss), s) == -1   # n_part
    assert lib.sbi_b200_reduce_partials(L.ptr(gp), 0, 8, L.ptr(grad), s) == -1
    p = torch.full((8,), 3.0, device="cuda")
    state = torch.zeros(16, device="cuda")
    step = torch.zeros(2, dtype=torch.int32, device="cuda")
    args = (L.ptr(p), L.ptr(grad), L.ptr(state), L.ptr(step), None)
    hyper = (LR, BETA1, BETA2, EPS, 5.0, 1.0)
    assert lib.sbi_b200_adam_clip_step_norm(*args, 8, *hyper, L.ptr(ss), 0, s) == -1       # partials, none counted
    assert lib.sbi_b200_adam_clip_step_norm(*args, 0, *hyper, L.ptr(ss), 2, s) == -1
    assert lib.sbi_b200_adam_clip_step(*args, 0, *hyper, s) == -1
    assert lib.sbi_b200_nll_stats(L.ptr(grad), -1, L.ptr(ss), s) == -1
    torch.cuda.synchronize()
    assert torch.all(grad == 7.0) and torch.all(ss == 7.0) and torch.all(p == 3.0)
    assert torch.all(state == 0) and step.cpu().tolist() == [0, 0]
