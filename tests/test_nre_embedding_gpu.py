"""Learned embedding nets in the NRE `resnet` classifier on the GPU: the input gradients of the ratio VJP kernel
and the pair -> row gradient sum against fp64 oracles, `_RatioFn` with index gathers, the graph-captured NRE
trainers against an eager replay of the reference's repeated-row step, best-epoch restore / resume, posterior fits
and the reference trainer driving the estimator."""
import copy
import ctypes as C_
import math
import warnings

import pytest
import torch
from torch import nn

from oracle import ref_shim, sbi_port
from oracle.nflows_port.nn.nets import ResidualNet

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")


def _fc(d_in, d_out, seed=5):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(d_in, 32), nn.ReLU(), nn.Linear(32, d_out))


def _theta_net(seed=8):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(2, 6), nn.Tanh())


class _Conv(nn.Module):
    def __init__(self):
        super().__init__()
        torch.manual_seed(6)
        self.conv = nn.Conv1d(2, 4, 5)
        self.fc = nn.Linear(4 * 21, 6)

    def forward(self, x):
        return self.fc(torch.relu(self.conv(x)).flatten(1))


def _copies_task(n, seed=0):
    """theta ~ N(0, I_2), x = 25 noisy copies of theta (50-d, sigma 1): posterior N(sum_k x_k / 26, I / 26)."""
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(n, 2, generator=g)
    x = theta.repeat(1, 25) + torch.randn(n, 50, generator=g)
    return theta, x


def _oracle_of(est, perturb=0.0, seed=0):
    """An independent fp32 copy of `est` in the oracle's classes (nflows ResidualNet behind sbi's RatioEstimator),
    with the same weights; `perturb` first moves every classifier weight by N(0, perturb^2) (through the state
    dict, so the packed buffer's padding stays zero) and loads the result back into `est`."""
    lay = est.layout
    net = ResidualNet(in_features=lay.Dt + lay.Dx, out_features=1, hidden_features=lay.H, context_features=None,
                      num_blocks=lay.NB, activation=torch.relu)
    ref = sbi_port.RatioEstimator(net, est.theta_shape, est.x_shape, copy.deepcopy(est.embedding_net_theta).cpu(),
                                  copy.deepcopy(est.embedding_net_x).cpu())
    ref.load_state_dict({k: v.cpu() for k, v in est.state_dict().items()})
    if perturb:
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            for p in ref.net.parameters():
                p.add_(perturb * torch.randn(p.shape, generator=g))
        est.load_state_dict(ref.state_dict())
    return ref


def _rel_err(got, r32, r64, scale=0.0):
    sc = max(r64.abs().max().item(), scale, 1e-30)
    return (got.cpu().double() - r64).abs().max().item() / sc, (r32.double() - r64).abs().max().item() / sc


def _assert_grad(what, got, r32, r64, scale=0.0):
    """Error relative to the max-norm of the reference gradient, or `scale` when that is larger (tensors whose exact
    gradient is 0, like the final bias under a softmax loss)."""
    err, err32 = _rel_err(got, r32, r64, scale)
    print(f"{what}: rel err {err:.2e} (torch fp32 {err32:.2e})")
    assert err <= max(2e-3, 4 * err32), (what, err, err32)


# ---------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("Dt,Dx,R", [(1, 1, 64), (3, 5, 77), (4, 6, 200), (7, 13, 1000), (1, 9, 33), (10, 2, 4099)])
def test_vjp_input_gradients_match_oracle(cuda_lib, Dt, Dx, R):
    """gtheta and gx of `sbi_b200_ratio_vjp_inputs` (identity embeddings: raw rows z-scored in-kernel, so the
    gradients pass the 1/std) against fp64 autograd of the oracle; partials, logits and gtheta bit-identical to
    `sbi_b200_ratio_vjp`; two calls bit-identical."""
    from sbi_b200 import _lib as L
    from sbi_b200.ratio import classifier_nn
    g = torch.Generator().manual_seed(Dt * 100 + Dx)
    theta = 0.7 * torch.randn(R, Dt, generator=g) + 0.3
    x = 1.5 * torch.randn(R, Dx, generator=g) - 0.2
    torch.manual_seed(0)
    est = classifier_nn("resnet")(theta, x).cuda()
    ref = _oracle_of(est, perturb=0.1)
    w = torch.randn(R, generator=g)

    def oracle(dtype):
        r = copy.deepcopy(ref).to(dtype)
        t, xx = theta.to(dtype).clone().requires_grad_(True), x.to(dtype).clone().requires_grad_(True)
        (r(t, xx) * w.to(dtype)).sum().backward()
        return t.grad, xx.grad

    (t32, x32), (t64, x64) = oracle(torch.float32), oracle(torch.float64)
    tc, xc = theta.cuda().requires_grad_(True), x.cuda().requires_grad_(True)
    (est(tc, xc) * w.cuda()).sum().backward()
    _assert_grad(f"gtheta Dt={Dt} Dx={Dx} R={R}", tc.grad, t32, t64)
    _assert_grad(f"gx Dt={Dt} Dx={Dx} R={R}", xc.grad, x32, x64)

    lib = cuda_lib
    n_part = lib.sbi_b200_ratio_vjp_parts(R)
    th, xx, wc = theta.cuda().contiguous(), x.cuda().contiguous(), w.cuda().contiguous()
    m = est._model(nbuf=3)
    pr = L.Pairs(th.data_ptr(), xx.data_ptr(), None, None, R, 0)

    def run(with_gx, old_entry=False):
        gp = torch.zeros(n_part, est.layout.n_params, device="cuda")
        lg = torch.zeros(R, device="cuda")
        gt = torch.zeros(R, Dt, device="cuda")
        gx = torch.zeros(R, Dx, device="cuda") if with_gx else None
        if old_entry:
            rc = lib.sbi_b200_ratio_vjp(C_.byref(m), C_.byref(pr), L.ptr(wc), L.ptr(lg), L.ptr(gp), L.ptr(gt),
                                        L.stream_ptr())
        else:
            rc = lib.sbi_b200_ratio_vjp_inputs(C_.byref(m), C_.byref(pr), L.ptr(wc), L.ptr(lg), L.ptr(gp), L.ptr(gt),
                                               L.ptr(gx), L.stream_ptr())
        L.check(rc, "ratio_vjp")
        torch.cuda.synchronize()
        return gp, lg, gt, gx

    a, b, c = run(True), run(True), run(False, old_entry=True)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    for u, v in zip(a[:3], c[:3]):
        assert torch.equal(u, v)


@pytest.mark.parametrize("n_pairs,n_rows,width", [(1000, 37, 8), (4096, 4096, 3), (50, 200, 1), (20000, 500, 13)])
def test_pair_rows_sum_matches_index_add(cuda_lib, n_pairs, n_rows, width):
    """`sbi_b200_pair_rows_sum` == fp64 index_add_ to fp32 rounding; rows no pair touches are zero; repeat calls are
    bit-identical; consecutive segments (order NULL) give the same sums as the sorted general path."""
    from sbi_b200.ratio import pair_rows_sum
    g = torch.Generator().manual_seed(n_pairs + width)
    gp = torch.randn(n_pairs, width, generator=g).cuda()
    idx = torch.randint(0, max(n_rows // 2, 1), (n_pairs,), generator=g).cuda()     # upper rows untouched
    ref = torch.zeros(n_rows, width, dtype=torch.float64).index_add_(0, idx.cpu(), gp.cpu().double())
    a, b = pair_rows_sum(gp, idx, n_rows), pair_rows_sum(gp, idx, n_rows)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    cnt = torch.bincount(idx.cpu(), minlength=n_rows)
    assert (a.cpu()[cnt == 0] == 0).all()
    err = (a.cpu().double() - ref).abs().max().item()
    absum = torch.zeros(n_rows, width, dtype=torch.float64).index_add_(0, idx.cpu(), gp.cpu().double().abs())
    bound = 2.0 ** -23 * max(int(cnt.max()), 1) * absum.max().item()      # sequential fp32 summation bound
    assert err <= bound, (err, bound)
    srt = idx.sort().values
    s1 = pair_rows_sum(gp, srt, n_rows, sorted_index=True)
    s2 = pair_rows_sum(gp, srt, n_rows)
    torch.cuda.synchronize()
    assert torch.equal(s1, s2)


# ---------------------------------------------------------------------------------------- _RatioFn
def _nre_trainer(theta, x):
    from sbi_b200.inference import NRE_B
    tr = NRE_B(classifier="resnet")
    tr.append_simulations(theta, x)
    tr._x2d = tr._x.reshape(theta.shape[0], -1)
    return tr


@pytest.mark.parametrize("sides", ["x", "theta", "both", "conv"])
def test_ratio_fn_with_gathers_matches_oracle(cuda_lib, sides):
    """NRE-B loss and gradients of `flat`, every embedding parameter and the raw theta, through `_loss_on` with a
    fixed contrastive table (the embedded sides paired by batch-local index, raw sides gathered from the whole
    set), against the reference's `_classifier_logits` on repeated rows in fp64."""
    from sbi_b200.ratio import classifier_nn
    theta, x = _copies_task(600)
    kw = {}
    if sides in ("x", "both"):
        kw["embedding_net_x"] = _fc(50, 8)
    if sides in ("theta", "both"):
        kw["embedding_net_theta"] = _theta_net()
    if sides == "conv":
        x, kw["embedding_net_x"] = x.reshape(-1, 2, 25), _Conv()
    torch.manual_seed(0)
    est = classifier_nn("resnet", **kw)(theta, x).cuda()
    ref = _oracle_of(est, perturb=0.05)
    tr = _nre_trainer(theta, x)
    tr._theta = tr._theta.clone().requires_grad_(True)
    B, A = 128, 10
    idx = torch.randperm(600, generator=torch.Generator().manual_seed(2))[:B]
    choices = tr._contrastive_choices(B, A - 1, "cuda")
    loss = tr._loss_on(est, idx.cuda(), A, choices=choices)
    loss.backward()

    def oracle(dtype):
        r = copy.deepcopy(ref).to(dtype)
        t = theta.to(dtype).clone().requires_grad_(True)
        l = sbi_port.nre_b_loss(r, t[idx], x[idx].to(dtype), A, choices=choices.cpu())
        l.backward()
        return l, t.grad, {k: p.grad for k, p in r.named_parameters()}

    (l32, t32, p32), (l64, t64, p64) = oracle(torch.float32), oracle(torch.float64)
    print(f"{sides}: loss {loss.item():.6f}, oracle fp64 {l64.item():.6f}, fp32 {l32.item():.6f}")
    assert abs(loss.item() - l64.item()) <= max(1e-5, 4 * abs(l32.item() - l64.item())) * max(1.0, abs(l64.item()))
    _assert_grad(f"{sides}: raw theta", tr._theta.grad, t32, t64)
    ours = dict(est.layout.unpack(est.flat.grad))
    ours.update({k: p.grad for k, p in est.named_parameters() if k != "net.flat"})
    assert set(ours) == set(p64), set(ours) ^ set(p64)
    scale = max(g.abs().max().item() for g in p64.values())
    for k in p64:
        _assert_grad(f"{sides}: {k}", ours[k], p32[k], p64[k], scale)


# ---------------------------------------------------------------------------------------- trainers
def _fixed_choices(B, k, device, rows=None):
    lo, hi = rows if rows is not None else (0, B)
    own = torch.arange(lo, hi, device=device).unsqueeze(1)
    return (own + 1 + torch.arange(k, device=device)) % B


def _eager_loss(cls, ref, th, xx, A, gamma=1.0, reg=100.0):
    from sbi_b200.multiround import bnre_loss, nre_a_loss, nre_c_loss
    B = th.shape[0]

    def logits(a):
        return sbi_port.nre_b_logits(ref, th, xx, a, choices=_fixed_choices(B, a - 1, "cpu").to(th.device)
                                     ).reshape(B, a)
    if cls == "NRE_B":
        lg = logits(A)
        return -torch.mean(lg[:, 0] - torch.logsumexp(lg, dim=-1))
    if cls == "NRE_A":
        return nre_a_loss(logits(2))
    if cls == "BNRE":
        return bnre_loss(logits(2), reg)
    return nre_c_loss(logits(A), logits(A - 1), gamma)


@pytest.mark.parametrize("cls,sides", [("NRE_B", "x"), ("NRE_B", "both"), ("NRE_B", "conv"), ("NRE_A", "x"),
                                       ("BNRE", "theta"), ("NRE_C", "x")])
def test_nre_trainers_with_embedding_match_eager(cuda_lib, monkeypatch, cls, sides):
    """3 full-batch epochs of the graph-captured trainer against an eager replay from the same weights: the
    reference's `_classifier_logits` on B x num_atoms repeated rows, the loss, backward, clip_grad_norm_(5.0) and
    torch Adam over the kernel AND embedding parameters.  Entries whose gradient is about 0 in some step are
    excluded (Adam's first steps are sign-like).  The last epoch's weights are compared, whichever epoch validated
    best; cuDNN runs in full fp32 (its TF32 convolutions would round B and B x num_atoms rows differently)."""
    import sbi_b200.inference as inference
    from sbi_b200.ratio import classifier_nn
    monkeypatch.setattr(inference.NRE_B, "_contrastive_choices", staticmethod(_fixed_choices))
    monkeypatch.setattr(inference._Trainer, "_load_best", lambda self, net: None)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    theta, x = _copies_task(400)
    kw = {}
    if sides in ("x", "both"):
        kw["embedding_net_x"] = _fc(50, 8)
    if sides in ("theta", "both"):
        kw["embedding_net_theta"] = _theta_net()
    if sides == "conv":
        x, kw["embedding_net_x"] = x.reshape(-1, 2, 25), _Conv()
    torch.manual_seed(0)
    est0 = classifier_nn("resnet", **kw)(theta, x)
    n_train, epochs = 360, 3
    inf = getattr(inference, cls)(classifier=lambda th, xx: copy.deepcopy(est0), device="cuda")
    inf.append_simulations(theta, x)
    # the identity permutation: every epoch's one batch is the training split in order, as in the replay
    randperm = torch.randperm
    monkeypatch.setattr(torch, "randperm", lambda n, **k: torch.arange(n, device=k.get("device")))
    with pytest.warns(UserWarning, match="Maximum number of epochs"):
        kwargs = dict(training_batch_size=n_train, max_num_epochs=epochs - 1, stop_after_epochs=1000)
        if cls == "NRE_C":
            kwargs["num_classes"] = 5
        est = inf.train(**kwargs)
    monkeypatch.setattr(torch, "randperm", randperm)
    tr = inf.train_indices
    assert torch.equal(tr, torch.arange(n_train))
    ref = _oracle_of(est0).cuda()
    opt = torch.optim.Adam(list(ref.parameters()), lr=5e-4)
    th, xx = theta[tr].cuda(), x[tr].cuda()
    A = 6 if cls == "NRE_C" else 10
    grads = []
    for _ in range(epochs):
        opt.zero_grad()
        _eager_loss(cls, ref, th, xx, A).backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), max_norm=5.0)
        grads.append({k: p.grad.clone() for k, p in ref.named_parameters()})
        opt.step()
    sd = est.state_dict()
    errs, n_small, n_emb = [], 0, 0
    for k, p in ref.named_parameters():
        small = torch.stack([g[k].abs() <= 1e-4 * max(max(gg.abs().max().item() for gg in g.values()), 1e-30)
                             for g in grads]).any(0)
        n_small += int(small.sum())
        n_emb += p.numel() if k.startswith("embedding") else 0
        d = (sd[k].cuda() - p.detach()).abs()[~small]
        if d.numel():
            errs.append(d.max().item())
    print(f"{cls} ({sides}): max |dparam| {max(errs):.2e}, {n_emb} embedding entries, {n_small} excluded")
    assert max(errs) <= 2e-5
    if sides != "theta":
        moved = (sd["embedding_net_x.1.fc.weight" if sides == "conv" else "embedding_net_x.1.0.weight"].cpu()
                 - est0.state_dict()["embedding_net_x.1.fc.weight" if sides == "conv" else "embedding_net_x.1.0.weight"])
        assert moved.abs().max() > 0


def test_nre_trainer_with_embedding_is_deterministic(cuda_lib):
    from sbi_b200.inference import NRE_B
    from sbi_b200.ratio import classifier_nn
    theta, x = _copies_task(2000)
    outs = []
    for _ in range(2):
        torch.manual_seed(3)
        inf = NRE_B(classifier=classifier_nn("resnet", embedding_net_x=_fc(50, 8)), device="cuda")
        with pytest.warns(UserWarning, match="Maximum number of epochs"):
            est = inf.append_simulations(theta, x).train(max_num_epochs=3)
        outs.append({k: v.clone() for k, v in est.state_dict().items()})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k


def test_best_epoch_and_resume_cover_both_embeddings(cuda_lib):
    """Early stopping restores both embeddings' weights of the best validation epoch, resume_training continues
    the joint Adam state of size 2 (P + P_theta + P_x); a frozen embedding only transforms its side."""
    from sbi_b200.inference import NRE_B, _weights
    from sbi_b200.ratio import classifier_nn
    theta, x = _copies_task(600)
    inf = NRE_B(classifier=classifier_nn("resnet", embedding_net_x=_fc(50, 8), embedding_net_theta=_theta_net()),
                device="cuda")
    inf.append_simulations(theta, x)
    seen = []
    record = inf._record_epoch

    def spy(tl, vl):
        seen.append((vl, [t.clone() for t in _weights(inf._neural_net)]))
        record(tl, vl)
    inf._record_epoch = spy
    inf.train(training_batch_size=50, learning_rate=5e-3, stop_after_epochs=2, max_num_epochs=500)
    best = min(range(len(seen)), key=lambda i: seen[i][0])
    assert best < len(seen) - 1
    net = inf._neural_net
    final = _weights(net)
    P_t = sum(p.numel() for p in net.embedding_net_theta.parameters())
    P_x = sum(p.numel() for p in net.embedding_net_x.parameters())
    assert len(final) == 1 + len(list(net.embedding_net_theta.parameters())) + len(list(net.embedding_net_x.parameters()))
    for w, b in zip(final, seen[best][1]):
        assert torch.equal(w, b)
    steps_before = int(inf._opt_step[0])
    inf._record_epoch = record
    with pytest.warns(UserWarning, match="Maximum number of epochs"):
        inf.train(training_batch_size=50, learning_rate=5e-3, max_num_epochs=len(seen) + 1, resume_training=True)
    steps_per_epoch = int(0.9 * 600) // 50
    assert int(inf._opt_step[0]) == steps_before + steps_per_epoch * (inf.epoch - len(seen))
    assert inf._opt_state.shape[0] == 2 * (net.layout.n_params + P_t + P_x)

    frozen = _fc(50, 8)
    for p in frozen.parameters():
        p.requires_grad_(False)
    inf = NRE_B(classifier=classifier_nn("resnet", embedding_net_x=frozen), device="cuda")
    with pytest.warns(UserWarning, match="Maximum number of epochs"):
        est = inf.append_simulations(theta, x).train(max_num_epochs=2)
    assert inf._opt_state.shape[0] == 2 * est.layout.n_params
    assert torch.equal(est.embedding_net_x[1][0].weight.cpu(), _fc(50, 8)[0].weight)


def test_data_parallel_with_embedding_raises_on_gpu(cuda_lib, tmp_path):
    import torch.distributed as dist
    from sbi_b200.inference import NRE_B
    from sbi_b200.ratio import classifier_nn
    dist.init_process_group("gloo", init_method=f"file://{tmp_path}/store", rank=0, world_size=1)
    try:
        theta, x = _copies_task(300)
        inf = NRE_B(classifier=classifier_nn("resnet", embedding_net_x=_fc(50, 8)), device="cuda").data_parallel()
        with pytest.raises(NotImplementedError, match="embedding"):
            inf.append_simulations(theta, x).train(max_num_epochs=1)
    finally:
        dist.destroy_process_group()


# ---------------------------------------------------------------------------------------- fits
@pytest.fixture(scope="module")
def trained(cuda_lib):
    from torch.distributions import MultivariateNormal
    from sbi_b200.inference import NRE_B
    from sbi_b200.ratio import classifier_nn
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(2), torch.eye(2))
    theta, x = _copies_task(60000)
    inf = NRE_B(prior, classifier=classifier_nn("resnet", embedding_net_x=_fc(50, 8)), device="cuda")
    inf.append_simulations(theta, x).train(max_num_epochs=200)
    return inf, prior


def _posterior_moments(x_o):
    return x_o.reshape(25, 2).sum(0) / 26, 1 / math.sqrt(26)


@pytest.mark.parametrize("how", ["rejection", "mcmc"])
def test_nre_with_embedding_fits_analytic_posterior(trained, how):
    """NRE-B `resnet` with an FC embedding on x (50 -> 8): |mean error| <= 0.35 posterior std and std within 25 % at
    3 observations, by rejection and by slice MCMC.  Measured on an H100 80GB HBM3 (700 W): |mean error| / std
    0.014, 0.063, 0.306 (rejection) and 0.014, 0.067, 0.304 (MCMC); |std ratio - 1| 0.057, 0.015, 0.057 and 0.040,
    0.044, 0.068.  The two samplers agree, so the third observation's 0.3 std is the trained classifier's bias there,
    not the sampler's; the flows reach 0.22 on the same observation (test_embedding_gpu)."""
    inf, _ = trained
    post = (inf.build_posterior(sample_with="rejection") if how == "rejection"
            else inf.build_posterior(mcmc_parameters=dict(num_chains=100, warmup_steps=100, thin=2)))
    _, xs = _copies_task(3, seed=7)
    for x_o in xs:
        s = post.sample((4000,), x=x_o[None]).cpu()
        mu, sd = _posterior_moments(x_o)
        dm, rs = ((s.mean(0) - mu).abs().max() / sd).item(), (s.std(0) / sd - 1).abs().max().item()
        print(f"NRE+embedding {how} fit: |dmean|/sd {dm:.3f}, |std ratio - 1| {rs:.3f}")
        assert dm <= 0.35 and rs <= 0.25


def test_sbc_takes_the_batched_mcmc_path(trained, recwarn):
    from sbi_b200.diagnostics import run_sbc
    inf, prior = trained
    post = inf.build_posterior(mcmc_parameters=dict(num_chains=20, warmup_steps=50, thin=1))
    torch.manual_seed(7)
    th = prior.sample((100,))
    xs = th.repeat(1, 25) + torch.randn(100, 50)
    ranks, dap = run_sbc(th, xs, post, num_posterior_samples=100)
    assert ranks.shape == (100, 2) and torch.isfinite(ranks.float()).all()
    assert not [w for w in recwarn if "Falling back" in str(w.message)]


def test_embedded_logits_take_the_wgmma_kernel(trained, monkeypatch):
    """At >= 32 768 pairs the embedded model's potential runs the wgmma logits kernel (its embedded widths fit
    RatioLayout.tc_plan), within 2e-4 of the SIMT kernel; the observation is embedded once per set_x."""
    from sbi_b200 import _lib as L
    from sbi_b200.potentials import ratio_estimator_based_potential
    inf, prior = trained
    est = copy.deepcopy(inf._neural_net)
    _, xs = _copies_task(1, seed=7)
    pot, _ = ratio_estimator_based_potential(est, prior, x_o=xs.cuda())
    th = torch.randn(40000, 2).cuda()
    calls, tc_calls = [], []
    hook = est.embedding_net_x.register_forward_hook(lambda *a: calls.append(1))
    lib = L.load()
    tc_entry = lib.sbi_b200_ratio_forward_tc
    monkeypatch.setattr(lib, "sbi_b200_ratio_forward_tc", lambda *a: tc_calls.append(1) or tc_entry(*a))
    a = pot(th, track_gradients=False)
    torch.cuda.synchronize()
    assert tc_calls
    monkeypatch.setenv("SBI_B200_TC", "0")
    b = pot(th, track_gradients=False)
    hook.remove()
    assert not calls                      # x_o was embedded by set_x, not per call
    err = ((a - b).abs() / b.abs().clamp_min(1.0)).max().item()
    print(f"wgmma vs SIMT logits (embedded model): max rel err {err:.2e}")
    assert err <= 2e-4


def test_iid_potential_pairs_by_index(trained):
    """n iid observations: the potential pairs theta with the embedded trials by index; it equals the sum of the
    single-observation potentials, with gradients."""
    from sbi_b200.potentials import ratio_estimator_based_potential
    inf, prior = trained
    est = copy.deepcopy(inf._neural_net)
    _, xs = _copies_task(3, seed=11)
    th = torch.randn(500, 2).cuda().requires_grad_(True)
    pot, _ = ratio_estimator_based_potential(est, prior, x_o=xs.cuda())
    v = pot(th, track_gradients=True)
    (g,) = torch.autograd.grad(v.sum(), th)
    lp = prior.log_prob(th.detach().cpu()).cuda()
    singles, gs = [], []
    for x in xs:
        pot.set_x(x[None].cuda())
        t = th.detach().clone().requires_grad_(True)
        s = pot(t, track_gradients=True)
        singles.append(s - prior.log_prob(t.cpu()).cuda())
        gs.append(torch.autograd.grad(s.sum(), t)[0])
    ref = torch.stack(singles).sum(0) + lp
    assert (v - ref).abs().max().item() <= 1e-3 * max(1.0, ref.abs().max().item())
    gref = sum(gs) - 2 * torch.autograd.functional.jacobian(lambda t: prior.log_prob(t).sum(), th.detach().cpu()).cuda()
    assert (g - gref).abs().max().item() <= 1e-3 * max(1.0, gref.abs().max().item())


# ---------------------------------------------------------------------------------------- drop-in
@needs_ref
def test_reference_nre_b_trains_b200_resnet_with_embedding(cuda_lib):
    """Drop-in: the unmodified reference NRE_B trains `classifier_nn("resnet", embedding_net_x=...)` from this
    package and samples by rejection."""
    assert ref_shim.install()
    from torch.distributions import MultivariateNormal
    from sbi.inference import NRE_B
    from sbi_b200.ratio import RatioEstimator, classifier_nn
    torch.manual_seed(0)
    prior = MultivariateNormal(torch.zeros(2, device="cuda"), torch.eye(2, device="cuda"))
    theta, x = _copies_task(5000)
    _, xs = _copies_task(1, seed=7)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        inf = NRE_B(prior, classifier=classifier_nn("resnet", embedding_net_x=_fc(50, 8)), device="cuda",
                    show_progress_bars=False)
        est = inf.append_simulations(theta.cuda(), x.cuda()).train(training_batch_size=200, max_num_epochs=20)
        assert isinstance(est, RatioEstimator) and est.flat.is_cuda and len(est.embedding_nets) == 1
        s = inf.build_posterior(sample_with="rejection").sample((1000,), x=xs.cuda(), show_progress_bars=False)
    assert s.shape == (1000, 2) and torch.isfinite(s).all()
    mu, sd = _posterior_moments(xs[0])
    assert ((s.cpu().mean(0) - mu).abs().max() / sd).item() <= 1.0
