"""The flow-matching kernels (csrc/fm.cu: `fm_forward`, `fm_forward_div`, `fm_loss_vjp`, `fm_loss_vjp_cond` and
`fm_net_vjp`) across the hyperparameter range one compiled kernel serves, for FMPE and for the three NPSE score
estimators (the kernels' bare-network mode), against the oracle's `VectorFieldMLP` in float64.

* Shapes: one thing at a time varied from D=5, C=7, H=100, num_layers=5, time_embedding_dim=32, including widths
  that are not a multiple of 4 (padded features must stay out of LayerNorm and out of the gradient).
* Row counts around the 16- and 32-row tiles and the SM count, up to ~3 x 32 x SMs rows, where every CTA of every
  kernel loops over >= 3 tiles and the VJP adds each tile after its first into the CTA's gradient slab.
* The weight-ring plans `fm_tune` picks (printed for every case), and the shared-memory limit of each kernel per
  num_layers: the largest model that fits matches the oracle, the next one raises a named SBI_ESMEM error on
  the host while the kernels it still fits keep working.

Bars (fp32 kernels vs the fp64 oracle): velocities, loss values and network outputs <= 2e-3 * max(1, max|ref|);
divergence and Jacobian diagonal <= 3e-3 * max(1, max|ref|); parameter and condition gradients: max-norm error
<= max(2e-3, 4 x torch-fp32's error) relative to the max-norm of the reference; padding entries of the parameter
gradient exactly 0.  torch-fp32's error is printed next to the kernel's.
"""
import copy
import ctypes as C

import pytest
import torch
from torch import nn

from oracle import sbi_port

pytestmark = pytest.mark.gpu
VEL_TOL, DIV_TOL, GRAD_TOL = 2e-3, 3e-3, 2e-3
SMEM_MAX = 227 * 1024
KERNELS = ("forward", "loss/net VJP", "forward+divergence")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------ bars
def _abs(tag, got, r32, r64, tol):
    got = got.detach().cpu().double()
    scale = max(1.0, r64.abs().max().item())
    err = (got - r64).abs().max().item()
    err32 = (r32.double() - r64).abs().max().item()
    print(f"{tag}: kernel err {err:.3e}  torch-fp32 err {err32:.3e}  (bar {tol * scale:.3e})")
    assert torch.isfinite(got).all(), tag
    assert err <= tol * scale, (tag, err, err32)


def _rel(tag, got, r32, r64):
    got = got.detach().cpu().double()
    scale = r64.abs().max().item()
    err = (got - r64).abs().max().item() / scale
    err32 = (r32.double() - r64).abs().max().item() / scale
    print(f"{tag}: kernel rel err {err:.3e}  torch-fp32 rel err {err32:.3e}")
    assert err <= max(GRAD_TOL, 4 * err32), (tag, err, err32)


def _assert_esmem(fn, *dims):
    from sbi_b200._lib import SbiB200Error
    with pytest.raises(SbiB200Error) as ei:
        fn()
    msg = str(ei.value)
    print(f"expected error: {msg}")
    assert "SBI_ESMEM" in msg and "CUDA error" not in msg, msg
    for d in dims:
        assert d in msg, (d, msg)


def _pack64(lay, module):
    """The `net.*` gradients of an oracle module in the packed layout, in float64 (padding 0)."""
    flat = torch.zeros(lay.n_params, dtype=torch.float64)
    for k, p in module.named_parameters():
        if k.startswith("net."):
            flat[torch.as_tensor(lay.index[k].reshape(-1))] = p.grad.detach().double().reshape(-1)
    return flat


def _padding(lay):
    real = torch.zeros(lay.n_params, dtype=torch.bool)
    for ix in lay.index.values():
        real[torch.as_tensor(ix.reshape(-1))] = True
    return ~real


def _param_grad(tag, lay, got, r32, r64):
    """Padding entries exactly 0; the whole vector (real entries unmasked) against the oracle."""
    got = got.detach().cpu().double()
    pad = _padding(lay)
    assert (got[pad] == 0).all(), f"{tag}: padding entries must receive zero gradient"
    _rel(f"{tag} param-grad", got, r32, r64)


# ---------------------------------------------------------------------------------- ring plans
def _plans(lay):
    """`sbi_b200_fm_plan` of the three kernels: [nbuf, wcap, rpc_i, rpc_c, rpc_m, rpc_t, rpc_h, rpc_o, bytes, RN]."""
    from sbi_b200 import _lib as L
    s = L.FmModel()
    lay.fill_struct(s, 2)
    out = []
    for kernel in range(3):
        v = (C.c_int32 * 10)()
        assert L.load().sbi_b200_fm_plan(C.byref(s), kernel, v) == 0
        out.append(list(v))
    return out


def _fits(plan):
    return plan[8] <= SMEM_MAX


def _show_plans(tag, lay):
    plans = _plans(lay)
    for k, p in enumerate(plans):
        print(f"{tag} plan {KERNELS[k]}: nbuf={p[0]} wcap={p[1]} rpc_i/c/m/t/h/o={p[2:8]} Hp={lay.Hp} "
              f"{p[8]} B{'' if _fits(p) else ' > 227 KB'}")
    return plans


def _layout(D, C, H, NL, TE):
    from sbi_b200.pack import FmLayout
    return FmLayout(D=D, C=C, H=H, NL=NL, TE=TE)


def _limit(kernel, D, C, NL, TE=32):
    """The largest hidden width whose plan for `kernel` fits 227 KB (plans depend on round4(H) only)."""
    fit = [H for H in range(4, 512, 4) if _fits(_plans(_layout(D, C, H, NL, TE))[kernel])]
    assert fit and fit[-1] < 508
    return fit[-1]


# -------------------------------------------------------------------------------------- models
def _oracle_fm(D, C, H, NL, TE, freq, zx, zy, seed, perturb):
    """The oracle estimator built from its parts, every weight perturbed off its initial value (the output layer
    is zero-initialised), and the data its z-scoring was fitted on."""
    g = torch.Generator().manual_seed(seed)
    theta, x = 0.7 * torch.randn(500, D, generator=g) + 0.4, 1.5 * torch.randn(500, C, generator=g) - 0.3
    torch.manual_seed(seed)
    net = sbi_port.VectorFieldMLP(D, C, TE, H, NL, sinusoidal_max_freq=freq)
    dox, sx = sbi_port.z_score_parser(zx)
    doy, sy = sbi_port.z_score_parser(zy)
    mean_0, std_0 = sbi_port.z_standardization(theta, sx) if dox else (0.0, 1.0)
    emb = nn.Sequential(sbi_port.standardizing_net(x, sy), nn.Identity()) if doy else nn.Identity()
    ref = sbi_port.FlowMatchingEstimator(net, theta[0].shape, x[0].shape, emb, mean_0, std_0)
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(perturb * torch.randn(p.shape, generator=g))
    return ref, theta, x


def _fm_pair(D=5, C=7, H=100, NL=5, TE=32, freq=1000.0, zx="independent", zy="independent", seed=0, perturb=0.1):
    from sbi_b200.flowmatching import build_vector_field_estimator
    ref, theta, x = _oracle_fm(D, C, H, NL, TE, freq, zx, zy, seed, perturb)
    est = build_vector_field_estimator(theta, x, z_score_x=zx, z_score_y=zy, hidden_features=H, num_layers=NL,
                                       time_embedding_dim=TE, sinusoidal_max_freq=freq)
    est.load_state_dict(ref.state_dict())
    return ref, est.cuda()


def _score_pair(sde, D=5, C=7, H=100, NL=5, TE=32, seed=0, perturb=0.15):
    """(score estimator on the device, {dtype: (CPU twin of the estimator with the oracle network behind it,
    the oracle estimator)} for float64 and float32)."""
    from sbi_b200.score import build_score_estimator
    ref, theta, x = _oracle_fm(D, C, H, NL, TE, 1000.0, "independent", "independent", seed, perturb)
    kw = dict(sde_type=sde, hidden_features=H, num_layers=NL, time_embedding_dim=TE)
    est = build_score_estimator(theta, x, **kw)
    est.net.load_state_dict({k[len("net."):]: v for k, v in ref.state_dict().items() if k.startswith("net.")})
    twins = {}
    for dtype in (torch.float64, torch.float32):
        port = copy.deepcopy(ref).to(dtype)
        chk = build_score_estimator(theta, x, **kw).to(dtype)
        chk._net_call = (lambda p: lambda enc, cond, tenc: p.net(enc, p._embedding_net(cond).expand(enc.shape[0], -1),
                                                                 tenc))(port)
        twins[dtype] = (chk, port)
    return est.cuda(), twins


def _inputs(R, D, C, seed=2):
    """Rows with per-row condition and time; t = 0 and t = 1 exactly are among the times."""
    g = torch.Generator().manual_seed(seed)
    inp = 1.2 * torch.randn(R, D, generator=g) + 0.3
    cond = 1.5 * torch.randn(R, C, generator=g) - 0.3
    t = torch.rand(R, generator=g)
    t[0] = 0.0
    if R > 1:
        t[-1] = 1.0
    eps = torch.randn(R, D, generator=g)
    w = torch.randn(R, generator=g)
    return inp, cond, t, eps, w


# ---------------------------------------------------------------------------------- FMPE checks
def _oracle_v(ref, inp, cond, t, dtype):
    with torch.no_grad():
        return ref.to(dtype).forward(inp.to(dtype), cond.to(dtype), t.to(dtype))


def _check_forward(tag, ref, est, inp, cond, t):
    """Velocity with per-row / shared condition and per-row / shared time."""
    R = inp.shape[0]
    for name, c, tt in (("per-row cond, per-row t", cond, t), ("shared cond, shared t=0", cond[:1], torch.tensor(0.0)),
                        ("shared cond, per-row t", cond[:1], t), ("per-row cond, shared t=1", cond, torch.tensor(1.0))):
        r64, r32 = _oracle_v(ref, inp, c, tt, torch.float64), _oracle_v(ref, inp, c, tt, torch.float32)
        with torch.no_grad():
            got = est.forward(inp.cuda(), c.cuda(), tt.cuda())
        assert got.shape == (R, inp.shape[1])
        _abs(f"{tag} forward ({name})", got, r32, r64, VEL_TOL)


def _oracle_loss(ref, lay, inp, cond, t, eps, w, dtype):
    r = ref.to(dtype)
    r.zero_grad()
    c = cond.detach().to(dtype).clone().requires_grad_(True)
    loss = r.loss(inp.to(dtype), c, times=t.to(dtype), theta_1=eps.to(dtype))
    (loss * w.to(dtype)).sum().backward()
    return loss.detach().double(), _pack64(lay, r), c.grad.double()


def _kernel_loss(est, inp, cond, t, eps, w):
    from sbi_b200.flowmatching import _FmLoss
    est.zero_grad()
    cc = cond.cuda().requires_grad_(True)
    loss = _FmLoss.apply(est.net.flat, inp.cuda(), cc, t.cuda(), eps.cuda(), est)
    (loss * w.cuda()).sum().backward()
    return loss.detach(), est.flat.grad.clone(), cc.grad


def _check_loss(tag, ref, est, inp, cond, t, eps, w):
    """Per-row loss, parameter gradient and condition gradient of sum_r w_r loss_r (the autograd Function)."""
    lay = est.layout
    l32, g32, c32 = _oracle_loss(ref, lay, inp, cond, t, eps, w, torch.float32)
    l64, g64, c64 = _oracle_loss(ref, lay, inp, cond, t, eps, w, torch.float64)
    loss, gflat, gcond = _kernel_loss(est, inp, cond, t, eps, w)
    _abs(f"{tag} loss", loss, l32, l64, VEL_TOL)
    _param_grad(tag, lay, gflat, g32, g64)
    _rel(f"{tag} cond-grad", gcond.cpu().double(), c32, c64)
    return gflat


def _check_trainer_call(tag, ref, est, inp, cond, t, eps, B):
    """The training loop's call: B rows gathered by index from the data set, g = 1/B for every row, the loss sum
    and the non-finite row count accumulated on the device, the condition gradient of the gathered rows."""
    from sbi_b200 import _lib as L
    lay = est.layout
    idx = torch.randint(0, inp.shape[0], (B,), generator=torch.Generator().manual_seed(11))
    tb, eb = t[:B].clone(), eps[:B].clone()
    wb = torch.full((B,), 1.0 / B, dtype=torch.float64)
    l32, g32, c32 = _oracle_loss(ref, lay, inp[idx], cond[idx], tb, eb, wb, torch.float32)
    l64, g64, c64 = _oracle_loss(ref, lay, inp[idx], cond[idx], tb, eb, wb, torch.float64)
    loss_acc = torch.zeros(2, device="cuda")
    gcond = torch.empty(B, lay.C, device="cuda")
    loss, gpart, n_part = est.loss_raw(inp.cuda(), cond.cuda(), tb.cuda(), eb.cuda(), index=idx.cuda(),
                                       g_const=1.0 / B, loss_acc=loss_acc, gcond=gcond)
    gflat = L.reduce_partials(gpart, n_part, lay.n_params)
    acc = loss_acc.cpu().double()
    assert acc[1].item() == 0, f"{tag}: {acc[1].item()} non-finite rows"
    _abs(f"{tag} indexed loss", loss, l32, l64, VEL_TOL)
    _abs(f"{tag} indexed loss sum", acc[:1], l32.sum().reshape(1), l64.sum().reshape(1), VEL_TOL)
    _param_grad(f"{tag} indexed", lay, gflat, g32, g64)
    _rel(f"{tag} indexed cond-grad", gcond.cpu().double(), c32, c64)


def _oracle_div(ref, inp, cond, t, dtype):
    """(v, exact divergence): rows are independent, so D reverse passes of sum_r v_ri give every row's trace."""
    r = ref.to(dtype)
    with torch.enable_grad():
        x = inp.detach().to(dtype).clone().requires_grad_(True)
        v = r.forward(x, cond.to(dtype), t.to(dtype))
        tr = torch.zeros(inp.shape[0], dtype=dtype)
        for i in range(inp.shape[1]):
            gi, = torch.autograd.grad(v[:, i].sum(), x, retain_graph=True)
            tr += gi[:, i]
    return v.detach().double(), tr.double()


def _check_div(tag, ref, est, inp, cond, t, shared=True):
    cases = [("per-row cond, per-row t", cond, t)]
    if shared:
        cases.append(("shared cond, shared t=0.5", cond[:1], torch.tensor(0.5)))
    for name, c, tt in cases:
        v64, d64 = _oracle_div(ref, inp, c, tt, torch.float64)
        v32, d32 = _oracle_div(ref, inp, c, tt, torch.float32)
        with torch.no_grad():
            v, div = est.forward_and_divergence(inp.cuda(), c.cuda(), tt.cuda())
        _abs(f"{tag} forward_and_divergence v ({name})", v, v32, v64, VEL_TOL)
        _abs(f"{tag} divergence ({name})", div, d32, d64, DIV_TOL)


def _fm_kernel_check(kernel, tag, ref, est, R=300):
    inp, cond, t, eps, w = _inputs(R, est.layout.D, est.layout.C)
    if kernel == 0:
        _check_forward(tag, ref, est, inp, cond, t)
    elif kernel == 1:
        _check_loss(tag, ref, est, inp, cond, t, eps, w)
        _check_trainer_call(tag, ref, est, inp, cond, t, eps, R // 2)
    else:
        _check_div(tag, ref, est, inp, cond, t)


def _fm_esmem_call(kernel, est, R=64):
    inp, cond, t, eps, w = [a.cuda() if isinstance(a, torch.Tensor) else a
                            for a in _inputs(R, est.layout.D, est.layout.C)]
    if kernel == 0:
        return lambda: est.forward(inp, cond, t)
    if kernel == 1:
        return lambda: est.loss(inp, cond, times=t).mean().backward()
    return lambda: est.forward_and_divergence(inp, cond, t)


def _dims(lay):
    return f"D={lay.D}", f"C={lay.C}", f"H={lay.H}", f"num_layers={lay.NL}"


# ------------------------------------------------------------------------------------ shape cases
# (id, D, C, H, num_layers, time_embedding_dim, extra builder kwargs); H=None: the largest H the training
# kernel fits at that num_layers (found from the plans, not hard-coded)
FM_CASES = [
    ("default", 5, 7, 100, 5, 32, {}),
    ("H7", 5, 7, 7, 5, 32, {}),
    ("H33", 5, 7, 33, 5, 32, {}),
    ("H64", 5, 7, 64, 5, 32, {}),
    ("H_train_max_NL2", 5, 7, None, 2, 32, {}),
    ("H_train_max_NL5", 5, 7, None, 5, 32, {}),
    ("NL2", 5, 7, 100, 2, 32, {}),
    ("NL3", 5, 7, 100, 3, 32, {}),
    ("NL8", 5, 7, 100, 8, 32, {}),            # training / divergence do not fit: named SBI_ESMEM
    ("NL12", 5, 7, 100, 12, 32, {}),          # training / divergence do not fit: named SBI_ESMEM
    ("NL8_H64", 5, 7, 64, 8, 32, {}),
    ("NL12_H48", 5, 7, 48, 12, 32, {}),
    ("TE2", 5, 7, 100, 5, 2, {}),
    ("TE6", 5, 7, 100, 5, 6, {}),             # odd number of frequencies (3), TEp = 8
    ("TE16", 5, 7, 100, 5, 16, {}),
    ("TE64", 5, 7, 100, 5, 64, {}),
    ("maxfreq10", 5, 7, 100, 5, 32, dict(freq=10.0)),
    ("D1", 1, 7, 100, 5, 32, {}),
    ("D2", 2, 7, 100, 5, 32, {}),
    ("D13", 13, 7, 100, 5, 32, {}),
    ("D50", 50, 7, 100, 5, 32, {}),
    ("C1", 5, 1, 100, 5, 32, {}),
    ("C17", 5, 17, 100, 5, 32, {}),
    ("C64", 5, 64, 100, 5, 32, {}),
    ("zs_none", 5, 7, 100, 5, 32, dict(zx="none", zy="none")),
    ("zs_structured", 5, 7, 100, 5, 32, dict(zx="structured", zy="structured")),
    ("H33_D13", 13, 7, 33, 5, 32, {}),
]


def _case_H(D, C, H, NL, TE):
    return _limit(1, D, C, NL, TE) if H is None else H


@pytest.mark.parametrize("D,C,H,NL,TE,kw", [c[1:] for c in FM_CASES], ids=[c[0] for c in FM_CASES])
def test_fm_shapes_match_oracle(cuda_lib, D, C, H, NL, TE, kw):
    H = _case_H(D, C, H, NL, TE)
    ref, est = _fm_pair(D, C, H, NL, TE, **kw)
    tag = f"fm D={D} C={C} H={H} NL={NL} TE={TE} {kw}"
    plans = _show_plans(tag, est.layout)
    for kernel, plan in enumerate(plans):
        if _fits(plan):
            _fm_kernel_check(kernel, tag, ref, est)
        else:
            _assert_esmem(_fm_esmem_call(kernel, est), *_dims(est.layout))


# ------------------------------------------------------------------------------------ score checks
def _oracle_net(port, enc, cond, tenc, w, dtype):
    port = port.to(dtype)
    port.zero_grad()
    out = port.net(enc.to(dtype), port._embedding_net(cond.to(dtype)).expand(enc.shape[0], -1), tenc.to(dtype))
    (out * w.to(dtype)).sum().backward()
    return out.detach().double(), port


def _oracle_diag(port, enc, cond, tenc, dtype):
    port = port.to(dtype)
    with torch.enable_grad():
        e = enc.detach().to(dtype).clone().requires_grad_(True)
        out = port.net(e, port._embedding_net(cond.to(dtype)).expand(enc.shape[0], -1), tenc.to(dtype))
        diag = torch.zeros_like(e)
        for i in range(enc.shape[1]):
            gi, = torch.autograd.grad(out[:, i].sum(), e, retain_graph=True)
            diag[:, i] = gi[:, i]
    return out.detach().double(), diag.double()


def _oracle_ode_div(chk, th, cond, t):
    with torch.enable_grad():
        x = th.detach().to(chk.mean_0.dtype).clone().requires_grad_(True)
        f = chk.ode_fn(x, cond.to(x.dtype), t.to(x.dtype))
        tr = torch.zeros(th.shape[0], dtype=x.dtype)
        for i in range(th.shape[1]):
            gi, = torch.autograd.grad(f[:, i].sum(), x, retain_graph=True)
            tr += gi[:, i]
    return f.detach().double(), tr.double()


def _score_inputs(est, twins, R, seed=3):
    chk = twins[torch.float64][0]
    g = torch.Generator().manual_seed(seed)
    D, Cn = est.layout.D, est.layout.C
    enc = torch.randn(R, D, generator=g)
    cond = 1.5 * torch.randn(R, Cn, generator=g) - 0.3
    t = torch.rand(R, generator=g) * (est.t_max - est.t_min) + est.t_min
    t[0] = est.t_min
    if R > 1:
        t[-1] = est.t_max
    tenc = chk.std_fn(t.double()).reshape(-1).float()        # VE: up to sigma_max = 10
    w = torch.randn(R, D, generator=g)
    return enc, cond, t, tenc, w


def _check_score_net(tag, est, twins, enc, cond, tenc, w):
    """The bare network (fm_forward, raw) and its parameter gradient for a given output gradient (fm_net_vjp)."""
    lay = est.layout
    o64, p64 = _oracle_net(twins[torch.float64][1], enc, cond, tenc, w, torch.float64)
    o32, p32 = _oracle_net(twins[torch.float32][1], enc, cond, tenc, w, torch.float32)
    est.net.flat.grad = None
    out = est._net_call(enc.cuda(), cond.cuda(), tenc.cuda())
    (out * w.cuda()).sum().backward()
    _abs(f"{tag} net output", out, o32, o64, VEL_TOL)
    gflat = est.net.flat.grad.clone()
    _param_grad(f"{tag} net_vjp", lay, gflat, _pack64(lay, p32), _pack64(lay, p64))
    return gflat


def _check_score_diag(tag, est, twins, enc, cond, tenc):
    o64, d64 = _oracle_diag(twins[torch.float64][1], enc, cond, tenc, torch.float64)
    o32, d32 = _oracle_diag(twins[torch.float32][1], enc, cond, tenc, torch.float32)
    with torch.no_grad():
        out, diag = est._raw_forward_diag(enc.cuda(), cond.cuda().contiguous(), tenc.cuda())
    _abs(f"{tag} raw forward (diag kernel)", out, o32, o64, VEL_TOL)
    _abs(f"{tag} Jacobian diagonal", diag, d32, d64, DIV_TOL)


def _check_score_ode(tag, est, twins, th, cond, t):
    f64, d64 = _oracle_ode_div(twins[torch.float64][0], th, cond, t)
    f32, d32 = _oracle_ode_div(twins[torch.float32][0], th, cond, t)
    with torch.no_grad():
        f, div = est.ode_fn_and_divergence(th.cuda(), cond.cuda(), t.cuda())
    _abs(f"{tag} ode_fn", f, f32, f64, DIV_TOL)
    _abs(f"{tag} ode divergence", div, d32, d64, DIV_TOL)


SCORE_CASES = [
    ("ve_H33", "ve", 5, 7, 33, 5, 32),
    ("ve_D1", "ve", 1, 7, 100, 5, 32),
    ("vp_TE6", "vp", 5, 7, 100, 5, 6),
    ("subvp_D13", "subvp", 13, 7, 100, 5, 32),
]


@pytest.mark.parametrize("sde,D,C,H,NL,TE", [c[1:] for c in SCORE_CASES], ids=[c[0] for c in SCORE_CASES])
def test_score_shapes_match_oracle(cuda_lib, sde, D, C, H, NL, TE):
    est, twins = _score_pair(sde, D, C, H, NL, TE)
    tag = f"score {sde} D={D} C={C} H={H} NL={NL} TE={TE}"
    _show_plans(tag, est.layout)
    R = 300
    enc, cond, t, tenc, w = _score_inputs(est, twins, R)
    print(f"{tag}: time encodings in [{tenc.min().item():.3g}, {tenc.max().item():.3g}]")
    _check_score_net(tag, est, twins, enc, cond, tenc, w)
    _check_score_net(f"{tag} shared cond", est, twins, enc, cond[:1], tenc, w)
    _check_score_diag(tag, est, twins, enc, cond, tenc)
    th = 0.7 * enc + 0.4
    _check_score_ode(f"{tag} (per-row cond)", est, twins, th, cond, t)
    _check_score_ode(f"{tag} (shared cond)", est, twins, th, cond[:1], t)


# ------------------------------------------------------------------------------------- row counts
def _row_counts():
    S = _sms()
    return [1, 15, 16, 17, 31, 32, 33, 16 * S - 1, 16 * S, 16 * S + 1, 32 * S - 1, 32 * S + 1, 3 * 32 * S + 7]


@pytest.mark.parametrize("D,C,H", [(5, 7, 100), (13, 7, 33)], ids=["default", "H33_D13"])
def test_fm_row_counts_match_oracle(cuda_lib, D, C, H):
    """Every R around the 16- and 32-row tiles and the SM count.  From 16 x SMs + 1 rows a CTA of the VJP kernel
    runs a second tile and adds it into its gradient slab; at 3 x 32 x SMs + 7 rows every CTA of every kernel runs
    >= 3 tiles.  There all five entry points are checked, and a second VJP gives a bit-identical gradient (one
    writer per slab, fixed reduction order)."""
    ref, est = _fm_pair(D, C, H)
    sest, twins = _score_pair("vp", D, C, H)
    Rs = _row_counts()
    Rmax = Rs[-1]
    tag0 = f"fm D={D} C={C} H={H}"
    _show_plans(tag0, est.layout)
    inp, cond, t, eps, w = _inputs(Rmax, D, C)
    v64, v32 = _oracle_v(ref, inp, cond, t, torch.float64), _oracle_v(ref, inp, cond, t, torch.float32)
    dv64, d64 = _oracle_div(ref, inp, cond, t, torch.float64)
    dv32, d32 = _oracle_div(ref, inp, cond, t, torch.float32)
    enc, scond, _, tenc, sw = _score_inputs(sest, twins, Rmax)
    so64, sd64 = _oracle_diag(twins[torch.float64][1], enc, scond, tenc, torch.float64)
    so32, sd32 = _oracle_diag(twins[torch.float32][1], enc, scond, tenc, torch.float32)
    for R in Rs:
        tag = f"{tag0} R={R}"
        with torch.no_grad():
            v = est.forward(inp[:R].cuda(), cond[:R].cuda(), t[:R].cuda())
            fv, div = est.forward_and_divergence(inp[:R].cuda(), cond[:R].cuda(), t[:R].cuda())
            so, sd = sest._raw_forward_diag(enc[:R].cuda(), scond[:R].cuda(), tenc[:R].cuda())
        _abs(f"{tag} forward", v, v32[:R], v64[:R], VEL_TOL)
        _abs(f"{tag} forward_and_divergence v", fv, dv32[:R], dv64[:R], VEL_TOL)
        _abs(f"{tag} divergence", div, d32[:R], d64[:R], DIV_TOL)
        _abs(f"{tag} score raw forward (diag kernel)", so, so32[:R], so64[:R], VEL_TOL)
        _abs(f"{tag} score Jacobian diagonal", sd, sd32[:R], sd64[:R], DIV_TOL)
        g1 = _check_loss(tag, ref, est, inp[:R], cond[:R], t[:R], eps[:R], w[:R])
        s1 = _check_score_net(f"{tag} score", sest, twins, enc[:R], scond[:R], tenc[:R], sw[:R])
        if R == Rmax:
            _check_trainer_call(tag, ref, est, inp, cond, t, eps, R)
            g2 = _kernel_loss(est, inp, cond, t, eps, w)[1]
            sest.net.flat.grad = None
            (sest._net_call(enc.cuda(), scond.cuda(), tenc.cuda()) * sw.cuda()).sum().backward()
            assert torch.equal(g1, g2), "loss VJP: a second run changed the parameter gradient"
            assert torch.equal(s1, sest.net.flat.grad), "net VJP: a second run changed the parameter gradient"


# ------------------------------------------------------------------------------- shared-memory limit
@pytest.mark.parametrize("NL", [2, 5, 12])
def test_fm_shared_memory_limit(cuda_lib, NL):
    """D = C = 20, TE = 32.  For each kernel, the largest H whose plan fits 227 KB matches the oracle; at the next H
    (a multiple of 4) that kernel raises SBI_ESMEM naming the model, from the host check before any launch, and
    every kernel whose plan still fits matches the oracle."""
    D = Cn = 20
    limits = [_limit(k, D, Cn, NL) for k in range(3)]
    print(f"NL={NL}: largest H per kernel {dict(zip(KERNELS, limits))}")
    assert limits[0] >= limits[1] and limits[0] >= limits[2], "evaluation fits at least what training fits"
    for kernel, Hmax in enumerate(limits):
        ref, est = _fm_pair(D, Cn, Hmax, NL)
        tag = f"inside {KERNELS[kernel]}: fm D={D} C={Cn} H={Hmax} NL={NL}"
        assert _fits(_show_plans(tag, est.layout)[kernel])
        _fm_kernel_check(kernel, tag, ref, est, R=200)
        H = Hmax + 4
        ref, est = _fm_pair(D, Cn, H, NL)
        tag = f"outside {KERNELS[kernel]}: fm D={D} C={Cn} H={H} NL={NL}"
        plans = _show_plans(tag, est.layout)
        assert not _fits(plans[kernel])
        for k, plan in enumerate(plans):
            if _fits(plan):
                _fm_kernel_check(k, f"{tag}, {KERNELS[k]}", ref, est, R=100)
            else:
                _assert_esmem(_fm_esmem_call(k, est), *_dims(est.layout))


def test_fm_model_past_training_limit_samples_but_does_not_train(cuda_lib):
    """posterior_flow_nn(hidden_features=128) at D = C = 20: the 32-row evaluation kernel fits, so ODE sampling
    runs; training and the exact-trace log-probability do not, and say which model does not fit."""
    from sbi_b200.flowmatching import log_prob_ode, posterior_flow_nn, sample_ode
    from sbi_b200.score import posterior_score_nn
    g = torch.Generator().manual_seed(0)
    theta, x = torch.randn(500, 20, generator=g), torch.randn(500, 20, generator=g)
    torch.manual_seed(0)
    est = posterior_flow_nn(hidden_features=128)(theta, x).cuda()
    dims = ("D=20", "C=20", "H=128", "num_layers=5")
    s = sample_ode(est, 64, x[:1].cuda())
    assert s.shape == (64, 20) and torch.isfinite(s).all()
    _assert_esmem(lambda: est.loss(theta[:64].cuda(), x[:64].cuda()), *dims)
    _assert_esmem(lambda: log_prob_ode(est, theta[:8].cuda(), x[:1].cuda()), *dims)
    # the score estimators run the same kernels in bare-network mode
    sc = posterior_score_nn(sde_type="ve", hidden_features=128)(theta, x).cuda()
    with torch.no_grad():
        assert torch.isfinite(sc(theta[:64].cuda(), x[:1].cuda(), torch.tensor(0.5, device="cuda"))).all()
    _assert_esmem(lambda: sc.loss(theta[:64].cuda(), x[:64].cuda()).mean().backward(), *dims)
    _assert_esmem(lambda: sc.ode_fn_and_divergence(theta[:8].cuda(), x[:1].cuda(), torch.full((8,), 0.5).cuda()),
                  *dims)


# ------------------------------------------------------------------------------------- ring regimes
def test_fm_ring_plans_cover_every_regime(lib):
    """The plans the cases above run against the oracle cover a hidden layer streamed whole, a ragged last chunk,
    a ring deeper than two stages, and the smallest chunks `fm_tune` leaves at the shared-memory edge (the merge
    layer, the largest matrix, in 4-row chunks).  A retune that stops reaching one of them fails here."""
    shapes = [(c[0], c[1], c[2], _case_H(c[1], c[2], c[3], c[4], c[5]), c[4], c[5]) for c in FM_CASES]
    shapes += [(c[0], c[2], c[3], c[4], c[5], c[6]) for c in SCORE_CASES]
    shapes += [(f"limit_NL{NL}_{KERNELS[k]}", 20, 20, _limit(k, 20, 20, NL), NL, 32)
               for NL in (2, 5, 12) for k in range(3)]
    regimes = {"hidden layer whole": [], "ragged last chunk": [], "ring deeper than 2": [],
               "smallest chunks at the edge": []}
    for tag, D, Cn, H, NL, TE in shapes:
        lay = _layout(D, Cn, H, NL, TE)
        for k, p in enumerate(_show_plans(tag, lay)):
            if not _fits(p):
                continue
            nbuf, rpc_m, rpc_h = p[0], p[4], p[6]
            where = f"{tag}/{KERNELS[k]}"
            if rpc_h == lay.Hp:
                regimes["hidden layer whole"].append(where)
            if lay.Hp % rpc_h:
                regimes["ragged last chunk"].append(where)
            if nbuf > 2:
                regimes["ring deeper than 2"].append(where)
            if rpc_m == 4 < lay.Hp:
                regimes["smallest chunks at the edge"].append(where)
    for name, where in regimes.items():
        print(f"{name}: {len(where)} plans, e.g. {where[:4]}")
        assert where, f"no case runs a plan with {name}"
