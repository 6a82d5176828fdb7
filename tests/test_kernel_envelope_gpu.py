"""The NSF, MAF, MAF-RQS and `resnet` ratio kernels across the hyperparameter range one compiled kernel
serves (hidden width, residual blocks, bins, transforms, dims, z-scoring, tail bound, embedding net), at
row counts around every tile switch, with the VJP regime and the weight-ring chunking pinned, at both
sides of the tensor-core envelope, and for models no tile fits (a named SBI_ESMEM error).

Bars (fp32 kernels vs the fp64 oracle, as in test_nsf_gpu.py): log-probs and logits <= 2e-3 absolute;
samples <= 2e-3, log|det| <= 5e-3; gradients <= max(2e-3, 4 x torch-fp32's error) of the max-norm;
padding entries of the parameter gradient exactly 0.  torch-fp32's error is printed next to the kernel's.
"""
import copy
import ctypes as C
import os
import re
import subprocess
import sys

import pytest
import torch
from torch import nn

from oracle import sbi_port
from tests.helpers import (b200_from_oracle, b200_maf_from_oracle, nsf_vjp_raw, oracle_maf, oracle_nsf, use_vjp_path,
                           vjp_step)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGP_TOL, X_TOL, LAD_TOL, GRAD_TOL, TC_TOL = 2e-3, 2e-3, 5e-3, 2e-3, 2e-4


def _big_tile_rows():
    """Rows from which the SIMT evaluation kernels switch from 32- to 64-row tiles (64 x 2 x SMs)."""
    return 128 * torch.cuda.get_device_properties(0).multi_processor_count


def _abs(tag, got, r32, r64, tol):
    got = got.detach().cpu().double()
    err = (got - r64).abs().max().item()
    err32 = (r32.double() - r64).abs().max().item()
    print(f"{tag}: kernel err {err:.3e}  torch-fp32 err {err32:.3e}")
    assert torch.isfinite(got).all(), tag
    # log|det| of 32+ features over 16k rows: torch's own fp32 misses 5e-3, so 2x its error is the bar there
    assert err <= max(tol, 2 * err32), (tag, err, err32)


def _rel(tag, got, r32, r64):
    scale = r64.abs().max().item()
    err = (got - r64).abs().max().item() / scale
    err32 = (r32 - r64).abs().max().item() / scale
    print(f"{tag}: kernel rel err {err:.3e}  torch-fp32 rel err {err32:.3e}")
    assert err <= max(GRAD_TOL, 4 * err32), (tag, err, err32)


# ------------------------------------------------------------------------------------ flow checks
def _flow_logprob(tag, flow, est, inp, cond):
    with torch.no_grad():
        r64 = flow.double().log_prob(inp.double(), cond.double())[0]
        r32 = flow.float().log_prob(inp.float(), cond.float())[0]
        got = est.log_prob(inp.cuda(), cond.cuda())[0]
    _abs(f"{tag} log_prob", got, r32, r64, LOGP_TOL)
    return got


def _oracle_inverse(flow, noise, cond, dtype):
    f = flow.to(dtype)
    with torch.no_grad():
        return f.net._transform.inverse(noise.to(dtype), context=f.net._embedding_net(cond.to(dtype)))


def _flow_inverse(tag, flow, est, noise, cond):
    x64, lad64 = _oracle_inverse(flow, noise, cond, torch.float64)
    x32, lad32 = _oracle_inverse(flow, noise, cond, torch.float32)
    x, lad = est.inverse_flow(noise.cuda(), cond.cuda())
    _abs(f"{tag} inverse x", x, x32, x64, X_TOL)
    _abs(f"{tag} inverse logabsdet", lad, lad32, lad64, LAD_TOL)
    return x, lad


def _oracle_grads(flow, est, inp, cond, g, dtype):
    f = flow.to(dtype)
    f.zero_grad()
    i = inp.to(dtype).detach().requires_grad_(True)
    c = cond.to(dtype).detach().requires_grad_(True)
    (f.log_prob(i, c)[0] * g.to(dtype)).sum().backward()
    return est.layout.pack({k: p.grad for k, p in f.named_parameters()}).double(), i.grad.double(), c.grad.double()


def _kernel_grads(est, inp, cond, g):
    ic = inp.float().cuda().requires_grad_(True)
    cc = cond.float().cuda().requires_grad_(True)
    est.zero_grad()
    (est.log_prob(ic, cc)[0] * g.float().cuda()).sum().backward()
    return est.flat.grad.cpu().double(), ic.grad.cpu().double(), cc.grad.cpu().double()


def _padding(est):
    real = torch.zeros(est.layout.n_params, dtype=torch.bool)
    for ix in est.layout.index.values():
        real[torch.as_tensor(ix.reshape(-1))] = True
    return ~real


def _flow_vjp(tag, flow, est, inp, cond):
    g = torch.randn(inp.shape[0], dtype=torch.float64, generator=torch.Generator().manual_seed(7))
    r32 = _oracle_grads(flow, est, inp, cond, g, torch.float32)
    r64 = _oracle_grads(flow, est, inp, cond, g, torch.float64)
    got = _kernel_grads(est, inp, cond, g)
    assert (got[0][_padding(est)] == 0).all(), f"{tag}: padding entries must receive zero gradient"
    # MADE weights: the kernels compute dense gradients, masked-out entries are frozen by the Adam mask
    mask = est.net._mask.cpu().double()
    for name, a, b32, b64 in zip(("param", "input", "cond"), got, r32, r64):
        if name == "param":
            a, b32, b64 = a * mask, b32 * mask, b64 * mask
        _rel(f"{tag} {name}-grad", a, b32, b64)


def _assert_esmem(fn, *dims):
    from sbi_b200._lib import SbiB200Error
    with pytest.raises(SbiB200Error) as ei:
        fn()
    msg = str(ei.value)
    print(f"expected error: {msg}")
    assert "SBI_ESMEM" in msg and "CUDA error" not in msg, msg
    for d in dims:
        assert d in msg, (d, msg)


# -------------------------------------------------------------------------------------------- NSF
# (id, D, C, builder kwargs, input scale, does the SIMT VJP fit a 32- or 16-row tile)
NSF_CASES = [
    ("H7", 10, 10, dict(hidden_features=7), 1.3, True),
    ("H33", 10, 10, dict(hidden_features=33), 1.3, True),
    ("H68", 10, 10, dict(hidden_features=68), 1.3, True),         # ring chunks 60+8 / 48+20; 16-row VJP
    ("H128", 10, 10, dict(hidden_features=128), 1.3, False),      # ring chunks 32 / 28; no VJP tile fits
    ("NB0", 10, 10, dict(num_blocks=0), 1.3, True),
    ("NB1", 10, 10, dict(num_blocks=1), 1.3, True),
    ("NB4", 10, 10, dict(num_blocks=4), 1.3, True),               # 16-row VJP
    ("NB8", 10, 10, dict(num_blocks=8), 1.3, False),
    ("KB2", 10, 10, dict(num_bins=2), 1.3, True),
    ("KB5", 10, 10, dict(num_bins=5), 1.3, True),
    ("KB16", 10, 10, dict(num_bins=16), 1.3, True),               # 16-row VJP
    ("T1", 10, 10, dict(num_transforms=1), 1.3, True),
    ("T2", 10, 10, dict(num_transforms=2), 1.3, True),
    ("T7", 10, 10, dict(num_transforms=7), 1.3, True),
    ("tail1", 10, 10, dict(tail_bound=1.0), 1.5, True),
    ("tail6", 10, 10, dict(tail_bound=6.0), 4.0, True),
    ("zs_none", 10, 10, dict(z_score_x="none", z_score_y="none"), 1.3, True),
    ("zs_structured", 10, 10, dict(z_score_x="structured", z_score_y="structured"), 1.3, True),
    ("D2", 2, 10, {}, 1.3, True),
    ("D3", 3, 10, {}, 1.3, True),
    ("D13", 13, 10, {}, 1.3, True),                               # 16-row VJP
    ("C1", 10, 1, {}, 1.3, True),
    ("C17", 10, 17, {}, 1.3, True),
]


@pytest.mark.parametrize("D,C,kw,scale,vjp_fits", [c[1:] for c in NSF_CASES], ids=[c[0] for c in NSF_CASES])
def test_nsf_hyperparameters_match_oracle(cuda_lib, D, C, kw, scale, vjp_fits):
    R = 300
    flow, theta, x = oracle_nsf(D, C, n=500, **kw)
    est = b200_from_oracle(flow, theta, x, **kw)
    inp, cond = theta[:R] * scale, x[:R]
    tag = f"nsf D={D} C={C} {kw}"
    _flow_logprob(tag, flow, est, inp, cond)
    noise = torch.randn(R, D, generator=torch.Generator().manual_seed(5)) * scale
    _flow_inverse(tag, flow, est, noise, cond)
    if vjp_fits:
        _flow_vjp(tag, flow, est, inp, cond)
    else:
        _assert_esmem(lambda: _kernel_grads(est, inp, cond, torch.ones(R, dtype=torch.float64)),
                      f"D={D}", f"C={C}", f"H={est.layout.H}", f"num_blocks={est.layout.NB}")


def test_nsf_embedding_net_matches_oracle(cuda_lib):
    """A non-identity embedding (Linear 10 -> 6, tanh) in front of the conditioner: the kernels see the
    embedded context; gradients flow back through torch into the raw condition."""
    emb = nn.Sequential(nn.Linear(10, 6), nn.Tanh())
    with torch.no_grad():
        emb[0].weight.mul_(2.0)
    flow, theta, x = oracle_nsf(10, 10, n=500, embedding_net=emb)
    est = b200_from_oracle(flow, theta, x, embedding_net=copy.deepcopy(emb))
    assert est.layout.C == 6 and not est._embed_identity
    R = 300
    inp, cond = theta[:R] * 1.3, x[:R]
    _flow_logprob("nsf embedding", flow, est, inp, cond)
    _flow_inverse("nsf embedding", flow, est, torch.randn(R, 10, generator=torch.Generator().manual_seed(5)), cond)
    _flow_vjp("nsf embedding", flow, est, inp, cond)


# ------------------------------------------------------------------------------------- row tiles
def _row_tiles(tag, flow, est, theta, x):
    T0 = _big_tile_rows()
    n = T0 + 1
    inp, cond = theta[:n] * 1.3, x[:n]
    noise = torch.randn(n, theta.shape[1], generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        lp64 = flow.double().log_prob(inp.double(), cond.double())[0]
        lp32 = flow.float().log_prob(inp.float(), cond.float())[0]
    x64, lad64 = _oracle_inverse(flow, noise, cond, torch.float64)
    x32, lad32 = _oracle_inverse(flow, noise, cond, torch.float32)
    for R in (1, 31, 33, T0 - 1, T0, T0 + 1):
        with torch.no_grad():
            lp = est.log_prob(inp[:R].cuda(), cond[:R].cuda())[0]
        _abs(f"{tag} R={R} log_prob", lp, lp32[:R], lp64[:R], LOGP_TOL)
        xs, lad = est.inverse_flow(noise[:R].cuda(), cond[:R].cuda())
        _abs(f"{tag} R={R} inverse x", xs, x32[:R], x64[:R], X_TOL)
        _abs(f"{tag} R={R} inverse logabsdet", lad, lad32[:R], lad64[:R], LAD_TOL)


@pytest.mark.parametrize("D,C,kw", [(10, 10, {}), (32, 10, dict(hidden_features=64, num_blocks=1)),
                                    (36, 10, dict(num_blocks=1))], ids=["default", "D32_H64_NB1", "D36_NB1"])
def test_nsf_row_tiles_match_oracle(cuda_lib, monkeypatch, D, C, kw):
    """R around 1, the 32-row tile and the 64-row switch.  D=32/H=64/NB=1 and D=36/NB=1 fit a 32-row tile
    (141 / 148 KB) but not a 64-row one (231 / 246 KB): large batches must stay on 32-row tiles."""
    monkeypatch.setenv("SBI_B200_TC", "0")       # the SIMT tiles at every R (H=50 would go to wgmma from 1024)
    flow, theta, x = oracle_nsf(D, C, n=_big_tile_rows() + 1, **kw)
    est = b200_from_oracle(flow, theta, x, **kw)
    _row_tiles(f"nsf D={D} C={C} {kw}", flow, est, theta, x)


@pytest.mark.parametrize("kw", [dict(hidden_features=240), dict(rqs=True, num_bins=16, D=13)],
                         ids=["maf_H240", "maf_rqs_D13_KB16"])
def test_maf_row_tiles_match_oracle(cuda_lib, kw):
    """MAF H=240 (135 KB at 32 rows, 228 KB at 64; it trains at 223 KB) and MAF-RQS D=13 KB=16
    (147 / 249 KB) evaluate large batches on 32-row tiles."""
    kw = dict(kw)
    D = kw.pop("D", 3)
    flow, theta, x = oracle_maf(D, 2, n=_big_tile_rows() + 1, **kw)
    est = b200_maf_from_oracle(flow, theta, x, **kw)
    _row_tiles(f"maf D={D} {kw}", flow, est, theta, x)


# ------------------------------------------------------------------------------------ VJP regimes
_VJP_KERNEL = re.compile(r"nsf_vjp_kernel<\d+, \d+, \d+, (true|false)>")


def _vjp_kernels_seen(fn, repeat=1, attempts=3):
    """(the NSF VJP kernels `repeat` calls of `fn()` launch, what the last call returns).  The window is padded on
    both sides: a kernel that starts right after the profiler does is now and then missing from its trace.  Late in a
    long test session the profiler also now and then returns a trace without any of the window's kernels.  Every call
    of `fn` launches an NSF VJP kernel, so an empty result is such a lost trace, and the window is taken again, up to
    `attempts` times."""
    import time
    from torch.profiler import ProfilerActivity, profile
    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.02)
            for _ in range(repeat):
                out = fn()
            torch.cuda.synchronize()
            time.sleep(0.02)
        seen = sorted({m.group(0) for e in prof.key_averages() for m in [_VJP_KERNEL.search(e.key)] if m})
        if seen:
            break
    return seen, out


@pytest.mark.parametrize("kw,want", [({}, "nsf_vjp_kernel<32, 2, 2, true>"),
                                     (dict(hidden_features=64), "nsf_vjp_kernel<16, 2, 2, false>"),
                                     (dict(num_blocks=4), "nsf_vjp_kernel<16, 2, 2, false>")],
                         ids=["32row_spill", "16row_H64", "16row_NB4"])
def test_nsf_vjp_regime_kernels(cuda_lib, kw, want):
    flow, theta, x = oracle_nsf(10, 10, n=500, **kw)
    est = b200_from_oracle(flow, theta, x, **kw)
    ic = (theta[:300] * 1.3).cuda().requires_grad_(True)
    seen, _ = _vjp_kernels_seen(lambda: est.log_prob(ic, x[:300].cuda())[0].sum().backward())
    print(f"{kw}: VJP kernels seen {seen}")
    assert seen == [want]
    _flow_vjp(f"vjp regime {kw}", flow, est, theta[:300] * 1.3, x[:300])


def test_nsf_vjp_kernel_follows_the_callers_scratch(cuda_lib):
    """With the caller's activation scratch the 32-row VJP spills (nsf_vjp_kernel<32, 2, 2, true>); without one the
    32-row recompute kernel runs and its gradients match the fp64 oracle."""
    from sbi_b200 import _lib as L
    flow, theta, x = oracle_nsf(10, 10, n=500)
    est = b200_from_oracle(flow, theta, x)
    R = 300
    inp, cond = theta[:R] * 1.3, x[:R]
    g = torch.randn(R, dtype=torch.float64, generator=torch.Generator().manual_seed(7))
    ic, cc, gc = inp.float().cuda(), cond.float().cuda(), g.float().cuda()
    save = torch.empty(cuda_lib.sbi_b200_nsf_vjp_save_bytes(C.byref(est._model(nbuf=3)), R) // 4, device="cuda")
    seen, _ = _vjp_kernels_seen(lambda: nsf_vjp_raw(est, ic, cc, gc, save), repeat=3)
    assert seen == ["nsf_vjp_kernel<32, 2, 2, true>"], seen
    seen, (rc, gpart, ginp, gcond, _) = _vjp_kernels_seen(lambda: nsf_vjp_raw(est, ic, cc, gc, None), repeat=3)
    print(f"no scratch: VJP kernels seen {seen}")
    assert seen == ["nsf_vjp_kernel<32, 2, 2, false>"] and rc == 0
    r32 = _oracle_grads(flow, est, inp, cond, g, torch.float32)
    r64 = _oracle_grads(flow, est, inp, cond, g, torch.float64)
    gflat = L.reduce_partials(gpart, gpart.shape[0], est.layout.n_params).cpu().double()
    assert (gflat[_padding(est)] == 0).all(), "padding entries must receive zero gradient"
    for name, a, b32, b64 in zip(("param", "input", "cond"), (gflat, ginp.cpu().double(), gcond.cpu().double()),
                                 r32, r64):
        _rel(f"vjp recompute {name}-grad", a, b32, b64)


def _run_script(script, env_extra, out):
    env = dict(os.environ, **env_extra)
    subprocess.run([sys.executable, "-c", script, ROOT, str(out)], check=True, env=env, timeout=600)
    return torch.load(out)


# --------------------------------------------------------------------------------- weight ring
def test_nsf_weight_ring_chunking(cuda_lib, tmp_path):
    """SBI_B200_WCAP=0 shrinks every weight-ring slot to the smallest the layout allows (read at import ->
    subprocess): the default model's hidden layers then stream in 32+20 / 24+24+4 row chunks instead of
    one.  In the forward sweep a chunk splits output rows, never a K sum, so log-probs and samples are
    bit-identical.  The backward sweep's dX = W^T dY sums over W's rows, which the chunks split
    (stages.cuh accumulates it chunk by chunk), so gradients agree to fp32 reassociation only."""
    script = r'''
import sys, torch
sys.path.insert(0, sys.argv[1])
from tests.helpers import b200_from_oracle, oracle_nsf
flow, theta, x = oracle_nsf(10, 10, n=500)
est = b200_from_oracle(flow, theta, x)
lay = est.layout
R = 300
inp, cond = (theta[:R] * 1.3).cuda(), x[:R].cuda()
with torch.no_grad():
    lp = est.log_prob(inp, cond)[0]
    xs, lad = est.inverse_flow(torch.randn(R, 10, generator=torch.Generator().manual_seed(5)).cuda(), cond)
ic, cc = inp.clone().requires_grad_(True), cond.clone().requires_grad_(True)
w = torch.randn(R, generator=torch.Generator().manual_seed(9)).cuda()
(est.log_prob(ic, cc)[0] * w).sum().backward()
torch.save({"rpc": (lay.rpc0, lay.rpc1, lay.rpc2, lay.nf_chunk), "lp": lp.cpu(), "x": xs.cpu(), "lad": lad.cpu(),
            "flat": est.flat.grad.cpu(), "inp": ic.grad.cpu(), "cond": cc.grad.cpu()}, sys.argv[2])
'''
    env = {"SBI_B200_TC": "0", "SBI_B200_VJP_TC": "0"}
    one = _run_script(script, env, tmp_path / "default.pt")
    small = _run_script(script, dict(env, SBI_B200_WCAP="0"), tmp_path / "small.pt")
    print(f"ring rows per chunk (rpc0, rpc1, rpc2, nf_chunk): default {one['rpc']}, SBI_B200_WCAP=0 {small['rpc']}")
    assert one["rpc"] == (52, 52, 52, 2) and small["rpc"] == (52, 32, 24, 1)
    for k in ("lp", "x", "lad"):
        assert torch.equal(one[k], small[k]), k
    assert one["flat"].abs().max() > 0
    for k in ("flat", "inp", "cond"):
        d = ((one[k] - small[k]).abs().max() / one[k].abs().max()).item()
        print(f"{k}-grad: chunked vs one-slot rel diff {d:.3e}")
        assert d <= 1e-4, k


# ------------------------------------------------------------------------------------ MAF / RQS
MAF_CASES = [
    ("H7", 3, dict(hidden_features=7)), ("H33", 3, dict(hidden_features=33)), ("H100", 3, dict(hidden_features=100)),
    ("NB1", 3, dict(num_blocks=1)), ("NB3", 3, dict(num_blocks=3)),
    ("T1", 3, dict(num_transforms=1)), ("T3", 3, dict(num_transforms=3)),
    ("D2", 2, {}), ("D13", 13, {}),
]
RQS_CASES = MAF_CASES + [("KB2", 3, dict(num_bins=2)), ("KB16", 3, dict(num_bins=16))]


@pytest.mark.parametrize("rqs,D,kw", [(False,) + c[1:] for c in MAF_CASES] + [(True,) + c[1:] for c in RQS_CASES],
                         ids=[f"maf_{c[0]}" for c in MAF_CASES] + [f"maf_rqs_{c[0]}" for c in RQS_CASES])
def test_maf_hyperparameters_match_oracle(cuda_lib, rqs, D, kw):
    R = 300
    flow, theta, x = oracle_maf(D, 2, n=500, rqs=rqs, **kw)
    est = b200_maf_from_oracle(flow, theta, x, rqs=rqs, **kw)
    inp, cond = theta[:R] * 1.5, x[:R]
    tag = f"{'maf_rqs' if rqs else 'maf'} D={D} {kw}"
    _flow_logprob(tag, flow, est, inp, cond)
    _flow_inverse(tag, flow, est, torch.randn(R, D, generator=torch.Generator().manual_seed(5)), cond)
    _flow_vjp(tag, flow, est, inp, cond)


# ------------------------------------------------------------------------------------ resnet ratio
def _ratio_pair(Dt, Dx, seed=0, **kw):
    from sbi_b200.ratio import build_resnet_classifier
    g = torch.Generator().manual_seed(seed)
    theta, x = torch.randn(600, Dt, generator=g) + 0.5, 2 * torch.randn(600, Dx, generator=g)
    torch.manual_seed(seed)
    ref = sbi_port.build_resnet_classifier(theta, x, **kw)
    with torch.no_grad():
        for p in ref.parameters():
            p.add_(0.1 * torch.randn(p.shape, generator=g))
    est = build_resnet_classifier(theta, x, **kw)
    est.load_state_dict(ref.state_dict())
    return ref, est.cuda()


def _ratio_oracle(ref, est, th, xx, w, dtype):
    r = ref.to(dtype)
    r.zero_grad()
    t = th.detach().to(dtype).clone().requires_grad_(True)
    o = r(t, xx.to(dtype))
    (o * w.to(dtype)).sum().backward()
    gp = est.layout.pack({k: p.grad for k, p in r.named_parameters() if k.startswith("net.")}).double()
    return o.detach().double(), gp, t.grad.double()


RATIO_CASES = [("H7", 3, 5, dict(hidden_features=7)), ("H33", 3, 5, dict(hidden_features=33)),
               ("H100", 3, 5, dict(hidden_features=100)), ("NB1", 3, 5, dict(num_blocks=1)),
               ("NB4", 3, 5, dict(num_blocks=4)), ("Dx1", 3, 1, {}), ("Dx100", 3, 100, {})]


@pytest.mark.parametrize("Dt,Dx,kw", [c[1:] for c in RATIO_CASES], ids=[c[0] for c in RATIO_CASES])
def test_ratio_hyperparameters_match_oracle(cuda_lib, Dt, Dx, kw):
    from sbi_b200.ratio import _RatioFn
    ref, est = _ratio_pair(Dt, Dx, **kw)
    R = 500
    g0 = torch.Generator().manual_seed(1)
    th, xx, w = torch.randn(R, Dt, generator=g0), torch.randn(R, Dx, generator=g0), torch.randn(R, generator=g0)
    tag = f"ratio Dt={Dt} Dx={Dx} {kw}"
    # pairs given directly
    o32, gp32, gt32 = _ratio_oracle(ref, est, th, xx, w, torch.float32)
    o64, gp64, gt64 = _ratio_oracle(ref, est, th, xx, w, torch.float64)
    tc = th.cuda().requires_grad_(True)
    est.zero_grad()
    out = est(tc, xx.cuda())
    (out * w.cuda()).sum().backward()
    _abs(f"{tag} logits", out, o32, o64, LOGP_TOL)
    assert (est.flat.grad.cpu()[_padding(est)] == 0).all(), "padding entries must receive zero gradient"
    _rel(f"{tag} param-grad", est.flat.grad.cpu().double(), gp32, gp64)
    _rel(f"{tag} theta-grad", tc.grad.cpu().double(), gt32, gt64)
    # pairs through index gathers
    gi = torch.Generator().manual_seed(2)
    ti, xi = torch.randint(0, R, (R,), generator=gi), torch.randint(0, R, (R,), generator=gi)
    o32i, gp32i, _ = _ratio_oracle(ref, est, th[ti], xx[xi], w, torch.float32)
    o64i, gp64i, _ = _ratio_oracle(ref, est, th[ti], xx[xi], w, torch.float64)
    est.zero_grad()
    out = _RatioFn.apply(est.net.flat, th.cuda(), xx.cuda(), est, ti.cuda(), xi.cuda(), False)
    (out * w.cuda()).sum().backward()
    _abs(f"{tag} indexed logits", out, o32i, o64i, LOGP_TOL)
    _rel(f"{tag} indexed param-grad", est.flat.grad.cpu().double(), gp32i, gp64i)
    # one shared x
    with torch.no_grad():
        o64s = ref.double()(th.double(), xx[:1].double().expand(R, -1))
        o32s = ref.float()(th, xx[:1].expand(R, -1))
    _abs(f"{tag} shared-x logits", est.logits_raw(th.cuda(), xx[:1].cuda(), x_shared=True), o32s, o64s, LOGP_TOL)


def test_ratio_row_tiles_match_oracle(cuda_lib):
    """resnet Dt=2, Dx=640 (134 KB at 32 rows, 235 KB at 64) and mlp Dt=2, Dx=700 (139 / 241 KB): logits
    of batches from the 64-row switch on stay on 32-row tiles."""
    from sbi_b200.ratio import build_mlp_classifier
    T0 = _big_tile_rows()
    g0 = torch.Generator().manual_seed(1)
    ref, est = _ratio_pair(2, 640)
    n = T0 + 1
    th, xx = torch.randn(n, 2, generator=g0), torch.randn(n, 640, generator=g0)
    with torch.no_grad():
        o64, o32 = ref.double()(th.double(), xx.double()), ref.float()(th, xx)
        for R in (T0 - 1, T0, T0 + 1):
            _abs(f"resnet Dx=640 R={R} logits", est.logits_raw(th[:R].cuda(), xx[:R].cuda()), o32[:R], o64[:R],
                 LOGP_TOL)
    # mlp classifier without z-scoring; its oracle is the torch stack the reference builds
    Dx = 700
    th, xx = torch.randn(n, 2, generator=g0), torch.randn(n, Dx, generator=g0)
    torch.manual_seed(0)
    mlp = build_mlp_classifier(th[:600], xx[:600], z_score_x=None, z_score_y=None).cuda()
    oracle = nn.Sequential(nn.Linear(2 + Dx, 50), nn.LayerNorm(50), nn.ReLU(), nn.Linear(50, 50), nn.LayerNorm(50),
                           nn.ReLU(), nn.Linear(50, 1))
    sd = {k[len("net."):]: v.cpu() for k, v in mlp.state_dict().items() if k.startswith("net.")}
    oracle.load_state_dict(sd)
    with torch.no_grad():
        u = torch.cat([th, xx], 1)
        o64, o32 = oracle.double()(u.double())[:, 0], oracle.float()(u)[:, 0]
        for R in (T0 - 1, T0, T0 + 1):
            _abs(f"mlp Dx={Dx} R={R} logits", mlp.logits_raw(th[:R].cuda(), xx[:R].cuda()), o32[:R], o64[:R],
                 LOGP_TOL)


# ------------------------------------------------------------------------------- tensor-core edges
def _nsf_lib_tc_ok(est):
    """The library's verdict on the wgmma evaluation path: with the host plan's descriptor when there is
    one, else with a well-formed placeholder (the library must decline on the model's dims alone)."""
    from sbi_b200 import _lib as L
    m = est._model(nbuf=2)
    plan = est.layout.tc_plan()
    tc = (L.NsfTc(plan["n_words"], plan["stage_cap"], None, None, None) if plan else L.NsfTc(32, 32, None, None, None))
    return bool(L.load().sbi_b200_nsf_tc_supported(C.byref(m), C.byref(tc)))


@pytest.mark.parametrize("D,C,NB", [(2, 14, 1), (2, 14, 3), (16, 12, 1)], ids=["HC64", "HC64_NB3", "D16_C12"])
def test_nsf_tensor_core_edge_inside(cuda_lib, monkeypatch, D, C, NB):
    """The largest models the wgmma kernels take: H + C = 64, D = 16, and the 112 KB shared-memory budget
    (one of two CTAs per SM), which at T=5 caps D=16 at C=12 and H + C = 64 at 3 blocks.  The host plan and
    the library both accept; wgmma and SIMT agree to 2e-4 and both match the oracle (log_prob, sampling,
    training VJP)."""
    flow, theta, x = oracle_nsf(D, C, n=2000, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    assert est.layout.tc_plan() is not None and est.layout.tc_bwd_plan() is not None and _nsf_lib_tc_ok(est)
    R = 2000
    inp, cond = theta[:R] * 1.3, x[:R]
    noise = torch.randn(R, D, generator=torch.Generator().manual_seed(5))
    res = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("SBI_B200_TC", mode)
        assert (est._tc_state(est._model(nbuf=2)) is not None) == (mode == "1")
        res[mode] = (_flow_logprob(f"nsf tc={mode} D={D} C={C} NB={NB}", flow, est, inp, cond),
                     *_flow_inverse(f"nsf tc={mode} D={D} C={C} NB={NB}", flow, est, noise, cond))
    # log|det| (16 features x 5 layers) keeps the 2.5x looser ratio its oracle bar has (5e-3 vs 2e-3):
    # at D=16 each path is ~1.6e-4 from fp64, as far as torch's own fp32
    for name, a, b, tol in zip(("log_prob", "x", "logabsdet"), res["1"], res["0"],
                               (TC_TOL, TC_TOL, TC_TOL * LAD_TOL / LOGP_TOL)):
        d = (a - b).abs().max().item()
        print(f"D={D} C={C} NB={NB} {name}: |wgmma - SIMT| {d:.3e}")
        assert d <= tol, name
    use_vjp_path(monkeypatch, est, True)
    g = torch.randn(R, dtype=torch.float64, generator=torch.Generator().manual_seed(7))
    got = vjp_step(est, inp.cuda(), cond.cuda(), g.float().cuda()).grad.double()
    r32 = _oracle_grads(flow, est, inp, cond, g, torch.float32)[0]
    r64 = _oracle_grads(flow, est, inp, cond, g, torch.float64)[0]
    assert (got[_padding(est)] == 0).all()
    _rel(f"nsf tc VJP D={D} C={C} NB={NB} param-grad", got, r32, r64)


@pytest.mark.parametrize("D,C,NB,plan", [(16, 15, 1, False), (17, 10, 1, False), (16, 13, 1, True), (2, 14, 4, True)],
                         ids=["HC65", "D17", "D16_C13_smem", "NB4_smem"])
def test_nsf_tensor_core_edge_outside(cuda_lib, monkeypatch, D, C, NB, plan):
    """Just outside: H + C = 65 and D = 17 the host plan and the library both decline; D=16/C=13 and
    NB=4 pass the host plan's dimension checks but exceed the library's 112 KB budget, so the library
    declines.  Forcing the tensor cores leaves the SIMT kernels, which match the oracle."""
    flow, theta, x = oracle_nsf(D, C, n=2000, num_blocks=NB)
    est = b200_from_oracle(flow, theta, x, num_blocks=NB)
    assert (est.layout.tc_plan() is not None) == plan and not _nsf_lib_tc_ok(est)
    monkeypatch.setenv("SBI_B200_TC", "1")
    monkeypatch.setenv("SBI_B200_VJP_TC", "1")
    assert est._tc_state(est._model(nbuf=2)) is None and not est._vjp_uses_tc(2000, True)
    inp, cond = theta * 1.3, x
    _flow_logprob(f"nsf outside D={D} C={C}", flow, est, inp, cond)
    _flow_inverse(f"nsf outside D={D} C={C}", flow, est, torch.randn(2000, D, generator=torch.Generator().manual_seed(5)),
                  cond)


def _ratio_lib_tc_ok(est):
    from sbi_b200 import _lib as L
    m = est._model(nbuf=2)
    plan = est.layout.tc_plan()
    tc = (L.NsfTc(plan["n_words"], plan["stage_cap"], None, None, None) if plan else L.NsfTc(32, 32, None, None, None))
    return bool(L.load().sbi_b200_ratio_tc_supported(C.byref(m), C.byref(tc)))


@pytest.mark.parametrize("Dt,Dx,NB,plan,inside", [(4, 48, 1, True, True), (4, 40, 8, True, True),
                                                  (6, 50, 1, True, False), (4, 44, 8, True, False),
                                                  (7, 50, 2, False, False)],
                         ids=["52_NB1", "44_NB8", "56_NB1_smem", "48_NB8_smem", "57"])
def test_ratio_tensor_core_edge(cuda_lib, monkeypatch, Dt, Dx, NB, plan, inside):
    """The host plan takes Dt + Dx <= 56; the library also needs the padded inputs of a 128-row tile and the
    weight ring in 112 KB, i.e. Dtp + Dxp <= 52 with one block and <= 44 with eight.  Inside, wgmma and
    SIMT agree to 2e-4; outside, forcing the tensor cores leaves SIMT; both match the oracle."""
    ref, est = _ratio_pair(Dt, Dx, num_blocks=NB)
    assert (est.layout.tc_plan() is not None) == plan and _ratio_lib_tc_ok(est) == inside
    R = 2000
    g0 = torch.Generator().manual_seed(1)
    th, xx = torch.randn(R, Dt, generator=g0), torch.randn(R, Dx, generator=g0)
    with torch.no_grad():
        o64, o32 = ref.double()(th.double(), xx.double()), ref.float()(th, xx)
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("SBI_B200_TC", mode)
        assert (est._tc_state(est._model(nbuf=2)) is not None) == (inside and mode == "1")
        out[mode] = est.logits_raw(th.cuda(), xx.cuda())
        _abs(f"ratio Dt+Dx={Dt + Dx} NB={NB} tc={mode} logits", out[mode], o32, o64, LOGP_TOL)
    d = (out["1"] - out["0"]).abs().max().item()
    print(f"ratio Dt+Dx={Dt + Dx} NB={NB}: |wgmma - SIMT| {d:.3e}")
    assert d <= TC_TOL


# ------------------------------------------------------------------------------ models no tile fits
def test_models_that_fit_no_tile_raise_named_esmem(cuda_lib):
    """Training an NSF with H=128 (374 KB at 32 rows, 230 KB at 16) or a MAF with H=300 (263 KB at 32 rows,
    no 16-row VJP) has no tile: the error names SBI_ESMEM and the model's dimensions."""
    flow, theta, x = oracle_nsf(10, 10, n=500, hidden_features=128)
    est = b200_from_oracle(flow, theta, x, hidden_features=128)
    _assert_esmem(lambda: est.loss(theta[:100].cuda(), x[:100].cuda()).mean().backward(),
                  "D=10", "C=10", "H=128", "num_blocks=2")
    flow, theta, x = oracle_maf(3, 2, n=500, hidden_features=300)
    est = b200_maf_from_oracle(flow, theta, x, hidden_features=300)
    _assert_esmem(lambda: est.loss(theta[:100].cuda(), x[:100].cuda()).mean().backward(),
                  "D=3", "C=2", "H=300", "num_blocks=2")
