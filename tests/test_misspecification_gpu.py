"""The MMD misspecification test on the device: every null MMD and the observed one against an fp64 evaluation of
the reference's formulas on the same index tables (torch fp32's own error printed beside), the radix-selected
bandwidths against torch.median(torch.cdist(.)) and the lower-median rank, p-value parity with the UNMODIFIED
reference for the same seed (near-tie flips counted), bit-determinism, and the reference's acceptance cases."""
import pytest
import torch
from torch import nn

from oracle import ref_shim
from sbi_b200 import misspecification as M
from sbi_b200.diagnostics import calc_misspecification_mmd

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")


def _sets(out, z, z_obs, n_obs, m):
    """(X, Y) of every set of `_null_and_observed`: null sets, then the observed one."""
    nx = min(n_obs, m)
    sets = [(z[p[:nx]], z[p[nx:m]]) for p in out["table"]]
    return sets + [(z_obs, z[:m])]


def _reference_formulas(x, y, mode, cdist_mode="donot_use_mm_for_euclid_dist"):
    """misspecification.py:19-53 as written, in the dtype of x and y."""
    h = torch.median(torch.cdist(x, y, compute_mode=cdist_mode)).item()

    def k(a, b):
        return torch.exp(-(torch.cdist(a, b, compute_mode=cdist_mode) ** 2) / (2.0 * h ** 2))
    kx, ky, kxy = k(x, x), k(y, y), k(x, y)
    if mode == "biased":
        return (kx.mean() + ky.mean() - 2 * kxy.mean()).item(), h
    return (kx.sum() / (kx.shape[0] * (kx.shape[0] - 1)) + ky.sum() / (ky.shape[0] * (ky.shape[0] - 1))
            - 2 * kxy.mean()).item(), h


def _data(n, d, n_obs, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_obs, d, generator=g).cuda() + 0.3, torch.randn(n, d, generator=g).cuda()


def _check(sub, n_obs, m, d, S, mode, seed=0, n=None):
    n = n if n is not None else max(m, n_obs) + 17
    z_obs, z = _data(n, d, n_obs, seed)
    torch.manual_seed(seed)
    out = M._null_and_observed(z_obs, z, n_obs, S - 1, m, mode)
    sets = _sets(out, z, z_obs, n_obs, m)
    assert out["mmd"].shape == (S,)
    check = sorted({0, 1, S // 2, S - 2, S - 1} & set(range(S)))[:sub]
    err = err32 = 0.0
    for s in check:
        x, y = sets[s]
        want, h64 = _reference_formulas(x.double(), y.double(), mode)
        got = out["mmd"][s].item()
        if want == float("inf"):
            assert got == float("inf"), (s, got)
            continue
        err = max(err, abs(got - want))
        err32 = max(err32, abs(_reference_formulas(x, y, mode, "use_mm_for_euclid_dist_if_necessary")[0] - want))
        assert abs(out["bandwidth"][s].item() - h64) <= 1e-6 * h64, (s, out["bandwidth"][s].item(), h64)
    print(f"n_obs={n_obs} M={m} d={d} S={S} {mode}: max |device - fp64| = {err:.2e}, torch fp32 {err32:.2e}")
    assert err <= 2e-6, err
    return out


@pytest.mark.parametrize("n_obs,m,d,S,mode", [
    (1, 3, 1, 1, "biased"), (2, 3, 2, 7, "unbiased"), (2, 1000, 37, 40, "biased"), (100, 1000, 2, 5000, "biased"),
    (100, 1000, 300, 30, "unbiased"), (1, 4097, 2, 12, "biased"), (100, 4097, 37, 6, "unbiased"),
    (2, 4097, 300, 3, "biased"), (100, 1000, 1, 700, "unbiased"),
])
def test_values_match_fp64_reference_formulas(cuda_lib, n_obs, m, d, S, mode):
    _check(5, n_obs, m, d, S, mode)


def test_single_observation_unbiased_is_inf_with_p_one(cuda_lib):
    out = _check(5, 1, 1000, 2, 50, "unbiased")
    assert torch.isinf(out["mmd"]).all()
    z_obs, z = _data(2000, 2, 1, 1)
    p, (null, obs) = M.calculate_p_misspecification(z_obs, z, n_shuffle=20, mode="unbiased")
    assert p == 1.0 and torch.isinf(null).all() and torch.isinf(obs)


@pytest.mark.parametrize("nx,ny,d,dup", [(3, 4, 2, False), (5, 7, 3, False), (40, 61, 5, True),
                                         (100, 900, 20, True), (64, 64, 1, True), (33, 97, 300, False)])
def test_bandwidth_is_the_lower_median(cuda_lib, nx, ny, d, dup):
    g = torch.Generator().manual_seed(nx * ny + d)
    pts = torch.randn(nx + ny, d, generator=g)
    if dup:   # rows drawn from 7 distinct points: many X-Y distances tie at the median
        pts = pts[torch.randint(0, 7, (nx + ny,), generator=g)]
    x, y = pts[:nx].cuda(), pts[nx:].cuda()
    h = M.median_heuristic(x, y)
    d64 = torch.cdist(x.double(), y.double(), compute_mode="donot_use_mm_for_euclid_dist").flatten()
    want = torch.median(d64).item()
    assert abs(h - want) <= 1e-6 * want, (h, want)
    k = (d64.numel() - 1) // 2
    assert int((d64 < h * (1 - 1e-6)).sum()) <= k < int((d64 <= h * (1 + 1e-6)).sum())


def test_empty_y_block_and_empty_observation_are_nan(cuda_lib):
    """The reference takes the median and the mean of an empty matrix: NaN, not an error."""
    z_obs, z = _data(50, 2, 30, 2)
    p, (null, obs) = M.calculate_p_misspecification(z_obs, z, n_shuffle=3, max_samples=30)
    assert p == 1.0 and torch.isnan(null).all() and torch.isfinite(obs)
    p, (null, obs) = M.calculate_p_misspecification(z_obs[:0], z, n_shuffle=3)
    assert torch.isnan(null).all() and torch.isnan(obs)


def test_public_pair_functions(cuda_lib):
    x, y = torch.randn(30, 4).cuda(), torch.randn(50, 4).cuda()
    k = M.rbf_kernel(x, y, 1.7)
    want = torch.exp(-torch.cdist(x.double(), y.double(), compute_mode="donot_use_mm_for_euclid_dist") ** 2
                     / (2 * 1.7 ** 2))
    assert k.shape == (30, 50) and k.dtype == torch.float32 and (k.double() - want).abs().max() < 1e-6
    for mode in ("biased", "unbiased"):
        got = M.compute_rbf_mmd(x, y, 1.7, mode)
        kx = torch.exp(-torch.cdist(x.double(), x.double()) ** 2 / (2 * 1.7 ** 2))
        ky = torch.exp(-torch.cdist(y.double(), y.double()) ** 2 / (2 * 1.7 ** 2))
        if mode == "biased":
            ref = kx.mean() + ky.mean() - 2 * want.mean()
        else:
            ref = kx.sum() / (30 * 29) + ky.sum() / (50 * 49) - 2 * want.mean()
        assert got.shape == () and got.dtype == torch.float32 and abs(got.item() - ref.item()) < 2e-6
        med = M.compute_rbf_mmd_median_heuristic(x, y, mode)
        assert abs(med.item() - _reference_formulas(x.double(), y.double(), mode)[0]) < 2e-6
    assert M.rbf_kernel(x.cpu(), y.cpu(), 1.0).device.type == "cpu"


def test_deterministic_and_independent_of_other_sets(cuda_lib):
    z_obs, z = _data(3000, 5, 20, 4)
    zz = torch.cat([z, z_obs])
    perms = torch.stack([torch.randperm(3000)[:1000] for _ in range(40)]).to(torch.int32)
    nxy = torch.tensor([[20, 980]]).expand(40, 2)
    a, ha = M._mmd_sets(zz, perms, nxy)
    b, hb = M._mmd_sets(zz, perms, nxy)
    assert torch.equal(a, b) and torch.equal(ha, hb)
    sub, hsub = M._mmd_sets(zz, perms[7:9], nxy[7:9])
    assert torch.equal(sub, a[7:9]) and torch.equal(hsub, ha[7:9])
    # next to a set of other sizes (the observed set), in a wider table
    obs = torch.cat([torch.arange(3000, 3020), torch.arange(1000)]).to(torch.int32)
    wide = torch.cat([torch.nn.functional.pad(perms[:3], (0, 20)), obs.unsqueeze(0)])
    c, hc = M._mmd_sets(zz, wide, torch.cat([nxy[:3], torch.tensor([[20, 1000]])]))
    assert torch.equal(c[:3], a[:3]) and torch.equal(hc[:3], ha[:3])
    torch.manual_seed(9)
    r1 = calc_misspecification_mmd(z_obs, z, n_shuffle=100)
    torch.manual_seed(9)
    r2 = calc_misspecification_mmd(z_obs, z, n_shuffle=100)
    assert r1[0] == r2[0] and torch.equal(r1[1][0], r2[1][0]) and torch.equal(r1[1][1], r2[1][1])


@needs_ref
@pytest.mark.parametrize("n_obs,d,mode,offset", [(1, 2, "biased", 0.0), (1, 2, "biased", 2.0),
                                                 (10, 3, "unbiased", 0.3), (100, 20, "biased", 0.05)])
def test_p_value_parity_with_reference(cuda_lib, n_obs, d, mode, offset):
    assert ref_shim.install()
    from sbi.diagnostics import misspecification as R
    g = torch.Generator().manual_seed(n_obs + d)
    x, x_o = torch.randn(3000, d, generator=g), torch.randn(n_obs, d, generator=g) + offset
    torch.manual_seed(11)
    p, (null, obs) = calc_misspecification_mmd(x_o.cuda(), x.cuda(), n_shuffle=200, max_samples=600, mmd_mode=mode)
    torch.manual_seed(11)
    p_ref, (null_ref, obs_ref) = R.calc_misspecification_mmd(x_o, x, n_shuffle=200, max_samples=600, mmd_mode=mode)
    assert null.dtype == null_ref.dtype == torch.float32 and null.device.type == "cpu" and obs.shape == ()
    assert obs.device.type == "cuda"
    err = max((null - null_ref).abs().max().item(), abs(obs.item() - obs_ref.item()))
    ours, theirs = null < obs.cpu(), null_ref < obs_ref
    flips = int((ours != theirs).sum())
    near = (null_ref - obs_ref).abs() <= 1e-5
    print(f"n_obs={n_obs} d={d} {mode}: p {p:.4f} vs reference {p_ref:.4f}, max |MMD - reference| {err:.2e}, "
          f"{flips} near-tie flips")
    assert bool(near[ours != theirs].all())
    assert abs(p - p_ref) <= flips / 200 + 1e-12
    assert err <= 2e-5


def _gauss_case(seed=2025, d=2):
    torch.manual_seed(seed)
    prior = torch.distributions.MultivariateNormal(torch.zeros(d), torch.eye(d))
    prior_mis = torch.distributions.MultivariateNormal(torch.zeros(d) + 4, torch.eye(d))

    def sim(t):
        return t + torch.randn_like(t)
    theta_train = prior.sample((1000,))
    x_train = sim(theta_train)
    x_val = sim(prior.sample((1000,)))
    x_o = sim(prior.sample((1,)))
    x_o_mis = sim(prior_mis.sample((1,)))
    return prior, theta_train, x_train, x_val, x_o, x_o_mis


def test_acceptance_x_space(cuda_lib):
    _, _, _, x_val, x_o, x_o_mis = _gauss_case()
    p_well, _ = calc_misspecification_mmd(inference=None, x_obs=x_o, x=x_val, mode="x_space")
    p_mis, _ = calc_misspecification_mmd(inference=None, x_obs=x_o_mis, x=x_val, mode="x_space")
    print(f"x_space: p well specified {p_well:.3f}, misspecified {p_mis:.3f}")
    assert p_well > 0.05 and p_mis < 0.05


def test_acceptance_embedding(cuda_lib):
    from sbi_b200.inference import NPE
    from sbi_b200.neural_nets import posterior_nn
    prior, theta_train, x_train, x_val, x_o, x_o_mis = _gauss_case()
    emb = nn.Sequential(nn.Linear(2, 20), nn.ReLU(), nn.Linear(20, 20), nn.ReLU(), nn.Linear(20, 2))
    inf = NPE(prior=prior, density_estimator=posterior_nn("nsf", embedding_net=emb), device="cuda")
    inf.append_simulations(theta_train, x_train).train()
    p_well, (null, obs) = calc_misspecification_mmd(x_o, x_val, inference=inf, mode="embedding")
    p_mis, _ = calc_misspecification_mmd(x_o_mis, x_val, inference=inf, mode="embedding")
    print(f"embedding: p well specified {p_well:.3f}, misspecified {p_mis:.3f}")
    assert null.shape == (1000,) and obs.shape == ()
    assert p_well > 0.05 and p_mis < 0.05
