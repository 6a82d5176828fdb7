"""Host-side logic on the CPU: builder/initialisation parity with the reference builder, the packed
layout's invariants, reference-format (de)serialisation, and the accept/reject control flow."""
import copy
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import sbi_port
from sbi_b200.neural_nets import build_maf, build_nsf, likelihood_nn, posterior_nn
from sbi_b200.pack import NsfLayout
from sbi_b200.posteriors import accept_reject_sample, within_support

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("D,C", [(10, 10), (3, 2), (2, 7), (17, 4)])
def test_builder_matches_reference_builder_bitwise(D, C):
    theta, x = torch.randn(400, D) * 2 + 1, torch.randn(400, C) - 3
    torch.manual_seed(3)
    ref = sbi_port.build_nsf(theta, x)
    torch.manual_seed(3)
    est = build_nsf(theta, x)
    sr, se = ref.state_dict(), est.state_dict()
    assert set(sr) == set(se)
    for k in sr:
        assert torch.equal(sr[k].float(), se[k].float().cpu()), k
    assert est.layout.num_real_params() == sum(p.numel() for p in ref.parameters())


@pytest.mark.parametrize("D,C", [(3, 2), (10, 10), (1, 4)])
def test_maf_builder_matches_reference_builder_bitwise(D, C):
    theta, x = torch.randn(300, D) + 1, torch.randn(300, C) * 2
    torch.manual_seed(8)
    ref = sbi_port.build_maf(theta, x)
    torch.manual_seed(8)
    est = build_maf(theta, x)
    sr, se = ref.state_dict(), est.state_dict()
    assert set(sr) == set(se)
    for k in sr:
        assert torch.equal(sr[k].float(), se[k].float()), k
    g = torch.load(os.path.join(GOLD, "maf_d3c2.pt"))
    e2 = build_maf(g["theta"], g["x"])
    e2.load_state_dict(g["state_dict"])
    out = e2.state_dict()
    for k, v in g["state_dict"].items():
        assert torch.equal(out[k].float(), v.float()), k
    # masked-out weights never reach the kernels: the packed buffer holds W * M
    lay = e2.layout
    for k, mk in lay._wm().items():
        packed = e2.flat.detach()[torch.as_tensor(lay.index[k].reshape(-1))].reshape(mk.shape)
        assert (packed[torch.as_tensor(mk) == 0] == 0).all()


def test_state_dict_roundtrip_with_reference_fixture():
    g = torch.load(os.path.join(GOLD, "nsf_d10.pt"))
    est = build_nsf(g["theta"], g["x"])
    missing, unexpected = est.load_state_dict(g["state_dict"])
    assert not missing and not unexpected
    out = est.state_dict()
    for k, v in g["state_dict"].items():
        assert torch.equal(out[k].float(), v.float()), k
    e2 = copy.deepcopy(est)
    e3 = pickle.loads(pickle.dumps(est))
    assert torch.equal(e2.flat, est.flat) and torch.equal(e3.flat, est.flat)
    # padding stays exactly zero and is frozen by the mask
    mask = est.net._mask.bool()
    assert (est.flat.detach()[~mask] == 0).all()
    assert int(mask.sum()) == est.layout.num_real_params()


@pytest.mark.parametrize("D,C,H,NB,KB,T", [(10, 10, 50, 2, 10, 5), (3, 2, 50, 2, 10, 5), (5, 33, 64, 3, 8, 4),
                                            (31, 7, 128, 1, 16, 2)])
def test_layout_invariants(D, C, H, NB, KB, T):
    lay = NsfLayout(D=D, C=C, H=H, NB=NB, KB=KB, T=T)
    allidx = np.concatenate([v.reshape(-1) for v in lay.index.values()])
    assert len(np.unique(allidx)) == len(allidx), "tensors overlap in the packed buffer"
    assert allidx.max() < lay.n_params and lay.n_params % 4 == 0
    for l in range(T):
        row = lay.layer_tab[l]
        for f in (2, 3, 4, 5, 6, 7, 8, 9):
            assert row[f] % 4 == 0, "16-byte alignment for cp.async.bulk"
        assert row[0] + row[1] == D
    # every chunk fits a ring slot
    assert lay.rpc0 * lay.K0p <= lay.wcap and lay.rpc1 * lay.Hp <= lay.wcap
    assert lay.rpc2 * (lay.Hp + lay.Cp) <= lay.wcap and lay.nf_chunk * lay.PR * lay.Hp <= lay.wcap
    assert lay.rpc0 % 4 == 0 and lay.rpc1 % 4 == 0 and lay.rpc2 % 4 == 0


def test_factories_mirror_reference_roles():
    theta, x = torch.randn(100, 4), torch.randn(100, 6)
    p = posterior_nn("nsf", hidden_features=32, num_transforms=2)(theta, x)
    assert p.input_shape == (4,) and p.condition_shape == (6,) and p.layout.T == 2 and p.layout.H == 32
    l = likelihood_nn("nsf")(theta, x)
    assert l.input_shape == (6,) and l.condition_shape == (4,)
    with pytest.raises(NotImplementedError):
        posterior_nn("mdn")(theta, x)
    with pytest.raises(ValueError):
        posterior_nn("nsf", z_score_theta="bogus")(theta, x)


def test_estimator_shape_errors_match_reference_messages():
    theta, x = torch.randn(100, 4), torch.randn(100, 6)
    est = build_nsf(theta, x)
    with pytest.raises(ValueError, match="does not match the expected input dimensionality"):
        est.log_prob(torch.randn(5, 3), x[:5])
    with pytest.raises(ValueError, match="Shape of condition"):
        est.log_prob(theta[:5], torch.randn(5, 5))


class _FakeProposal:
    """Deterministic proposal: counts how many draws were requested (rejection_sampling_test.py:11-17)."""

    def __init__(self):
        self.calls = []
        self.g = torch.Generator().manual_seed(0)

    def __call__(self, shape, **kw):
        n = torch.Size(shape).numel()
        self.calls.append(n)
        return torch.rand(n, 1, 2, generator=self.g) * 2 - 1


def test_accept_reject_control_flow():
    prop = _FakeProposal()
    accept = lambda th: (th[..., 0] > 0).reshape(-1)   # noqa: E731  ~50 % acceptance
    s, rate = accept_reject_sample(prop, accept, num_samples=1000, max_sampling_batch_size=400)
    assert s.shape == (1000, 1, 2) and (s[..., 0] > 0).all()
    assert 0.4 < rate.item() < 0.6
    # first batch = min(num_samples, max_batch); afterwards 1.5 * remaining / rate, floor 100, cap 400
    assert prop.calls[0] == 400 and all(100 <= c <= 400 for c in prop.calls[1:])
    with pytest.raises(RuntimeError, match="max_sampling_time"):
        accept_reject_sample(_FakeProposal(), lambda th: torch.zeros(th.shape[0], dtype=torch.bool),
                             num_samples=10, max_sampling_time=0.05)


def test_within_support_matches_reference_semantics():
    from torch.distributions import Uniform, Independent
    prior = Independent(Uniform(-torch.ones(2), torch.ones(2), validate_args=False), 1)
    th = torch.tensor([[0.0, 0.5], [1.5, 0.0], [-0.2, -1.2]])
    assert within_support(prior, th).tolist() == [True, False, False]


def test_vector_field_trainers_refuse_later_rounds_like_the_reference():
    """base_vf_inference.py:451-496: FMPE / NPSE have the first-round loss only."""
    from sbi_b200.inference import FMPE, NPSE
    for cls in (FMPE, NPSE):
        t = object.__new__(cls)
        t._vf_check_rounds({})                                   # nothing appended yet
        t._data_round_index = [0, 0]
        t._vf_check_rounds({})
        t._data_round_index = [0, 1]
        with pytest.raises(NotImplementedError, match=f"Multi-round {cls.__name__}"):
            t._vf_check_rounds({})
        t._vf_check_rounds({"force_first_round_loss": True})


def _nsf_model_on_host(lay):
    """The kernels' model struct of `lay` with its pointers on host buffers: enough for the host-side queries,
    which read the struct and never dereference its pointers."""
    from sbi_b200 import _lib as L
    keep = [torch.zeros(lay.n_params), *(torch.from_numpy(t) for t in lay.tables()),
            torch.ones(2 * lay.Dp + 2 * lay.Cp)]
    m = lay.fill_struct(L.NsfModel(), 3)
    m.d_params, m.d_layer_tab, m.d_feat_tab, m.d_stats = (t.data_ptr() for t in keep)
    return m, keep


def test_nsf_vjp_save_bytes(lib):
    """The SIMT VJP's activation scratch: one slab of (4 NB + 1) Hp + TRmax PR rows of 36 floats per layer and
    partial-gradient slab; none for the models that run 16-row tiles, an invalid model or R < 1."""
    import ctypes as C
    m, _keep = _nsf_model_on_host(NsfLayout(D=10, C=10))
    slab = ((4 * m.NB + 1) * m.Hp + m.TRmax * m.PR) * 36
    query = lambda R: lib.sbi_b200_nsf_vjp_save_bytes(C.byref(m), R)   # noqa: E731
    for R in (1, 31, 32, 33, 300, 4096, 10 ** 6):
        assert query(R) == 4 * slab * m.T * lib.sbi_b200_nsf_vjp_parts(R), R
    n_sat = lib.sbi_b200_nsf_vjp_parts(10 ** 9)
    assert n_sat > 1
    sizes = [query(32 * k) for k in range(1, n_sat + 3)]
    assert all(a < b for a, b in zip(sizes[:n_sat], sizes[1:n_sat])), "grows with R while the parts count does"
    assert sizes[n_sat - 1] == sizes[n_sat] == sizes[n_sat + 1] == query(10 ** 9)
    assert query(0) == 0 and query(-5) == 0
    assert lib.sbi_b200_nsf_vjp_save_bytes(None, 4096) == 0
    m.d_params = None
    assert query(4096) == 0
    for kw in (dict(H=64), dict(NB=4)):
        m16, _keep16 = _nsf_model_on_host(NsfLayout(D=10, C=10, **kw))
        assert lib.sbi_b200_nsf_vjp_save_bytes(C.byref(m16), 4096) == 0, kw
