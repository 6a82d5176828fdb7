"""The host side that the flow, ratio and vector-field estimators share (`estimators.PackedNet` and
`_PackedEstimator`), on the CPU: the kernels' statistics vector against the layout include/sbi_b200.h documents,
when it is rebuilt, copies without the derived-data cache, and state_dict round trips between differently seeded
estimators."""
import copy
import pickle

import pytest
import torch
from torch import nn

from sbi_b200.estimators import Standardize
from sbi_b200.flowmatching import FlowMatchingEstimator, build_vector_field_estimator
from sbi_b200.neural_nets import build_made, build_maf, build_maf_rqs, build_nsf
from sbi_b200.ratio import RatioEstimator, build_linear_classifier, build_mlp_classifier, build_resnet_classifier
from sbi_b200.score import build_score_estimator


def _data(D, C, n=200):
    g = torch.Generator().manual_seed(0)
    return 0.7 * torch.randn(n, D, generator=g) + 0.3, 1.3 * torch.randn(n, C, generator=g) - 0.2


# every builder takes z_score_x (input / theta) and z_score_y (condition / x)
BUILDERS = {
    "nsf": lambda **kw: build_nsf(*_data(3, 2), hidden_features=16, num_transforms=2, **kw),
    "nsf_1d": lambda **kw: build_nsf(*_data(1, 3), hidden_features=32, num_transforms=2, **kw),
    "maf": lambda **kw: build_maf(*_data(4, 2), hidden_features=16, num_transforms=3, **kw),
    "maf_rqs": lambda **kw: build_maf_rqs(*_data(4, 3), hidden_features=16, num_transforms=2, **kw),
    "made": lambda **kw: build_made(*_data(3, 2), hidden_features=16, **kw),
    "resnet": lambda **kw: build_resnet_classifier(*_data(3, 5), hidden_features=16, **kw),
    "mlp": lambda **kw: build_mlp_classifier(*_data(3, 5), hidden_features=16, **kw),
    "linear": lambda **kw: build_linear_classifier(*_data(3, 5), **kw),
    "fm": lambda **kw: build_vector_field_estimator(*_data(3, 5), hidden_features=16, num_layers=2, **kw),
    "ve": lambda **kw: build_score_estimator(*_data(3, 5), sde_type="ve", hidden_features=16, num_layers=2, **kw),
    "vp": lambda **kw: build_score_estimator(*_data(3, 5), sde_type="vp", hidden_features=16, num_layers=2, **kw),
    "subvp": lambda **kw: build_score_estimator(*_data(3, 5), sde_type="subvp", hidden_features=16, num_layers=2,
                                                **kw),
}
FLOWS = ("nsf", "nsf_1d", "maf", "maf_rqs", "made")


def _block(values, n, n_pad, pad):
    """n real entries (a scalar is repeated), padded to n_pad with `pad`."""
    return torch.cat([torch.as_tensor(values, dtype=torch.float32).reshape(-1).expand(n), torch.full((n_pad - n,), pad)])


def _zscore(emb):
    return (emb[0]._mean, emb[0]._std) if isinstance(emb, nn.Sequential) else (0.0, 1.0)


def _expected(est, raw_condition=False):
    """The statistics vector restated from include/sbi_b200.h:
    flows  [shift (Dp) | scale (Dp) | ctx_mean (Cp) | ctx_std (Cp)], `made` with feature 0 (the dummy) at 0 / 1;
    ratio  [theta_mean (Dtp) | theta_std (Dtp) | x_mean (Dxp) | x_std (Dxp)];
    fm     [mean_0 (Dp) | std_0 (Dp) | ctx_mean (Cp) | ctx_std (Cp) | div_term (TEp/2) | 4 more],
    with the condition at 0 / 1 when an embedding net runs in torch first, or for `raw_condition`."""
    lay = est.layout
    if isinstance(est, RatioEstimator):
        (tm, ts), (xm, xs) = _zscore(est.embedding_net_theta), _zscore(est.embedding_net_x)
        return torch.cat([_block(tm, lay.Dt, lay.Dtp, 0.0), _block(ts, lay.Dt, lay.Dtp, 1.0),
                          _block(xm, lay.Dx, lay.Dxp, 0.0), _block(xs, lay.Dx, lay.Dxp, 1.0)])
    cm, cs = _zscore(est.embedding_net) if est._embed_identity and not raw_condition else (0.0, 1.0)
    cond = [_block(cm, lay.C, lay.Cp, 0.0), _block(cs, lay.C, lay.Cp, 1.0)]
    if isinstance(est, FlowMatchingEstimator):
        tail = _block(est.net._div_term, lay.TE // 2, lay.TEp // 2 + 4, 0.0)
        return torch.cat([_block(est.mean_0, lay.D, lay.Dp, 0.0), _block(est.std_0, lay.D, lay.Dp, 1.0)] + cond + [tail])
    if lay.family == "made":
        shift = torch.cat([torch.zeros(1), _block(est.net._shift, lay.D - 1, lay.D - 1, 0.0)])
        scale = torch.cat([torch.ones(1), _block(est.net._scale, lay.D - 1, lay.D - 1, 1.0)])
    else:
        shift, scale = est.net._shift, est.net._scale
    return torch.cat([_block(shift, lay.D, lay.Dp, 0.0), _block(scale, lay.D, lay.Dp, 1.0)] + cond)


def _ld_zscore(est):
    n = est.layout.D - (1 if est.layout.family == "made" else 0)
    return float(torch.log(torch.abs(est.net._scale.double())).reshape(-1).expand(n).sum())


@pytest.mark.parametrize("zscore", [True, False], ids=["zscored", "raw"])
@pytest.mark.parametrize("name", BUILDERS)
def test_statistics_vector_has_the_header_layout(name, zscore):
    z = {} if zscore else dict(z_score_x=None, z_score_y=None)
    est = BUILDERS[name](**z)
    st, ld = est._stats()
    want = _expected(est)
    assert st.dtype == torch.float32 and torch.equal(st, want), (st, want)
    if name in FLOWS:
        assert ld == _ld_zscore(est) and (ld != 0.0) == zscore
        raw, ld_raw = est._stats(raw_condition=True)
        assert torch.equal(raw, _expected(est, raw_condition=True)) and ld_raw == ld
        assert {"stats", "stats_raw"} <= set(est._cache)
    else:
        assert ld == 0.0


@pytest.mark.parametrize("name", FLOWS + ("fm",))
def test_statistics_vector_with_an_embedding_net(name):
    """The embedding net runs in torch behind the condition z-score, so the kernels get identity statistics."""
    C = BUILDERS[name]().condition_shape.numel()
    est = BUILDERS[name](embedding_net=nn.Linear(C, 4))
    assert not est._embed_identity and isinstance(est.embedding_net[0], Standardize)
    assert torch.equal(est._stats()[0], _expected(est))


def _sources(est):
    """Tensors the statistics vector is built from: input scale, condition std (and FM's div_term)."""
    if isinstance(est, RatioEstimator):
        return [est.embedding_net_theta[0]._std, est.embedding_net_x[0]._std]
    if isinstance(est, FlowMatchingEstimator):
        return [est.std_0, est.embedding_net[0]._std, est.net._div_term]
    return [est.net._scale, est.embedding_net[0]._std]


@pytest.mark.parametrize("name", BUILDERS)
def test_statistics_vector_is_rebuilt_after_an_in_place_change_of_a_source(name):
    est = BUILDERS[name]()
    st, _ = est._stats()
    assert est._stats()[0] is st                      # cached while nothing changes
    for src in _sources(est):
        with torch.no_grad():
            src.mul_(1.5)
        new, ld = est._stats()
        assert new is not st and torch.equal(new, _expected(est)), src
        if name in FLOWS:
            assert ld == _ld_zscore(est)
        st = new
        assert est._stats()[0] is st


@pytest.mark.parametrize("name", BUILDERS)
def test_deepcopy_and_pickle_drop_the_cache(name):
    est = BUILDERS[name]()
    st, _ = est._stats()
    est._gpart(2)
    for twin in (copy.deepcopy(est), pickle.loads(pickle.dumps(est))):
        assert twin._cache == {}
        assert torch.equal(twin.flat, est.flat) and twin.flat.data_ptr() != est.flat.data_ptr()
        assert torch.equal(twin._stats()[0], st)
    assert set(est._cache) >= {"stats", "gpart"}


@pytest.mark.parametrize("name", BUILDERS)
def test_state_dict_loads_into_a_differently_seeded_estimator(name):
    torch.manual_seed(1)
    a = BUILDERS[name]()
    torch.manual_seed(2)
    b = BUILDERS[name]()
    assert not torch.equal(a.flat, b.flat)
    if name == "made":       # masked-out raw weights: kept aside, not in the flat buffer
        assert a.net._raw.abs().sum() > 0 and not torch.equal(a.net._raw, b.net._raw)
    if name.startswith("maf"):
        assert any((pa != pb).any() for pa, pb in zip(a.layout.perms, b.layout.perms))
    b.load_state_dict(a.state_dict())
    assert torch.equal(b.flat, a.flat) and torch.equal(b.net._raw, a.net._raw)
    if name.startswith("maf"):   # the loaded permutations are adopted, tables included
        assert all((pa == pb).all() for pa, pb in zip(a.layout.perms, b.layout.perms))
    for ta, tb in zip(a.net.tables(), b.net.tables()):
        assert torch.equal(ta, tb)
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    # only the reference's keys load: a dict holding the flat buffer alone is missing all of them
    with pytest.raises(RuntimeError, match="Missing key"):
        b.load_state_dict({"net.flat": a.flat.detach().clone()})
