"""The `mlp` and `linear` NRE classifiers without a GPU: packed layout, reference keys and initial
weights (tests/golden/ratio_mlp_d4x6.pt), state_dict round trip, factory errors, C ABI symbols.

The fixture comes from the UNMODIFIED reference sbi (the copy staged under oracle/_ref, through
oracle.ref_shim); `python tests/test_ratio_mlp_cpu.py` writes it with `make_fixture`:

  ratio_mlp_d4x6.pt  reference `classifier_nn("mlp")`, `classifier_nn("mlp", norm_layer=nn.Identity)` and
                     `classifier_nn("linear")` (theta-dim 4, x-dim 6): initial state_dict under the seed and
                     the RNG draw that follows it, a perturbed state_dict, pairs, logits (also with a shared
                     x), and the fp64 parameter / theta gradients of sum_r w_r logit_r.
"""
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "ratio_mlp_d4x6.pt")
MODELS = {"mlp": ("mlp", {}), "mlp_identity": ("mlp", dict(norm_layer=nn.Identity)), "linear": ("linear", {})}
HAVE_REF = os.path.isdir(os.path.join(os.path.dirname(HERE), "oracle", "_ref", "sbi"))


def make_fixture(Dt=4, Dx=6, seed=17, n=400):
    """The contents of ratio_mlp_d4x6.pt, computed by the reference's own classifiers."""
    from oracle import ref_shim
    assert ref_shim.install(), "needs the staged reference sbi"
    from sbi.neural_nets import classifier_nn
    g = torch.Generator().manual_seed(seed)
    theta = 0.7 * torch.randn(n, Dt, generator=g) + 0.3
    x = 1.3 * torch.randn(n, Dx, generator=g) - 0.2
    th, xx = theta[:96] * 1.2, x[:96]
    w = torch.randn(96, generator=g)
    out = dict(theta=theta, x=x, th=th, xx=xx, w=w, Dt=Dt, Dx=Dx, seed=seed)
    for name, (model, kw) in MODELS.items():
        torch.manual_seed(seed)
        est = classifier_nn(model, **kw)(theta, x)
        init = {k: v.clone() for k, v in est.state_dict().items()}
        next_draw = torch.randn(4)
        with torch.no_grad():
            for p in est.parameters():
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            logits = est(th, xx)
            logits_shared = est(th, xx[:1].expand(96, -1))
        est64 = est.double()
        t = th.double().clone().requires_grad_(True)
        (est64(t, xx.double()) * w.double()).sum().backward()
        out[name] = dict(init_state_dict=init, next_draw=next_draw,
                         state_dict={k: v.float() for k, v in est64.state_dict().items()},
                         logits=logits, logits_shared=logits_shared,
                         grad_params={k: p.grad.clone() for k, p in est64.named_parameters()},
                         grad_theta=t.grad.clone())
    return out


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.mark.parametrize("Dt,Dx,H,NL,norm", [(4, 6, 50, 2, "layer"), (1, 1, 50, 2, None), (5, 100, 128, 2, "layer"),
                                             (2, 3, 30, 2, "layer"), (4, 6, 50, 0, None), (5, 100, 50, 0, None)])
def test_layout_covers_every_key_once_and_masks_pads(Dt, Dx, H, NL, norm):
    from sbi_b200.pack import MlpRatioLayout
    lay = MlpRatioLayout(Dt=Dt, Dx=Dx, H=H, NL=NL, norm=norm)
    pos = np.concatenate([v.reshape(-1) for v in lay.index.values()])
    assert len(np.unique(pos)) == pos.size == lay.num_real_params()
    assert pos.min() >= 0 and pos.max() < lay.n_params
    mask = lay.trainable_mask()
    assert int(mask.sum()) == pos.size and bool(mask[torch.as_tensor(pos)].all())
    want = {"net.weight", "net.bias"} if NL == 0 else (
        {f"net.{i}.{p}" for i in ((0, 1, 3, 4, 6) if norm else (0, 3, 6)) for p in ("weight", "bias")})
    assert set(lay.index) == want
    K = Dt + Dx
    n_real = K + 1 if NL == 0 else (K * H + H) + (H * H + H) + (H + 1) + (4 * H if norm else 0)
    assert pos.size == n_real
    # pack / unpack round trip
    g = torch.Generator().manual_seed(0)
    state = {k: torch.randn(v.shape, generator=g) for k, v in lay.index.items()}
    flat = lay.pack(state)
    assert all(torch.equal(t, state[k]) for k, t in lay.unpack(flat).items())
    assert flat[mask == 0].abs().max() == 0


@pytest.mark.parametrize("name", list(MODELS))
def test_build_reproduces_reference_initial_state(gold, name):
    from sbi_b200.ratio import classifier_nn
    model, kw = MODELS[name]
    torch.manual_seed(gold["seed"])
    est = classifier_nn(model, **kw)(gold["theta"], gold["x"])
    draw = torch.randn(4)
    want = gold[name]["init_state_dict"]
    got = est.state_dict()
    assert set(got) == set(want)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    assert torch.equal(draw, gold[name]["next_draw"])


@pytest.mark.parametrize("name", list(MODELS))
def test_state_dict_round_trip_with_reference_keys(gold, name):
    from sbi_b200.ratio import RatioEstimator, classifier_nn
    model, kw = MODELS[name]
    est = classifier_nn(model, **kw)(gold["theta"], gold["x"])
    assert isinstance(est, RatioEstimator)
    est.load_state_dict(gold[name]["state_dict"], strict=True)
    got = est.state_dict()
    assert set(got) == set(gold[name]["state_dict"])
    for k, v in gold[name]["state_dict"].items():
        assert torch.equal(got[k], v), k
    with pytest.raises(RuntimeError):
        est.load_state_dict({k: v for k, v in gold[name]["state_dict"].items() if "net." not in k}, strict=True)


def test_layernorm_eps_is_read_from_the_built_module():
    from functools import partial
    from sbi_b200.ratio import classifier_nn
    theta, x = torch.randn(50, 2), torch.randn(50, 3)
    est = classifier_nn("mlp", norm_layer=partial(nn.LayerNorm, eps=1e-3))(theta, x)
    assert est.layout.norm == "layer" and est.layout.eps == pytest.approx(1e-3)
    assert classifier_nn("mlp", norm_layer=nn.Identity)(theta, x).layout.norm is None


def test_classifier_nn_errors_match_reference():
    from sbi_b200.ratio import classifier_nn
    theta, x = torch.randn(50, 2), torch.randn(50, 3)
    with pytest.raises(ValueError, match=r"\['num_blocks'\] are not used by model='mlp'"):
        classifier_nn("mlp", num_blocks=3)
    with pytest.raises(ValueError, match=r"\['hidden_features'\] are not used by model='linear'"):
        classifier_nn("linear", hidden_features=30)
    with pytest.raises(ValueError, match=r"\['norm_layer'\] are not used by model='resnet'"):
        classifier_nn("resnet", norm_layer=nn.Identity)
    with pytest.raises(ValueError, match="Unknown classifier model"):
        classifier_nn("mdn")
    for bad in (nn.BatchNorm1d, lambda h: nn.LayerNorm(h, elementwise_affine=False)):
        with pytest.raises(NotImplementedError, match="LayerNorm"):
            classifier_nn("mlp", norm_layer=bad)(theta, x)
    for model in ("mlp", "linear"):
        with pytest.raises(ValueError, match="transform_to_unconstrained"):
            classifier_nn(model, z_score_theta="transform_to_unconstrained")(theta, x)
        with pytest.raises(NotImplementedError, match="embedding"):
            classifier_nn(model, embedding_net_x=nn.Linear(3, 3))(theta, x)


def _assert_same(a, b, path="fixture"):
    if isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            _assert_same(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape, path
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-7), path
    else:
        assert a == b, path


@pytest.mark.skipif(not HAVE_REF, reason="no staged copy of the reference sbi")
def test_fixture_is_what_the_reference_computes(gold):
    _assert_same(make_fixture(), gold)


@pytest.mark.skipif(not HAVE_REF, reason="no staged copy of the reference sbi")
@pytest.mark.parametrize("args", [dict(model="mlp", num_blocks=3), dict(model="linear", hidden_features=30),
                                  dict(model="linear", norm_layer=nn.Identity)])
def test_classifier_nn_rejects_what_the_reference_rejects(args):
    from oracle import ref_shim
    assert ref_shim.install()
    from sbi.neural_nets import classifier_nn as ref_classifier_nn
    from sbi_b200.ratio import classifier_nn
    with pytest.raises(ValueError) as ref_err:
        ref_classifier_nn(**args)
    with pytest.raises(ValueError) as err:
        classifier_nn(**args)
    assert str(err.value) in str(ref_err.value)


def test_mlp_entry_points_exported(lib):
    from sbi_b200 import _lib
    hdr = open(os.path.join(os.path.dirname(HERE), "include", "sbi_b200.h")).read()
    for name in ("sbi_b200_ratio_mlp_forward", "sbi_b200_ratio_mlp_vjp_parts", "sbi_b200_ratio_mlp_vjp"):
        assert f"{name}(" in hdr and name in _lib.exported_symbols()
        assert getattr(lib, name) is not None
    assert lib.sbi_b200_ratio_mlp_forward(None, None, None, None) == -1
    assert lib.sbi_b200_ratio_mlp_vjp_parts(1) == 1


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    torch.save(make_fixture(), GOLD)
    print(GOLD, os.path.getsize(GOLD))
