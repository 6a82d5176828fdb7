"""Embedding nets in the flow-matching builder on the CPU: parity with the UNMODIFIED reference builder (through
oracle.ref_shim) for initial weights and state_dict keys, reference checkpoints load, and the score estimators
keep rejecting embedding nets."""
import copy

import pytest
import torch
from torch import nn

from oracle import ref_shim


def _emb(seed=3):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(12, 16), nn.ReLU(), nn.Linear(16, 4))


def _data():
    g = torch.Generator().manual_seed(0)
    return 0.8 * torch.randn(300, 3, generator=g) + 0.2, torch.randn(300, 12, generator=g) - 0.5


@pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
def test_fmpe_builder_with_embedding_matches_reference():
    assert ref_shim.install()
    from sbi.neural_nets import posterior_flow_nn as ref_posterior_flow_nn
    from sbi_b200.flowmatching import posterior_flow_nn
    theta, x = _data()
    emb = _emb()
    torch.manual_seed(9)
    a = ref_posterior_flow_nn("mlp", embedding_net=copy.deepcopy(emb))(theta, x)
    torch.manual_seed(9)
    b = posterior_flow_nn("mlp", embedding_net=copy.deepcopy(emb))(theta, x)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) == set(sb), set(sa) ^ set(sb)
    assert "_embedding_net.1.0.weight" in sb and "_embedding_net.0._mean" in sb
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    assert b.layout.C == 4
    # a reference checkpoint loads into a freshly built estimator
    torch.manual_seed(1)
    c = posterior_flow_nn("mlp", embedding_net=_emb(seed=4))(theta, x)
    c.load_state_dict(sa)
    sc = c.state_dict()
    for k in sa:
        assert torch.equal(sa[k], sc[k]), k


def test_embedded_condition_width_and_identity_statistics():
    """With an embedding net the kernels see the embedded width, and the condition z-score runs in torch
    (Standardize ahead of the user's module), not in the kernel."""
    from sbi_b200.flowmatching import build_vector_field_estimator
    theta, x = _data()
    est = build_vector_field_estimator(theta, x, embedding_net=_emb())
    assert est.layout.C == 4 and not est._embed_identity
    ident = build_vector_field_estimator(theta, x)
    assert ident.layout.C == 12 and ident._embed_identity
    ctx = est._embed(x[:5])
    ref = est.embedding_net[1](est.embedding_net[0](x[:5]))
    assert ctx.shape == (5, 4) and torch.equal(ctx, ref)


def test_score_estimators_keep_rejecting_embedding_nets():
    from sbi_b200.score import posterior_score_nn
    theta, x = _data()
    with pytest.raises(NotImplementedError, match="embedding"):
        posterior_score_nn("mlp", embedding_net=_emb())(theta, x)
    posterior_score_nn("mlp")(theta, x)      # identity embedding still builds
