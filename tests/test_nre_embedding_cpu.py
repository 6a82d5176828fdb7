"""Embedding nets in the NRE `resnet` classifier on the CPU: the network is built on the embedded widths, its
initial weights and state_dict keys equal the UNMODIFIED reference builder's (through oracle.ref_shim), reference
checkpoints load, the two new C entries are declared and bound, and data-parallel training with an embedding
raises."""
import copy
import os
import re

import pytest
import torch
from torch import nn

from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emb_x(seed=3):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(12, 16), nn.ReLU(), nn.Linear(16, 5))


def _emb_theta(seed=4):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Linear(3, 7), nn.Tanh())


def _data():
    g = torch.Generator().manual_seed(0)
    return 0.8 * torch.randn(300, 3, generator=g) + 0.2, torch.randn(300, 12, generator=g) - 0.5


@pytest.mark.parametrize("sides", ["x", "theta", "both"])
def test_resnet_builds_on_embedded_widths(sides):
    from sbi_b200.ratio import classifier_nn
    theta, x = _data()
    kw = {}
    if sides in ("x", "both"):
        kw["embedding_net_x"] = _emb_x()
    if sides in ("theta", "both"):
        kw["embedding_net_theta"] = _emb_theta()
    est = classifier_nn("resnet", **kw)(theta, x)
    lay = est.layout
    assert (lay.Dt, lay.Dx) == (7 if sides != "x" else 3, 5 if sides != "theta" else 12)
    assert est.theta_shape == (3,) and est.x_shape == (12,)
    assert len(est.embedding_nets) == (2 if sides == "both" else 1)
    # an embedded side standardises in torch: the kernels get identity statistics for it
    th_stats, x_stats, _ = est._stat_sources(False)
    assert (th_stats is None) == (sides != "x") and (x_stats is None) == (sides != "theta")
    rows = est.embed_x(x[:4])
    if sides == "theta":
        assert torch.equal(rows, x[:4])
    else:
        assert torch.equal(rows, est.embedding_net_x[1](est.embedding_net_x[0](x[:4])))
    assert rows.shape == (4, lay.Dx)


def test_conv_embedding_sees_event_shape():
    """x of event shape (2, 6) reaches a Conv1d embedding unflattened; the classifier sees its output width."""
    from sbi_b200.ratio import classifier_nn
    theta, x = _data()
    x = x.reshape(-1, 2, 6)
    torch.manual_seed(0)
    emb = nn.Sequential(nn.Conv1d(2, 3, 3), nn.Flatten())
    est = classifier_nn("resnet", embedding_net_x=emb)(theta, x)
    assert est.layout.Dx == 12 and est.x_shape == (2, 6)
    assert est.embed_x(x[:5]).shape == (5, 12)


@pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
@pytest.mark.parametrize("z_score", ["independent", "structured", "none"])
def test_resnet_builder_with_embeddings_matches_reference(z_score):
    assert ref_shim.install()
    from sbi.neural_nets import classifier_nn as ref_classifier_nn
    from sbi_b200.ratio import classifier_nn
    theta, x = _data()
    et, ex = _emb_theta(), _emb_x()
    kw = dict(z_score_theta=z_score, z_score_x=z_score)
    torch.manual_seed(9)
    a = ref_classifier_nn("resnet", embedding_net_theta=copy.deepcopy(et), embedding_net_x=copy.deepcopy(ex),
                          **kw)(theta, x)
    torch.manual_seed(9)
    b = classifier_nn("resnet", embedding_net_theta=copy.deepcopy(et), embedding_net_x=copy.deepcopy(ex),
                      **kw)(theta, x)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) == set(sb), set(sa) ^ set(sb)
    if z_score != "none":
        assert "embedding_net_x.0._mean" in sb and "embedding_net_x.1.0.weight" in sb
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    # a reference checkpoint loads into a freshly built estimator
    torch.manual_seed(1)
    c = classifier_nn("resnet", embedding_net_theta=_emb_theta(seed=6), embedding_net_x=_emb_x(seed=7),
                      **kw)(theta, x)
    c.load_state_dict(sa)
    sc = c.state_dict()
    for k in sa:
        assert torch.equal(sa[k], sc[k]), k


def test_mlp_and_linear_keep_rejecting_embedding_nets():
    from sbi_b200.ratio import classifier_nn
    theta, x = _data()
    for model in ("mlp", "linear"):
        with pytest.raises(NotImplementedError, match="embedding"):
            classifier_nn(model, embedding_net_theta=_emb_theta())(theta, x)


def test_new_entries_declared_and_bound():
    from sbi_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "sbi_b200.h")).read()
    for name in ("sbi_b200_ratio_vjp_inputs", "sbi_b200_pair_rows_sum"):
        assert re.search(rf"\bint\s+{name}\s*\(", hdr), name
        assert name in _lib.exported_symbols()


def test_data_parallel_with_embedding_raises(monkeypatch, tmp_path):
    import torch.distributed as dist
    import sbi_b200.inference as inference
    from sbi_b200.ratio import classifier_nn
    # the check comes before any kernel runs, so it is reachable on a host without a GPU
    monkeypatch.setattr(inference, "_process_device", lambda device: "cpu")
    dist.init_process_group("gloo", init_method=f"file://{tmp_path}/store", rank=0, world_size=1)
    try:
        theta, x = _data()
        inf = inference.NRE_B(classifier=classifier_nn("resnet", embedding_net_x=_emb_x())).data_parallel()
        with pytest.raises(NotImplementedError, match="embedding"):
            inf.append_simulations(theta, x).train(max_num_epochs=1)
    finally:
        dist.destroy_process_group()
