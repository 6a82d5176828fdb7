"""L-C2ST without a GPU: the constructor, validation and state-machine errors with the reference's messages, the
classifier kwargs, and everything drawn on the host -- initial weights, validation splits, KFold, null permutations,
z-scoring -- against scikit-learn and the UNMODIFIED reference (through oracle.ref_shim); the unsupported
classifiers, kwargs and network sizes; and the refusal to train without a CUDA device."""
import numpy as np
import pytest
import torch

pytest.importorskip("sklearn")
from sklearn.ensemble import RandomForestClassifier  # noqa: E402
from sklearn.neural_network import MLPClassifier  # noqa: E402
from sklearn.neural_network import _multilayer_perceptron as skmlp  # noqa: E402

from oracle import ref_shim  # noqa: E402
from sbi_b200 import lc2st as L  # noqa: E402
from sbi_b200.diagnostics import LC2ST, LC2ST_NF, LC2STState  # noqa: E402

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")


@pytest.fixture(scope="module")
def ref():
    assert ref_shim.install()
    from sbi.diagnostics import lc2st as R
    return R


def _data(n=50, dt=2, dx=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, dt, generator=g), torch.randn(n, dx, generator=g), torch.randn(n, dt, generator=g) + .3


def _errors_equal(ours, theirs):
    with pytest.raises(Exception) as a:
        ours()
    with pytest.raises(Exception) as b:
        theirs()
    assert type(a.value) is type(b.value) and str(a.value) == str(b.value), (a.value, b.value)


@needs_ref
@pytest.mark.parametrize("case", [
    dict(prior_samples=None), dict(xs=None), dict(posterior_samples=None),
    dict(prior_samples=torch.randn(10, 2), xs=torch.randn(10, 3), posterior_samples=torch.randn(10, 4)),
    dict(prior_samples=torch.randn(100, 2), xs=torch.randn(50, 3), posterior_samples=torch.randn(100, 2)),
    dict(num_folds=0), dict(num_folds=60), dict(classifier="invalid"), dict(seed=1.5),
    dict(prior_samples=np.zeros((10, 2))), dict(xs=torch.zeros(0, 3)), dict(classifier=int),
])
def test_constructor_errors_match_reference(ref, case):
    t, x, p = _data()
    kw = {**dict(prior_samples=t, xs=x, posterior_samples=p), **case}
    _errors_equal(lambda: LC2ST(**kw), lambda: ref.LC2ST(**kw))


@needs_ref
def test_nf_and_deprecation_errors_match_reference(ref):
    t, x, p = _data()
    inv = lambda th, xx: th  # noqa: E731
    base = torch.distributions.MultivariateNormal(torch.zeros(2), torch.eye(2))
    for kw in (dict(flow_inverse_transform=None, flow_base_dist=base), dict(flow_inverse_transform=inv)):
        _errors_equal(lambda: LC2ST_NF(t, x, p, **kw), lambda: ref.LC2ST_NF(t, x, p, **kw))
    with pytest.warns(FutureWarning, match="thetas.*deprecated"):
        _errors_equal(lambda: LC2ST(prior_samples=t, thetas=t, xs=x, posterior_samples=p),
                      lambda: ref.LC2ST(prior_samples=t, thetas=t, xs=x, posterior_samples=p))
    with pytest.warns(FutureWarning, match="thetas.*deprecated"):
        assert torch.equal(LC2ST(thetas=t, xs=x, posterior_samples=p).theta_q, t)


@needs_ref
def test_state_machine_errors_match_reference(ref):
    t, x, p = _data()
    ours, theirs = LC2ST(t, x, p, num_trials_null=2), ref.LC2ST(t, x, p, num_trials_null=2)
    assert ours.state == LC2STState.INITIALIZED and theirs.state.name == "INITIALIZED"
    for name in ("p_value", "get_statistic_on_observed_data", "get_statistics_under_null_hypothesis"):
        _errors_equal(lambda: getattr(ours, name)(theta_o=p[:5], x_o=x[0]),
                      lambda: getattr(theirs, name)(theta_o=p[:5], x_o=x[0]))
    for st in ("OBSERVED_TRAINED", "NULL_TRAINED"):
        ours._state, theirs._state = LC2STState[st], ref.LC2STState[st]
        _errors_equal(lambda: ours.p_value(theta_o=p[:5], x_o=x[0]), lambda: theirs.p_value(theta_o=p[:5], x_o=x[0]))
    ours._state, theirs._state = LC2STState.READY, ref.LC2STState.READY
    ours.trained_clfs_null, theirs.trained_clfs_null = {0: []}, {0: []}
    _errors_equal(lambda: ours.get_statistics_under_null_hypothesis(theta_o=p[:5], x_o=x[0]),
                  lambda: theirs.get_statistics_under_null_hypothesis(theta_o=p[:5], x_o=x[0]))
    _errors_equal(ours.train_under_null_hypothesis, theirs.train_under_null_hypothesis)
    no_null = LC2ST(t, x, p, permutation=False, num_trials_null=2)
    ref_no_null = ref.LC2ST(t, x, p, permutation=False, num_trials_null=2)
    _errors_equal(no_null.train_under_null_hypothesis, ref_no_null.train_under_null_hypothesis)


@needs_ref
def test_nan_rows_and_zscore_match_reference(ref):
    t, x, p = _data(n=40)
    x[3, 1], x[7, 0] = float("nan"), float("inf")
    p[:, 0] = 0.25   # a constant dimension keeps std 1
    with pytest.warns(UserWarning, match="Found 1 NaNs and 1 Infs") as w_ours:
        ours = LC2ST(t, x, p, z_score=True)
    with pytest.warns(UserWarning) as w_ref:
        theirs = ref.LC2ST(t, x, p, z_score=True)
    assert str(w_ours[0].message) == str(w_ref[0].message)
    for name in ("theta_p", "theta_q", "x_p", "theta_p_mean", "theta_p_std", "x_p_mean", "x_p_std"):
        assert torch.equal(getattr(ours, name), getattr(theirs, name)), name
    assert ours.theta_p_std[0] == 1.0
    assert torch.equal(ours._normalize_theta(t), theirs._normalize_theta(t))
    assert torch.equal(ours._normalize_x(ours.x_p), theirs._normalize_x(ours.x_p))


@needs_ref
@pytest.mark.parametrize("kw", [None, dict(max_iter=7, alpha=0.1), dict(hidden_layer_sizes=(5,), random_state=3)])
def test_classifier_kwargs_merge_like_reference(ref, kw):
    t, x, p = _data(dt=3)
    ours, theirs = LC2ST(t, x, p, classifier_kwargs=kw), ref.LC2ST(t, x, p, classifier_kwargs=kw)
    assert ours.clf_kwargs == theirs.clf_kwargs
    assert ours.clf_class is MLPClassifier and theirs.clf_class is MLPClassifier
    assert LC2ST(t, x, p, classifier="mlp", device="cuda").clf_class is MLPClassifier


def test_unsupported_classifiers_and_kwargs():
    t, x, p = _data()
    with pytest.raises(NotImplementedError, match="random_forest.*supported"):
        LC2ST(t, x, p, classifier="random_forest")
    with pytest.raises(NotImplementedError, match="RandomForestClassifier.*supported"):
        LC2ST(t, x, p, classifier=RandomForestClassifier)
    with pytest.raises(TypeError, match="subclass of BaseEstimator"):
        LC2ST(t, x, p, classifier=dict)
    for kw in (dict(activation="tanh"), dict(solver="sgd"), dict(momentum=0.5), dict(warm_start=True)):
        with pytest.raises(NotImplementedError, match="does not support"):
            LC2ST(t, x, p, classifier_kwargs=kw)
    with pytest.raises(TypeError, match="fitted sklearn MLPClassifiers"):
        L._as_classifier(RandomForestClassifier(), torch.device("cpu"))


def test_network_envelope(lib):
    L._Net(64, (100, 100))                      # the default widths at dim_theta = 10, dim_theta + dim_x = 64
    L._Net(64, (128, 128))
    L._Net(3, (7,))
    L._Net(8, (16, 16, 16, 16))
    with pytest.raises(NotImplementedError, match="at most 64 inputs"):
        L._Net(65, (10, 10))
    with pytest.raises(NotImplementedError, match="1 to 4 hidden layers"):
        L._Net(4, (8,) * 5)
    with pytest.raises(NotImplementedError, match="at most 256 units"):
        L._Net(4, (257, 8))
    with pytest.raises(NotImplementedError, match="shared memory"):
        L._Net(64, (256, 256))
    out = (L.C.c_int32 * 3)()
    net = L._Net(64, (100, 100))
    assert lib.sbi_b200_lc2st_plan(L.C.byref(net.c), out) == 0 and out[0] == 32 and out[1] >= 8
    bad = L._lib.Lc2stNet(F=4, L=2, P=1)
    assert lib.sbi_b200_lc2st_plan(L.C.byref(bad), out) == -1


class _InitOnly(MLPClassifier):
    """sklearn's fit up to the optimizer: the initial weights stay in coefs_ / intercepts_."""

    def _fit_stochastic(self, *a, **k):
        pass


@pytest.mark.parametrize("random_state", [0, 1, 7, 12345])
@pytest.mark.parametrize("hidden", [(20, 20), (5,), (30, 10, 4)])
def test_initial_weights_bit_equal_to_sklearn(random_state, hidden):
    X = np.random.default_rng(0).normal(size=(40, 5)).astype(np.float32)
    y = np.r_[np.zeros(20, np.int64), np.ones(20, np.int64)]
    sk = _InitOnly(hidden_layer_sizes=hidden, random_state=random_state).fit(X, y)
    net = L._Net(5, hidden)
    ours = net.init_params(np.random.RandomState(random_state))
    assert np.array_equal(ours, net.pack(sk.coefs_, sk.intercepts_))
    assert ours.dtype == np.float32


def test_global_numpy_state_used_when_random_state_is_none():
    net = L._Net(4, (6, 6))
    np.random.seed(11)
    a = net.init_params(np.random.mtrand._rand)
    np.random.seed(11)
    X = np.random.default_rng(0).normal(size=(30, 4)).astype(np.float32)
    sk = _InitOnly(hidden_layer_sizes=(6, 6)).fit(X, np.r_[np.zeros(15), np.ones(15)].astype(np.int64))
    assert np.array_equal(a, net.pack(sk.coefs_, sk.intercepts_))


@needs_ref
@pytest.mark.parametrize("rs,E", [(None, 3), (5, 3), (None, 1), (2, 1)])
def test_ensemble_random_states_follow_reference(ref, rs, E):
    t, x, p = _data()
    kw = None if rs is None else dict(random_state=rs)
    ours = LC2ST(t, x, p, num_ensemble=E, classifier_kwargs=kw)
    seen = []

    class Rec(MLPClassifier):
        def fit(self, X, y):
            seen.append(self.random_state)
            return self

    ens = ref.EnsembleClassifier(Rec(random_state=rs), E, verbosity=0)
    (ens if E > 1 else Rec(random_state=rs)).fit(np.zeros((4, 2)), np.r_[0, 0, 1, 1])
    assert ours._member_states() == seen


@pytest.mark.parametrize("n,vf,rs", [(200, 0.1, 0), (2000, 0.1, 3), (38, 0.1, 1), (100, 0.25, 9)])
def test_validation_split_equals_sklearn(monkeypatch, n, vf, rs):
    """The training / validation samples (in their order) equal sklearn's own train_test_split inside fit."""
    seen = {}
    real = skmlp.train_test_split

    def spy(*a, **k):
        out = real(*a, **k)
        seen["train"], seen["val"] = out[0][:, 0].astype(int), out[1][:, 0].astype(int)
        return out

    monkeypatch.setattr(skmlp, "train_test_split", spy)
    X = np.c_[np.arange(n), np.random.default_rng(1).normal(size=(n, 2))].astype(np.float32)
    y = np.r_[np.zeros(n // 2), np.ones(n - n // 2)].astype(np.int64)
    MLPClassifier(hidden_layer_sizes=(4,), max_iter=1, early_stopping=True, validation_fraction=vf,
                  random_state=rs).fit(X, y)
    s = L._clf_settings(dict(hidden_layer_sizes=(4,), max_iter=1, early_stopping=True, validation_fraction=vf))
    mdl = L._Model(np.zeros((n, 2), np.int32), y.astype(np.float32), rs)
    _, idx, n_train, _ = L.prepare_model(L._Net(3, (4,)), mdl, s)
    assert np.array_equal(idx[:n_train], seen["train"]) and np.array_equal(idx[n_train:], seen["val"])


def test_validation_set_too_small():
    """Too few samples for a stratified 2-row validation set: sklearn's own error."""
    s = L._clf_settings(dict(early_stopping=True))
    y = np.r_[np.zeros(5), np.ones(5)].astype(np.int64)
    mdl = L._Model(np.zeros((10, 2), np.int32), y.astype(np.float32), 0)
    with pytest.raises(ValueError) as ours:
        L.prepare_model(L._Net(3, (4,)), mdl, s)
    with pytest.raises(ValueError) as theirs:
        MLPClassifier(hidden_layer_sizes=(4,), early_stopping=True, random_state=0).fit(np.zeros((10, 3)), y)
    assert str(ours.value) == str(theirs.value)
    mdl = L._Model(np.zeros((20, 2), np.int32), np.r_[np.zeros(10), np.ones(10)].astype(np.float32), 0)
    assert len(L.prepare_model(L._Net(3, (4,)), mdl, s)[1]) - L.prepare_model(L._Net(3, (4,)), mdl, s)[2] == 2


@needs_ref
@pytest.mark.parametrize("folds,seed", [(1, 1), (3, 1), (5, 42)])
def test_kfold_indices_equal_reference(ref, folds, seed):
    t, x, p = _data(n=23)
    ours = LC2ST(t, x, p, num_folds=folds, seed=seed)._fold_indices()
    if folds == 1:
        assert len(ours) == 1 and np.array_equal(ours[0], np.arange(23))
        return
    theirs = [tr for tr, _ in ref.KFold(n_splits=folds, shuffle=True, random_state=seed).split(p.numpy())]
    assert all(np.array_equal(a, b) for a, b in zip(ours, theirs)) and len(ours) == len(theirs)


@needs_ref
@pytest.mark.parametrize("t", [0, 1, 17, 99])
def test_null_permutations_equal_reference_and_leave_global_rng(ref, t):
    n = 31
    jp, jq = torch.randn(n, 4), torch.randn(n, 4)
    state = torch.random.get_rng_state()
    perm = L.permutation_indices(n, t)
    assert torch.equal(torch.random.get_rng_state(), state)
    rp, rq = ref.permute_data(jp, jq, seed=t)
    joint = torch.cat([jp, jq])
    assert torch.equal(joint[perm[:n]], rp) and torch.equal(joint[perm[n:]], rq)


def test_training_needs_a_cuda_device():
    if torch.cuda.is_available():
        pytest.skip("checks the no-GPU behaviour")
    t, x, p = _data()
    lc = LC2ST(t, x, p, num_trials_null=2)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        lc.train_on_observed_data()
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        lc.train_under_null_hypothesis()
    assert lc.state == LC2STState.INITIALIZED
