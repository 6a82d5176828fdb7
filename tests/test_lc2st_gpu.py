"""L-C2ST on the H100: the training kernel against scikit-learn's MLPClassifier when fed sklearn's own epoch orders,
the evaluation kernel against sklearn's predict_proba, batching independence and determinism, the test's
statistical behaviour on a linear-Gaussian task with an analytic posterior, and the null statistics against the
UNMODIFIED reference's sklearn path."""
import math
import warnings

import numpy as np
import pytest
import torch

pytest.importorskip("sklearn")
from scipy.stats import binomtest, ks_2samp  # noqa: E402
from sklearn.exceptions import ConvergenceWarning  # noqa: E402
from sklearn.model_selection import train_test_split  # noqa: E402
from sklearn.neural_network import MLPClassifier  # noqa: E402
from sklearn.utils import shuffle as sk_shuffle  # noqa: E402

from oracle import ref_shim  # noqa: E402
from sbi_b200 import lc2st as L  # noqa: E402
from sbi_b200.diagnostics import LC2ST, LC2ST_NF  # noqa: E402

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="no copy of the reference sbi")
DEV = torch.device("cuda")


def _two_samples(n, dt, dx, seed, shift=0.6):
    """n rows per class: P = (theta, x), Q = (theta + shift, x); features float32, labels 0 / 1."""
    r = np.random.default_rng(seed)
    x = r.normal(size=(n, dx))
    tp = r.normal(size=(n, dt)) + 0.5 * x[:, :1]
    tq = r.normal(size=(n, dt)) + shift
    X = np.r_[np.c_[tp, x], np.c_[tq, x]].astype(np.float32)
    y = np.r_[np.zeros(n), np.ones(n)].astype(np.int64)
    return X, y


def _replay_orders(net, n, y, kw, seed):
    """sklearn's epoch orders for MLPClassifier(random_state=seed).fit: replay its RandomState draws."""
    rs = np.random.RandomState(seed)
    net.init_params(rs)
    n_train = n
    if kw.get("early_stopping"):
        yb = (y == 1).reshape(-1, 1)
        tr, _ = train_test_split(np.arange(n), yb, random_state=rs, test_size=kw.get("validation_fraction", 0.1),
                                 stratify=yb)[:2]
        n_train = len(tr)
    idx, out = np.arange(n_train), []
    for _ in range(kw["max_iter"]):
        idx = sk_shuffle(idx, random_state=rs)
        out.append(idx)
    return np.stack(out)


def _fit_ours(X, y, dt, kw, seed, orders=None):
    n = len(y)
    i = np.arange(n)
    mdl = L._Model(np.stack([i, i], 1).astype(np.int32), y.astype(np.float32), seed)
    X = torch.from_numpy(X)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        return L.train_classifiers(X[:, :dt], X[:, dt:], [mdl], kw, DEV,
                                   epoch_orders=None if orders is None else [orders])[0]


CASES = {
    "dt1_dx1_ntrain135": (1, 1, 75, dict(early_stopping=True)),
    "dt2_dx3_partial_batch": (2, 3, 500, dict(early_stopping=True)),
    "dt5_dx5_no_early_stop": (5, 5, 350, dict(early_stopping=False)),
    "dt2_dx4_alpha_lr_bs": (2, 4, 250, dict(early_stopping=True, alpha=1e-2, learning_rate_init=3e-3,
                                            batch_size=64)),
    "dt5_dx20_bs37_no_es": (5, 20, 150, dict(early_stopping=False, batch_size=37, alpha=0.0)),
}


class _MarginMLP(MLPClassifier):
    """sklearn's MLPClassifier, recording per epoch the smallest |logit| over the validation rows with the weights
    that score them: the margin by which the accuracy (and so the stopping decision) is matched."""

    def _update_no_improvement_count(self, early_stopping, X, y, sample_weight):
        if early_stopping:
            z = X
            for i, (W, b) in enumerate(zip(self.coefs_, self.intercepts_)):
                z = z @ W + b
                z = np.maximum(z, 0) if i < len(self.coefs_) - 1 else z
            self.margins_ = getattr(self, "margins_", []) + [float(np.abs(z).min())]
        super()._update_no_improvement_count(early_stopping, X, y, sample_weight)


def _replay_case(dt, dx, n, kw, seed=3):
    X, y = _two_samples(n, dt, dx, seed=7)
    net = L._Net(dt + dx, kw["hidden_layer_sizes"])
    ours = _fit_ours(X, y, dt, kw, seed, _replay_orders(net, len(y), y, kw, seed))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        sk = _MarginMLP(random_state=seed, **kw).fit(X, y)
    err = max(float(np.abs(a - b).max()) for a, b in zip(ours.coefs_ + ours.intercepts_, sk.coefs_ + sk.intercepts_))
    margin = min(getattr(sk, "margins_", [math.inf]))
    print(f"{kw}: n_iter {sk.n_iter_}, max |coef diff| = {err:.2e}, smallest validation |z| = {margin:.2e}")
    assert ours.n_iter_ == sk.n_iter_
    if kw.get("early_stopping"):
        assert ours.validation_scores_ == [float(v) for v in sk.validation_scores_]
        assert ours.best_validation_score_ == sk.best_validation_score_
    else:
        assert np.allclose(ours.loss_curve_, sk.loss_curve_, rtol=1e-5)
        assert ours.best_loss_ == pytest.approx(sk.best_loss_, rel=1e-5)
    return err, sk


@pytest.mark.parametrize("max_iter", [1, 3, 5])
@pytest.mark.parametrize("case", list(CASES))
def test_training_replays_sklearn(cuda_lib, case, max_iter):
    dt, dx, n, extra = CASES[case]
    kw = dict(hidden_layer_sizes=(10 * dt, 10 * dt), max_iter=max_iter, n_iter_no_change=50, **extra)
    err, _ = _replay_case(dt, dx, n, kw)
    assert err <= 1e-5


@pytest.mark.parametrize("n_iter_no_change", [1, 2, 3])
@pytest.mark.parametrize("early_stopping", [True, False], ids=["val_score", "train_loss"])
def test_stop_rule_replays_sklearn(cuda_lib, early_stopping, n_iter_no_change):
    """Runs that sklearn stops before max_iter: the stopping epoch, the curves and the restored weights agree."""
    kw = dict(hidden_layer_sizes=(20, 20), max_iter=60, n_iter_no_change=n_iter_no_change,
              early_stopping=early_stopping, tol=1e-4 if early_stopping else 2e-3)
    err, sk = _replay_case(2, 3, 300, kw)
    assert sk.n_iter_ < kw["max_iter"]
    assert err <= 1e-5


def test_evaluation_matches_predict_proba(cuda_lib):
    """141 fitted sklearn classifiers (ensembles of 1 and of 3) on 1061 rows: one launch each."""
    dt, dx, S = 3, 4, 1061
    X, y = _two_samples(200, dt, dx, seed=1)
    fitted = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        for k in range(141):
            fitted.append(MLPClassifier(hidden_layer_sizes=(30, 30), max_iter=2, random_state=k).fit(X, y))
    rows = np.random.default_rng(2).normal(size=(S, dt + dx)).astype(np.float32)
    clfs = [L._as_classifier(c, DEV) for c in fitted]
    theta = torch.from_numpy(rows[:, :dt]).reshape(1, S, dt)
    x_o = torch.from_numpy(rows[0, dt:])
    rows[:, dt:] = rows[0, dt:]
    probs, scores = L._evaluate(clfs, theta, None, x_o)
    want = np.stack([c.predict_proba(rows)[:, 0] for c in fitted])
    want_s = ((want - np.full(S, 0.5)) ** 2).mean(axis=1)
    assert np.abs(probs - want).max() <= 1e-6
    assert np.abs(scores / want_s - 1).max() <= 1e-5
    ens = [L.TrainedEnsemble(clfs[3 * i:3 * i + 3]) for i in range(47)]
    probs_e, scores_e = L._evaluate(ens, theta, None, x_o)
    want_e = np.stack([np.mean([c.predict_proba(rows) for c in fitted[3 * i:3 * i + 3]], axis=0)[:, 0]
                       for i in range(47)])
    assert np.abs(probs_e - want_e).max() <= 1e-6
    assert np.abs(scores_e / ((want_e - 0.5) ** 2).mean(axis=1) - 1).max() <= 1e-5


def test_batching_independence_and_determinism(cuda_lib):
    """A model trained alone equals the same model inside a launch of 300 with very different stopping epochs."""
    dt, dx = 2, 3
    X, y = _two_samples(400, dt, dx, seed=5)
    Xt = torch.from_numpy(X)
    kw = dict(hidden_layer_sizes=(20, 20), max_iter=300, n_iter_no_change=10, early_stopping=True)
    i = np.arange(len(y))
    models = []
    for k in range(300):
        keep = i if k % 3 == 0 else np.r_[i[:40 + k], i[400:440 + k]]
        models.append(L._Model(np.stack([keep, keep], 1).astype(np.int32), y[keep].astype(np.float32), k))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        many = L.train_classifiers(Xt[:, :dt], Xt[:, dt:], models, kw, DEV)
        for k in (0, 7, 299):
            alone = L.train_classifiers(Xt[:, :dt], Xt[:, dt:], [models[k]], kw, DEV)[0]
            assert torch.equal(alone._flat, many[k]._flat)
            assert alone.n_iter_ == many[k].n_iter_ and alone.validation_scores_ == many[k].validation_scores_
    iters = [m.n_iter_ for m in many]
    print(f"stopping epochs in the launch: min {min(iters)}, max {max(iters)}")
    assert max(iters) - min(iters) >= 20


def _run_lc2st(seed_data, **kw):
    t, x, p = _lg_calibration(300, seed_data, shift=0.0)
    lc = LC2ST(t, x, p, num_trials_null=20, classifier_kwargs=dict(random_state=4), **kw)
    lc.train_on_observed_data().train_under_null_hypothesis()
    return lc


def test_full_runs_are_bit_identical(cuda_lib):
    a, b = _run_lc2st(0, num_folds=2, num_ensemble=2), _run_lc2st(0, num_folds=2, num_ensemble=2)
    for ca, cb in zip(a.trained_clfs, b.trained_clfs):
        assert all(torch.equal(m._flat, n._flat) for m, n in zip(ca.members, cb.members))
    for t in range(a.num_trials_null):
        for ca, cb in zip(a.trained_clfs_null[t], b.trained_clfs_null[t]):
            assert all(torch.equal(m._flat, n._flat) for m, n in zip(ca.members, cb.members))
    th, xo = _lg_posterior(torch.zeros(2), 500, shift=0.0, seed=3), torch.zeros(2)
    sa, sb = a.get_statistics_under_null_hypothesis(th, xo), b.get_statistics_under_null_hypothesis(th, xo)
    assert np.array_equal(sa.scores, sb.scores) and np.array_equal(sa.probabilities, sb.probabilities)
    assert sa.probabilities.shape == (20, 2, 500) and sa.scores.shape == (20,)
    obs = a.get_scores(th, xo, a.trained_clfs)
    assert obs.scores.shape == (2,) and obs.probabilities.shape == (2, 500)
    assert a.p_value(th, xo) == b.p_value(th, xo)


# ---- linear Gaussian: theta ~ N(0, I), x = theta + N(0, s^2 I); posterior N(x / (1 + s^2), s^2 / (1 + s^2) I)
S2 = 0.5


def _lg_posterior(x, n, shift, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    mean = x / (1 + S2) + shift
    return mean + scale * (S2 / (1 + S2)) ** 0.5 * torch.randn(n, x.shape[-1], generator=g)


def _lg_calibration(n, seed, shift, scale=1.0, d=2):
    g = torch.Generator().manual_seed(seed)
    theta = torch.randn(n, d, generator=g)
    x = theta + S2 ** 0.5 * torch.randn(n, d, generator=g)
    post = x / (1 + S2) + shift + scale * (S2 / (1 + S2)) ** 0.5 * torch.randn(n, d, generator=g)
    return theta, x, post


def _inverse(shift, scale):
    """The analytic flow of the (possibly wrong) posterior estimate: z = (theta - mean(x)) / std."""
    return lambda theta, x: (theta - x / (1 + S2) - shift) / (scale * (S2 / (1 + S2)) ** 0.5)


@pytest.mark.parametrize("kind", ["exact", "shifted", "overdispersed"])
@pytest.mark.parametrize("nf", [False, True], ids=["LC2ST", "LC2ST_NF"])
def test_linear_gaussian_rejection_rates(cuda_lib, kind, nf):
    shift, scale = {"exact": (0.0, 1.0), "shifted": (0.5, 1.0), "overdispersed": (0.0, 2.0)}[kind]
    theta, x, post = _lg_calibration(1000, 11, shift, scale)
    base = torch.distributions.MultivariateNormal(torch.zeros(2), torch.eye(2))
    if nf:
        lc = LC2ST_NF(theta, x, post, flow_inverse_transform=_inverse(shift, scale), flow_base_dist=base,
                      num_eval=1000)
    else:
        lc = LC2ST(theta, x, post)
    lc.train_on_observed_data(seed=0).train_under_null_hypothesis()
    g = torch.Generator().manual_seed(12)
    rejects = 0
    for k in range(100):
        th_true = torch.randn(2, generator=g)
        x_o = th_true + S2 ** 0.5 * torch.randn(2, generator=g)
        if nf:
            rejects += lc.reject_test(x_o=x_o)
        else:
            rejects += lc.reject_test(theta_o=_lg_posterior(x_o, 1000, shift, 100 + k, scale), x_o=x_o)
    print(f"{'LC2ST_NF' if nf else 'LC2ST'} {kind}: {rejects} / 100 rejected")
    if kind == "exact":
        assert binomtest(rejects, 100, 0.05, alternative="greater").pvalue > 0.01
    else:
        assert rejects > 95


def test_lc2st_nf_on_a_one_epoch_nsf_npe(cuda_lib):
    """LC2ST_NF on what a user passes in: an sbi_b200 NSF NPE trained for one epoch, its `inverse_transform`
    (device tensors next to host xs, host base draws and host theta_o) and its standard-normal base.  The
    barely trained flow must be rejected at (almost) every observation."""
    from sbi_b200.inference import NPE
    prior = torch.distributions.MultivariateNormal(torch.zeros(2), torch.eye(2))
    g = torch.Generator().manual_seed(31)
    theta = torch.randn(3000, 2, generator=g)
    x = theta + S2 ** 0.5 * torch.randn(3000, 2, generator=g)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est = NPE(prior, density_estimator="nsf", device="cuda").append_simulations(theta, x).train(
            training_batch_size=200, max_num_epochs=1)
    theta_cal, x_cal = theta[:1000], x[:1000]
    with torch.no_grad():
        post = est.sample((1,), x_cal.cuda())[0]
        lc = LC2ST_NF(theta_cal, x_cal, post, flow_base_dist=prior, num_eval=1000,
                      flow_inverse_transform=lambda t, xx: est.inverse_transform(t.cuda(), xx.cuda()))
    assert lc.theta_p.is_cuda and not lc.x_p.is_cuda and not lc.theta_o.is_cuda
    lc.train_on_observed_data(seed=0).train_under_null_hypothesis()
    rejects = 0
    for k in range(100):
        th_true = torch.randn(2, generator=g)
        rejects += lc.reject_test(x_o=th_true + S2 ** 0.5 * torch.randn(2, generator=g))
    print(f"LC2ST_NF on a 1-epoch NSF NPE: {rejects} / 100 rejected")
    assert rejects > 95


@needs_ref
def test_null_statistics_match_reference(cuda_lib):
    """dim_theta 2, N 1000, 100 null trials: our null statistics and the reference's sklearn ones are one
    distribution, and both decide a clearly good and a clearly bad case alike."""
    assert ref_shim.install()
    from sbi.diagnostics.lc2st import LC2ST as RefLC2ST
    theta, x, post = _lg_calibration(1000, 21, 0.0)
    _, _, bad = _lg_calibration(1000, 21, 0.7)
    x_o = torch.tensor([0.3, -0.2])
    good_o, bad_o = _lg_posterior(x_o, 1000, 0.0, 5), _lg_posterior(x_o, 1000, 0.7, 5)
    out = {}
    for name, cls in (("ours", LC2ST), ("ref", RefLC2ST)):
        res = []
        for samples, theta_o in ((post, good_o), (bad, bad_o)):   # the estimator under test made both
            lc = cls(theta, x, samples)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                lc.train_on_observed_data(seed=1, verbosity=0).train_under_null_hypothesis(verbosity=0)
            if not res:
                res.append(lc.get_statistics_under_null_hypothesis(theta_o=theta_o, x_o=x_o).scores)
            res.append(lc.reject_test(theta_o=theta_o, x_o=x_o))
        out[name] = tuple(res)
    p = ks_2samp(out["ours"][0], out["ref"][0]).pvalue
    print(f"KS p = {p:.3f}; null mean ours {out['ours'][0].mean():.3e} ref {out['ref'][0].mean():.3e}")
    assert p > 0.01
    print(f"decisions (good, bad): ours {out['ours'][1:]}, reference {out['ref'][1:]}")
    assert out["ours"][1:] == out["ref"][1:] == (False, True)


@pytest.mark.parametrize("dt,dx,hidden", [(10, 54, None), (2, 62, (128, 128)), (3, 2, (8, 8, 8, 8))])
def test_envelope_sizes_train_and_evaluate(cuda_lib, dt, dx, hidden):
    theta, x, post = _lg_calibration(400, 3, 0.4, d=dt)
    xs = torch.cat([x, torch.randn(400, dx - dt)], 1) if dx > dt else x[:, :dx]
    kw = dict(max_iter=20) if hidden is None else dict(max_iter=20, hidden_layer_sizes=hidden)
    lc = LC2ST(theta, xs, post, num_trials_null=3, classifier_kwargs=kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        lc.train_on_observed_data(seed=0).train_under_null_hypothesis()
    assert lc.trained_clfs[0].coefs_[0].shape == (dt + dx, hidden[0] if hidden else 10 * dt)
    assert 0.0 <= lc.p_value(theta_o=post[:100], x_o=xs[0]) <= 1.0


def test_smallest_validation_set(cuda_lib):
    """10 samples per class: a stratified 2-row validation set; 5 per class leave sklearn's 1-row one, an error."""
    theta, x, post = _lg_calibration(10, 4, 0.4)
    lc = LC2ST(theta, x, post, num_trials_null=2, classifier_kwargs=dict(max_iter=30))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        lc.train_on_observed_data(seed=0).train_under_null_hypothesis()
    v = lc.trained_clfs[0].validation_scores_
    assert len(v) == lc.trained_clfs[0].n_iter_ and set(v) <= {0.0, 0.5, 1.0}
    with pytest.raises(ValueError):
        LC2ST(theta[:5], x[:5], post[:5], classifier_kwargs=dict(max_iter=3)).train_on_observed_data()


def test_pretrained_sklearn_null_classifiers(cuda_lib):
    """LC2ST_NF accepts fitted sklearn MLPClassifiers as its null classifiers (NULL_TRAINED at construction)."""
    theta, x, post = _lg_calibration(300, 6, 0.0)
    base = torch.distributions.MultivariateNormal(torch.zeros(2), torch.eye(2))
    X, y = _two_samples(100, 2, 2, seed=0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        null = {t: [MLPClassifier(hidden_layer_sizes=(20, 20), max_iter=3, random_state=t).fit(X, y)]
                for t in range(5)}
    lc = LC2ST_NF(theta, x, post, flow_inverse_transform=_inverse(0.0, 1.0), flow_base_dist=base, num_eval=200,
                  trained_clfs_null=null, num_trials_null=5)
    assert lc.state.name == "NULL_TRAINED"
    lc.train_on_observed_data(seed=0)
    assert lc.state.name == "READY"
    assert 0.0 <= lc.p_value(x_o=x[0]) <= 1.0
    with pytest.raises(TypeError):
        LC2ST_NF(theta, x, post, flow_inverse_transform=_inverse(0.0, 1.0), flow_base_dist=base,
                 trained_clfs_null={0: [object()]})
