"""The local classifier two-sample test (L-C2ST) with the reference's classes, signatures, messages and state machine
(the reference sbi's `sbi/diagnostics/lc2st.py`).  The classifiers are scikit-learn's `MLPClassifier(solver="adam")` with
ReLU hidden layers, but trained on the device: one launch of `sbi_b200_lc2st_train` trains every classifier a call
needs (observed: folds x ensemble; null: trials x folds x ensemble) with sklearn's algorithm in float32, early
stopping included, and one launch of `sbi_b200_lc2st_eval` evaluates every classifier a statistic needs.

Everything sklearn and the reference draw on the host is drawn the same way here: each model's initial weights and
its stratified validation split come from `check_random_state(random_state)` in sklearn's order, KFold and the null
permutations match, and `null_distribution` is sampled in the reference's order.  The deviations:
  * the epoch orders are keyed bijections drawn on the device; their key is drawn from the model's RandomState
    after the split, so a fixed `random_state` (or a seeded numpy) makes a run deterministic, but the RandomState
    is left in a different state than sklearn's per-epoch `shuffle` leaves it;
  * the null permutations come from a local torch generator seeded with the trial index, so, unlike the
    reference's `torch.manual_seed(t)`, the global torch RNG is left alone;
  * there is no skorch branch: `classifier="mlp"` runs this trainer whatever `device` says, and no CPU path.
"""
from __future__ import annotations

import ctypes as C
import warnings
from dataclasses import dataclass
from enum import Enum, auto
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Type, Union

import numpy as np
import torch
from torch import Tensor

try:
    from sklearn.base import BaseEstimator
    from sklearn.exceptions import ConvergenceWarning
    from sklearn.model_selection import KFold, train_test_split
    from sklearn.neural_network import MLPClassifier
    from sklearn.utils import check_random_state
except ModuleNotFoundError as e:   # the classifiers, their seeding and their splits are scikit-learn's
    raise ImportError("sbi_b200's LC2ST / LC2ST_NF need scikit-learn (`pip install scikit-learn`): they train "
                      "sklearn's MLPClassifier and draw its seeds, splits and folds with sklearn") from e

from . import _lib

DEFAULT_MLP_ACTIVATION = "relu"
DEFAULT_MLP_HIDDEN_LAYER_MULTIPLIER = 10
DEFAULT_MLP_MAX_ITER = 1000
DEFAULT_MLP_SOLVER = "adam"
DEFAULT_MLP_EARLY_STOPPING = True
DEFAULT_MLP_N_ITER_NO_CHANGE = 50

# MLPClassifier hyperparameters the trainer implements, with sklearn's defaults
SUPPORTED_KWARGS = {
    "hidden_layer_sizes": (100,), "max_iter": 200, "n_iter_no_change": 10, "tol": 1e-4, "early_stopping": False,
    "validation_fraction": 0.1, "alpha": 1e-4, "learning_rate_init": 1e-3, "batch_size": "auto", "beta_1": 0.9,
    "beta_2": 0.999, "epsilon": 1e-8, "shuffle": True, "random_state": None,
}
_FIXED_KWARGS = {"activation": "relu", "solver": "adam"}


class LC2STState(Enum):
    """Lifecycle states of LC2ST (INITIALIZED -> OBSERVED_TRAINED / NULL_TRAINED -> READY)."""

    INITIALIZED = auto()
    OBSERVED_TRAINED = auto()
    NULL_TRAINED = auto()
    READY = auto()


@dataclass
class LC2STScores:
    """Scores, shape (num_folds,) or (num_trials_null,), and the class-0 probabilities behind them."""

    scores: np.ndarray
    probabilities: Optional[np.ndarray] = None


# ---------------------------------------------------------------------------------------------------------------
# networks and the device entry points
class _Net:
    """One classifier architecture: F inputs, ReLU hidden widths, one logistic output."""

    def __init__(self, F: int, hidden: Sequence[int]):
        self.F, self.hidden = int(F), tuple(int(h) for h in hidden)
        if not (1 <= self.F <= _lib.SBI_LC2ST_MAX_F and 1 <= len(self.hidden) <= _lib.SBI_LC2ST_MAX_HIDDEN
                and all(1 <= h <= _lib.SBI_LC2ST_MAX_WIDTH for h in self.hidden)):
            raise NotImplementedError(
                f"LC2ST classifier with {self.F} inputs (dim_theta + dim_x) and hidden_layer_sizes={self.hidden}: "
                f"the device trainer supports at most {_lib.SBI_LC2ST_MAX_F} inputs and 1 to "
                f"{_lib.SBI_LC2ST_MAX_HIDDEN} hidden layers of at most {_lib.SBI_LC2ST_MAX_WIDTH} units")
        units = (self.F, *self.hidden, 1)
        self.shapes = [(units[i], units[i + 1]) for i in range(len(units) - 1)]
        self.P = sum(a * b + b for a, b in self.shapes)
        self.c = _lib.Lc2stNet(F=self.F, L=len(self.hidden), P=self.P)
        for i, h in enumerate(self.hidden):
            self.c.H[i] = h
        out = (C.c_int32 * 3)()
        rc = _lib.load().sbi_b200_lc2st_plan(C.byref(self.c), out)
        if rc == -2:
            raise NotImplementedError(
                f"LC2ST classifier with {self.F} inputs and hidden_layer_sizes={self.hidden} does not fit the "
                "shared memory of one CTA (its weights and gradient must fit 227 KB next to an 8-row tile)")
        _lib.check(rc, "lc2st_plan")
        self.key = (self.F, self.hidden)

    def pack(self, coefs: Sequence[np.ndarray], intercepts: Sequence[np.ndarray]) -> np.ndarray:
        parts = []
        for (a, b), W, bias in zip(self.shapes, coefs, intercepts):
            parts += [np.asarray(W, np.float32).reshape(a * b), np.asarray(bias, np.float32).reshape(b)]
        return np.concatenate(parts)

    def unpack(self, flat: np.ndarray) -> Tuple[List[np.ndarray], List[np.ndarray]]:
        coefs, intercepts, o = [], [], 0
        for a, b in self.shapes:
            coefs.append(flat[o:o + a * b].reshape(a, b).copy())
            o += a * b
            intercepts.append(flat[o:o + b].copy())
            o += b
        return coefs, intercepts

    def init_params(self, rs: np.random.RandomState) -> np.ndarray:
        """sklearn's `_init_coef` per layer in order: coefs then intercepts, uniform in +-sqrt(6 / (in + out))."""
        coefs, intercepts = [], []
        for a, b in self.shapes:
            bound = np.sqrt(6.0 / (a + b))
            coefs.append(rs.uniform(-bound, bound, (a, b)).astype(np.float32))
            intercepts.append(rs.uniform(-bound, bound, b).astype(np.float32))
        return self.pack(coefs, intercepts)


def _device(device: str) -> torch.device:
    if not torch.cuda.is_available():
        raise RuntimeError("sbi_b200: LC2ST trains and evaluates its classifiers on a CUDA (sm_90a) device and there "
                           "is no CPU fallback")
    try:
        d = torch.device(device)
    except (RuntimeError, TypeError):
        d = torch.device("cuda")
    return d if d.type == "cuda" else torch.device("cuda", torch.cuda.current_device())


class TrainedMLP:
    """A trained classifier with sklearn's fitted attributes (`coefs_`, `intercepts_`, `n_iter_`, `loss_curve_`,
    `validation_scores_`, `best_validation_score_`, `best_loss_`) and a `predict_proba` on the device."""

    activation = "relu"
    out_activation_ = "logistic"

    def __init__(self, net: _Net, flat: Tensor, n_iter: int = 0, loss_curve=None, validation_scores=None,
                 best_validation_score=None, best_loss=None, host: Optional[np.ndarray] = None):
        self._net, self._flat = net, flat
        self.coefs_, self.intercepts_ = net.unpack(flat.detach().cpu().numpy() if host is None else host)
        self.n_layers_ = len(self.coefs_) + 1
        self.n_outputs_ = 1
        self.classes_ = np.array([0, 1])
        self.n_iter_ = n_iter
        self.loss_curve_ = loss_curve
        self.validation_scores_ = validation_scores
        self.best_validation_score_ = best_validation_score
        self.best_loss_ = best_loss

    @property
    def members(self) -> List["TrainedMLP"]:
        return [self]

    def predict_proba(self, X) -> np.ndarray:
        X = torch.as_tensor(np.asarray(X, dtype=np.float32))
        prob0, _ = _evaluate([self], X.reshape(1, *X.shape), None, torch.zeros(0))
        return np.stack([prob0[0], 1.0 - prob0[0]], axis=1)


class TrainedEnsemble:
    """`num_ensemble` classifiers whose class probabilities are averaged (the reference's EnsembleClassifier)."""

    def __init__(self, trained_clfs: List[TrainedMLP]):
        self.trained_clfs = trained_clfs
        self.num_ensemble = len(trained_clfs)

    @property
    def members(self) -> List[TrainedMLP]:
        return self.trained_clfs

    def predict_proba(self, X) -> np.ndarray:
        X = torch.as_tensor(np.asarray(X, dtype=np.float32))
        prob0, _ = _evaluate([self], X.reshape(1, *X.shape), None, torch.zeros(0))
        return np.stack([prob0[0], 1.0 - prob0[0]], axis=1)


def _from_sklearn(clf: MLPClassifier, device: torch.device) -> TrainedMLP:
    if getattr(clf, "activation", None) != "relu" or getattr(clf, "out_activation_", None) != "logistic" \
            or list(getattr(clf, "classes_", [])) != [0, 1]:
        raise NotImplementedError("only fitted binary MLPClassifiers with activation='relu' (classes 0 and 1) can "
                                  "be evaluated by the device kernel")
    coefs = clf.coefs_
    net = _Net(coefs[0].shape[0], [c.shape[1] for c in coefs[:-1]])
    flat = torch.from_numpy(net.pack(coefs, clf.intercepts_)).to(device)
    return TrainedMLP(net, flat, n_iter=getattr(clf, "n_iter_", 0), loss_curve=getattr(clf, "loss_curve_", None),
                      validation_scores=getattr(clf, "validation_scores_", None),
                      best_validation_score=getattr(clf, "best_validation_score_", None),
                      best_loss=getattr(clf, "best_loss_", None))


def _as_classifier(clf, device: torch.device):
    """Our trained classifiers as they are; fitted sklearn MLPClassifiers (or an ensemble of them, an object with a
    `trained_clfs` list) packed for the device; anything else is a TypeError."""
    if isinstance(clf, (TrainedMLP, TrainedEnsemble)):
        return clf
    if isinstance(clf, MLPClassifier):
        return _from_sklearn(clf, device)
    members = getattr(clf, "trained_clfs", None)
    if isinstance(members, list) and members and all(isinstance(c, (MLPClassifier, TrainedMLP)) for c in members):
        return TrainedEnsemble([c if isinstance(c, TrainedMLP) else _from_sklearn(c, device) for c in members])
    raise TypeError(f"LC2ST classifiers must be classifiers trained by LC2ST or fitted sklearn MLPClassifiers, got "
                    f"{type(clf).__name__}.")


def _evaluate(clfs: Sequence, theta_blocks: Tensor, group: Optional[Sequence[int]], x_o: Tensor
              ) -> Tuple[np.ndarray, np.ndarray]:
    """Class-0 probabilities (len(clfs), S) and scores (len(clfs),) of classifiers on rows [theta_blocks[g], x_o],
    g = group[c] (0 when None): one `sbi_b200_lc2st_eval` launch per architecture and ensemble size involved
    (one launch in every LC2ST workflow)."""
    G, S, dt = theta_blocks.shape
    x_o = x_o.reshape(-1)
    groups: Dict[tuple, List[int]] = {}
    for i, c in enumerate(clfs):
        m = c.members
        groups.setdefault((m[0]._net.key, len(m)), []).append(i)
    probs = np.empty((len(clfs), S), np.float32)
    scores = np.empty(len(clfs), np.float64)
    lib = _lib.load()
    for (_, E), idx in groups.items():
        net = clfs[idx[0]].members[0]._net
        if net.F != dt + x_o.numel():
            raise ValueError(f"classifier expects {net.F} features, got {dt + x_o.numel()}")
        members = [m for i in idx for m in clfs[i].members]
        if any(m._net.key != net.key for m in members):
            raise ValueError("the members of an ensemble must share one architecture")
        dev = members[0]._flat.device
        params = torch.stack([m._flat for m in members]).contiguous()
        th = theta_blocks.to(dev, torch.float32).contiguous()
        xo = x_o.to(dev, torch.float32).contiguous()
        g = None if group is None else torch.tensor([group[i] for i in idx], dtype=torch.int32, device=dev)
        nchunk = lib.sbi_b200_lc2st_eval_chunks(C.byref(net.c), S)
        _lib.check(nchunk if nchunk < 0 else 0, "lc2st_eval_chunks")
        n = len(idx)
        prob = torch.empty(n, S, dtype=torch.float32, device=dev)
        part = torch.empty(n, nchunk, dtype=torch.float64, device=dev)
        score = torch.empty(n, dtype=torch.float64, device=dev)
        _lib.call("lc2st_eval", net.c, params, n, E, th if dt else None, dt, S, g, xo if xo.numel() else None,
                  xo.numel(), prob, part, score)
        probs[idx] = prob.cpu().numpy()
        scores[idx] = score.cpu().numpy()
    return probs, scores


@dataclass
class _Model:
    """One classifier to fit: its samples (pairs of theta-table and x-table rows) with labels, and its
    random_state (sklearn's `check_random_state` argument)."""

    rows: np.ndarray     # (n, 2) int32
    labels: np.ndarray   # (n,) float32
    random_state: Any


def _clf_settings(kw: Dict[str, Any]) -> Dict[str, Any]:
    """sklearn's defaults under the caller's kwargs, after checking that the trainer implements them."""
    bad = [k for k in kw if k not in SUPPORTED_KWARGS and k not in _FIXED_KWARGS]
    for k, v in _FIXED_KWARGS.items():
        if k in kw and kw[k] != v:
            bad.append(f"{k}={kw[k]!r}")
    if bad:
        raise NotImplementedError(
            f"LC2ST's device trainer does not support the MLPClassifier arguments {sorted(map(str, bad))}; it "
            f"supports activation='relu', solver='adam' and {sorted(SUPPORTED_KWARGS)}")
    s = {**SUPPORTED_KWARGS, **{k: v for k, v in kw.items() if k in SUPPORTED_KWARGS}}
    h = s["hidden_layer_sizes"]
    s["hidden_layer_sizes"] = list(h) if hasattr(h, "__iter__") else [h]
    if any(int(v) <= 0 for v in s["hidden_layer_sizes"]):
        raise ValueError(f"hidden_layer_sizes must be > 0, got {s['hidden_layer_sizes']}.")
    if int(s["max_iter"]) < 1:
        raise ValueError(f"max_iter must be >= 1, got {s['max_iter']}.")
    if int(s["n_iter_no_change"]) < 1:   # as sklearn's parameter validation
        raise ValueError(f"n_iter_no_change must be >= 1, got {s['n_iter_no_change']}.")
    return s


def prepare_model(net: _Net, mdl: _Model, s: Dict[str, Any]) -> Tuple[np.ndarray, np.ndarray, int, int]:
    """What sklearn draws on the host for one fit, from `check_random_state(random_state)` in its order: the
    initial parameters, then (early stopping) the stratified validation split; then the device shuffle key.
    Returns (packed initial parameters, sample order: training then validation samples, n_train, key)."""
    rs = check_random_state(mdl.random_state)
    init = net.init_params(rs)
    idx = np.arange(len(mdl.labels))
    n_train = len(idx)
    if s["early_stopping"]:
        yb = (mdl.labels == 1).reshape(-1, 1)   # sklearn stratifies on the binarized (n, 1) labels
        tr, va = train_test_split(idx, yb, random_state=rs, test_size=s["validation_fraction"], stratify=yb)[:2]
        if va.shape[0] < 2:
            raise ValueError("The validation set is too small. Increase 'validation_fraction' or the size of "
                             "your dataset.")
        idx, n_train = np.concatenate([tr, va]), len(tr)
    key = int(rs.randint(0, np.iinfo(np.int64).max, dtype=np.int64))
    return init, idx, n_train, key


def train_classifiers(theta_table: Tensor, x_table: Tensor, models: List[_Model], clf_kwargs: Dict[str, Any],
                      device: torch.device, epoch_orders: Optional[List[np.ndarray]] = None) -> List[TrainedMLP]:
    """Fit every model in one `sbi_b200_lc2st_train` launch.  `epoch_orders[m]` (max_iter, n_train), if given,
    replaces the device shuffle of model m by the caller's per-epoch orders of its training samples."""
    s = _clf_settings(clf_kwargs)
    dt, dx = theta_table.shape[1], x_table.shape[1]
    net = _Net(dt + dx, s["hidden_layer_sizes"])
    max_iter, early = int(s["max_iter"]), bool(s["early_stopping"])
    M = len(models)
    init = np.empty((M, net.P), np.float32)
    rows, labels, orders = [], [], []
    jobs = (_lib.Lc2stJob * max(M, 1))()
    row0, order0 = 0, 0
    for i, mdl in enumerate(models):
        init[i], idx, n_train, key = prepare_model(net, mdl, s)
        n = len(idx)
        if s["batch_size"] != "auto" and not 1 <= s["batch_size"] <= n_train:
            warnings.warn("Got `batch_size` less than 1 or larger than sample size. It is going to be clipped")
        rows.append(mdl.rows[idx])
        labels.append(mdl.labels[idx])
        jobs[i].row0, jobs[i].n_train, jobs[i].n_val, jobs[i].key = row0, n_train, n - n_train, key
        jobs[i].order0 = -1
        if epoch_orders is not None:
            o = np.asarray(epoch_orders[i], np.int32)
            assert o.shape == (max_iter, n_train), (o.shape, max_iter, n_train)
            orders.append(o.reshape(-1))
            jobs[i].order0 = order0
            order0 += o.size
        row0 += n
    opt = _lib.Lc2stOpt(
        max_iter=max_iter, n_iter_no_change=int(s["n_iter_no_change"]), early_stopping=int(early),
        shuffle=int(bool(s["shuffle"])),
        # sklearn's "auto" is min(200, n_train); an explicit size is clipped to [1, n_train] per model on the device
        batch_size=0 if s["batch_size"] == "auto" else max(1, int(s["batch_size"])),
        beta1=np.float32(s["beta_1"]), beta2=np.float32(s["beta_2"]), one_minus_beta1=np.float32(1 - s["beta_1"]),
        one_minus_beta2=np.float32(1 - s["beta_2"]), eps=np.float32(s["epsilon"]), alpha=np.float32(s["alpha"]),
        lr_d=float(s["learning_rate_init"]), beta1_d=float(s["beta_1"]), beta2_d=float(s["beta_2"]),
        tol=float(s["tol"]))
    lib = _lib.load()
    th = theta_table.to(device, torch.float32).contiguous()
    xt = x_table.to(device, torch.float32).contiguous()
    d_rows = torch.from_numpy(np.concatenate(rows).astype(np.int32)).to(device)
    d_lab = torch.from_numpy(np.concatenate(labels).astype(np.float32)).to(device)
    d_jobs = torch.frombuffer(bytearray(jobs), dtype=torch.uint8).to(device)
    d_order = torch.from_numpy(np.concatenate(orders)).to(device) if orders else None
    params = torch.from_numpy(init).to(device)
    ws = torch.empty(lib.sbi_b200_lc2st_ws_floats(C.byref(net.c), M), dtype=torch.float32, device=device)
    n_iter = torch.empty(M, dtype=torch.int32, device=device)
    val_curve = torch.zeros(M, max_iter, dtype=torch.float64, device=device)
    loss_curve = torch.zeros(M, max_iter, dtype=torch.float64, device=device)
    best = torch.empty(M, dtype=torch.float64, device=device)
    _lib.call("lc2st_train", net.c, opt, d_jobs, M, th if dt else None, dt, xt if dx else None, dx, d_rows, d_lab,
              d_order, params, ws, n_iter, val_curve, loss_curve, best)
    n_iter_h, params_h = n_iter.cpu().numpy(), params.cpu().numpy()
    val_h, loss_h, best_h = val_curve.cpu().numpy(), loss_curve.cpu().numpy(), best.cpu().numpy()
    out = []
    for i in range(M):
        k = int(n_iter_h[i])
        out.append(TrainedMLP(net, params[i], n_iter=k, loss_curve=[float(v) for v in loss_h[i, :k]],
                              validation_scores=[float(v) for v in val_h[i, :k]] if early else None,
                              best_validation_score=float(best_h[i]) if early else None,
                              best_loss=None if early else float(best_h[i]), host=params_h[i]))
    hit = int((n_iter_h == max_iter).sum())
    if hit:
        warnings.warn(f"Stochastic Optimizer: Maximum iterations ({max_iter}) reached and the optimization hasn't "
                      f"converged yet ({hit} of {M} classifiers).", ConvergenceWarning, stacklevel=3)
    return out


def permutation_indices(n: int, t: int) -> Tensor:
    """The reference's `permute_data(seed=t)` permutation of the 2n joint rows, from a local generator."""
    return torch.randperm(2 * n, generator=torch.Generator().manual_seed(t))


# ---------------------------------------------------------------------------------------------------------------
class LC2ST:
    r"""L-C2ST: Local Classifier Two-Sample Test (Linhart et al. 2023), with the reference's interface; see the
    module docstring for how the classifiers are trained and where the run differs from the reference."""

    def __init__(
        self,
        prior_samples: Optional[Tensor] = None,
        xs: Optional[Tensor] = None,
        posterior_samples: Optional[Tensor] = None,
        seed: int = 1,
        num_folds: int = 1,
        num_ensemble: int = 1,
        classifier: Union[str, Type[BaseEstimator]] = MLPClassifier,
        z_score: bool = False,
        classifier_kwargs: Optional[Dict[str, Any]] = None,
        num_trials_null: int = 100,
        permutation: bool = True,
        device: str = "cpu",
        *,
        thetas: Optional[Tensor] = None,
    ) -> None:
        if thetas is not None:
            warnings.warn(
                "Parameter 'thetas' is deprecated and will be removed in a future "
                "version. Use 'prior_samples' instead.",
                FutureWarning,
                stacklevel=2,
            )
            if prior_samples is not None:
                raise ValueError("Cannot specify both 'thetas' and 'prior_samples'. Use 'prior_samples' only.")
            prior_samples = thetas
        if prior_samples is None:
            raise ValueError("prior_samples is required.")
        if xs is None:
            raise ValueError("xs is required.")
        if posterior_samples is None:
            raise ValueError("posterior_samples is required.")

        self._validate_inputs(prior_samples, xs, posterior_samples, num_folds, seed)
        xf = xs.reshape(xs.shape[0], -1)
        x_is_nan, x_is_inf = torch.isnan(xf).any(dim=1), torch.isinf(xf).any(dim=1)
        num_nans, num_infs = int(x_is_nan.sum().item()), int(x_is_inf.sum().item())
        is_valid_x = ~x_is_nan & ~x_is_inf
        if num_nans > 0 or num_infs > 0:
            warnings.warn(
                f"Found {num_nans} NaNs and {num_infs} Infs in xs. "
                f"These rows will be removed from all input tensors. "
                f"Only {is_valid_x.sum()} / {len(xs)} samples remain.",
                stacklevel=2,
            )
        prior_samples = prior_samples[is_valid_x.to(prior_samples.device)]
        xs = xs[is_valid_x]
        posterior_samples = posterior_samples[is_valid_x.to(posterior_samples.device)]
        self._validate_inputs(prior_samples, xs, posterior_samples, num_folds, seed)

        self.theta_p = posterior_samples
        self.x_p = xs
        self.theta_q = prior_samples
        self.x_q = xs
        self.z_score = z_score
        self._setup_normalization()

        self._base_seed = seed
        self.seed = seed
        self.num_folds = num_folds
        self.num_ensemble = num_ensemble
        self.device = device

        self.clf_class = self._resolve_classifier(classifier)
        self.clf_kwargs = self._get_classifier_kwargs(classifier_kwargs, prior_samples.shape[-1])
        _clf_settings(self.clf_kwargs)

        self._state = LC2STState.INITIALIZED
        self.trained_clfs: Optional[List[Any]] = None
        self.trained_clfs_null: Optional[Dict[int, List[Any]]] = None
        self.num_trials_null = num_trials_null
        self.permutation = permutation
        self.null_distribution: Optional[torch.distributions.Distribution] = None

    def _validate_inputs(self, prior_samples: Tensor, xs: Tensor, posterior_samples: Tensor, num_folds: int,
                         seed: int) -> None:
        if not isinstance(prior_samples, Tensor):
            raise TypeError(f"prior_samples must be a torch.Tensor, got {type(prior_samples)}.")
        if not isinstance(xs, Tensor):
            raise TypeError(f"xs must be a torch.Tensor, got {type(xs)}.")
        if not isinstance(posterior_samples, Tensor):
            raise TypeError(f"posterior_samples must be a torch.Tensor, got {type(posterior_samples)}.")
        if prior_samples.shape[0] == 0:
            raise ValueError("prior_samples cannot be empty.")
        if xs.shape[0] == 0:
            raise ValueError("xs cannot be empty.")
        if posterior_samples.shape[0] == 0:
            raise ValueError("posterior_samples cannot be empty.")
        if not (prior_samples.shape[0] == xs.shape[0] == posterior_samples.shape[0]):
            raise ValueError(
                f"Sample size mismatch: prior_samples has {prior_samples.shape[0]}, "
                f"xs has {xs.shape[0]}, posterior_samples has "
                f"{posterior_samples.shape[0]}. All must have the same number "
                f"of samples."
            )
        if prior_samples.shape[-1] != posterior_samples.shape[-1]:
            raise ValueError(
                f"Dimension mismatch: prior_samples has dimension "
                f"{prior_samples.shape[-1]}, but posterior_samples has dimension "
                f"{posterior_samples.shape[-1]}."
            )
        if num_folds < 1:
            raise ValueError(f"num_folds must be >= 1, got {num_folds}.")
        if num_folds > prior_samples.shape[0]:
            raise ValueError(f"num_folds ({num_folds}) cannot exceed sample size ({prior_samples.shape[0]}).")
        if not isinstance(seed, int):
            raise TypeError(f"seed must be an integer, got {type(seed)}.")

    def _setup_normalization(self) -> None:
        """z-score statistics of P; constant dimensions keep std 1 (mean-centering only)."""
        self.theta_p_mean = torch.mean(self.theta_p, dim=0)
        theta_std = torch.std(self.theta_p, dim=0)
        self.theta_p_std = theta_std.masked_fill(theta_std == 0, 1.0)
        self.x_p_mean = torch.mean(self.x_p, dim=0)
        x_std = torch.std(self.x_p, dim=0)
        self.x_p_std = x_std.masked_fill(x_std == 0, 1.0)

    def _resolve_classifier(self, classifier: Union[str, Type[BaseEstimator]]) -> Type[BaseEstimator]:
        supported = ('supported: classifier=MLPClassifier or "mlp" (scikit-learn\'s MLPClassifier algorithm, trained '
                     'on the device)')
        if isinstance(classifier, str):
            if classifier.lower() == "mlp":
                return MLPClassifier
            if classifier.lower() == "random_forest":
                raise NotImplementedError(f'classifier="random_forest" is not implemented; {supported}.')
            raise ValueError(
                f'Invalid classifier: "{classifier}". '
                'Expected "mlp", "random_forest", '
                "or a valid scikit-learn classifier class."
            )
        if not (isinstance(classifier, type) and issubclass(classifier, BaseEstimator)):
            raise TypeError(
                f"classifier must be a string or a subclass of BaseEstimator, got {type(classifier).__name__}."
            )
        if classifier is not MLPClassifier:
            raise NotImplementedError(f"classifier={classifier.__name__} is not implemented; {supported}.")
        return classifier

    def _get_classifier_kwargs(self, classifier_kwargs: Optional[Dict[str, Any]], ndim: int) -> Dict[str, Any]:
        hidden_size = DEFAULT_MLP_HIDDEN_LAYER_MULTIPLIER * ndim
        defaults = {
            "activation": DEFAULT_MLP_ACTIVATION,
            "hidden_layer_sizes": (hidden_size, hidden_size),
            "max_iter": DEFAULT_MLP_MAX_ITER,
            "solver": DEFAULT_MLP_SOLVER,
            "early_stopping": DEFAULT_MLP_EARLY_STOPPING,
            "n_iter_no_change": DEFAULT_MLP_N_ITER_NO_CHANGE,
        }
        if classifier_kwargs is not None:
            defaults.update(classifier_kwargs)
        return defaults

    # The statistics follow the samples to their device: a flow's `inverse_transform` may return device tensors
    # next to host `xs`, host base-distribution draws and host `theta_o`.
    def _normalize_theta(self, theta: Tensor) -> Tensor:
        if self.z_score:
            return (theta - self.theta_p_mean.to(theta.device)) / self.theta_p_std.to(theta.device)
        return theta

    def _normalize_x(self, x: Tensor) -> Tensor:
        if self.z_score:
            return (x - self.x_p_mean.to(x.device)) / self.x_p_std.to(x.device)
        return x

    def _host(self, t: Tensor) -> Tensor:
        return t.detach().to("cpu", torch.float32)

    @property
    def state(self) -> LC2STState:
        return self._state

    # -- training ------------------------------------------------------------------------------------------------
    def _member_states(self) -> List[Any]:
        """EnsembleClassifier's rule: member n gets random_state + n, or n + 1 when random_state is None."""
        rs = self.clf_kwargs.get("random_state")
        if self.num_ensemble <= 1:
            return [rs]
        return [(rs + n) if rs is not None else n + 1 for n in range(self.num_ensemble)]

    def _fold_indices(self) -> List[np.ndarray]:
        n = self.theta_p.shape[0]
        if self.num_folds > 1:
            kf = KFold(n_splits=self.num_folds, shuffle=True, random_state=self.seed)
            return [train_idx for train_idx, _ in kf.split(np.zeros((n, 1)))]
        return [np.arange(n)]

    def _train_blocks(self, blocks: List[Tuple[np.ndarray, np.ndarray]], theta_table: Tensor) -> List[Any]:
        """Train one classifier (or ensemble) per (block, fold) in one launch.  A block gives the (theta row, x row)
        pairs of P's and of Q's samples; returns per block the list over folds."""
        folds = self._fold_indices()
        states = self._member_states()
        models = []
        for p_rows, q_rows in blocks:
            for tr in folds:
                pairs = np.concatenate([p_rows[tr], q_rows[tr]]).astype(np.int32)
                lab = np.concatenate([np.zeros(len(tr), np.float32), np.ones(len(tr), np.float32)])
                models += [_Model(pairs, lab, st) for st in states]
        x_table = self._host(self._normalize_x(self.x_p))
        fitted = train_classifiers(theta_table, x_table, models, self.clf_kwargs, _device(self.device))
        E, out, k = len(states), [], 0
        for _ in blocks:
            per_fold = []
            for _ in folds:
                mem = fitted[k:k + E]
                k += E
                per_fold.append(TrainedEnsemble(mem) if self.num_ensemble > 1 else mem[0])
            out.append(per_fold)
        return out

    def _observed_table(self) -> Tensor:
        return torch.cat([self._host(self._normalize_theta(self.theta_p)), self._host(self._normalize_theta(self.theta_q))])

    def train_on_observed_data(self, seed: Optional[int] = None, verbosity: int = 1) -> "LC2ST":
        """Trains the classifier(s) on the observed data (one per fold)."""
        if seed is not None:
            if "random_state" in self.clf_kwargs:
                warnings.warn(
                    "Overwriting 'random_state' in classifier_kwargs because "
                    "a 'seed' was provided to train_on_observed_data().",
                    UserWarning,
                    stacklevel=2,
                )
            self.clf_kwargs["random_state"] = seed
        n = self.theta_p.shape[0]
        i = np.arange(n)
        self.trained_clfs = self._train_blocks([(np.stack([i, i], 1), np.stack([n + i, i], 1))],
                                               self._observed_table())[0]
        if self._state in (LC2STState.NULL_TRAINED, LC2STState.READY):
            self._state = LC2STState.READY
        else:
            self._state = LC2STState.OBSERVED_TRAINED
        return self

    def train_under_null_hypothesis(self, verbosity: int = 1) -> "LC2ST":
        """Trains the classifiers of every null trial, all in one launch."""
        if self.trained_clfs_null is not None:
            raise ValueError(
                "Classifiers under the null hypothesis are already trained. "
                "To retrain, create a new instance or reset `trained_clfs_null` "
                "explicitly. Note that for LC2ST_NF the null classifiers are "
                "data-independent and can be reused with new estimators."
            )
        n = self.theta_p.shape[0]
        blocks = []
        if self.permutation:
            table = self._observed_table()
            for t in range(self.num_trials_null):
                perm = permutation_indices(n, t).numpy()
                pairs = np.stack([perm, perm % n], 1)
                blocks.append((pairs[:n], pairs[n:]))
        else:
            if self.null_distribution is None:
                raise ValueError(
                    "A null distribution must be provided when permutation=False. "
                    "Set null_distribution or use permutation=True."
                )
            parts, i = [], np.arange(n)
            for t in range(self.num_trials_null):
                theta_p_t = self.null_distribution.sample((n,))
                theta_q_t = self.null_distribution.sample((n,))
                parts += [self._host(self._normalize_theta(theta_p_t)), self._host(self._normalize_theta(theta_q_t))]
                blocks.append((np.stack([2 * n * t + i, i], 1), np.stack([2 * n * t + n + i, i], 1)))
            table = torch.cat(parts).to(torch.float32) if parts else torch.zeros(0, self.theta_p.shape[1])
        trained = self._train_blocks(blocks, table) if blocks else []
        self.trained_clfs_null = {t: clfs for t, clfs in enumerate(trained)}
        if self._state == LC2STState.OBSERVED_TRAINED:
            self._state = LC2STState.READY
        elif self._state == LC2STState.INITIALIZED:
            self._state = LC2STState.NULL_TRAINED
        return self

    # -- statistics ----------------------------------------------------------------------------------------------
    def _prepare_eval(self, theta_o: Tensor, x_o: Tensor) -> Tuple[Tensor, Tensor]:
        if x_o.shape == self.x_p_mean.shape:
            x_o = x_o.unsqueeze(0)
        return self._host(self._normalize_theta(theta_o)), self._host(self._normalize_x(x_o))

    def _null_thetas(self, theta_o: Tensor) -> List[Tensor]:
        """Per trial: theta_o (permutation) or a fresh draw from the null distribution, in the reference's order."""
        if self.permutation:
            return [theta_o] * self.num_trials_null
        if self.null_distribution is None:
            raise ValueError("A null distribution must be provided when permutation=False.")
        return [self.null_distribution.sample((theta_o.shape[0],)) for _ in range(self.num_trials_null)]

    def _scores(self, theta_o: Tensor, x_o: Tensor, observed: Optional[List[Any]], null_thetas: Optional[List[Tensor]]
                ) -> Tuple[Optional[Tuple[np.ndarray, np.ndarray]], Optional[Tuple[np.ndarray, np.ndarray]]]:
        """Probabilities and scores of the observed classifiers on theta_o and of every null trial's classifiers on
        its theta, from one batched evaluation."""
        dev = _device(self.device)
        observed = [_as_classifier(c, dev) for c in observed] if observed is not None else []
        blocks = [theta_o] if observed else []
        clfs, group = list(observed), [0] * len(observed)
        null = []
        if null_thetas is not None:
            shared = self.permutation
            if shared and not blocks:
                blocks = [theta_o]
            for t in range(self.num_trials_null):
                cl = [_as_classifier(c, dev) for c in self.trained_clfs_null[t]]
                if not shared:
                    blocks.append(null_thetas[t])
                null.append(len(cl))
                clfs += cl
                group += [0 if shared else len(blocks) - 1] * len(cl)
        xo = self._prepare_eval(theta_o, x_o)[1]
        tb = torch.stack([self._host(self._normalize_theta(b)) for b in blocks])
        probs, scores = _evaluate(clfs, tb, group, xo)
        k = len(observed)
        obs = (probs[:k], scores[:k]) if observed else None
        if null_thetas is None:
            return obs, None
        P, Sc, o = [], [], k
        for c in null:
            P.append(probs[o:o + c])
            Sc.append(scores[o:o + c].mean())
            o += c
        return obs, (np.array(P), np.array(Sc))

    def get_scores(self, theta_o: Tensor, x_o: Tensor, trained_clfs: List[Any], return_probs: bool = False
                   ) -> Union[LC2STScores, Tuple[np.ndarray, np.ndarray]]:
        """L-C2ST scores (mean squared distance of the class-0 probability to 1/2 over (theta_o, x_o)) of the given
        classifiers, all evaluated in one launch."""
        (probs_arr, scores_arr), _ = self._scores(theta_o, x_o, list(trained_clfs), None)
        if return_probs:
            warnings.warn(
                "The 'return_probs' parameter is deprecated and will be "
                "removed in a future release. It returns a (probs, scores) "
                "tuple; use LC2STScores.probabilities and LC2STScores.scores "
                "from the default return value instead.",
                FutureWarning,
                stacklevel=2,
            )
            return probs_arr, scores_arr
        return LC2STScores(scores=scores_arr, probabilities=probs_arr)

    def _require_observed(self):
        if self._state not in (LC2STState.OBSERVED_TRAINED, LC2STState.READY):
            raise RuntimeError(
                "Classifiers have not been trained on observed data. "
                "Call train_on_observed_data() before computing statistics."
            )

    def _require_null(self):
        if self._state not in (LC2STState.NULL_TRAINED, LC2STState.READY):
            raise RuntimeError(
                "Classifiers have not been trained under the null hypothesis. "
                "Call train_under_null_hypothesis() first."
            )
        if self.trained_clfs_null is None or len(self.trained_clfs_null) != self.num_trials_null:
            raise RuntimeError(
                f"Expected {self.num_trials_null} null classifiers, "
                f"got {len(self.trained_clfs_null) if self.trained_clfs_null else 0}."
            )

    def get_statistic_on_observed_data(self, theta_o: Tensor, x_o: Tensor) -> float:
        """The L-C2ST statistic at x_o: the mean over the folds' scores."""
        self._require_observed()
        result = self.get_scores(theta_o=theta_o, x_o=x_o, trained_clfs=self.trained_clfs)
        return float(result.scores.mean())

    def p_value(self, theta_o: Tensor, x_o: Tensor) -> float:
        r"""$1/H \sum_h I(T_h > T_o)$ over the null trials; observed and null classifiers in one evaluation."""
        if self._state != LC2STState.READY:
            missing = []
            if self._state in (LC2STState.INITIALIZED, LC2STState.NULL_TRAINED):
                missing.append("train_on_observed_data()")
            if self._state in (LC2STState.INITIALIZED, LC2STState.OBSERVED_TRAINED):
                missing.append("train_under_null_hypothesis()")
            raise RuntimeError(f"LC2ST is not ready to compute p-values. Call {' and '.join(missing)} first.")
        self._require_observed()
        self._require_null()
        obs, null = self._scores(theta_o, x_o, self.trained_clfs, self._null_thetas(theta_o))
        stat_data = float(obs[1].mean())
        return float((stat_data < null[1]).mean())

    def reject_test(self, theta_o: Tensor, x_o: Tensor, alpha: float = 0.05) -> bool:
        """True if H0 is rejected at level alpha."""
        return bool(self.p_value(theta_o=theta_o, x_o=x_o) < alpha)

    def get_statistics_under_null_hypothesis(self, theta_o: Tensor, x_o: Tensor, return_probs: bool = False,
                                             verbosity: int = 0
                                             ) -> Union[LC2STScores, Tuple[np.ndarray, np.ndarray]]:
        """Per null trial: the mean over its folds' scores, all trials in one evaluation."""
        self._require_null()
        _, (probs_null_arr, stats_null_arr) = self._scores(theta_o, x_o, None, self._null_thetas(theta_o))
        if return_probs:
            warnings.warn(
                "The 'return_probs' parameter is deprecated and will be "
                "removed in a future release. It returns a (probs, scores) "
                "tuple; use LC2STScores.probabilities and LC2STScores.scores "
                "from the default return value instead.",
                FutureWarning,
                stacklevel=2,
            )
            return probs_null_arr, stats_null_arr
        return LC2STScores(scores=stats_null_arr, probabilities=probs_null_arr)


class LC2ST_NF(LC2ST):
    r"""L-C2ST in the base space of a normalizing flow: samples are mapped through `flow_inverse_transform`, the null
    is the base distribution (no permutation), `theta_o` is drawn once at construction, and null classifiers can be
    passed in pre-trained (ours, or fitted sklearn ReLU MLPClassifiers)."""

    def __init__(
        self,
        prior_samples: Optional[Tensor] = None,
        xs: Optional[Tensor] = None,
        posterior_samples: Optional[Tensor] = None,
        flow_inverse_transform: Optional[Callable[[Tensor, Tensor], Tensor]] = None,
        flow_base_dist: Optional[torch.distributions.Distribution] = None,
        num_eval: int = 10_000,
        trained_clfs_null: Optional[Dict[int, List[Any]]] = None,
        *,
        thetas: Optional[Tensor] = None,
        **kwargs: Any,
    ) -> None:
        if thetas is not None:
            warnings.warn(
                "Parameter 'thetas' is deprecated and will be removed in a future "
                "version. Use 'prior_samples' instead.",
                FutureWarning,
                stacklevel=2,
            )
            if prior_samples is not None:
                raise ValueError("Cannot specify both 'thetas' and 'prior_samples'. Use 'prior_samples' only.")
            prior_samples = thetas
        if prior_samples is None:
            raise ValueError("prior_samples is required.")
        if xs is None:
            raise ValueError("xs is required.")
        if posterior_samples is None:
            raise ValueError("posterior_samples is required.")
        if flow_inverse_transform is None:
            raise ValueError("flow_inverse_transform is required.")
        if flow_base_dist is None:
            raise ValueError("flow_base_dist is required.")

        self.flow_inverse_transform = flow_inverse_transform
        inverse_prior_samples = flow_inverse_transform(prior_samples, xs).detach()
        inverse_posterior_samples = flow_inverse_transform(posterior_samples, xs).detach()
        super().__init__(prior_samples=inverse_prior_samples, xs=xs, posterior_samples=inverse_posterior_samples,
                         **kwargs)
        self.null_distribution = flow_base_dist
        self.permutation = False
        if trained_clfs_null is not None:
            dev = _device(self.device)
            trained_clfs_null = {t: [_as_classifier(c, dev) for c in clfs] for t, clfs in trained_clfs_null.items()}
        self.trained_clfs_null = trained_clfs_null
        if trained_clfs_null is not None:
            self._state = LC2STState.NULL_TRAINED
        self.theta_o = flow_base_dist.sample(torch.Size([num_eval]))

    def get_scores(self, x_o: Tensor, trained_clfs: List[Any], return_probs: bool = False, **kwargs: Any
                   ) -> Union[LC2STScores, Tuple[np.ndarray, np.ndarray]]:
        return super().get_scores(theta_o=self.theta_o, x_o=x_o, trained_clfs=trained_clfs, return_probs=return_probs)

    def get_statistic_on_observed_data(self, x_o: Tensor, **kwargs: Any) -> float:
        return super().get_statistic_on_observed_data(theta_o=self.theta_o, x_o=x_o)

    def p_value(self, x_o: Tensor, **kwargs: Any) -> float:
        return super().p_value(theta_o=self.theta_o, x_o=x_o)

    def reject_test(self, x_o: Tensor, alpha: float = 0.05, **kwargs: Any) -> bool:
        return super().reject_test(theta_o=self.theta_o, x_o=x_o, alpha=alpha)

    def train_under_null_hypothesis(self, verbosity: int = 1) -> "LC2ST_NF":
        if self.trained_clfs_null is not None:
            raise ValueError(
                "Classifiers under the null hypothesis are already trained. "
                "To retrain, create a new instance or reset `trained_clfs_null` "
                "explicitly. Note that for LC2ST_NF the null classifiers are "
                "data-independent and can be reused with new estimators."
            )
        super().train_under_null_hypothesis(verbosity=verbosity)
        return self

    def get_statistics_under_null_hypothesis(self, x_o: Tensor, return_probs: bool = False, verbosity: int = 0,
                                             **kwargs: Any) -> Union[LC2STScores, Tuple[np.ndarray, np.ndarray]]:
        return super().get_statistics_under_null_hypothesis(theta_o=self.theta_o, x_o=x_o, return_probs=return_probs,
                                                            verbosity=verbosity)
