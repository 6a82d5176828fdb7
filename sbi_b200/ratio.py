"""Ratio estimator (NRE) at sbi's estimator boundary, backed by the sm_90a kernels.

`RatioEstimator` mirrors /root/reference/sbi/neural_nets/ratio_estimators.py:11-157 for the
`linear`, `mlp` and `resnet` classifiers of /root/reference/sbi/neural_nets/net_builders/classifier.py:
`forward(theta, x)` / `unnormalized_log_ratio` return logits of shape `(*batch_shape)` for
equally-prefixed `theta` and `x` (no broadcasting, same error), `state_dict()` uses the
reference's keys.  `classifier_nn` / `build_*_classifier` mirror factory.py:174-241.  The layout
selects the kernels: `RatioLayout` (resnet) csrc/ratio.cu and csrc/ratio_tc.cu, `MlpRatioLayout`
(mlp, linear) csrc/ratio_mlp.cu.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings
from typing import Any, Callable, Optional, Union

import torch
from torch import Tensor, nn
from torch.nn import init

from . import _lib as L
from .estimators import PackedNet, Standardize, _PackedEstimator, _zscore_of
from .neural_nets import _linear_init, check_data_device, standardizing_stats, z_score_parser
from .pack import MlpRatioLayout, RatioLayout


class RatioEstimator(_PackedEstimator):
    r"""log r(theta, x) = classifier logit; trained by NRE (ratio_estimators.py:11-157).

    Each side (theta, x) has its own embedding net.  An identity side hands its raw rows to the kernels, which
    z-score them in-kernel; an embedded side runs `Standardize` + the user's module in torch and the kernels read
    the embedded rows with identity statistics (`resnet` classifier only)."""

    def __init__(self, layout: Union[RatioLayout, MlpRatioLayout], theta_shape, x_shape, theta_stats, x_stats,
                 embedding_net_theta: nn.Module = None, embedding_net_x: nn.Module = None):
        super().__init__()
        self._input_shape = torch.Size(theta_shape)
        self._condition_shape = torch.Size(x_shape)
        self.theta_shape, self.x_shape = self._input_shape, self._condition_shape
        et = embedding_net_theta if embedding_net_theta is not None else nn.Identity()
        ex = embedding_net_x if embedding_net_x is not None else nn.Identity()
        self._embed_theta_identity = isinstance(et, nn.Identity)
        self._embed_x_identity = isinstance(ex, nn.Identity)
        if not (self._embed_theta_identity and self._embed_x_identity) and not isinstance(layout, RatioLayout):
            raise NotImplementedError("the sm_90a mlp / linear classifier kernels take nn.Identity() embedding nets "
                                      "(embedding nets are implemented for the resnet classifier)")
        self.embedding_net_theta = nn.Sequential(Standardize(*theta_stats), et) if theta_stats else et
        self.embedding_net_x = nn.Sequential(Standardize(*x_stats), ex) if x_stats else ex
        # sits where the reference keeps its ResidualNet / nn.Sequential
        self.net = PackedNet(layout)
        self.net.hidden_features = layout.H
        self._cache = {}

    @property
    def embedding_nets(self) -> list:
        """The embedding nets that run in torch ahead of the kernels (the non-identity sides)."""
        return [e for e, ident in ((self.embedding_net_theta, self._embed_theta_identity),
                                   (self.embedding_net_x, self._embed_x_identity)) if not ident]

    # ---- kernel views: [theta mean (Dtp) | theta std (Dtp) | x mean (Dxp) | x std (Dxp)]
    def _stat_widths(self):
        lay = self.layout
        return lay.Dtp, lay.Dt, lay.Dxp, lay.Dx, 0

    def _stat_sources(self, raw_condition: bool):
        th = _zscore_of(self.embedding_net_theta) if self._embed_theta_identity else None
        xx = _zscore_of(self.embedding_net_x) if self._embed_x_identity else None
        return th, xx, None

    def embed_theta(self, theta: Tensor) -> Tensor:
        """(N, *theta_shape) -> the (N, Dt) rows the kernels read: raw (z-scored in-kernel) for an identity
        embedding, else Standardize + the embedding net in torch."""
        n = theta.shape[0]
        if self._embed_theta_identity:
            return theta.reshape(n, -1).contiguous().float()
        return self.embedding_net_theta(theta).reshape(n, -1).contiguous().float()

    def embed_x(self, x: Tensor) -> Tensor:
        """(N, *x_shape) -> the (N, Dx) rows the kernels read (see `embed_theta`)."""
        n = x.shape[0]
        if self._embed_x_identity:
            return x.reshape(n, -1).contiguous().float()
        return self.embedding_net_x(x).reshape(n, -1).contiguous().float()

    # ---- shape checks: ratio_estimators.py:53-112
    def _check(self, theta: Tensor, x: Tensor):
        if theta.shape[-len(self.theta_shape):] != self.theta_shape:
            raise ValueError(f"The trailing dimensions of `theta` do not match the `theta_shape`: "
                             f"{theta.shape[-len(self.theta_shape):]} != {self.theta_shape}.")
        if x.shape[-len(self.x_shape):] != self.x_shape:
            raise ValueError(f"The trailing dimensions of `x` do not match the `x_shape`: "
                             f"{x.shape[-len(self.x_shape):]} != {self.x_shape}.")
        tp, xp = theta.shape[:-len(self.theta_shape)], x.shape[:-len(self.x_shape)]
        if tp != xp:
            raise ValueError(f"The shape prefixes of `theta` and `x` must match: {tuple(tp)=} != "
                             f"{tuple(xp)=}. Make them agree, since we do not broadcast for you.")
        return tp

    def unnormalized_log_ratio(self, theta: Tensor, x: Tensor) -> Tensor:
        prefix = self._check(theta, x)
        th = self.embed_theta(theta.reshape(-1, *self.theta_shape))
        xx = self.embed_x(x.reshape(-1, *self.x_shape))
        return _RatioFn.apply(self.net.flat, th, xx, self, None, None, False).reshape(*prefix)

    def forward(self, *args, **kwargs) -> Tensor:
        return self.unnormalized_log_ratio(*args, **kwargs)

    def loss(self, input: Tensor, condition: Tensor, **kwargs) -> Tensor:
        raise NotImplementedError()

    # ---- raw entry (no autograd): pairs given by optional index arrays / shared x
    def logits_raw(self, theta: Tensor, x: Tensor, ti: Optional[Tensor] = None,
                   xi: Optional[Tensor] = None, x_shared: bool = False, R: Optional[int] = None) -> Tensor:
        lib = L.load()
        L.require_cuda(theta, "theta")
        L.require_cuda(x, "x")
        R = (ti.shape[0] if ti is not None else theta.shape[0]) if R is None else R
        out = torch.empty(R, dtype=torch.float32, device=theta.device)
        m = self._model(nbuf=2)
        pr = L.Pairs(theta.data_ptr(), x.data_ptr(), None if ti is None else ti.data_ptr(),
                     None if xi is None else xi.data_ptr(), R, 1 if x_shared else 0)
        tc = self._tc_state(m) if (R >= self.TC_MIN_ROWS or os.environ.get("SBI_B200_TC", "") == "1") else None
        if tc is not None:
            L.check(lib.sbi_b200_ratio_forward_tc(C.byref(m), C.byref(tc), C.byref(pr), L.ptr(out),
                                                  L.stream_ptr()), "ratio_forward_tc")
            return out
        self._check_rc(self._entry("forward")(C.byref(m), C.byref(pr), L.ptr(out), L.stream_ptr()),
                    f"{self.layout.family}_forward")
        return out

    #: pairs from which the logits go through the wgmma kernel (csrc/ratio_tc.cu); the crossover against
    #: the SIMT kernel has not been measured for the wgmma kernel (profiles/tc_ratio_time.py measures it)
    TC_MIN_ROWS = int(os.environ.get("SBI_B200_RATIO_TC_MIN_ROWS", 32768))


class _RatioFn(torch.autograd.Function):
    """Logits of the pairs (theta[ti[r]], x[xi[r]]) (x[0] with `x_shared`) and their VJP.  The backward returns
    the gradients of the flat parameters and of the `theta` and `x` rows, each when asked for: per-pair input
    gradients from the VJP kernel, summed onto the gathered rows by `pair_rows_sum`.  `xi_sorted`: xi is
    non-decreasing (the rows' pairs are consecutive), so the x side needs no sort."""

    @staticmethod
    def forward(ctx, flat, theta, x, est: RatioEstimator, ti, xi, x_shared, xi_sorted=False):
        out = est.logits_raw(theta, x, ti, xi, x_shared)
        ctx.save_for_backward(theta, x)
        ctx.est, ctx.ti, ctx.xi, ctx.x_shared, ctx.xi_sorted = est, ti, xi, x_shared, xi_sorted
        return out

    @staticmethod
    def backward(ctx, g):
        theta, x = ctx.saved_tensors
        est = ctx.est
        R = g.shape[0]
        n_part = est._entry("vjp_parts")(R)
        gpart = est._gpart(n_part)
        need_flat, need_th, need_x = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        resnet = est.layout.family == "ratio"
        need_x = need_x and resnet
        gth = torch.empty(R, est.layout.Dt, dtype=torch.float32, device=theta.device) if need_th else None
        gx = torch.empty(R, est.layout.Dx, dtype=torch.float32, device=theta.device) if need_x else None
        m = est._model(nbuf=3)
        pr = L.Pairs(theta.data_ptr(), x.data_ptr(), None if ctx.ti is None else ctx.ti.data_ptr(),
                     None if ctx.xi is None else ctx.xi.data_ptr(), R, 1 if ctx.x_shared else 0)
        g = g.contiguous().float()
        if resnet:
            est._check_rc(L.load().sbi_b200_ratio_vjp_inputs(C.byref(m), C.byref(pr), L.ptr(g), None, L.ptr(gpart),
                                                            L.ptr(gth), L.ptr(gx), L.stream_ptr()), "ratio_vjp")
        else:   # per-pair theta gradients, summed onto the gathered rows below
            est._check_rc(est._entry("vjp")(C.byref(m), C.byref(pr), L.ptr(g), None, L.ptr(gpart), L.ptr(gth),
                                            L.stream_ptr()), f"{est.layout.family}_vjp")
        gflat = L.reduce_partials(gpart, n_part, est.layout.n_params) if need_flat else None
        if need_th and ctx.ti is not None:
            gth = pair_rows_sum(gth, ctx.ti, theta.shape[0])
        if need_x:
            if ctx.x_shared:
                gx = pair_rows_sum(gx, None, 1, torch.arange(2, dtype=torch.int64, device=gx.device) * R)
            elif ctx.xi is not None:
                gx = pair_rows_sum(gx, ctx.xi, x.shape[0], sorted_index=ctx.xi_sorted)
        return gflat, gth, gx, None, None, None, None, None


def pair_rows_sum(gpair: Tensor, index: Optional[Tensor], n_rows: int, row_ptr: Optional[Tensor] = None,
                  sorted_index: bool = False) -> Tensor:
    """(n_rows, W) gradients of gathered rows from the (R, W) gradients of their pairs: row j receives the sum of
    gpair[r] over the pairs r with index[r] == j (csrc/ratio.cu `pair_rows_sum_kernel`: one owner per entry, no
    atomics).  The CSR of the index is built on the device (stable sort + searchsorted, graph-capturable); a
    non-decreasing index (`sorted_index`) needs no sort.  `row_ptr` given: consecutive segments."""
    dev = gpair.device
    order = None
    if row_ptr is None:
        keys = index
        if not sorted_index:
            keys, order = torch.sort(index, stable=True)
            order = order.contiguous()
        row_ptr = torch.searchsorted(keys, torch.arange(n_rows + 1, dtype=keys.dtype, device=dev))
    out = torch.empty(n_rows, gpair.shape[1], dtype=torch.float32, device=dev)
    L.check(L.load().sbi_b200_pair_rows_sum(L.ptr(gpair.contiguous()), gpair.shape[1], L.ptr(order),
                                            L.ptr(row_ptr.contiguous()), n_rows, L.ptr(out), L.stream_ptr()),
            "pair_rows_sum")
    return out


def build_resnet_classifier(
    batch_x: Tensor, batch_y: Tensor, z_score_x: Optional[str] = "independent",
    z_score_y: Optional[str] = "independent", hidden_features: int = 50,
    embedding_net_x: nn.Module = nn.Identity(), embedding_net_y: nn.Module = nn.Identity(),
    num_blocks: int = 2, dropout_probability: float = 0.0, use_batch_norm: bool = False,
) -> RatioEstimator:
    """classifier.py:172-235 (in the classifier's view x = theta, y = x).  Parameters are drawn in
    nflows' construction order (initial layer, per block two linears with the second re-drawn
    U(-1e-3, 1e-3), final layer), so a seed reproduces the reference's initial weights.  With embedding
    nets the network is built on the embedded widths, each probed with one batch row like the reference."""
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("Ratio-based classifiers (NRE) do not implement `transform_to_unconstrained`.")
    if dropout_probability != 0.0 or use_batch_norm:
        raise NotImplementedError("dropout / batch norm are not implemented in the sm_90a ratio kernels")
    # get_numel (nn_utils.py:17-47): the widths the classifier sees are those of the embedded rows
    Dt = embedding_net_x.to(batch_x.device)(batch_x[:1]).numel()
    Dx = embedding_net_y.to(batch_y.device)(batch_y[:1]).numel()
    H = hidden_features
    lay = RatioLayout(Dt=Dt, Dx=Dx, H=H, NB=num_blocks)
    state = {}
    state["net.initial_layer.weight"], state["net.initial_layer.bias"] = _linear_init(H, Dt + Dx)
    for b in range(num_blocks):
        state[f"net.blocks.{b}.linear_layers.0.weight"], state[f"net.blocks.{b}.linear_layers.0.bias"] = _linear_init(H, H)
        w, bb = _linear_init(H, H)
        init.uniform_(w, -1e-3, 1e-3)
        init.uniform_(bb, -1e-3, 1e-3)
        state[f"net.blocks.{b}.linear_layers.1.weight"], state[f"net.blocks.{b}.linear_layers.1.bias"] = w, bb
    state["net.final_layer.weight"], state["net.final_layer.bias"] = _linear_init(1, H)
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    t_stats = standardizing_stats(batch_x, sx) if zx else None
    x_stats = standardizing_stats(batch_y, sy) if zy else None
    est = RatioEstimator(lay, batch_x[0].shape, batch_y[0].shape, t_stats, x_stats,
                         embedding_net_x, embedding_net_y)
    with torch.no_grad():
        lay.pack(state, out=est.net.flat.data)
    return est


def _input_stats(batch_x: Tensor, batch_y: Tensor, z_score_x, z_score_y):
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    return (standardizing_stats(batch_x, sx) if zx else None), (standardizing_stats(batch_y, sy) if zy else None)


def _norm_params(mod: nn.Module, H: int):
    """(kind, eps, {weight, bias}) of a module built by `norm_layer(H)`; the kernels implement
    nn.LayerNorm(H) with affine parameters (row-local) and nn.Identity."""
    if type(mod) is nn.Identity:
        return None, None, {}
    if (type(mod) is nn.LayerNorm and tuple(mod.normalized_shape) == (H,) and mod.elementwise_affine
            and mod.bias is not None):
        return "layer", float(mod.eps), {"weight": mod.weight.detach(), "bias": mod.bias.detach()}
    raise NotImplementedError(
        f"the sm_90a mlp classifier kernels implement norm_layer=nn.LayerNorm (affine) or nn.Identity; got {mod!r}")


def build_linear_classifier(
    batch_x: Tensor, batch_y: Tensor, z_score_x: Optional[str] = "independent",
    z_score_y: Optional[str] = "independent", embedding_net_x: nn.Module = nn.Identity(),
    embedding_net_y: nn.Module = nn.Identity(), **kwargs,
) -> RatioEstimator:
    """classifier.py:49-104: logit = Linear(Dt + Dx, 1)(u); one nn.Linear draw from the global RNG.
    Like the reference, other keyword arguments are ignored."""
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("Ratio-based classifiers (NRE) do not implement `transform_to_unconstrained`.")
    Dt, Dx = batch_x[0].numel(), batch_y[0].numel()
    lay = MlpRatioLayout(Dt=Dt, Dx=Dx, NL=0, norm=None)
    state = {}
    state["net.weight"], state["net.bias"] = _linear_init(1, Dt + Dx)
    t_stats, x_stats = _input_stats(batch_x, batch_y, z_score_x, z_score_y)
    est = RatioEstimator(lay, batch_x[0].shape, batch_y[0].shape, t_stats, x_stats,
                         embedding_net_x, embedding_net_y)
    with torch.no_grad():
        lay.pack(state, out=est.net.flat.data)
    return est


def build_mlp_classifier(
    batch_x: Tensor, batch_y: Tensor, z_score_x: Optional[str] = "independent",
    z_score_y: Optional[str] = "independent", hidden_features: int = 50,
    embedding_net_x: nn.Module = nn.Identity(), embedding_net_y: nn.Module = nn.Identity(),
    norm_layer: Callable[[int], nn.Module] = nn.LayerNorm,
) -> RatioEstimator:
    """classifier.py:107-169: Sequential(Linear(Dt+Dx, H), norm_layer(H), ReLU, Linear(H, H),
    norm_layer(H), ReLU, Linear(H, 1)).  Modules are constructed in that order, so a seed reproduces
    the reference's initial weights; the norm layers' own parameters are taken as built."""
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("Ratio-based classifiers (NRE) do not implement `transform_to_unconstrained`.")
    Dt, Dx, H = batch_x[0].numel(), batch_y[0].numel(), hidden_features
    state, norms = {}, []
    for l, fan_in in enumerate((Dt + Dx, H)):
        state[f"net.{3 * l}.weight"], state[f"net.{3 * l}.bias"] = _linear_init(H, fan_in)
        kind, eps, p = _norm_params(norm_layer(H), H)
        norms.append((kind, eps))
        state.update({f"net.{3 * l + 1}.{k}": v for k, v in p.items()})
    if norms[0] != norms[1]:
        raise NotImplementedError("the sm_90a mlp classifier kernels need both norm layers of the same kind and eps")
    state["net.6.weight"], state["net.6.bias"] = _linear_init(1, H)
    kind, eps = norms[0]
    lay = MlpRatioLayout(Dt=Dt, Dx=Dx, H=H, NL=2, norm=kind, eps=eps if eps is not None else 1e-5)
    t_stats, x_stats = _input_stats(batch_x, batch_y, z_score_x, z_score_y)
    est = RatioEstimator(lay, batch_x[0].shape, batch_y[0].shape, t_stats, x_stats,
                         embedding_net_x, embedding_net_y)
    with torch.no_grad():
        lay.pack(state, out=est.net.flat.data)
    return est


_BUILDERS = {"linear": build_linear_classifier, "mlp": build_mlp_classifier, "resnet": build_resnet_classifier}
#: the model-specific arguments of estimator_configs.py:1375-1419 (`hidden_features` is a factory argument)
_MODEL_ARGS = {"linear": set(), "mlp": {"hidden_features", "norm_layer"},
               "resnet": {"hidden_features", "num_blocks", "dropout_probability", "use_batch_norm"}}


def classifier_nn(
    model: str, z_score_theta: Optional[str] = "independent", z_score_x: Optional[str] = "independent",
    hidden_features: int = 50, embedding_net_theta: nn.Module = nn.Identity(),
    embedding_net_x: nn.Module = nn.Identity(), **kwargs: Any,
) -> Callable:
    """factory.py:174-241: build function for the NRE classifier `linear`, `mlp` or `resnet`.  An
    argument that belongs to another model (or a non-default `hidden_features` for `linear`) raises
    ValueError, as in the reference."""
    if model not in _BUILDERS:
        raise ValueError(f"Unknown classifier model {model!r}. Must be one of {sorted(_BUILDERS)}.")
    given = set(kwargs) | ({"hidden_features"} if hidden_features != 50 else set())
    unused = sorted((given & set().union(*_MODEL_ARGS.values())) - _MODEL_ARGS[model])
    if unused:
        raise ValueError(f"Argument(s) {unused} are not used by model={model!r} and would be silently ignored.")
    unknown = sorted(set(kwargs) - set().union(*_MODEL_ARGS.values()))
    if unknown:
        warnings.warn(f"Unknown kwargs passed to the {model!r} classifier: {unknown}. These will be forwarded "
                      "to the underlying builder. If this is unintentional, check for typos.", stacklevel=2)
    if model != "linear":
        kwargs["hidden_features"] = hidden_features

    def build_fn(batch_theta, batch_x):
        from ._refabc import register_with_reference
        register_with_reference()
        return _BUILDERS[model](
            batch_x=batch_theta, batch_y=batch_x, z_score_x=z_score_theta, z_score_y=z_score_x,
            embedding_net_x=embedding_net_theta, embedding_net_y=embedding_net_x, **kwargs)

    return build_fn
