"""Builder API: `posterior_nn`, `likelihood_nn` and the per-model build functions.

Same names, argument meaning and defaults as the reference factories
(/root/reference/sbi/neural_nets/factory.py:323-430 `posterior_nn`, :244-320
`likelihood_nn`) and builders (/root/reference/sbi/neural_nets/net_builders/flow.py:333-460
`build_nsf`).  Each factory returns `build_fn(batch_theta, batch_x)`; the returned estimator
implements sbi's ConditionalDensityEstimator interface on the sm_90a kernels, so it can be
passed to the reference trainers (`NPE(prior, density_estimator=posterior_nn("nsf"))`) or to
this package's device-resident trainers (`sbi_b200.inference`).
"""
from __future__ import annotations

from typing import Any, Callable, Optional

import numpy as np
import torch
from torch import Tensor, nn
from torch.nn import init

from .estimators import FlowEstimator, MadeEstimator, NSFEstimator
from .pack import MadeLayout, MafLayout, Nsf1dLayout, NsfLayout

_NSF_MODELS = ("nsf",)


# ---- z-scoring statistics: sbiutils.py:376-415 / :431-488 ----------------------------------------
def _valid_rows(t: Tensor) -> Tensor:
    flat = t.reshape(t.shape[0], -1)
    ok = ~torch.isnan(flat).any(1) & ~torch.isinf(flat).any(1)
    assert ok.sum() > 0, "No valid data entries left after excluding NaNs and Infs."
    return ok


def z_standardization(batch_t: Tensor, structured: bool = False, min_std: float = 1e-14):
    """Mean / std for the input z-score transform (sbiutils.py:376-415)."""
    ok = _valid_rows(batch_t)
    if structured:
        t_mean = torch.mean(batch_t[ok])
        sample_std = torch.std(batch_t[ok], dim=1)
        sample_std[sample_std < min_std] = min_std
        t_std = torch.mean(sample_std)
    else:
        t_mean = torch.mean(batch_t[ok], dim=0)
        t_std = torch.std(batch_t[ok], dim=0)
        t_std[t_std < min_std] = min_std
    return t_mean, t_std


def standardizing_stats(batch_t: Tensor, structured: bool = False, min_std: float = 1e-7):
    """Mean / std of the condition `Standardize` net (sbiutils.py:431-488)."""
    ok = _valid_rows(batch_t)
    t_mean = torch.mean(batch_t[ok]) if structured else torch.mean(batch_t[ok], dim=0)
    if len(batch_t) > 1:
        if structured:
            sample_std = torch.std(batch_t[ok], dim=1)
            sample_std[sample_std < min_std] = min_std
            t_std = torch.mean(sample_std)
        else:
            t_std = torch.std(batch_t[ok], dim=0)
            t_std[t_std < min_std] = min_std
    else:
        t_std = torch.ones(1)
    assert not (torch.isnan(t_mean).any() or torch.isnan(t_std).any()), (
        "Training data mean or std for standardizing net must not contain NaNs.")
    return t_mean, t_std


def z_score_parser(flag):
    if type(flag) is bool:
        return flag, False
    if flag in (None, "none"):
        return False, False
    if flag == "independent":
        return True, False
    if flag == "structured":
        return True, True
    raise ValueError(
        f"Invalid z-scoring option {flag!r}. Use 'none', 'independent', or 'structured'.")


def check_data_device(a: Tensor, b: Tensor):
    """user_input_checks.py:464-477."""
    assert a.device == b.device, (
        f"Mismatch in fed data's device: datum_1 has device {a.device}, whereas datum_2 has "
        f"device {b.device}. Please use data from a common device.")


def _linear_init(out_f: int, in_f: int):
    """Fresh nn.Linear weights/bias: consumes the global torch RNG exactly like the
    reference's module construction does."""
    lin = nn.Linear(in_f, out_f)
    return lin.weight.detach(), lin.bias.detach()


def build_nsf(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_transforms: int = 5, num_bins: int = 10,
    embedding_net: nn.Module = nn.Identity(), tail_bound: float = 3.0,
    hidden_layers_spline_context: int = 1, num_blocks: int = 2,
    dropout_probability: float = 0.0, use_batch_norm: bool = False, **kwargs,
) -> NSFEstimator:
    """Builds NSF p(x|y); same arguments as the reference (flow.py:333-460).

    Parameters are initialised by constructing the same torch modules in the same order as
    nflows does (ResidualNet: initial layer, per block context layer + two linears with the
    last re-drawn U(-1e-3,1e-3), final layer; LULinear identity init), so a given global seed
    yields the reference's initial weights.
    """
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("`transform_to_unconstrained` is not supported by build_nsf.")
    if dropout_probability != 0.0 or use_batch_norm:
        raise NotImplementedError("dropout / batch norm are not implemented in the sm_90a "
                                  "NSF kernels (reference defaults are 0.0 / False)")
    x_numel = batch_x[0].numel()
    with torch.no_grad():
        y_numel = embedding_net(batch_y[:1]).numel()
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    if x_numel == 1:
        # scalar x (flow.py:401-408): a dummy mask and spline parameters learnt from the condition alone
        # (ContextSplineMap: Linear, [one shared Linear] x hidden_layers, Linear -- constructed in that order)
        H, C, hl = hidden_features, y_numel, int(hidden_layers_spline_context)
        lay = Nsf1dLayout(C=C, H=H, NB=hl, KB=num_bins, T=num_transforms, tail_bound=float(tail_bound),
                          zscore_input=zx, zscore_cond=zy, embed_is_identity=isinstance(embedding_net, nn.Identity))
        state = {}
        base = 1 if zx else 0
        for l in range(num_transforms):
            pn = f"net._transform._transforms.{base + l}.transform_net.spline_predictor."
            state[pn + "0.weight"], state[pn + "0.bias"] = _linear_init(H, C)
            w, b = _linear_init(H, H)        # constructed (RNG consumed) even when it is repeated zero times
            if hl > 0:
                for k in range(hl):
                    state[pn + f"{2 + 2 * k}.weight"], state[pn + f"{2 + 2 * k}.bias"] = w, b
            state[pn + f"{2 + 2 * hl}.weight"], state[pn + f"{2 + 2 * hl}.bias"] = _linear_init(3 * num_bins - 1, H)
        if zx:
            t_mean, t_std = z_standardization(batch_x.reshape(batch_x.shape[0], -1), sx)
            shift, scale = -t_mean / t_std, 1 / t_std
        else:
            shift, scale = torch.zeros(()), torch.ones(())
        c_mean, c_std = standardizing_stats(batch_y, sy) if zy else (None, None)
        est = NSFEstimator(lay, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape, shift=shift,
                           scale=scale, cond_mean=c_mean, cond_std=c_std, embedding_net=embedding_net)
        with torch.no_grad():
            lay.pack(state, out=est.net.flat.data)
        return est
    lay = NsfLayout(D=x_numel, C=y_numel, H=hidden_features, NB=num_blocks, KB=num_bins,
                    T=num_transforms, tail_bound=float(tail_bound), zscore_input=zx,
                    zscore_cond=zy, embed_is_identity=isinstance(embedding_net, nn.Identity))
    H, C = hidden_features, y_numel
    state = {}
    base = 1 if zx else 0
    for l in range(num_transforms):
        n_id, n_tr = len(lay.id_feats[l]), len(lay.tr_feats[l])
        pc = f"net._transform._transforms.{base + 2 * l}.transform_net."
        pl = f"net._transform._transforms.{base + 2 * l + 1}."
        state[pc + "initial_layer.weight"], state[pc + "initial_layer.bias"] = _linear_init(H, n_id + C)
        for b in range(num_blocks):
            pb = pc + f"blocks.{b}."
            state[pb + "context_layer.weight"], state[pb + "context_layer.bias"] = _linear_init(H, C)
            state[pb + "linear_layers.0.weight"], state[pb + "linear_layers.0.bias"] = _linear_init(H, H)
            w, bb = _linear_init(H, H)
            init.uniform_(w, -1e-3, 1e-3)
            init.uniform_(bb, -1e-3, 1e-3)
            state[pb + "linear_layers.1.weight"], state[pb + "linear_layers.1.bias"] = w, bb
        state[pc + "final_layer.weight"], state[pc + "final_layer.bias"] = _linear_init(
            n_tr * (3 * num_bins - 1), H)
        ntri = x_numel * (x_numel - 1) // 2
        state[pl + "lower_entries"] = torch.zeros(ntri)
        state[pl + "upper_entries"] = torch.zeros(ntri)
        state[pl + "unconstrained_upper_diag"] = torch.full((x_numel,), float(np.log(np.exp(1 - 1e-3) - 1)))
        state[pl + "bias"] = torch.zeros(x_numel)

    if zx:
        t_mean, t_std = z_standardization(batch_x.reshape(batch_x.shape[0], -1), sx)
        shift, scale = -t_mean / t_std, 1 / t_std
    else:
        shift, scale = torch.zeros(()), torch.ones(())
    if zy:
        c_mean, c_std = standardizing_stats(batch_y, sy)
    else:
        c_mean = c_std = None
    est = NSFEstimator(lay, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape,
                       shift=shift, scale=scale, cond_mean=c_mean, cond_std=c_std,
                       embedding_net=embedding_net)
    with torch.no_grad():
        lay.pack(state, out=est.net.flat.data)
    return est


def build_maf(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_transforms: int = 5, embedding_net: nn.Module = nn.Identity(),
    num_blocks: int = 2, dropout_probability: float = 0.0, use_batch_norm: bool = False,
    num_bins: int = 10, **kwargs,
) -> FlowEstimator:
    """Builds MAF p(x|y); same arguments as the reference (flow.py:115-209): per transform a
    `MaskedAffineAutoregressiveTransform(hidden, context, num_blocks, use_residual_blocks=False,
    tanh)` followed by a `RandomPermutation`.  The global torch RNG is consumed in nflows' order
    (MADE: initial masked layer, context layer, blocks, final layer; then `torch.randperm`), so
    a seed yields the reference's initial weights AND permutations."""
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("`transform_to_unconstrained` is not supported by build_maf.")
    if dropout_probability != 0.0 or use_batch_norm:
        raise NotImplementedError("dropout / batch norm are not implemented in the sm_90a MAF kernels")
    x_numel = batch_x[0].numel()
    with torch.no_grad():
        y_numel = embedding_net(batch_y[:1]).numel()
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    H, C, D = hidden_features, y_numel, x_numel
    state, perms = {}, []
    base = 1 if zx else 0
    for l in range(num_transforms):
        pa = f"net._transform._transforms.{base + 2 * l}.autoregressive_net."
        state[pa + "initial_layer.weight"], state[pa + "initial_layer.bias"] = _linear_init(H, D)
        state[pa + "context_layer.weight"], state[pa + "context_layer.bias"] = _linear_init(H, C)
        for b in range(num_blocks):
            state[pa + f"blocks.{b}.linear.weight"], state[pa + f"blocks.{b}.linear.bias"] = _linear_init(H, H)
        state[pa + "final_layer.weight"], state[pa + "final_layer.bias"] = _linear_init(2 * D, H)
        perms.append(torch.randperm(D).numpy())
    lay = MafLayout(D=D, C=C, H=H, NB=num_blocks, T=num_transforms, perms=perms, zscore_input=zx,
                    zscore_cond=zy, embed_is_identity=isinstance(embedding_net, nn.Identity),
                    scale_softplus=bool(kwargs.get("maf_scale_softplus", True)))
    if zx:
        t_mean, t_std = z_standardization(batch_x.reshape(batch_x.shape[0], -1), sx)
        shift, scale = -t_mean / t_std, 1 / t_std
    else:
        shift, scale = torch.zeros(()), torch.ones(())
    c_mean, c_std = standardizing_stats(batch_y, sy) if zy else (None, None)
    est = FlowEstimator(lay, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape,
                        shift=shift, scale=scale, cond_mean=c_mean, cond_std=c_std,
                        embedding_net=embedding_net)
    with torch.no_grad():
        lay.pack(state, out=est.net.flat.data, raw_out=est.net._raw)
    return est


def build_maf_rqs(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_transforms: int = 5, embedding_net: nn.Module = nn.Identity(),
    num_blocks: int = 2, num_bins: int = 10, tails: Optional[str] = "linear", tail_bound: float = 3.0,
    dropout_probability: float = 0.0, use_batch_norm: bool = False, min_bin_width: float = 1e-3,
    min_bin_height: float = 1e-3, min_derivative: float = 1e-3, **kwargs,
) -> FlowEstimator:
    """Builds MAF p(x|y) whose element-wise maps are rational-quadratic splines; same arguments as the
    reference (flow.py:212-330): per transform a `MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
    hidden, context, num_bins, tails="linear", tail_bound, num_blocks, use_residual_blocks=False, tanh)`
    followed by a `RandomPermutation`.  Same MADE and RNG order as `build_maf`; the final masked layer
    emits 3*num_bins - 1 raw spline parameters per feature."""
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("`transform_to_unconstrained` is not supported by build_maf_rqs.")
    if dropout_probability != 0.0 or use_batch_norm:
        raise NotImplementedError("dropout / batch norm are not implemented in the sm_90a MAF kernels")
    if tails != "linear":
        raise NotImplementedError("the sm_90a spline code implements tails='linear' (the reference default)")
    x_numel = batch_x[0].numel()
    with torch.no_grad():
        y_numel = embedding_net(batch_y[:1]).numel()
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    H, C, D = hidden_features, y_numel, x_numel
    mult = 3 * num_bins - 1
    state, perms = {}, []
    base = 1 if zx else 0
    for l in range(num_transforms):
        pa = f"net._transform._transforms.{base + 2 * l}.autoregressive_net."
        state[pa + "initial_layer.weight"], state[pa + "initial_layer.bias"] = _linear_init(H, D)
        state[pa + "context_layer.weight"], state[pa + "context_layer.bias"] = _linear_init(H, C)
        for b in range(num_blocks):
            state[pa + f"blocks.{b}.linear.weight"], state[pa + f"blocks.{b}.linear.bias"] = _linear_init(H, H)
        state[pa + "final_layer.weight"], state[pa + "final_layer.bias"] = _linear_init(mult * D, H)
        perms.append(torch.randperm(D).numpy())
    lay = MafLayout(D=D, C=C, H=H, NB=num_blocks, T=num_transforms, perms=perms, zscore_input=zx,
                    zscore_cond=zy, embed_is_identity=isinstance(embedding_net, nn.Identity),
                    head="rqs", KB=num_bins, tail_bound=float(tail_bound), min_bin_width=float(min_bin_width),
                    min_bin_height=float(min_bin_height), min_derivative=float(min_derivative))
    if zx:
        t_mean, t_std = z_standardization(batch_x.reshape(batch_x.shape[0], -1), sx)
        shift, scale = -t_mean / t_std, 1 / t_std
    else:
        shift, scale = torch.zeros(()), torch.ones(())
    c_mean, c_std = standardizing_stats(batch_y, sy) if zy else (None, None)
    est = FlowEstimator(lay, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape,
                        shift=shift, scale=scale, cond_mean=c_mean, cond_std=c_std,
                        embedding_net=embedding_net)
    with torch.no_grad():
        lay.pack(state, out=est.net.flat.data, raw_out=est.net._raw)
    return est


def build_made(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_mixture_components: int = 10, embedding_net: nn.Module = nn.Identity(),
    **kwargs,
) -> MadeEstimator:
    """Builds MADE p(x|y); same arguments as the reference (flow.py:37-112): z-scoring + MADEMoGWrapper(
    features, hidden, context, num_blocks=5, num_mixture_components, use_residual_blocks=True, relu,
    custom_initialization=True).  Modules are initialised in nflows' construction order (MADE: initial masked
    layer, context layer, per block context layer + two masked linears with the last re-drawn U(-1e-3, 1e-3),
    final masked layer; then MixtureOfGaussiansMADE._initialize), so a seed yields the reference's weights."""
    check_data_device(batch_x, batch_y)
    if z_score_x == "transform_to_unconstrained":
        raise ValueError("`transform_to_unconstrained` is not supported by build_made.")
    x_numel = batch_x[0].numel()
    with torch.no_grad():
        y_numel = embedding_net(batch_y[:1]).numel()
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    H, C, F, M, NB = hidden_features, y_numel, x_numel + 1, num_mixture_components, 5
    eps = 1e-2
    lay = MadeLayout(D=F, C=C, H=H, NB=NB, M=M, epsilon=eps, zscore_input=zx, zscore_cond=zy,
                     embed_is_identity=isinstance(embedding_net, nn.Identity))
    pm = "net._distribution._made."
    st = {}
    st[pm + "initial_layer.weight"], st[pm + "initial_layer.bias"] = _linear_init(H, F)
    st[pm + "context_layer.weight"], st[pm + "context_layer.bias"] = _linear_init(H, C)
    for b in range(NB):
        pb = pm + f"blocks.{b}."
        st[pb + "context_layer.weight"], st[pb + "context_layer.bias"] = _linear_init(H, C)
        st[pb + "linear_layers.0.weight"], st[pb + "linear_layers.0.bias"] = _linear_init(H, H)
        w, bb = _linear_init(H, H)
        init.uniform_(w, -1e-3, 1e-3)
        init.uniform_(bb, -1e-3, 1e-3)
        st[pb + "linear_layers.1.weight"], st[pb + "linear_layers.1.bias"] = w, bb
    wf, bf = _linear_init(3 * M * F, H)
    wf, bf = wf.clone(), bf.clone()
    wf[::3, :] = eps * torch.randn(F * M, H)
    bf[::3] = eps * torch.randn(F * M)
    wf[2::3] = eps * torch.randn(F * M, H)
    bf[2::3] = torch.log(torch.exp(torch.Tensor([1 - eps])) - 1) * torch.ones(F * M) + eps * torch.randn(F * M)
    st[pm + "final_layer.weight"], st[pm + "final_layer.bias"] = wf, bf
    if zx:
        t_mean, t_std = z_standardization(batch_x.reshape(batch_x.shape[0], -1), sx)
        shift, scale = -t_mean / t_std, 1 / t_std
    else:
        shift, scale = torch.zeros(()), torch.ones(())
    c_mean, c_std = standardizing_stats(batch_y, sy) if zy else (None, None)
    est = MadeEstimator(lay, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape,
                        shift=shift, scale=scale, cond_mean=c_mean, cond_std=c_std, embedding_net=embedding_net)
    with torch.no_grad():
        lay.pack(st, out=est.net.flat.data, raw_out=est.net._raw)
    return est


_BUILDERS = {"nsf": build_nsf, "maf": build_maf, "maf_rqs": build_maf_rqs, "made": build_made}


def _density_build_fn(model: str, input_is_theta: bool, **kw) -> Callable:
    if model not in _BUILDERS:
        raise NotImplementedError(
            f"sbi_b200 implements {sorted(_BUILDERS)} density estimators on sm_90a; "
            f"got model={model!r}.")
    builder = _BUILDERS[model]

    def build_fn(batch_theta, batch_x):
        from ._refabc import register_with_reference
        register_with_reference()   # virtual subclass of the reference's ABCs if sbi is imported
        if input_is_theta:   # NPE models p(theta | x)
            return builder(batch_x=batch_theta, batch_y=batch_x, **kw)
        return builder(batch_x=batch_x, batch_y=batch_theta, **kw)   # NLE: p(x | theta)

    return build_fn


def posterior_nn(
    model: str, z_score_theta: Optional[str] = "independent", z_score_x: Optional[str] = "independent",
    hidden_features: int = 50, num_transforms: int = 5, num_bins: int = 10,
    embedding_net: nn.Module = nn.Identity(), num_components: int = 10, **kwargs: Any,
) -> Callable:
    """factory.py:323-430: build function for p(theta | x) (NPE)."""
    return _density_build_fn(
        model, True, z_score_x=z_score_theta, z_score_y=z_score_x,
        hidden_features=hidden_features, num_transforms=num_transforms, num_bins=num_bins,
        embedding_net=embedding_net, **kwargs)


def likelihood_nn(
    model: str, z_score_theta: Optional[str] = "independent", z_score_x: Optional[str] = "independent",
    hidden_features: int = 50, num_transforms: int = 5, num_bins: int = 10,
    embedding_net: nn.Module = nn.Identity(), num_components: int = 10, **kwargs: Any,
) -> Callable:
    """factory.py:244-320: build function for p(x | theta) (NLE); roles swapped (:316-318)."""
    return _density_build_fn(
        model, False, z_score_x=z_score_x, z_score_y=z_score_theta,
        hidden_features=hidden_features, num_transforms=num_transforms, num_bins=num_bins,
        embedding_net=embedding_net, **kwargs)
