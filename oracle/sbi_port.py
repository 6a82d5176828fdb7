"""CPU restatement of the sbi-owned part of the hot path (TEST INFRASTRUCTURE).

/root/reference does not exist on the GPU box, so the parity checker used by the
``-m gpu`` tests, ``__graft_entry__.smoke()`` and the timed CPU baseline in ``bench.py``
cannot import the reference there.  This module restates, on top of
``oracle.nflows_port``, exactly the reference code that sits between sbi's public API and
nflows for this path.  Every function cites the reference file:line it follows.  In the
build container it is cross-checked against the UNMODIFIED reference (imported through
``oracle.ref_shim``) by ``tests/test_oracle_vs_reference.py``.
"""
from __future__ import annotations

import math
import time
from copy import deepcopy
from functools import partial
from typing import Optional, Tuple

import torch
from torch import Tensor, nn
from torch.nn.utils.clip_grad import clip_grad_norm_
from torch.optim import Adam
from torch.utils import data
from torch.utils.data.sampler import SubsetRandomSampler

from .nflows_port import distributions as distributions_
from .nflows_port import flows, transforms
from .nflows_port.nn import nets


# ----------------------------------------------------------------------------- z-scoring
def handle_invalid_x(x: Tensor, exclude_invalid_x: bool = True):
    """sbi/utils/sbiutils.py:491-525."""
    batch_size = x.shape[0]
    x = x.reshape(batch_size, -1)
    x_is_nan = torch.isnan(x).any(dim=1)
    x_is_inf = torch.isinf(x).any(dim=1)
    if exclude_invalid_x:
        is_valid = ~x_is_nan & ~x_is_inf
    else:
        is_valid = torch.ones(batch_size, dtype=torch.bool)
    return is_valid, int(x_is_nan.sum()), int(x_is_inf.sum())


def z_standardization(batch_t: Tensor, structured_dims: bool = False, min_std: float = 1e-14):
    """sbi/utils/sbiutils.py:376-415."""
    is_valid_t, *_ = handle_invalid_x(batch_t, True)
    if structured_dims:
        t_mean = torch.mean(batch_t[is_valid_t])
        sample_std = torch.std(batch_t[is_valid_t], dim=1)
        sample_std[sample_std < min_std] = min_std
        t_std = torch.mean(sample_std)
    else:
        t_mean = torch.mean(batch_t[is_valid_t], dim=0)
        t_std = torch.std(batch_t[is_valid_t], dim=0)
        t_std[t_std < min_std] = min_std
    return t_mean, t_std


def standardizing_transform(batch_t: Tensor, structured_dims: bool = False, min_std: float = 1e-14):
    """sbi/utils/sbiutils.py:226-247."""
    t_mean, t_std = z_standardization(batch_t, structured_dims, min_std)
    return transforms.PointwiseAffineTransform(shift=-t_mean / t_std, scale=1 / t_std)


class Standardize(nn.Module):
    """sbi/utils/sbiutils.py:418-428."""

    def __init__(self, mean, std):
        super().__init__()
        mean, std = map(torch.as_tensor, (mean, std))
        self.mean = mean
        self.std = std
        self.register_buffer("_mean", mean)
        self.register_buffer("_std", std)

    def forward(self, tensor):
        return (tensor - self._mean) / self._std


def standardizing_net(batch_t: Tensor, structured_dims: bool = False, min_std: float = 1e-7):
    """sbi/utils/sbiutils.py:431-488."""
    is_valid_t, *_ = handle_invalid_x(batch_t, True)
    if structured_dims:
        t_mean = torch.mean(batch_t[is_valid_t])
    else:
        t_mean = torch.mean(batch_t[is_valid_t], dim=0)
    if len(batch_t) > 1:
        if structured_dims:
            sample_std = torch.std(batch_t[is_valid_t], dim=1)
            sample_std[sample_std < min_std] = min_std
            t_std = torch.mean(sample_std)
        else:
            t_std = torch.std(batch_t[is_valid_t], dim=0)
            t_std[t_std < min_std] = min_std
    else:
        t_std = torch.ones(1)
    assert not (torch.isnan(t_mean).any() or torch.isnan(t_std).any())
    return Standardize(t_mean, t_std)


def z_score_parser(z_score_flag) -> Tuple[bool, bool]:
    """sbi/utils/sbiutils.py:z_score_parser -- (do z-score?, structured?)."""
    if type(z_score_flag) is bool:
        return z_score_flag, False
    if z_score_flag in (None, "none"):
        return False, False
    if z_score_flag == "independent":
        return True, False
    if z_score_flag == "structured":
        return True, True
    raise ValueError(f"Invalid z-scoring option {z_score_flag!r}")


def create_alternating_binary_mask(features: int, even: bool = True) -> Tensor:
    """sbi/utils/torchutils.py:396-410."""
    mask = torch.zeros(features).byte()
    start = 0 if even else 1
    mask[start::2] += 1
    return mask


def searchsorted(bin_locations: Tensor, inputs: Tensor, eps: float = 1e-6) -> Tensor:
    """sbi/utils/torchutils.py:449-463 (the one known-answer test of the path pins this)."""
    bin_locations[..., -1] += eps
    return torch.sum(inputs[..., None] >= bin_locations, dim=-1) - 1


def get_base_dist(num_dims: int, dtype=torch.float32):
    """sbi/neural_nets/net_builders/flow.py:1481-1488."""
    base = distributions_.StandardNormal((num_dims,))
    base._log_z = base._log_z.to(dtype)
    return base


# ----------------------------------------------------------------------------- estimator wrapper
class NFlowsFlow(nn.Module):
    """sbi/neural_nets/estimators/nflows_flow.py:14-151 on top of
    sbi/neural_nets/estimators/base.py:35-306 (shape handling)."""

    def __init__(self, net, input_shape, condition_shape):
        super().__init__()
        self.net = net
        self._input_shape = torch.Size(input_shape)
        self._condition_shape = torch.Size(condition_shape)

    input_shape = property(lambda self: self._input_shape)
    condition_shape = property(lambda self: self._condition_shape)

    @property
    def embedding_net(self):
        return self.net._embedding_net

    def _broadcast_and_align(self, input: Tensor, condition: Tensor):
        """base.py:142-198."""
        input_event_dims = len(self.input_shape)
        condition_event_dims = len(self.condition_shape)
        if input.dim() <= input_event_dims + 1:
            input = input.unsqueeze(0)
        sample_dim = input.shape[0]
        input_batch_dim = input.shape[1]
        condition_has_sample_dim = condition.dim() > condition_event_dims + 1
        condition_batch_dim = condition.shape[1] if condition_has_sample_dim else condition.shape[0]
        try:
            batch_dim = torch.broadcast_shapes((input_batch_dim,), (condition_batch_dim,))[0]
        except RuntimeError as err:
            raise RuntimeError(
                "Expected `input` and `condition` to have broadcastable batch "
                "dimensions: their batch sizes must match, or one of them must be 1. "
                f"Got input={input_batch_dim} and condition={condition_batch_dim}."
            ) from err
        input = input.expand(sample_dim, batch_dim, *self.input_shape)
        if condition_has_sample_dim:
            condition = condition.expand(sample_dim, batch_dim, *self.condition_shape)
        else:
            condition = (
                condition.expand(batch_dim, *self.condition_shape)
                .unsqueeze(0)
                .expand(sample_dim, batch_dim, *self.condition_shape)
            )
        return input, condition, batch_dim

    def inverse_transform(self, input: Tensor, condition: Tensor) -> Tensor:
        condition_dims = len(self.condition_shape)
        batch_shape_in = input.shape[:-1]
        batch_shape_cond = condition.shape[:-condition_dims]
        batch_shape = torch.broadcast_shapes(batch_shape_in, batch_shape_cond)
        input = input.expand(batch_shape + (input.shape[-1],))
        condition = condition.expand(batch_shape + self.condition_shape)
        input = input.reshape(-1, input.shape[-1])
        condition = condition.reshape(-1, *self.condition_shape)
        # NB: exactly like the reference (nflows_flow.py:73) the RAW condition is passed -- the
        # embedding net / condition z-scoring is NOT applied on this code path.
        noise, _ = self.net._transform(input, context=condition)
        return noise.reshape(batch_shape + (noise.shape[-1],))

    def log_prob(self, input: Tensor, condition: Tensor) -> Tensor:
        input, condition, batch_dim = self._broadcast_and_align(input, condition)
        sample_dim = input.shape[0]
        input = input.reshape(sample_dim * batch_dim, -1)
        condition = condition.reshape(sample_dim * batch_dim, *self.condition_shape)
        log_probs = self.net.log_prob(input, context=condition)
        return log_probs.reshape(sample_dim, batch_dim)

    def loss(self, input: Tensor, condition: Tensor) -> Tensor:
        return -self.log_prob(input.unsqueeze(0), condition)[0]

    def sample(self, sample_shape, condition: Tensor) -> Tensor:
        condition_batch_dim = condition.shape[0]
        num_samples = torch.Size(sample_shape).numel()
        samples = self.net.sample(num_samples, context=condition)
        samples = samples.transpose(0, 1)
        return samples.reshape((*sample_shape, condition_batch_dim, *self.input_shape))

    def sample_and_log_prob(self, sample_shape, condition: Tensor):
        condition_batch_dim = condition.shape[0]
        num_samples = torch.Size(sample_shape).numel()
        samples, log_probs = self.net.sample_and_log_prob(num_samples, context=condition)
        samples = samples.reshape((*sample_shape, condition_batch_dim, -1))
        log_probs = log_probs.reshape((*sample_shape, -1))
        return samples, log_probs


# ----------------------------------------------------------------------------- builders
def build_nsf(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_transforms: int = 5, num_bins: int = 10,
    embedding_net: nn.Module = None, tail_bound: float = 3.0, num_blocks: int = 2,
    dropout_probability: float = 0.0, use_batch_norm: bool = False, **kwargs,
) -> NFlowsFlow:
    """sbi/neural_nets/net_builders/flow.py:333-460 (x_numel > 1 branch)."""
    embedding_net = embedding_net if embedding_net is not None else nn.Identity()
    x_numel = batch_x[0].numel()
    y_numel = embedding_net(batch_y[:1]).numel()
    if x_numel == 1:
        raise NotImplementedError("1-D NSF (ContextSplineMap) is not restated yet")

    def mask_in_layer(i):
        return create_alternating_binary_mask(features=x_numel, even=(i % 2 == 0))

    conditioner = partial(
        nets.ResidualNet, hidden_features=hidden_features, context_features=y_numel,
        num_blocks=num_blocks, activation=torch.relu,
        dropout_probability=dropout_probability, use_batch_norm=use_batch_norm,
    )
    transform_list = []
    for i in range(num_transforms):
        transform_list.append(
            transforms.PiecewiseRationalQuadraticCouplingTransform(
                mask=mask_in_layer(i), transform_net_create_fn=conditioner,
                num_bins=num_bins, tails="linear", tail_bound=tail_bound,
                apply_unconditional_transform=False,
            )
        )
        transform_list.append(transforms.LULinear(x_numel, identity_init=True))

    z_score_x_bool, structured_x = z_score_parser(z_score_x)
    if z_score_x_bool:
        transform_list = [standardizing_transform(batch_x, structured_x)] + transform_list
    z_score_y_bool, structured_y = z_score_parser(z_score_y)
    if z_score_y_bool:
        embedding_net = nn.Sequential(standardizing_net(batch_y, structured_y), embedding_net)
    distribution = get_base_dist(x_numel)
    transform = transforms.CompositeTransform(transform_list)
    neural_net = flows.Flow(transform, distribution, embedding_net)
    return NFlowsFlow(neural_net, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape)


def build_maf(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_transforms: int = 5, embedding_net: nn.Module = None,
    num_blocks: int = 2, dropout_probability: float = 0.0, use_batch_norm: bool = False,
    **kwargs,
) -> NFlowsFlow:
    """sbi/neural_nets/net_builders/flow.py:115-209."""
    return _build_made_flow(batch_x, batch_y, z_score_x, z_score_y, embedding_net, num_transforms, partial(
        transforms.MaskedAffineAutoregressiveTransform, hidden_features=hidden_features, num_blocks=num_blocks,
        use_residual_blocks=False, random_mask=False, activation=torch.tanh,
        dropout_probability=dropout_probability, use_batch_norm=use_batch_norm))


def build_maf_rqs(
    batch_x: Tensor, batch_y: Tensor, z_score_x="independent", z_score_y="independent",
    hidden_features: int = 50, num_transforms: int = 5, embedding_net: nn.Module = None,
    num_blocks: int = 2, num_bins: int = 10, tail_bound: float = 3.0, dropout_probability: float = 0.0,
    use_batch_norm: bool = False, **kwargs,
) -> NFlowsFlow:
    """sbi/neural_nets/net_builders/flow.py:212-330 (tails="linear", the reference default)."""
    return _build_made_flow(batch_x, batch_y, z_score_x, z_score_y, embedding_net, num_transforms, partial(
        transforms.MaskedPiecewiseRationalQuadraticAutoregressiveTransform, hidden_features=hidden_features,
        num_bins=num_bins, tails="linear", tail_bound=tail_bound, num_blocks=num_blocks,
        use_residual_blocks=False, random_mask=False, activation=torch.tanh,
        dropout_probability=dropout_probability, use_batch_norm=use_batch_norm))


def _build_made_flow(batch_x, batch_y, z_score_x, z_score_y, embedding_net, num_transforms, made_transform):
    """The flow both MAF builders assemble: per transform a MADE transform and a RandomPermutation."""
    embedding_net = embedding_net if embedding_net is not None else nn.Identity()
    x_numel = batch_x[0].numel()
    y_numel = embedding_net(batch_y[:1]).numel()
    if x_numel == 1:
        import warnings
        warnings.warn("In one-dimensional output space, this flow is limited to Gaussians",
                      stacklevel=3)
    transform_list = []
    for _ in range(num_transforms):
        block = [
            made_transform(features=x_numel, context_features=y_numel),
            transforms.RandomPermutation(features=x_numel),
        ]
        transform_list += block
    z_score_x_bool, structured_x = z_score_parser(z_score_x)
    if z_score_x_bool:
        transform_list = [standardizing_transform(batch_x, structured_x)] + transform_list
    z_score_y_bool, structured_y = z_score_parser(z_score_y)
    if z_score_y_bool:
        embedding_net = nn.Sequential(standardizing_net(batch_y, structured_y), embedding_net)
    distribution = get_base_dist(x_numel)
    transform = transforms.CompositeTransform(transform_list)
    neural_net = flows.Flow(transform, distribution, embedding_net)
    return NFlowsFlow(neural_net, input_shape=batch_x[0].shape, condition_shape=batch_y[0].shape)


# ----------------------------------------------------------------------------- ratio estimator (NRE)
class RatioEstimator(nn.Module):
    """sbi/neural_nets/ratio_estimators.py:11-157."""

    def __init__(self, net, theta_shape, x_shape, embedding_net_theta=None, embedding_net_x=None):
        super().__init__()
        self.net = net
        self.theta_shape, self.x_shape = torch.Size(theta_shape), torch.Size(x_shape)
        self.embedding_net_theta = embedding_net_theta if embedding_net_theta is not None else nn.Identity()
        self.embedding_net_x = embedding_net_x if embedding_net_x is not None else nn.Identity()

    def combine_theta_and_x(self, theta: Tensor, x: Tensor) -> Tensor:
        prefix = theta.shape[:-len(self.theta_shape)]
        if prefix != x.shape[:-len(self.x_shape)]:
            raise ValueError("The shape prefixes of `theta` and `x` must match")
        et = self.embedding_net_theta(theta.reshape(-1, *self.theta_shape))
        ex = self.embedding_net_x(x.reshape(-1, *self.x_shape))
        return torch.cat([et, ex], dim=-1).reshape(*prefix, -1)

    def unnormalized_log_ratio(self, theta: Tensor, x: Tensor) -> Tensor:
        return self.net(self.combine_theta_and_x(theta, x)).squeeze(-1)

    def forward(self, *args, **kwargs):
        return self.unnormalized_log_ratio(*args, **kwargs)


def build_resnet_classifier(batch_x: Tensor, batch_y: Tensor, z_score_x="independent",
                            z_score_y="independent", hidden_features: int = 50, num_blocks: int = 2):
    """sbi/neural_nets/net_builders/classifier.py:172-235 (x = theta, y = x in its view)."""
    x_numel, y_numel = batch_x[0].numel(), batch_y[0].numel()
    neural_net = nets.ResidualNet(in_features=x_numel + y_numel, out_features=1,
                                  hidden_features=hidden_features, context_features=None,
                                  num_blocks=num_blocks, activation=torch.relu)
    zx, sx = z_score_parser(z_score_x)
    zy, sy = z_score_parser(z_score_y)
    ex = nn.Sequential(standardizing_net(batch_x, sx), nn.Identity()) if zx else nn.Identity()
    ey = nn.Sequential(standardizing_net(batch_y, sy), nn.Identity()) if zy else nn.Identity()
    return RatioEstimator(neural_net, batch_x[0].shape, batch_y[0].shape, ex, ey)


def nre_b_logits(net: RatioEstimator, theta: Tensor, x: Tensor, num_atoms: int, choices: Tensor = None):
    """sbi/inference/trainers/nre/nre_base.py:396-415 (`choices` may be supplied to pin the draw)."""
    batch_size = theta.shape[0]
    repeated_x = x.repeat_interleave(num_atoms, dim=0)
    if choices is None:
        probs = torch.ones(batch_size, batch_size) * (1 - torch.eye(batch_size)) / (batch_size - 1)
        choices = torch.multinomial(probs, num_samples=num_atoms - 1, replacement=False)
    contrasting_theta = theta[choices]
    atomic_theta = torch.cat((theta[:, None, :], contrasting_theta), dim=1).reshape(batch_size * num_atoms, -1)
    return net(atomic_theta, repeated_x)


def nre_b_loss(net: RatioEstimator, theta: Tensor, x: Tensor, num_atoms: int, choices: Tensor = None):
    """sbi/inference/trainers/nre/nre_b.py:157-182."""
    batch_size = theta.shape[0]
    logits = nre_b_logits(net, theta, x, num_atoms, choices).reshape(batch_size, num_atoms)
    log_prob = logits[:, 0] - torch.logsumexp(logits, dim=-1)
    return -torch.mean(log_prob)


# ----------------------------------------------------------------------------- flow matching (FMPE)
class SinusoidalTimeEmbedding(nn.Module):
    """sbi/neural_nets/net_builders/vector_field_nets.py:367-421."""

    def __init__(self, embed_dim: int = 16, max_freq: float = 0.01):
        super().__init__()
        self.embed_dim = embed_dim
        self.register_buffer("div_term", torch.exp(torch.arange(0, embed_dim, 2) * (-math.log(max_freq) / embed_dim)))

    def forward(self, t: Tensor) -> Tensor:
        if t.ndim == 1:
            t = t.unsqueeze(-1)
        emb = torch.zeros(t.shape[:-1] + (self.embed_dim,), device=t.device, dtype=t.dtype)
        emb[:, 0::2] = torch.sin(t * self.div_term)
        emb[:, 1::2] = torch.cos(t * self.div_term)
        return emb


class VectorFieldMLP(nn.Module):
    """sbi/neural_nets/net_builders/vector_field_nets.py:610-719 (GELU, LayerNorm, skip connections)."""

    def __init__(self, input_dim, condition_dim, time_emb_dim, hidden_features=100, num_layers=5,
                 sinusoidal_max_freq=1000.0):
        super().__init__()
        self.input_layer = nn.Linear(input_dim, hidden_features)
        self.condition_layer = nn.Linear(condition_dim, hidden_features)
        self.input_merge_layer = nn.Linear(2 * hidden_features, hidden_features)
        self.time_emb = SinusoidalTimeEmbedding(time_emb_dim, sinusoidal_max_freq)
        self.activation = nn.GELU()
        self.layers = nn.ModuleList([nn.Linear(hidden_features, hidden_features) for _ in range(num_layers)])
        self.layers_norm = nn.ModuleList([nn.LayerNorm(hidden_features) for _ in range(num_layers)])
        self.time_linear_layer = nn.Linear(time_emb_dim, hidden_features)
        self.output_layer = nn.Linear(hidden_features, input_dim)
        nn.init.zeros_(self.output_layer.weight)

    def forward(self, input, condition, t):
        h = self.input_merge_layer(self.activation(torch.cat([self.input_layer(input), self.condition_layer(condition)], -1)))
        t_emb = self.time_linear_layer(self.time_emb(t))
        h = self.activation(h)
        for lin, ln in zip(self.layers, self.layers_norm):
            h_old = h
            h = self.activation(lin(h))
            h = h + t_emb
            h = h + h_old
            h = ln(h)
        return self.output_layer(h)


class FlowMatchingEstimator(nn.Module):
    """sbi/neural_nets/estimators/flowmatching_estimator.py:120-347 (no gaussian baseline)."""

    def __init__(self, net, input_shape, condition_shape, embedding_net, mean_0, std_0, noise_scale=1e-3):
        super().__init__()
        self.net, self._embedding_net, self.noise_scale = net, embedding_net, noise_scale
        self.input_shape, self.condition_shape = torch.Size(input_shape), torch.Size(condition_shape)
        self.register_buffer("mean_0", torch.as_tensor(mean_0, dtype=torch.float32).expand(input_shape).clone())
        self.register_buffer("std_0", torch.as_tensor(std_0, dtype=torch.float32).expand(input_shape).clone())
        # base distribution N(mean_base, std_base) of the ODE (estimators/base.py: ConditionalVectorFieldEstimator)
        self.register_buffer("_mean_base", torch.zeros(1, *self.input_shape))
        self.register_buffer("_std_base", torch.ones(1, *self.input_shape))
        self.register_buffer("_theta_shift", torch.zeros(1, *self.input_shape, dtype=torch.float32))
        self.register_buffer("_theta_scale", torch.ones(1, *self.input_shape, dtype=torch.float32))
        self.register_buffer("_compose_standardization", torch.tensor(False), persistent=True)

    def _stats(self, time):
        t = time.view(-1, 1)
        mu_t = (1 - t) * self.mean_0.view(1, -1)
        std_t = torch.sqrt(((1 - t) * self.std_0.view(1, -1)) ** 2 + t ** 2 + 1e-6)
        return mu_t, std_t

    def forward(self, input, condition, time):
        bshape = torch.broadcast_shapes(input.shape[:-1], condition.shape[:-1])
        cond = torch.broadcast_to(self._embedding_net(condition), bshape + condition.shape[-1:]).reshape(-1, condition.shape[-1])
        inp = torch.broadcast_to(input, bshape + self.input_shape).reshape(-1, input.shape[-1])
        time = torch.broadcast_to(time, bshape).reshape(-1)
        mu_t, std_t = self._stats(time)
        v_out = self.net((inp - mu_t) / std_t, cond, time)
        v = v_out * torch.sqrt(1 + self.std_0.view(1, -1) ** 2) - self.mean_0.view(1, -1)
        return v.reshape(*bshape, *self.input_shape)

    def loss(self, input, condition, times=None, theta_1=None):
        if times is None:
            times = torch.rand(input.shape[:-1], device=input.device, dtype=input.dtype)
        times_ = times[..., None]
        if theta_1 is None:
            theta_1 = torch.randn_like(input)
        theta_t = (1 - times_) * input + (times_ + self.noise_scale) * theta_1
        vector_field = theta_1 - input
        cond = self._embedding_net(condition)
        mu_t, std_t = self._stats(times.reshape(-1))
        v_out = self.net((theta_t - mu_t) / std_t, cond, times.reshape(-1))
        target = (vector_field + self.mean_0.view(1, -1)) / torch.sqrt(1 + self.std_0.view(1, -1) ** 2)
        return torch.mean((v_out - target) ** 2, dim=-1)


def build_flow_matching_estimator(batch_x, batch_y, hidden_features=100, num_layers=5, time_embedding_dim=32):
    """vector_field_nets.py:136-338 with the FMPE defaults (mlp, sinusoidal time embedding max_freq 1000)."""
    net = VectorFieldMLP(batch_x[0].numel(), batch_y[0].numel(), time_embedding_dim, hidden_features, num_layers)
    mean_0, std_0 = z_standardization(batch_x, False)
    emb = nn.Sequential(standardizing_net(batch_y, False), nn.Identity())
    return FlowMatchingEstimator(net, batch_x[0].shape, batch_y[0].shape, emb, mean_0, std_0)


# ----------------------------------------------------------------------------- training loop
class ReferenceTrainer:
    """First-round NPE/NLE training exactly as the reference runs it on one device:
    sbi/inference/trainers/base.py:499-563 (get_dataloaders), :1060-1148
    (_run_training_loop), :1150-1193 (_train_epoch), :1195-1225 (_validate_epoch),
    :1254-1284 (_converged); loss = estimator.loss(theta, x)
    (npe/npe_base.py:542-575, calibration kernel = ones).
    """

    def __init__(self, build_fn, swap_roles: bool = False):
        self.build_fn = build_fn
        self.swap = swap_roles        # NLE: loss(x, condition=theta)
        self.net = None
        self.summary = dict(training_loss=[], validation_loss=[], epoch_durations_sec=[],
                            epochs_trained=[], best_validation_loss=[])

    def get_dataloaders(self, theta, x, training_batch_size=200, validation_fraction=0.1):
        masks = torch.ones(theta.shape[0], 1)
        dataset = data.TensorDataset(theta, x, masks)
        num_examples = theta.size(0)
        num_training_examples = int((1 - validation_fraction) * num_examples)
        num_validation_examples = num_examples - num_training_examples
        permuted_indices = torch.randperm(num_examples)
        self.train_indices = permuted_indices[:num_training_examples]
        self.val_indices = permuted_indices[num_training_examples:]
        train_loader = data.DataLoader(
            dataset, batch_size=min(training_batch_size, num_training_examples),
            drop_last=True, sampler=SubsetRandomSampler(self.train_indices.tolist()))
        val_loader = data.DataLoader(
            dataset, batch_size=min(training_batch_size, num_validation_examples),
            shuffle=False, drop_last=True, sampler=SubsetRandomSampler(self.val_indices.tolist()))
        return train_loader, val_loader

    def _losses(self, batch):
        theta_b, x_b = batch[0], batch[1]
        if self.swap:
            loss = self.net.loss(x_b, theta_b)
        else:
            loss = self.net.loss(theta_b, x_b)
        assert torch.isfinite(loss).all(), "NaN/Inf present in loss."
        return loss

    def train(self, theta, x, training_batch_size=200, learning_rate=5e-4,
              validation_fraction=0.1, stop_after_epochs=20, max_num_epochs=2 ** 31 - 1,
              clip_max_norm: Optional[float] = 5.0):
        train_loader, val_loader = self.get_dataloaders(
            theta, x, training_batch_size, validation_fraction)
        if self.net is None:
            self.net = self.build_fn(theta[self.train_indices], x[self.train_indices])
        net = self.net
        optimizer = Adam(list(net.parameters()), lr=learning_rate)
        epoch, val_loss = 0, float("Inf")
        best_val, best_state, since = float("Inf"), None, 0

        def converged():
            nonlocal best_val, best_state, since
            c = False
            if epoch == 0 or val_loss < best_val:
                best_val = val_loss
                since = 0
                best_state = deepcopy(net.state_dict())
            else:
                since += 1
            if since > stop_after_epochs - 1:
                net.load_state_dict(best_state)
                c = True
            return c

        while epoch <= max_num_epochs and not converged():
            net.train()
            t0 = time.time()
            train_loss_sum = 0
            for batch in train_loader:
                optimizer.zero_grad()
                losses = self._losses(batch)
                loss = torch.mean(losses)
                train_loss_sum += losses.sum().item()
                loss.backward()
                if clip_max_norm is not None:
                    clip_grad_norm_(net.parameters(), max_norm=clip_max_norm)
                optimizer.step()
            train_loss = train_loss_sum / (len(train_loader) * train_loader.batch_size)
            net.eval()
            val_sum = 0
            with torch.no_grad():
                for batch in val_loader:
                    val_sum += self._losses(batch).sum().item()
            val_loss = val_sum / (len(val_loader) * val_loader.batch_size)
            self.summary["training_loss"].append(train_loss)
            self.summary["validation_loss"].append(val_loss)
            self.summary["epoch_durations_sec"].append(time.time() - t0)
            epoch += 1
        if epoch > max_num_epochs:
            if val_loss < best_val:
                best_val = val_loss
                best_state = deepcopy(net.state_dict())
            elif best_state is not None:
                net.load_state_dict(best_state)
        self.summary["epochs_trained"].append(epoch)
        self.summary["best_validation_loss"].append(best_val)
        net.zero_grad(set_to_none=True)
        return net


# ----------------------------------------------------------------------------- workload
def linear_gaussian_data(num_sims: int, dim: int, seed: int = 0):
    """Synthetic (theta, x) of the mini-sbibm `gaussian_linear` task
    (tests/mini_sbibm/gaussian_linear.py:30-32; simulator
    sbi/simulators/linear_gaussian.py:15-26): prior N(0, 0.1 I), x = theta + sqrt(0.1) eps."""
    g = torch.Generator().manual_seed(seed)
    theta = math.sqrt(0.1) * torch.randn(num_sims, dim, generator=g)
    x = theta + math.sqrt(0.1) * torch.randn(num_sims, dim, generator=g)
    return theta, x
