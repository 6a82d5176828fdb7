"""Neural posterior score estimation (NPSE, SURVEY 8f-3) on the sm_90a kernels.

The score network is the same `VectorFieldMLP` as FMPE's (vector_field_nets.py:610-719), so it runs on the
flow-matching kernels in their bare-network mode (`sbi_fm_model.raw = 1`): forward = `sbi_b200_fm_forward`,
parameter gradient for a given output gradient = `sbi_b200_fm_net_vjp`.  Everything AROUND the network is the
element-wise arithmetic of the reference's estimators, restated here in the reference's operation order:

* `ConditionalScoreEstimator`  /root/reference/sbi/neural_nets/estimators/score_estimator.py:15-528
  (forward :149-215: time-dependent z-scoring, Gaussian skip term, -mean_t/std_t output scaling; loss :230-316:
  denoising score matching with the control variate; weight functions :478-509; ode_fn :511-528),
* `VPScoreEstimator` :531-641, `SubVPScoreEstimator` :644-769, `VEScoreEstimator` :772-1097 (incl. the lognormal
  training schedule and the power-law solve schedule),
* `posterior_score_nn` /root/reference/sbi/neural_nets/factory.py (score estimators, `net="mlp"`),
  builder vector_field_nets.py:136-338 with `estimator_type="score"`.

`tests/test_score_cpu.py` swaps the kernel call for the reference's own network on the CPU and checks forward,
loss, schedules, drift / diffusion against the UNMODIFIED reference classes exactly.
"""
from __future__ import annotations

import math
import warnings
from typing import Any, Callable, Optional, Union

import torch
from torch import Tensor, nn

from . import _lib as L
from .flowmatching import FlowMatchingEstimator, build_vector_field_estimator


class _RawNet(torch.autograd.Function):
    """VectorFieldMLP(input_enc, condition, time_enc) on the kernels; gradient w.r.t. the parameters only."""

    @staticmethod
    def forward(ctx, flat, inp, cond, tenc, est):
        out = est._raw_forward(inp, cond, tenc)
        ctx.save_for_backward(inp, cond, tenc)
        ctx.est = est
        return out

    @staticmethod
    def backward(ctx, g):
        inp, cond, tenc = ctx.saved_tensors
        est = ctx.est
        R = inp.shape[0]
        n_part = L.load().sbi_b200_fm_vjp_parts(R)
        gpart = est._gpart(n_part)
        m = est._model(nbuf=2)
        g = g.contiguous().float()
        est._call("fm_net_vjp", m, L.rows(inp, cond, shared=cond.shape[0] == 1 and R > 1), tenc, g, gpart)
        return L.reduce_partials(gpart, n_part, est.layout.n_params), None, None, None, None


class ConditionalScoreEstimator(FlowMatchingEstimator):
    """score_estimator.py:15-528.  t = t_min is (almost) data, t = t_max is noise."""

    SCORE_DEFINED, SDE_DEFINED, MARGINALS_DEFINED = True, True, True
    IS_SCORE = True

    def __init__(self, layout, input_shape, condition_shape, mean_0, std_0, cond_stats, div_term,
                 embedding_net: Optional[nn.Module] = None, weight_fn: Union[str, Callable] = "max_likelihood",
                 beta_min: float = 0.01, beta_max: float = 10.0, t_min: float = 1e-3, t_max: float = 1.0):
        super().__init__(layout, input_shape, condition_shape, mean_0, std_0, cond_stats, div_term, embedding_net)
        if not self._embed_identity:
            raise NotImplementedError("the sm_90a score estimators take nn.Identity() embedding nets")
        self.t_min, self.t_max = t_min, t_max
        self.beta_min, self.beta_max = beta_min, beta_max
        self._set_weight_fn(weight_fn)
        # mean_0 / std_0 keep the reference's shapes: (D,) from z-scoring, (1,) for the scalar defaults
        m0 = mean_0 if isinstance(mean_0, Tensor) else torch.tensor([mean_0])
        s0 = std_0 if isinstance(std_0, Tensor) else torch.tensor([std_0])
        self.mean_0 = m0.clone().detach().float()
        self.std_0 = s0.clone().detach().float()
        t_tensor = torch.as_tensor([t_max], device=self.mean_0.device)
        self._mean_base = torch.broadcast_to(self.approx_marginal_mean(t_tensor), (1, *self._input_shape)).clone()
        self._std_base = torch.broadcast_to(self.approx_marginal_std(t_tensor), (1, *self._input_shape)).clone()

    # ---- the bare network on the kernels ------------------------------------------------------------------
    def _fill_model(self, s, ld: float):
        super()._fill_model(s, ld)
        s.raw = 1

    def _raw_forward(self, inp: Tensor, cond: Tensor, tenc: Tensor) -> Tensor:
        L.require_cuda(inp, "input")
        out = torch.empty_like(inp)
        m = self._model(nbuf=2)
        self._call("fm_forward", m, L.rows(inp, cond, shared=cond.shape[0] == 1 and inp.shape[0] > 1), tenc, 0, out)
        return out

    def _raw_forward_diag(self, inp: Tensor, cond: Tensor, tenc: Tensor):
        """(net(inp), diag of d net / d inp): `sbi_b200_fm_forward_div` in bare-network mode."""
        L.require_cuda(inp, "input")
        out, diag = torch.empty_like(inp), torch.empty_like(inp)
        m = self._model(nbuf=2)
        self._call("fm_forward_div", m, L.rows(inp, cond, shared=cond.shape[0] == 1 and inp.shape[0] > 1), tenc, 0,
                   out, diag)
        return out, diag

    def _net_call(self, input_enc: Tensor, condition: Tensor, time_enc: Tensor) -> Tensor:
        """`self.net(input_enc, condition_emb, time_enc)` of the reference (condition standardised in-kernel).
        input_enc (R, D), condition (R, C) or (1, C), time_enc (R,)."""
        return _RawNet.apply(self.net.flat, input_enc.contiguous().float(), condition.contiguous().float(),
                             time_enc.contiguous().float(), self)

    # ---- reference API (score_estimator.py:149-228) ---------------------------------------------------------
    def forward(self, input: Tensor, condition: Tensor, time: Tensor) -> Tensor:
        bs_in = input.shape[:-len(self.input_shape)]
        bs_c = condition.shape[:-len(self.condition_shape)]
        batch_shape = torch.broadcast_shapes(bs_in, bs_c)
        input = torch.broadcast_to(input, batch_shape + self.input_shape)
        time = torch.as_tensor(time, dtype=input.dtype, device=input.device)
        time = torch.broadcast_to(time, batch_shape)
        mean = self.approx_marginal_mean(time)
        std = self.approx_marginal_std(time)
        time_enc = self.std_fn(time)
        input_enc = (input - mean) / std
        score_gaussian = (input - mean) / std ** 2
        D, Cn = self.layout.D, self.layout.C
        shared = int(torch.Size(bs_c).numel()) == 1
        cond2 = condition.reshape(-1, Cn) if shared else torch.broadcast_to(
            condition, batch_shape + self.condition_shape).reshape(-1, Cn)
        score_pred = self._net_call(input_enc.reshape(-1, D), cond2, time_enc.reshape(-1))
        score_pred = score_pred.reshape(*batch_shape, *self.input_shape)
        scale = self.mean_t_fn(time) / self.std_fn(time)
        return -scale * score_pred - score_gaussian

    def score(self, input: Tensor, condition: Tensor, t: Tensor) -> Tensor:
        return self(input=input, condition=condition, time=t)

    def loss(self, input: Tensor, condition: Tensor, times: Optional[Tensor] = None, control_variate=True,
             control_variate_threshold=0.3) -> Tensor:
        """Denoising score matching loss (:230-316), (batch,)."""
        if times is None:
            times = self.train_schedule(input.shape[0])
        times = times.to(input.device)
        eps = torch.randn_like(input)
        mean = self.mean_fn(input, times)
        std = self.std_fn(times)
        input_noised = mean + std * eps
        score_target = -eps / std
        if control_variate:      # both network evaluations (noised input, mean) in one launch of 2 B rows
            both = self.forward(torch.stack((input_noised, mean)), condition, times)
            score_pred, score_mean_pred = both[0], both[1]
        else:
            score_pred = self.forward(input_noised, condition, times)
        weights = self.weight_fn(times)
        loss = torch.sum((score_pred - score_target) ** 2.0, dim=-1)
        if control_variate:
            D = input.shape[-1]
            s = torch.squeeze(std, -1)
            term1 = 2 / s * torch.sum(eps * score_mean_pred, dim=-1)
            term2 = torch.sum(eps ** 2, dim=-1) / s ** 2
            term3 = D / s ** 2
            cv = term3 - term1 - term2
            cv = torch.where(s < control_variate_threshold, cv, 0.0)
            loss = loss + cv
        return weights * loss

    def approx_marginal_mean(self, times: Tensor) -> Tensor:
        return self.mean_t_fn(times) * self.mean_0

    def approx_marginal_std(self, times: Tensor) -> Tensor:
        var = self.mean_t_fn(times) ** 2 * self.std_0 ** 2 + self.std_fn(times) ** 2
        return torch.sqrt(var)

    def mean_t_fn(self, times: Tensor) -> Tensor:
        raise NotImplementedError

    def mean_fn(self, x0: Tensor, times: Tensor) -> Tensor:
        return self.mean_t_fn(times) * x0

    def std_fn(self, times: Tensor) -> Tensor:
        raise NotImplementedError

    def drift_fn(self, input: Tensor, times: Tensor) -> Tensor:
        raise NotImplementedError

    def diffusion_fn(self, input: Tensor, times: Tensor) -> Tensor:
        raise NotImplementedError

    def noise_schedule(self, times: Tensor) -> Tensor:
        return self.beta_min + (self.beta_max - self.beta_min) * times

    def train_schedule(self, num_samples: int, t_min: Optional[float] = None, t_max: Optional[float] = None) -> Tensor:
        t_min = self.t_min if t_min is None else t_min
        t_max = self.t_max if t_max is None else t_max
        return torch.rand(num_samples, device=self._mean_base.device) * (t_max - t_min) + t_min

    def solve_schedule(self, num_steps: int, t_min: Optional[float] = None, t_max: Optional[float] = None) -> Tensor:
        t_min = self.t_min if t_min is None else t_min
        t_max = self.t_max if t_max is None else t_max
        return torch.linspace(t_max, t_min, num_steps, device=self._mean_base.device)

    def _set_weight_fn(self, weight_fn: Union[str, Callable]):
        if weight_fn == "identity":
            self.weight_fn = self._identity_weight_fn
        elif weight_fn == "max_likelihood":
            self.weight_fn = self._max_likelihood_weight_fn
        elif weight_fn == "variance":
            self.weight_fn = self._variance_weight_fn
        elif callable(weight_fn):
            self.weight_fn = weight_fn
        else:
            raise ValueError(f"Weight function {weight_fn} not recognized.")

    def _identity_weight_fn(self, times):
        return 1

    def _max_likelihood_weight_fn(self, times):
        return self.diffusion_fn(torch.ones((1,), device=times.device), times) ** 2

    def _variance_weight_fn(self, times):
        return self.std_fn(times) ** 2

    def ode_fn(self, input: Tensor, condition: Tensor, times: Tensor) -> Tensor:
        """Probability-flow ODE, f - 0.5 g^2 score (:511-528)."""
        score = self.score(input=input, condition=condition, t=times)
        f = self.drift_fn(input, times)
        g = self.diffusion_fn(input, times)
        return f - 0.5 * g ** 2 * score

    def drift_divergence(self, input: Tensor, times: Tensor) -> Tensor:
        """sum_i d f_i / d theta_i of `drift_fn`, (R,)."""
        raise NotImplementedError

    @torch.no_grad()
    def ode_fn_and_divergence(self, input: Tensor, condition: Tensor, times: Tensor):
        """(ode_fn, its exact divergence w.r.t. the input): what zuko's FreeFormJacobianTransform(exact=True)
        obtains by D autograd passes (zuko_ode.py:80-124), here from one forward-mode kernel launch that returns
        the diagonal of the network's input Jacobian.  input (R, D), condition (1, C) or (R, C), times (R,).
            score_i = -scale net_i(enc) - (x_i - mean_i) / std_i^2 ,  enc = (x - mean) / std
            d score_i / d x_i = -scale J_ii / std_i - 1 / std_i^2"""
        D, Cn = self.layout.D, self.layout.C
        x = input.reshape(-1, D).float()
        times = torch.as_tensor(times, dtype=x.dtype, device=x.device).expand(x.shape[0])
        mean = self.approx_marginal_mean(times)
        std = self.approx_marginal_std(times)
        time_enc = self.std_fn(times)
        input_enc = (x - mean) / std
        score_gaussian = (x - mean) / std ** 2
        net, diag = self._raw_forward_diag(input_enc.contiguous(), condition.reshape(-1, Cn).contiguous().float(),
                                           time_enc.reshape(-1).contiguous())
        scale = self.mean_t_fn(times) / self.std_fn(times)
        score = -scale * net - score_gaussian
        dscore = (-scale * diag / std - 1.0 / std ** 2).expand(x.shape).sum(-1)
        f = self.drift_fn(x, times)
        g = self.diffusion_fn(x, times)
        rhs = f - 0.5 * g ** 2 * score
        div = self.drift_divergence(x, times) - 0.5 * g.reshape(-1) ** 2 * dscore
        return rhs, div

    def loss_raw(self, *a, **k):
        raise NotImplementedError("the fused flow-matching loss kernel does not apply to score estimators")

    def forward_and_divergence(self, *a, **k):
        raise NotImplementedError("score estimators expose `ode_fn_and_divergence`")


class VPScoreEstimator(ConditionalScoreEstimator):
    """Variance-preserving SDE (DDPM), score_estimator.py:531-641."""

    def _ex(self, t: Tensor) -> Tensor:
        for _ in range(len(self.input_shape)):
            t = t.unsqueeze(-1)
        return t

    def mean_t_fn(self, times: Tensor) -> Tensor:
        return self._ex(torch.exp(-0.25 * times ** 2.0 * (self.beta_max - self.beta_min) - 0.5 * times * self.beta_min))

    def std_fn(self, times: Tensor) -> Tensor:
        std = 1.0 - torch.exp(-0.5 * times ** 2.0 * (self.beta_max - self.beta_min) - times * self.beta_min)
        return torch.sqrt(self._ex(std))

    def drift_fn(self, input: Tensor, times: Tensor) -> Tensor:
        phi = -0.5 * self.noise_schedule(times)
        while len(phi.shape) < len(input.shape):
            phi = phi.unsqueeze(-1)
        return phi * input

    def diffusion_fn(self, input: Tensor, times: Tensor) -> Tensor:
        g = torch.sqrt(self.noise_schedule(times))
        while len(g.shape) < len(input.shape):
            g = g.unsqueeze(-1)
        return g

    def drift_divergence(self, input: Tensor, times: Tensor) -> Tensor:
        return -0.5 * self.noise_schedule(times) * self.layout.D


class SubVPScoreEstimator(VPScoreEstimator):
    """Sub-variance-preserving SDE, score_estimator.py:644-769 (same mean and drift as VP; t_min defaults to 1e-2)."""

    def __init__(self, layout, input_shape, condition_shape, mean_0, std_0, cond_stats, div_term,
                 embedding_net: Optional[nn.Module] = None, weight_fn: Union[str, Callable] = "max_likelihood",
                 beta_min: float = 0.01, beta_max: float = 10.0, t_min: float = 1e-2, t_max: float = 1.0):
        super().__init__(layout, input_shape, condition_shape, mean_0, std_0, cond_stats, div_term, embedding_net,
                         weight_fn=weight_fn, beta_min=beta_min, beta_max=beta_max, t_min=t_min, t_max=t_max)

    def std_fn(self, times: Tensor) -> Tensor:
        std = 1.0 - torch.exp(-0.5 * times ** 2.0 * (self.beta_max - self.beta_min) - times * self.beta_min)
        return self._ex(std)

    def diffusion_fn(self, input: Tensor, times: Tensor) -> Tensor:
        g = torch.sqrt(torch.abs(self.noise_schedule(times) * (
            1 - torch.exp(-2 * self.beta_min * times - (self.beta_max - self.beta_min) * times ** 2))))
        while len(g.shape) < len(input.shape):
            g = g.unsqueeze(-1)
        return g


class VEScoreEstimator(ConditionalScoreEstimator):
    """Variance-exploding SDE (SMLD), score_estimator.py:772-1097."""

    def __init__(self, layout, input_shape, condition_shape, mean_0, std_0, cond_stats, div_term,
                 embedding_net: Optional[nn.Module] = None, weight_fn: Union[str, Callable] = "max_likelihood",
                 sigma_min: float = 1e-4, sigma_max: float = 10.0, t_min: float = 1e-3, t_max: float = 1.0,
                 train_schedule: str = "uniform", solve_schedule: str = "uniform", lognormal_mean: float = -1.2,
                 lognormal_std: float = 1.2, power_law_exponent: float = 7.0):
        if sigma_min <= 0:
            raise ValueError(f"sigma_min must be positive, got {sigma_min}")
        if sigma_max <= sigma_min:
            raise ValueError(f"sigma_max ({sigma_max}) must be greater than sigma_min ({sigma_min})")
        if train_schedule not in ("uniform", "lognormal"):
            raise ValueError(f"train_schedule must be one of ('uniform', 'lognormal'), got '{train_schedule}'")
        if solve_schedule not in ("uniform", "power_law"):
            raise ValueError(f"solve_schedule must be one of ('uniform', 'power_law'), got '{solve_schedule}'")
        if train_schedule == "lognormal" and lognormal_std <= 0:
            raise ValueError(f"lognormal_std must be positive, got {lognormal_std}")
        if solve_schedule == "power_law" and power_law_exponent <= 0:
            raise ValueError(f"power_law_exponent must be positive, got {power_law_exponent}")
        self.sigma_min, self.sigma_max = sigma_min, sigma_max
        self._train_schedule_type, self._solve_schedule_type = train_schedule, solve_schedule
        self.lognormal_mean, self.lognormal_std = lognormal_mean, lognormal_std
        self.power_law_exponent = power_law_exponent
        super().__init__(layout, input_shape, condition_shape, mean_0, std_0, cond_stats, div_term, embedding_net,
                         weight_fn=weight_fn, t_min=t_min, t_max=t_max)
        self._warn_on_inappropriate_config()

    def _warn_on_inappropriate_config(self) -> None:
        """Share of lognormal draws that the clamp to [sigma_min, sigma_max] will move (:880-905)."""
        if self._train_schedule_type != "lognormal":
            return
        z_lo = (math.log(self.sigma_min) - self.lognormal_mean) / self.lognormal_std
        z_hi = (math.log(self.sigma_max) - self.lognormal_mean) / self.lognormal_std
        frac_clamped = 1.0 - 0.5 * (math.erf(z_hi / math.sqrt(2)) - math.erf(z_lo / math.sqrt(2)))
        if frac_clamped > 0.05:
            warnings.warn(f"Lognormal schedule: ~{100 * frac_clamped:.1f}% of samples will be clamped to "
                          f"[{self.sigma_min}, {self.sigma_max}]. Consider adjusting lognormal_mean="
                          f"{self.lognormal_mean} or lognormal_std={self.lognormal_std}.", UserWarning, stacklevel=3)

    def _ex(self, t: Tensor) -> Tensor:
        for _ in range(len(self.input_shape)):
            t = t.unsqueeze(-1)
        return t

    def mean_t_fn(self, times: Tensor) -> Tensor:
        return self._ex(torch.ones_like(times, device=times.device))

    def std_fn(self, times: Tensor) -> Tensor:
        return self._ex(self.sigma_min * (self.sigma_max / self.sigma_min) ** times)

    def noise_schedule(self, times: Tensor) -> Tensor:
        return self.sigma_min * (self.sigma_max / self.sigma_min) ** times

    def drift_fn(self, input: Tensor, times: Tensor) -> Tensor:
        return torch.zeros(1, device=input.device)      # (a fill, not a host copy: legal inside graph capture)

    def drift_divergence(self, input: Tensor, times: Tensor) -> Tensor:
        return torch.zeros(1, device=input.device)

    def diffusion_fn(self, input: Tensor, times: Tensor) -> Tensor:
        sigma_ratio = self.sigma_max / self.sigma_min
        sigmas = self.noise_schedule(times)
        g = sigmas * math.sqrt((2 * math.log(sigma_ratio)))
        while len(g.shape) < len(input.shape):
            g = g.unsqueeze(-1)
        return g.to(input.device)

    def train_schedule(self, num_samples: int, t_min: Optional[float] = None, t_max: Optional[float] = None) -> Tensor:
        t_min = self.t_min if t_min is None else t_min
        t_max = self.t_max if t_max is None else t_max
        if t_min >= t_max:
            raise ValueError(f"t_min ({t_min}) must be less than t_max ({t_max}).")
        if self._train_schedule_type == "uniform":
            return torch.rand(num_samples, device=self._mean_base.device) * (t_max - t_min) + t_min
        log_sigma = self.lognormal_mean + self.lognormal_std * torch.randn(num_samples, device=self._mean_base.device)
        log_sigma_min, log_sigma_max = math.log(self.sigma_min), math.log(self.sigma_max)
        log_sigma_clamped = torch.clamp(log_sigma, log_sigma_min, log_sigma_max)
        unit = (log_sigma_clamped - log_sigma_min) / (log_sigma_max - log_sigma_min)
        return torch.clamp(unit * (t_max - t_min) + t_min, t_min, t_max)

    def solve_schedule(self, num_steps: int, t_min: Optional[float] = None, t_max: Optional[float] = None) -> Tensor:
        t_min = self.t_min if t_min is None else t_min
        t_max = self.t_max if t_max is None else t_max
        if t_min >= t_max:
            raise ValueError(f"t_min ({t_min}) must be less than t_max ({t_max}).")
        if self._solve_schedule_type == "uniform":
            return torch.linspace(t_max, t_min, num_steps, device=self._mean_base.device)
        rho = self.power_law_exponent
        steps = torch.linspace(0, 1, num_steps, device=self._mean_base.device)
        a, b = self.sigma_max ** (1.0 / rho), self.sigma_min ** (1.0 / rho)
        sigmas = (a + steps * (b - a)) ** rho
        unit = torch.log(sigmas / self.sigma_min) / math.log(self.sigma_max / self.sigma_min)
        times = unit * (t_max - t_min) + t_min
        times[0] = t_max
        if num_steps > 1:
            times[-1] = t_min
        return times


_SDE = {"vp": VPScoreEstimator, "subvp": SubVPScoreEstimator, "ve": VEScoreEstimator}


def build_score_estimator(batch_x: Tensor, batch_y: Tensor, sde_type: str = "ve", z_score_x: Optional[str] = "independent",
                          z_score_y: Optional[str] = "independent", embedding_net: nn.Module = nn.Identity(),
                          hidden_features: int = 100, time_embedding_dim: int = 32, num_layers: int = 5,
                          net: str = "mlp", **kwargs) -> ConditionalScoreEstimator:
    """vector_field_nets.py:136-338 with estimator_type='score', net='mlp': the network is built (and the torch RNG
    consumed) exactly like the flow-matching one; the estimator class follows `sde_type`."""
    if sde_type not in _SDE:
        raise ValueError(f"Unknown SDE type: {sde_type}")
    if net != "mlp":
        raise NotImplementedError("sbi_b200 implements net='mlp' score networks on sm_90a")
    fm = build_vector_field_estimator(batch_x, batch_y, estimator_type="flow", z_score_x=z_score_x, z_score_y=z_score_y,
                                      embedding_net=embedding_net, hidden_features=hidden_features,
                                      time_embedding_dim=time_embedding_dim, num_layers=num_layers, net="mlp")
    emb = fm._embedding_net
    cond_stats = (emb[0]._mean, emb[0]._std) if isinstance(emb, nn.Sequential) else None
    keys = {"ve": ("sigma_min", "sigma_max", "train_schedule", "solve_schedule", "lognormal_mean", "lognormal_std",
                   "power_law_exponent"), "vp": ("beta_min", "beta_max"), "subvp": ("beta_min", "beta_max")}[sde_type]
    est_kw = {k: kwargs[k] for k in keys if k in kwargs}
    zx = z_score_x not in (None, "none", False)
    mean_0 = fm.mean_0.reshape(-1).clone() if zx else 0.0
    std_0 = fm.std_0.reshape(-1).clone() if zx else 1.0
    est = _SDE[sde_type](fm.layout, batch_x[0].shape, batch_y[0].shape, mean_0, std_0, cond_stats,
                         fm.net._div_term.clone(), embedding_net, **est_kw)
    with torch.no_grad():
        est.net.flat.copy_(fm.net.flat)
    return est


def posterior_score_nn(model: str = "mlp", sde_type: str = "ve", z_score_theta: Optional[str] = "independent",
                       z_score_x: Optional[str] = "independent", hidden_features: int = 100, num_layers: int = 5,
                       embedding_net: nn.Module = nn.Identity(), time_emb_type: str = "sinusoidal",
                       t_embedding_dim: int = 32, compose_standardization: bool = False, **kwargs: Any) -> Callable:
    """The reference's `posterior_score_nn` (factory.py:433-530): build function for a score estimator of
    p(theta | x)."""
    if time_emb_type != "sinusoidal" or compose_standardization:
        raise NotImplementedError("sinusoidal time embedding without composed standardization only")

    def build_fn(batch_theta, batch_x):
        from ._refabc import register_with_reference
        register_with_reference()
        return build_score_estimator(batch_x=batch_theta, batch_y=batch_x, sde_type=sde_type, z_score_x=z_score_theta,
                                     z_score_y=z_score_x, embedding_net=embedding_net, hidden_features=hidden_features,
                                     time_embedding_dim=t_embedding_dim, num_layers=num_layers, net=model,
                                     **kwargs)

    return build_fn
