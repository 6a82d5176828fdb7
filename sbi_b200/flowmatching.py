"""Flow-matching posterior estimation (FMPE) on the sm_90a kernels.

`FlowMatchingEstimator` mirrors /root/reference/sbi/neural_nets/estimators/flowmatching_estimator.py
(loss :270-347, forward :205-268, ode_fn :349-372) for the default `VectorFieldMLP`
(/root/reference/sbi/neural_nets/net_builders/vector_field_nets.py:610-719, sinusoidal time
embedding :367-421); `posterior_flow_nn` / `build_vector_field_estimator` mirror
factory.py:531-620 and vector_field_nets.py:136-338 for `net="mlp"`, `estimator_type="flow"`.
`sample_ode` integrates d theta/dt = v(theta, t; x_o) from t=1 (noise) to t=0 with an adaptive
Dormand-Prince 5(4) scheme (atol 1e-6, rtol 1e-5 as the reference passes to zuko,
samplers/ode_solvers/zuko_ode.py:29-31, :80-124); every right-hand-side evaluation is one
`sbi_b200_fm_forward` launch over all particles.
"""
from __future__ import annotations

import math
import warnings
from typing import Any, Callable, Optional, Tuple

import torch
from torch import Tensor, nn

from . import _lib as L
from .estimators import PackedNet, Standardize, _PackedEstimator, _zscore_of
from .neural_nets import (_linear_init, check_data_device, standardizing_stats, z_score_parser,
                          z_standardization)
from .pack import FmLayout


class FlowMatchingEstimator(_PackedEstimator):
    """Rectified-flow vector field v(theta_t, t; x); t=0 is data, t=1 is noise."""

    SCORE_DEFINED, SDE_DEFINED, MARGINALS_DEFINED = True, True, True
    t_min, t_max = 0.0, 1.0

    def __init__(self, layout: FmLayout, input_shape, condition_shape, mean_0, std_0, cond_stats,
                 div_term: Tensor, embedding_net: Optional[nn.Module] = None, noise_scale: float = 1e-3):
        super().__init__()
        self._input_shape, self._condition_shape = torch.Size(input_shape), torch.Size(condition_shape)
        user = embedding_net if embedding_net is not None else nn.Identity()
        # identity embedding: the kernels z-score the raw condition themselves; otherwise the embedding net
        # (behind the condition z-score) runs in torch and the kernels see its output with identity statistics
        self._embed_identity = isinstance(user, nn.Identity)
        self._embedding_net = nn.Sequential(Standardize(*cond_stats), user) if cond_stats else user
        self.noise_scale = noise_scale
        self.register_buffer("mean_0", torch.as_tensor(mean_0, dtype=torch.float32).expand(input_shape).clone())
        self.register_buffer("std_0", torch.as_tensor(std_0, dtype=torch.float32).expand(input_shape).clone())
        self.register_buffer("_mean_base", torch.zeros(1, *self._input_shape))
        self.register_buffer("_std_base", torch.ones(1, *self._input_shape))
        # boundary-affine buffers of the reference base class (estimators/base.py:389-398); composed
        # standardization itself is not implemented (always False)
        self.register_buffer("_theta_shift", torch.zeros(1, *self._input_shape, dtype=torch.float32))
        self.register_buffer("_theta_scale", torch.ones(1, *self._input_shape, dtype=torch.float32))
        self.register_buffer("_compose_standardization", torch.tensor(False), persistent=True)
        self.net = PackedNet(layout, dict(_div_term=div_term), tail=[("time_emb.div_term", "_div_term")])
        self._cache = {}

    embedding_net = property(lambda self: self._embedding_net)

    # ---- kernel views: [mean_0 (Dp) | std_0 (Dp) | ctx_mean (Cp) | ctx_std (Cp) | div_term (TEp/2) | 4 pad]
    def _stat_widths(self):
        lay = self.layout
        return lay.Dp, lay.D, lay.Cp, lay.C, lay.TEp // 2 + 4

    def _stat_sources(self, raw_condition: bool):
        cond = _zscore_of(self._embedding_net) if self._embed_identity else None
        return (self.mean_0, self.std_0), cond, self.net._div_term

    def _fill_model(self, s, ld: float):
        s.noise_scale = self.noise_scale

    def _embed(self, condition: Tensor) -> Tensor:
        """(n, *condition_shape) -> (n, C): the context the kernels read.  Identity embedding: the raw condition
        (z-scored in-kernel); otherwise the embedding net runs in torch, with autograd when enabled."""
        n = condition.shape[0]
        if self._embed_identity:
            return condition.reshape(n, self.layout.C).float()
        return self._embedding_net(condition).reshape(n, -1).float()

    # ---- reference API -------------------------------------------------------------------------
    def forward(self, input: Tensor, condition: Tensor, time: Tensor) -> Tensor:
        """Velocity in ORIGINAL space (flowmatching_estimator.py:205-268); batch shapes broadcast.  The condition
        is embedded once per distinct condition row, before broadcasting."""
        L.require_cuda(input, "input")
        bs_in = input.shape[:-len(self.input_shape)]
        bs_c = condition.shape[:-len(self.condition_shape)]
        bshape = torch.broadcast_shapes(bs_in, bs_c)
        inp = torch.broadcast_to(input, bshape + self.input_shape).reshape(-1, self.layout.D).contiguous().float()
        R = inp.shape[0]
        shared = int(torch.Size(bs_c).numel()) == 1
        ctx = self._embed(condition.reshape(-1, *self.condition_shape))
        cond = ctx if shared else torch.broadcast_to(ctx.reshape(*bs_c, self.layout.C),
                                                     bshape + (self.layout.C,)).reshape(-1, self.layout.C)
        cond = cond.contiguous()
        time = torch.as_tensor(time, dtype=torch.float32, device=inp.device)
        t_shared = time.numel() == 1
        tt = time.reshape(1) if t_shared else torch.broadcast_to(time, bshape).reshape(-1)
        tt = tt.contiguous()
        v = torch.empty_like(inp)
        m = self._model(nbuf=2)
        self._call("fm_forward", m, L.rows(inp, cond, shared=shared), tt, 1 if t_shared else 0, v)
        return v.reshape(*bshape, *self.input_shape)

    def forward_and_divergence(self, input: Tensor, condition: Tensor, time: Tensor):
        """(v, sum_i dv_i/dtheta_i): the velocity in ORIGINAL space and its exact divergence w.r.t. the
        input, one kernel (csrc/fm.cu `fm_trace_kernel`: forward + D forward-mode tangents).  input (R, D),
        condition (R, *condition_shape) or (1, *condition_shape) (embedded here), time scalar or (R,)."""
        L.require_cuda(input, "input")
        inp = input.reshape(-1, self.layout.D).contiguous().float()
        R = inp.shape[0]
        cond = self._embed(condition.reshape(-1, *self.condition_shape)).contiguous()
        shared = cond.shape[0] == 1
        time = torch.as_tensor(time, dtype=torch.float32, device=inp.device)
        t_shared = time.numel() == 1
        tt = (time.reshape(1) if t_shared else time.reshape(-1)).contiguous()
        v = torch.empty_like(inp)
        div = torch.empty(R, dtype=torch.float32, device=inp.device)
        m = self._model(nbuf=2)
        self._call("fm_forward_div", m, L.rows(inp, cond, shared=shared), tt, 1 if t_shared else 0, v, div)
        return v, div

    def ode_fn(self, input: Tensor, condition: Tensor, times: Tensor) -> Tensor:
        """flowmatching_estimator.py:349-372: the flow's ODE right-hand side is the velocity itself."""
        return self.forward(input, condition, times)

    # ---- SDE view of the flow (flowmatching_estimator.py:374-469) ----------------------------
    mean_base = property(lambda self: self._mean_base)
    std_base = property(lambda self: self._std_base)

    # boundary affine of the reference base class (estimators/base.py:460-475); composition is off
    compose_enabled = property(lambda self: bool(self._compose_standardization))

    def to_z(self, theta: Tensor) -> Tensor:
        return (theta - self._theta_shift) / self._theta_scale

    def from_z(self, z: Tensor) -> Tensor:
        return self._theta_shift + self._theta_scale * z

    def log_abs_det(self) -> Tensor:
        return torch.log(self._theta_scale).sum()

    def score(self, input: Tensor, condition: Tensor, t: Tensor) -> Tensor:
        """grad_theta log p_t(theta | x) = (-(1 - t) v - theta) / (t + sigma_min)   (:374-399)."""
        t = torch.as_tensor(t, dtype=torch.float32, device=input.device)
        v = self.forward(input, condition, t)
        return (-(1 - t) * v - input) / (t + self.noise_scale)

    def drift_fn(self, input: Tensor, times: Tensor, effective_t_max: float = 0.99) -> Tensor:
        """f(t) = -theta / (1 - t), with 1 - t floored at 1 - effective_t_max   (:401-434)."""
        times = torch.as_tensor(times, dtype=input.dtype, device=input.device)
        return -input / torch.maximum(1 - times, torch.tensor(1 - effective_t_max).to(input))

    def diffusion_fn(self, input: Tensor, times: Tensor, effective_t_max: float = 0.99) -> Tensor:
        """g(t) = sqrt(2 (t + sigma_min) / (1 - t))   (:436-469)."""
        times = torch.as_tensor(times, dtype=input.dtype, device=input.device)
        return torch.sqrt(2 * (times + self.noise_scale)
                          / torch.maximum(1 - times, torch.tensor(1 - effective_t_max).to(times)))

    def solve_schedule(self, num_steps: int, t_min: Optional[float] = None, t_max: Optional[float] = None) -> Tensor:
        """Uniform grid from t_max down to t_min (estimators/base.py:605-624)."""
        t_min = self.t_min if t_min is None else t_min
        t_max = self.t_max if t_max is None else t_max
        return torch.linspace(t_max, t_min, num_steps, device=self._mean_base.device)

    def loss(self, input: Tensor, condition: Tensor, times: Optional[Tensor] = None, **kwargs) -> Tensor:
        """(batch,) flow-matching losses; flowmatching_estimator.py:270-347.  t ~ U(0,1) and
        theta_1 ~ N(0, I) are drawn with torch on the device in the reference's order; the embedding net's
        gradient flows through the kernel's condition gradient."""
        if times is None:
            times = torch.rand(input.shape[:-1], device=input.device, dtype=input.dtype)
        theta_1 = torch.randn_like(input)
        ctx = self._embed(condition.reshape(-1, *self.condition_shape))
        return _FmLoss.apply(self.net.flat, input.reshape(-1, self.layout.D).contiguous().float(), ctx.contiguous(),
                             times.reshape(-1).contiguous().float(), theta_1.reshape(-1, self.layout.D).contiguous(),
                             self).reshape(input.shape[:-1])

    def loss_raw(self, inp, cond, times, eps, index=None, R=None, g_const=0.0, gpart=None, loss_acc=None,
                 want_loss=True, gcond=None):
        """Fused loss forward+backward on (optionally index-gathered) rows; returns the per-row loss.  `gcond`
        (R, C): receives the gradient with respect to the condition rows."""
        R = (index.shape[0] if index is not None else inp.shape[0]) if R is None else R
        loss = torch.empty(R, dtype=torch.float32, device=inp.device) if want_loss else None
        n_part = L.load().sbi_b200_fm_vjp_parts(R)
        gpart = self._gpart(n_part) if gpart is None else gpart
        m = self._model(nbuf=2)
        self._call("fm_loss_vjp_cond", m, L.rows(inp, cond, index, R), times, eps, None, g_const, loss, gpart,
                   loss_acc, gcond)
        return loss, gpart, n_part


class _FmLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flat, inp, cond, times, eps, est: FlowMatchingEstimator):
        R = inp.shape[0]
        loss = torch.empty(R, dtype=torch.float32, device=inp.device)
        gpart = est._gpart(L.load().sbi_b200_fm_vjp_parts(R))
        m = est._model(nbuf=2)
        # forward value only: g = 0 (the partial gradients written are zeros)
        est._call("fm_loss_vjp", m, L.rows(inp, cond), times, eps, None, 0.0, loss, gpart, None)
        ctx.save_for_backward(inp, cond, times, eps)
        ctx.est = est
        return loss

    @staticmethod
    def backward(ctx, g):
        inp, cond, times, eps = ctx.saved_tensors
        est = ctx.est
        n_part = L.load().sbi_b200_fm_vjp_parts(inp.shape[0])
        gpart = est._gpart(n_part)
        m = est._model(nbuf=2)
        g = g.contiguous().float()
        gcond = torch.empty_like(cond) if ctx.needs_input_grad[2] else None
        est._call("fm_loss_vjp_cond", m, L.rows(inp, cond), times, eps, g, 0.0, None, gpart, None, gcond)
        gflat = L.reduce_partials(gpart, n_part, est.layout.n_params) if ctx.needs_input_grad[0] else None
        return gflat, None, gcond, None, None, None


def build_vector_field_estimator(
    batch_x: Tensor, batch_y: Tensor, estimator_type: str = "flow", z_score_x: Optional[str] = "independent",
    z_score_y: Optional[str] = "independent", embedding_net: nn.Module = nn.Identity(),
    hidden_features: int = 100, time_embedding_dim: int = 32, num_layers: int = 5, net: str = "mlp",
    gaussian_baseline: bool = False, compose_standardization: bool = False,
    sinusoidal_max_freq: float = 1000.0, **kwargs,
) -> FlowMatchingEstimator:
    """vector_field_nets.py:136-338 for estimator_type='flow', net='mlp' (the FMPE default).  The
    torch RNG is consumed in VectorFieldMLP's construction order (:653-683), so a seed gives the
    reference's initial weights (the output layer's weight is zero-initialised, :683)."""
    check_data_device(batch_x, batch_y)
    if estimator_type != "flow" or net != "mlp" or gaussian_baseline or compose_standardization:
        raise NotImplementedError("sbi_b200 implements estimator_type='flow', net='mlp' without gaussian "
                                  "baseline / composed standardization")
    # the network's condition width is the embedded size (get_numel on the raw batch_y, like the reference)
    with torch.no_grad():
        Cn = embedding_net(batch_y[:1]).numel()
    D, H = batch_x[0].numel(), int(hidden_features)
    lay = FmLayout(D=D, C=Cn, H=H, NL=num_layers, TE=time_embedding_dim)
    st = {}
    st["net.input_layer.weight"], st["net.input_layer.bias"] = _linear_init(H, D)
    st["net.condition_layer.weight"], st["net.condition_layer.bias"] = _linear_init(H, Cn)
    st["net.input_merge_layer.weight"], st["net.input_merge_layer.bias"] = _linear_init(H, 2 * H)
    for i in range(num_layers):
        st[f"net.layers.{i}.weight"], st[f"net.layers.{i}.bias"] = _linear_init(H, H)
    for i in range(num_layers):
        st[f"net.layers_norm.{i}.weight"], st[f"net.layers_norm.{i}.bias"] = torch.ones(H), torch.zeros(H)
    st["net.time_linear_layer.weight"], st["net.time_linear_layer.bias"] = _linear_init(H, time_embedding_dim)
    w, b = _linear_init(D, H)
    st["net.output_layer.weight"], st["net.output_layer.bias"] = torch.zeros_like(w), b
    div_term = torch.exp(torch.arange(0, time_embedding_dim, 2) * (-math.log(sinusoidal_max_freq) / time_embedding_dim))
    zx, sx = z_score_parser(z_score_x)
    mean_0, std_0 = z_standardization(batch_x.reshape(batch_x.shape[0], -1), sx) if zx else (0.0, 1.0)
    zy, sy = z_score_parser(z_score_y)
    cstats = standardizing_stats(batch_y, sy) if zy else None
    est = FlowMatchingEstimator(lay, batch_x[0].shape, batch_y[0].shape, mean_0, std_0, cstats, div_term,
                                embedding_net)
    with torch.no_grad():
        lay.pack(st, out=est.net.flat.data)
    return est


def posterior_flow_nn(model: str = "mlp", z_score_theta: Optional[str] = "independent",
                      z_score_x: Optional[str] = "independent", hidden_features: int = 100, num_layers: int = 5,
                      embedding_net: nn.Module = nn.Identity(), time_emb_type: str = "sinusoidal",
                      t_embedding_dim: int = 32, gaussian_baseline: bool = False,
                      compose_standardization: bool = False, **kwargs: Any) -> Callable:
    """factory.py:531-620."""
    if time_emb_type != "sinusoidal":
        raise NotImplementedError("only the sinusoidal time embedding (FMPE default) is implemented")

    def build_fn(batch_theta, batch_x):
        from ._refabc import register_with_reference
        register_with_reference()
        return build_vector_field_estimator(
            batch_x=batch_theta, batch_y=batch_x, z_score_x=z_score_theta, z_score_y=z_score_x,
            hidden_features=hidden_features, num_layers=num_layers, embedding_net=embedding_net,
            time_embedding_dim=t_embedding_dim, net=model, gaussian_baseline=gaussian_baseline,
            compose_standardization=compose_standardization, **kwargs)

    return build_fn


# ---- ODE sampling --------------------------------------------------------------------------------
_A = [[], [1 / 5], [3 / 40, 9 / 40], [44 / 45, -56 / 15, 32 / 9],
      [19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729],
      [9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656],
      [35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84]]
_C = [0.0, 1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0, 1.0]
_B5 = [35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84, 0.0]
_B4 = [5179 / 57600, 0.0, 7571 / 16695, 393 / 640, -92097 / 339200, 187 / 2100, 1 / 40]


@torch.no_grad()
def odeint_dopri5(f: Callable[[Tensor, float], Tensor], y0: Tensor, t0: float, t1: float, atol: float = 1e-6,
                  rtol: float = 1e-5, max_steps: int = 10_000) -> Tuple[Tensor, int]:
    """Adaptive Dormand-Prince 5(4) from t0 to t1 (either direction), one step size for the whole
    batch, error norm = RMS over all entries of err / (atol + rtol * max(|y|, |y_new|)).
    Returns (y(t1), number of right-hand-side evaluations)."""
    direction = 1.0 if t1 >= t0 else -1.0
    t, y = float(t0), y0
    h = direction * min(abs(t1 - t0), 0.05)
    k1 = f(y, t)
    nfe = 1
    for _ in range(max_steps):
        if (t1 - t) * direction <= 1e-12:
            break
        if (t + h - t1) * direction > 0:
            h = t1 - t
        ks = [k1]
        for i in range(1, 7):
            yi = y + h * sum(a * k for a, k in zip(_A[i], ks))
            ks.append(f(yi, t + _C[i] * h))
        nfe += 6
        y5 = y + h * sum(b * k for b, k in zip(_B5, ks))
        err = h * sum((b5 - b4) * k for b5, b4, k in zip(_B5, _B4, ks))
        tol = atol + rtol * torch.maximum(y.abs(), y5.abs())
        en = float(torch.sqrt(torch.mean((err / tol) ** 2)).item())
        if en <= 1.0:
            t, y, k1 = t + h, y5, ks[6]     # FSAL
        fac = 0.9 * (1.0 / max(en, 1e-10)) ** 0.2
        h = h * min(5.0, max(0.2, fac))
    return y, nfe


class DeviceDopri5:
    """Adaptive Dormand-Prince 5(4) with the step control on the device (csrc/ode.cu; restates the solver
    the reference delegates to, zuko.utils.odeint, behind zuko_ode.py:80-124).  One step is a fixed launch
    sequence -- 6 x [stage combination -> right-hand side] -> error norm -> accept / commit / next step
    size -- captured once as a CUDA graph; the host replays it and polls the `done` flag every `poll`
    steps (one sync per `poll` steps instead of one `.item()` per step).

    rhs(y: Tensor (n,), t_ptr: int, out: Tensor (n,)) launches the right-hand side on the current stream,
    reading its time from the device scalar at address `t_ptr`."""

    _OFF_TSTAGE, _I_NFE, _I_NSTEPS, _I_NACC, _I_DONE, _I_MAX = 6, 8, 9, 10, 11, 12

    def __init__(self, n: int, device, rhs: Callable, atol: float = 1e-6, rtol: float = 1e-5,
                 max_steps: int = 10_000, poll: int = 4, use_graph: bool = True):
        self.device = torch.device(device)
        self.n, self.rhs, self.atol, self.rtol, self.max_steps, self.poll = n, rhs, atol, rtol, max_steps, poll
        self.y = torch.empty(n, dtype=torch.float32, device=device)
        self.yi = torch.empty(n, dtype=torch.float32, device=device)
        self.y5 = torch.empty(n, dtype=torch.float32, device=device)
        self.k = torch.empty(7, n, dtype=torch.float32, device=device)
        self.red = torch.empty(L.load().sbi_b200_ode_red_size(n), dtype=torch.float32, device=device)
        self.ctrl = torch.zeros(16, dtype=torch.float32, device=device)
        self.ctrl_i = self.ctrl.view(torch.int32)
        self.t_ptr = self.ctrl.data_ptr() + 4 * self._OFF_TSTAGE
        self.t_stage = self.ctrl[self._OFF_TSTAGE:self._OFF_TSTAGE + 1]     # the same device scalar as a tensor
        self._host = torch.zeros(16, dtype=torch.float32).pin_memory()
        self.use_graph = use_graph
        self.graph = None

    def _stage(self, i: int):
        L.call("ode_stage", self.y, self.k, self.yi, self.n, i, self.ctrl)

    def _step(self):
        for i in range(1, 7):
            self._stage(i)
            self.rhs(self.yi, self.t_ptr, self.k[i])
        L.call("ode_error_commit", self.y, self.k, self.y5, self.red, self.n, self.ctrl)

    def solve(self, y0: Tensor, t0: float, t1: float):
        """Integrate from t0 to t1 (either direction); returns (y(t1) as a view of the solver's state,
        right-hand-side evaluations, steps, accepted steps)."""
        import numpy as np
        direction = 1.0 if t1 >= t0 else -1.0
        h0 = direction * min(abs(t1 - t0), 0.05)
        c = np.zeros(16, np.float32)
        c[0:6] = [t0, h0, t1, direction, self.atol, self.rtol]
        ci = c.view(np.int32)
        ci[self._I_NFE], ci[self._I_MAX] = 1, self.max_steps
        if abs(t1 - t0) <= 1e-12:
            ci[self._I_DONE] = 1
        self.ctrl.copy_(torch.from_numpy(c))
        self.y.copy_(y0.reshape(-1))
        self._stage(0)                                   # yi = y, t_stage = t0
        self.rhs(self.yi, self.t_ptr, self.k[0])         # k_0 (also sets the kernel's attributes before capture)
        if self.use_graph and self.graph is None:
            snap = (self.y.clone(), self.k[0].clone(), self.ctrl.clone())
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                self._step()                             # warm-up outside capture
            torch.cuda.current_stream(self.device).wait_stream(side)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=torch.cuda.Stream(device=self.device)):
                self._step()
            self.y.copy_(snap[0]); self.k[0].copy_(snap[1]); self.ctrl.copy_(snap[2])
        while True:
            for _ in range(self.poll):
                if self.graph is not None:
                    self.graph.replay()
                else:
                    self._step()
            self._host.copy_(self.ctrl, non_blocking=True)
            torch.cuda.current_stream(self.device).synchronize()
            hi = self._host.view(torch.int32)
            done = int(hi[self._I_DONE])
            if done:
                break
        if done == 2:
            warnings.warn(f"dopri5: max_steps={self.max_steps} reached at t={float(self._host[0]):.4f}", stacklevel=2)
        return self.y, int(hi[self._I_NFE]), int(hi[self._I_NSTEPS]), int(hi[self._I_NACC])


def _fm_rhs(est: FlowMatchingEstimator, cond: Tensor, R: int, with_div: bool):
    """Right-hand side launcher for DeviceDopri5: state = theta (R, D) [| log|det| (R)]; `cond` is the embedded
    condition, one row shared by all R rows or one row per state row."""
    D = est.layout.D
    m = est._model(nbuf=2)
    shared = cond.shape[0] == 1

    def rhs(y: Tensor, t_ptr: int, out: Tensor):
        rows = L.rows(y, cond, n=R, shared=shared)
        if with_div:
            est._call("fm_forward_div", m, rows, t_ptr, 1, out, out.data_ptr() + 4 * R * D)
        else:
            est._call("fm_forward", m, rows, t_ptr, 1, out)
    return rhs


def _generic_rhs(est, cond: Tensor, R: int, with_div: bool, solver: "DeviceDopri5"):
    """Right-hand side for estimators whose ODE is `ode_fn` around the network kernel (score estimators,
    score.py): the element-wise arithmetic runs as torch ops on the solver's device-resident stage time, so
    the step still captures into one CUDA graph."""
    D = est.layout.D
    t_view = solver.t_stage

    def rhs(y: Tensor, t_ptr: int, out: Tensor):
        t = t_view.expand(R)
        th = y[:R * D].reshape(R, D)
        if with_div:
            f, dv = est.ode_fn_and_divergence(th, cond, t)
            out[:R * D].copy_(f.reshape(-1))
            out[R * D:].copy_(dv.reshape(-1))
        else:
            out.copy_(est.ode_fn(th, cond, t).reshape(-1))
    return rhs


def _make_solver(est, cond, R, n, dev, with_div, atol, rtol):
    """`cond`: the raw condition, (1, *condition_shape) shared by all R rows, or (B, *condition_shape) with state
    row r belonging to observation r % B.  The flow-matching kernels read the embedded condition, computed once
    per observation here and expanded to one row per state row."""
    B = cond.shape[0]
    if getattr(est, "IS_SCORE", False):
        solver = DeviceDopri5(n, dev, None, atol=atol, rtol=rtol)
        c = cond.reshape(B, -1)
        solver.rhs = _generic_rhs(est, (c if B == 1 else c.repeat(R // B, 1)).contiguous(), R, with_div, solver)
        return solver
    ctx = est._embed(cond.reshape(B, *est.condition_shape))
    ctx = (ctx if B == 1 else ctx.repeat(R // B, 1)).contiguous()
    return DeviceDopri5(n, dev, _fm_rhs(est, ctx, R, with_div), atol=atol, rtol=rtol)


@torch.no_grad()
def sample_ode(est: FlowMatchingEstimator, num_samples: int, condition: Tensor, atol: float = 1e-6,
               rtol: float = 1e-5, return_nfe: bool = False, device_control: bool = True, batched: bool = False):
    """Draw theta ~ q(theta | x): base N(mean_base, std_base) at t = t_max, integrate to t = t_min
    (VectorFieldPosterior.sample_via_ode, vector_field_posterior.py:436-465).  `device_control=False` keeps
    the host-side loop (`odeint_dopri5`) for comparison.  `batched=True`: `condition` holds B observations
    (B, *condition_shape) and the result is (num_samples, B, D), from ONE solve over all num_samples·B states with
    one step size for the whole state, as zuko's `odeint` takes it on a batched tensor."""
    dev = est.net.flat.device
    cond = condition.reshape(-1 if batched else 1, *est.condition_shape).to(dev).float()
    B = cond.shape[0]
    R = num_samples * B
    D = est.layout.D
    y0 = est._mean_base.to(dev) + est._std_base.to(dev) * torch.randn(R, D, device=dev)
    if not device_control:
        rows = cond if B == 1 else cond.repeat(num_samples, *([1] * len(est.condition_shape)))
        y, nfe = odeint_dopri5(lambda y, t: est.ode_fn(y, rows, torch.tensor(t, device=dev)), y0, est.t_max, est.t_min,
                               atol=atol, rtol=rtol)
    else:
        solver = _make_solver(est, cond, R, R * D, dev, False, atol, rtol)
        y, nfe, _, _ = solver.solve(y0, est.t_max, est.t_min)
        y = y.reshape(R, D).clone()
    if batched:
        y = y.reshape(num_samples, B, D)
    return (y, nfe) if return_nfe else y


@torch.no_grad()
def log_prob_ode(est: FlowMatchingEstimator, theta: Tensor, condition: Tensor, atol: float = 1e-6,
                 rtol: float = 1e-5, return_nfe: bool = False):
    """log q(theta | x) of the flow-matching posterior through the probability-flow ODE with the EXACT
    trace: integrate [theta, 0] from t_min to t_max with d log|det| / dt = div v, then
    log q = log N(z(t_max); mean_base, std_base) + log|det|   (zuko_ode.py:80-124 -> zuko
    NormalizingFlow(FreeFormJacobianTransform(exact=True), DiagNormal); vector_field_potential.py:145-212)."""
    dev = est.net.flat.device
    D = est.layout.D
    th = theta.reshape(-1, D).to(dev).float().contiguous()
    R = th.shape[0]
    cond = condition.reshape(1, *est.condition_shape).to(dev).float()
    y0 = torch.cat([th.reshape(-1), torch.zeros(R, device=dev)])
    solver = _make_solver(est, cond, R, R * D + R, dev, True, atol, rtol)
    y, nfe, _, _ = solver.solve(y0, est.t_min, est.t_max)
    z, ladj = y[:R * D].reshape(R, D), y[R * D:]
    mu, sd = est._mean_base.to(dev).reshape(1, D), est._std_base.to(dev).reshape(1, D)
    base = (-0.5 * ((z - mu) / sd) ** 2 - torch.log(sd) - 0.5 * math.log(2 * math.pi)).sum(1)
    lp = base + ladj
    return (lp, nfe) if return_nfe else lp


def factorised_iid_score(est, prior, theta: Tensor, cond: Tensor, t: Tensor, prior_score_weight=None) -> Tensor:
    """Score of the posterior given N iid observations, factorised approximation (FactorizedNPEScoreFunction,
    /root/reference/sbi/inference/potentials/vector_field_adaptor.py:725-813):
        sum_i score(theta | x_i, t) + (1 - N) w(t) grad_theta log prior(theta),   w(t) = (t_max - t) / t_max.
    theta (n, D), cond (N, C); the N per-observation scores of all n particles are ONE launch of n N rows."""
    n_iid = cond.shape[0]
    w = prior_score_weight(t) if prior_score_weight is not None else (est.t_max - t) / est.t_max
    with torch.enable_grad():          # compute_score (vector_field_adaptor.py:1329-1354)
        q = theta.detach().clone().requires_grad_(True)
        lp = prior.log_prob(q)
        prior_score = torch.autograd.grad(lp, q, grad_outputs=torch.ones_like(lp))[0].detach()
    base = est.score(theta[:, None, :], cond, t)                       # (n, N, D)
    return (1 - n_iid) * (w * prior_score) + base.sum(-2)


@torch.no_grad()
def sample_sde(est: FlowMatchingEstimator, num_samples: int, condition: Tensor, steps: int = 500,
               ts: Optional[Tensor] = None, eta: float = 1.0, fused: bool = True, corrector: Optional[str] = None,
               corrector_params: Optional[dict] = None, iid_method: Optional[str] = None, prior=None,
               iid_params: Optional[dict] = None, batched: bool = False) -> Tensor:
    """Draw theta ~ q(theta | x) with the reverse SDE, Euler-Maruyama predictor, no corrector
    (Diffuser.run, samplers/score/diffuser.py:124-180; EulerMaruyama.predict,
    samplers/score/predictors.py:112-120; driver VectorFieldPosterior._sample_via_diffusion,
    vector_field_posterior.py:331-433).  A step is [velocity kernel -> normal draw -> fused update kernel]
    (csrc/ode.cu `sde_em_step_kernel`), captured once as a CUDA graph and replayed for every grid point;
    `fused=False` keeps the step arithmetic in torch ops in the reference's order (for comparison).
    `corrector` in {None, "langevin", "gibbs"} (samplers/score/correctors.py) and several iid observations
    (`condition` of N rows, `iid_method="fnpe"`, inference/potentials/vector_field_adaptor.py:725-813) take the
    generic path: the same torch arithmetic as the reference around the network kernel.
    `batched=True`: `condition` holds B observations (B, *condition_shape), not iid trials; all num_samples·B
    particles (row n·B + b belongs to observation b) run in every step, and the result is (num_samples, B, D)."""
    assert eta > 0, "eta must be positive."
    dev = est.net.flat.device
    cond = condition.to(dev).float().reshape(-1, *est.condition_shape)
    B = cond.shape[0] if batched else 1
    n_iid = 1 if batched else cond.shape[0]
    R = num_samples * B
    if n_iid > 1 and iid_method != "fnpe":
        raise NotImplementedError(f"{n_iid} iid observations need iid_method='fnpe' (the factorised score, "
                                  "vector_field_adaptor.py:725-813); 'gauss' / 'auto_gauss' / 'jac_gauss' are not built")
    if n_iid > 1 and prior is None:
        raise AssertionError("Prior is required for iid methods.")
    ts = est.solve_schedule(steps) if ts is None else ts
    ts = ts.to(dev).float().contiguous()
    D = est.layout.D
    std0 = est._std_base.to(dev).reshape(1, D)
    if iid_method == "fnpe":        # Diffuser.initialize (diffuser.py:104-121) narrows the base for this method
        std0 = math.sqrt(1 / n_iid) * std0
    theta = est._mean_base.to(dev).reshape(1, D) + std0 * torch.randn(R, D, device=dev)
    score_of = lambda th, t: est.score(th, cond, t)
    if B > 1:       # (num_samples, B, D) against (1, B, C): each observation's condition is embedded once
        score_of = lambda th, t: est.score(th.reshape(num_samples, B, D), cond.unsqueeze(0), t).reshape(R, D)
    if n_iid > 1:
        w_fn = (iid_params or {}).get("prior_score_weight")
        score_of = lambda th, t: factorised_iid_score(est, prior, th, cond, t, w_fn)
    if corrector not in (None, "langevin", "gibbs"):
        raise NotImplementedError(f"corrector {corrector!r}: one of None, 'langevin', 'gibbs'")
    cp = dict(corrector_params or {})
    if not fused or corrector is not None or n_iid > 1 or getattr(est, "IS_SCORE", False):
        # generic path: the estimator's own score / drift / diffusion around the network kernel
        def predict(theta, t1, t0):            # EulerMaruyama.predict (predictors.py:112-120)
            dt = t1 - t0
            f = est.drift_fn(theta, t1)
            g = est.diffusion_fn(theta, t1)
            score = score_of(theta, t1)
            f_backward = f - (1 + eta ** 2) / 2 * g ** 2 * score
            return theta - f_backward * dt + (eta * g) * torch.randn_like(theta) * torch.sqrt(dt)

        def correct(theta, t0, t1):            # Diffuser.run calls corrector(samples, t_next, t_current)
            if corrector == "langevin":        # LangevinCorrector.correct (correctors.py:93-132): score at t1
                step = cp.get("step_size", 1e-4)
                std = math.sqrt(2 * step)
                for _ in range(cp.get("num_steps", 5)):
                    score = score_of(theta, t1)
                    theta = theta + step * score + std * torch.randn_like(theta)
                return theta
            for _ in range(cp.get("num_steps", 5)):   # GibbsCorrector (correctors.py:135-166): re-noise, predict back
                f = est.drift_fn(theta, t0)
                g = est.diffusion_fn(theta, t0)
                eps = torch.randn_like(theta)
                dt = t1 - t0
                theta = theta + f * dt + g * eps * torch.sqrt(dt)
                theta = predict(theta, t1, t0)
            return theta

        for i in range(1, ts.numel()):
            t1, t0 = ts[i - 1], ts[i]
            theta = predict(theta, t1, t0)
            if corrector is not None:
                theta = correct(theta, t0, t1)
        return theta.reshape(num_samples, B, D) if batched else theta
    theta = theta.contiguous()
    n = theta.numel()
    v = torch.empty_like(theta)
    z = torch.empty_like(theta)
    ctrl = torch.stack([ts[0], torch.ones((), device=dev)]).contiguous()       # [t_cur, next grid index]
    m = est._model(nbuf=2)
    cond = est._embed(cond)                       # x_o embedded once for all steps
    cond = (cond if B == 1 else cond.repeat(num_samples, 1)).contiguous()
    rows = L.rows(theta, cond, shared=B == 1)

    def step():
        est._call("fm_forward", m, rows, ctrl, 1, v)
        z.normal_()
        L.call("sde_em_step", theta, v, z, n, ts, ctrl, float(eta), float(est.noise_scale), 0.99)

    nsteps = ts.numel() - 1
    out = theta.reshape(num_samples, B, D) if batched else theta
    if nsteps < 1:
        return out
    step()                                        # first step eagerly (kernel attributes), the rest replayed
    if nsteps > 1:
        graph = torch.cuda.CUDAGraph()
        snap = (theta.clone(), ctrl.clone())
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            step()
        torch.cuda.current_stream(dev).wait_stream(side)
        theta.copy_(snap[0]); ctrl.copy_(snap[1])
        with torch.cuda.graph(graph, stream=torch.cuda.Stream(device=dev)):
            step()
        theta.copy_(snap[0]); ctrl.copy_(snap[1])
        for _ in range(nsteps - 1):
            graph.replay()
    return out
