"""The MMD misspecification test (reference sbi/diagnostics/misspecification.py:19-172) on sm_90a.

Is the observed data `x_o` something the simulator could have produced?  The test compares the median-heuristic
RBF MMD between `x_o` and simulated `x` with a permutation null: `n_shuffle` random splits of up to `max_samples`
simulations into an `n_obs`-row block and the rest.  The public functions keep the reference's signatures, return
types, error and warning texts.  The host draws every split with the reference's `torch.randperm(N)[:max_samples]`
calls, in its order and on the default generator, so a seed gives the reference's shuffles; the index table goes to
the device once, and every null statistic and the observed one come from one fixed sequence of launches
(csrc/mmd.cu): exact lower-median bandwidths by radix select, kernel sums combined in fp64 in a fixed order.

Differences from the reference: statistics are evaluated in fp32 from the inputs cast to fp32, with d^2 summed
directly rather than squared from `torch.cdist`, and combined in fp64 before the final rounding to fp32; there is no
CPU path.  `calc_misspecification_logprob` is not provided (it needs zuko-based marginal estimators).
"""
from __future__ import annotations

import warnings
from typing import Optional, Tuple

import torch
import torch.nn as nn
from torch import Tensor

from . import _lib

_MODES = ("biased", "unbiased")
_EMBED_CHUNK = 65536


def _cuda(t: Tensor, name: str) -> Tensor:
    """`t` as a contiguous fp32 tensor on a CUDA device (the kernels have no CPU path)."""
    if not t.is_cuda:
        if not torch.cuda.is_available():
            _lib.require_cuda(t, name)   # raises: no CPU fallback
        t = t.to("cuda")
    _lib.require_cuda(t, name)
    return t.float().contiguous()


def _check_pair(x: Tensor, y: Tensor):
    """The shape errors `torch.cdist` raises; batched (3-d and more) inputs are not supported."""
    for t, name in ((x, "X1"), (y, "X2")):
        if t.dim() < 2:
            raise RuntimeError(f"cdist only supports at least 2D tensors, {name} got: {t.dim()}D")
        if t.dim() > 2:
            raise NotImplementedError("the MMD kernels take 2-d (rows, features) inputs, got shape "
                                      f"{tuple(t.shape)}")
    if x.shape[1] != y.shape[1]:
        raise RuntimeError(f"X1 and X2 must have the same number of columns. X1: {x.shape[1]} X2: {y.shape[1]}")


def _mmd_sets(z: Tensor, table: Tensor, nxy: Tensor, mode: Optional[str] = "biased",
              bandwidth: Optional[float] = None) -> Tuple[Optional[Tensor], Tensor]:
    """MMDs (fp64, (S,)) and bandwidths (fp32, (S,)) of S index sets over the rows of `z` (R, D) on the device.

    Set s takes rows `table[s, :nx_s]` as X and `table[s, nx_s:nx_s + ny_s]` as Y, with `nxy[s] = (nx_s, ny_s)` (a
    host tensor).  The bandwidth is the lower median of the X-Y distances unless `bandwidth` is given; `mode=None`
    returns the bandwidths only."""
    S, L = (int(table.shape[0]), int(table.shape[1])) if table.dim() == 2 else (0, 0)
    R, D = int(z.shape[0]), int(z.shape[1])
    if not (1 <= S <= _lib.SBI_MMD_MAX_SETS and 1 <= L <= _lib.SBI_MMD_MAX_ROWS and 1 <= D and R < 2 ** 31):
        raise _lib.SbiB200Error(
            f"MMD: {S} index sets of {L} rows over a ({R}, {D}) matrix are outside the device envelope: 1 to "
            f"{_lib.SBI_MMD_MAX_SETS} sets of at most {_lib.SBI_MMD_MAX_ROWS} rows, at least one feature and "
            f"fewer than 2**31 rows")
    dev = z.device
    d_tab = table.to(device=dev, dtype=torch.int32).contiguous()
    d_nxy = nxy.to(device=dev, dtype=torch.int32).contiguous()
    bw = torch.empty(S, dtype=torch.float32, device=dev)
    if bandwidth is not None:
        bw.fill_(float(bandwidth))
    mmd = None if mode is None else torch.empty(S, dtype=torch.float64, device=dev)
    ws = torch.empty(max(1, _lib.load().sbi_b200_mmd_ws_bytes(S)), dtype=torch.uint8, device=dev)
    _lib.call("mmd", z, R, D, d_tab, L, d_nxy, S, int(nxy[:, 0].max()), int(nxy[:, 1].max()), int(mode == "unbiased"),
              int(bandwidth is not None), bw, mmd, ws)
    return mmd, bw


def _pair(x: Tensor, y: Tensor, mode: Optional[str], bandwidth: Optional[float] = None):
    _check_pair(x, y)
    z = torch.cat([_cuda(x, "x"), _cuda(y, "y")])
    nx, ny = int(x.shape[0]), int(y.shape[0])
    table = torch.arange(max(nx + ny, 1), dtype=torch.int32).unsqueeze(0)
    return _mmd_sets(z, table, torch.tensor([[nx, ny]]), mode, bandwidth)


def rbf_kernel(x: Tensor, y: Tensor, bandwidth: float):
    _check_pair(x, y)
    xd, yd = _cuda(x, "x"), _cuda(y, "y")
    out = torch.empty(x.shape[0], y.shape[0], dtype=torch.float32, device=xd.device)
    _lib.call("rbf_matrix", xd, xd.shape[0], yd, yd.shape[0], xd.shape[1], float(bandwidth), out)
    return out.to(x.device)


def median_heuristic(x: Tensor, y: Tensor):
    return _pair(x, y, None)[1].item()


def compute_rbf_mmd(x: Tensor, y: Tensor, bandwidth: float = 1.0, mode: str = "biased"):
    if mode not in _MODES:
        raise ValueError("mode should be either biased or unbiased")
    return _pair(x, y, mode, bandwidth)[0][0].float().to(x.device)


def compute_rbf_mmd_median_heuristic(x: Tensor, y: Tensor, mode: str = "biased"):
    """Median heuristic for bandwidth parameter.

    Described in
    `Large sample analysis of the median heuristic`, Garreau et al, 2018
    (https://arxiv.org/abs/1707.07269)
    """
    if mode not in _MODES:
        raise ValueError("mode should be either biased or unbiased")
    return _pair(x, y, mode)[0][0].float().to(x.device)


def shuffle_table(n: int, n_shuffle: int, max_samples: int) -> Tensor:
    """(n_shuffle, M) int64: the reference's `torch.randperm(n)[:max_samples]`, one call per shuffle, in order."""
    m = len(range(n)[:max_samples])
    if n_shuffle <= 0:
        return torch.empty(0, m, dtype=torch.int64)
    return torch.stack([torch.randperm(n)[:max_samples] for _ in range(n_shuffle)])


def _null_and_observed(z_obs: Optional[Tensor], z: Tensor, n_obs: int, n_shuffle: int, max_samples: int,
                       mode: str) -> dict:
    """Every null statistic, and with `z_obs` the observed one (`z_obs` against `z[:max_samples]`), in one call."""
    n = int(z.shape[0])
    if n_shuffle < 0:
        torch.zeros(n_shuffle)   # raises, as the reference's output buffer does
    if n_obs > n:
        raise ValueError("n of observed samples should be less than n of synthetic samples")
    if mode not in _MODES:
        if n_shuffle > 0:
            torch.randperm(n)   # the reference draws its first shuffle before it checks the mode
        raise ValueError("mode should be either biased or unbiased")
    if z_obs is not None:
        _check_pair(z_obs, z)
    elif z.dim() != 2:
        _check_pair(z, z)
    perms = shuffle_table(n, n_shuffle, max_samples)
    m = perms.shape[1]
    nx_null = min(max(n_obs, 0), m)
    rows = [perms.to(torch.int32)]
    nxy = [torch.tensor([[nx_null, m - nx_null]]).expand(perms.shape[0], 2)]
    zs = [_cuda(z, "x")]
    if z_obs is not None:
        obs_row = torch.cat([torch.arange(n, n + n_obs), torch.arange(m)]).to(torch.int32)
        width = max(m, obs_row.numel())
        rows = [torch.nn.functional.pad(rows[0], (0, width - m)), obs_row.unsqueeze(0)]
        nxy.append(torch.tensor([[n_obs, m]]))
        zs.append(_cuda(z_obs, "x_obs"))
    table = torch.cat(rows)
    mmd, bw = _mmd_sets(torch.cat(zs), table, torch.cat(nxy), mode)
    return dict(mmd=mmd, bandwidth=bw, table=perms, n_null=perms.shape[0])


def calculate_baseline_mmd(
    n_obs: int,
    y: Tensor,
    n_shuffle: int = 1_000,
    max_samples: int = 1_000,
    mode: str = "biased",
):
    """Calculates the MMD between two sets of synthetic data.

    Needed to compute the distribution of mmds under the null hypothesis
    that synthetic and observed samples come from the same distribution.

    Args:
        n_obs: number of observed data points,
            used to determine the number of samples for one set
        y: synthetic data
        n_shuffle: number of shuffles
        max_samples: maximum number of samples to use
        mode: mode of MMD calculation
    """
    if n_shuffle <= 0:
        mmds = torch.zeros(n_shuffle)
        if n_obs > y.shape[0]:
            raise ValueError("n of observed samples should be less than n of synthetic samples")
        return mmds
    out =_null_and_observed(None, y, n_obs, n_shuffle, max_samples, mode)
    return out["mmd"].float().cpu()


def _p_misspecification(x_obs: Tensor, x: Tensor, n_shuffle: int = 1_000, max_samples: int = 1_000,
                        mode: str = "biased") -> dict:
    """`calculate_p_misspecification` with the per-set bandwidths (null sets first, the observed set last) and the
    shuffle table beside the reference's outputs."""
    out = _null_and_observed(x_obs, x, int(x_obs.shape[0]), n_shuffle, max_samples, mode)
    k = out["n_null"]
    mmds_baseline = out["mmd"][:k].float().cpu()
    mmd = out["mmd"][k].float().to(x.device)
    p_val = 1 - (mmds_baseline < mmd.cpu()).sum().item() / n_shuffle
    return dict(p_val=p_val, mmds_baseline=mmds_baseline, mmd=mmd, bandwidths=out["bandwidth"], table=out["table"])


def calculate_p_misspecification(
    x_obs: Tensor,
    x: Tensor,
    n_shuffle: int = 1_000,
    max_samples: int = 1_000,
    mode: str = "biased",
):
    """Calculate the p-value of the misspecification test.

    Args:
        x_obs: observed data
        x: synthetic data
        n_shuffle: number of shuffles
        max_samples: maximum number of samples to use
        mode: mode of MMD calculation ("biased" or "unbiased")
    """
    out = _p_misspecification(x_obs, x, n_shuffle, max_samples, mode)
    return out["p_val"], (out["mmds_baseline"], out["mmd"])


def _embedding_device(net: nn.Module, inference, x: Tensor) -> torch.device:
    for t in list(net.parameters()) + list(net.buffers()):
        if t.is_cuda:
            return t.device
    if not torch.cuda.is_available():
        _lib.require_cuda(x, "x")   # raises: no CPU fallback
    dev = torch.device(getattr(inference, "_device", "cuda"))
    return dev if dev.type == "cuda" else torch.device("cuda")


def _embed(net: nn.Module, x: Tensor, dev: torch.device) -> Tensor:
    """The embedding net on the device, in chunks, without autograd."""
    with torch.no_grad():
        if x.shape[0] == 0:
            return net(x.to(dev)).detach()
        return torch.cat([net(x[i:i + _EMBED_CHUNK].to(dev)) for i in range(0, x.shape[0], _EMBED_CHUNK)])


def calc_misspecification_mmd(
    x_obs: Tensor,
    x: Tensor,
    inference=None,
    mode: str = "x_space",
    n_shuffle: int = 1_000,
    max_samples: int = 1_000,
    mmd_mode: str = "biased",
):
    """Misspecification test based on MMD in data- or embedding space.

    Args:
        x_obs: observed data
        x: synthetic data
        inference: sbi inference object (only used if mode == "embedding")
        mode: space of MMD calculation ("x_space" or "embedding")
        n_shuffle: number of shuffles for computing mmds under H_0
        max_samples: maximum number of samples to use
            (when we have too many synthetic samples x)
        mmd_mode: approximation of MMD calculation ("biased" or "unbiased")

    returns:
        p_val, (mmd_baseline,mmd): p-value of the misspecification test
        (MMDs under H_0, mmd)
    """
    if mode == "x_space":
        z_obs = x_obs
        z = x
    elif mode == "embedding":
        if inference is None:
            raise ValueError(
                "inference should not be None if mode is 'embedding'. "
                "Please provide an sbi inference object."
            )
        if getattr(inference, "_neural_net", None) is None:
            raise ValueError(
                "No neural net found. The inference object must be trained before "
                "computing the MMD in mode 'embedding'."
            )
        if isinstance(inference._neural_net.embedding_net, nn.modules.linear.Identity):
            warnings.warn(
                "The embedding net might be the identity function, "
                "in that case the MMD is computed in the x-space.",
                stacklevel=2,
            )
        if inference._neural_net.embedding_net is None:
            raise AttributeError(
                "embedding_net attribute is None but is required for misspecification"
                " detection."
            )
        net = inference._neural_net.embedding_net
        dev = _embedding_device(net, inference, x)
        z_obs = _embed(net, x_obs, dev)
        z = _embed(net, x, dev)
    else:
        raise ValueError("mode should be either 'x_space' or 'embedding'")

    p_val, (mmds_baseline, mmd) = calculate_p_misspecification(
        z_obs, z, n_shuffle=n_shuffle, max_samples=max_samples, mode=mmd_mode
    )
    return p_val, (mmds_baseline, mmd)
