"""Binding to the reference's estimator ABCs and the device hop for its CPU shape probe.

sbi's trainers gate on `isinstance(estimator, ConditionalEstimator)` /
`ConditionalDensityEstimator` / `ConditionalVectorFieldEstimator`
(/root/reference/sbi/inference/trainers/base.py:690, :985, :999) and build the network from
CPU batches, probe it with two CPU rows (`test_posterior_net_for_multi_d_x`,
/root/reference/sbi/utils/user_input_checks.py:767-795, called at
trainers/npe/npe_base.py:702-706) and only then move it to the training device
(trainers/base.py:1087).  The estimators of this package are plain `nn.Module`s that do not
import sbi; when the user's process HAS imported sbi they are registered as virtual subclasses
of those ABCs (`abc.ABCMeta.register`), so an unmodified `sbi.inference.NPE(prior,
density_estimator=sbi_b200.posterior_nn("nsf"))` accepts them.

There is still no CPU compute path: a call on an estimator whose parameters are on the CPU is
evaluated by a temporary copy on the CUDA device (`hop_to_device`) and the result is copied
back; without a CUDA device it raises.
"""
from __future__ import annotations

import copy
import sys

import torch

_registered = set()


def register_with_reference() -> bool:
    """Idempotent; a no-op unless `sbi` is already imported by the caller's process."""
    if "sbi" not in sys.modules:
        return False
    try:
        from sbi.neural_nets.estimators import base as ref_base
    except Exception:   # a partial / foreign `sbi` module: nothing to bind to
        return False
    from .estimators import FlowEstimator
    from .flowmatching import FlowMatchingEstimator
    from .ratio import RatioEstimator
    pairs = [(ref_base.ConditionalDensityEstimator, FlowEstimator),
             (ref_base.ConditionalVectorFieldEstimator, FlowMatchingEstimator)]
    try:
        from sbi.neural_nets.ratio_estimators import RatioEstimator as RefRatio
        pairs.append((RefRatio, RatioEstimator))
    except Exception:
        pairs.append((ref_base.ConditionalEstimator, RatioEstimator))
    for abc_cls, ours in pairs:
        key = (id(abc_cls), ours)
        if key in _registered:
            continue
        if hasattr(abc_cls, "register"):
            abc_cls.register(ours)
        _registered.add(key)
    return True


#: rows up to which a call on a CPU-resident estimator is hopped to the device (the reference's
#: probe uses 2; its `check_*` helpers never use more than a handful)
HOP_MAX_ROWS = 64


def hop_device():
    if not torch.cuda.is_available():
        raise RuntimeError(
            "sbi_b200: the estimator's parameters are on the CPU and no CUDA device is available; "
            "the kernels only run on a CUDA (sm_90a) device and there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())


def hop_to_device(est, method: str, *tensors, **kw):
    """Evaluate `est.<method>(*tensors)` on a temporary device copy of a CPU-resident estimator
    (no gradients); results come back on the CPU."""
    rows = max((t.reshape(-1, t.shape[-1]).shape[0] if t.dim() > 1 else 1) for t in tensors)
    if rows > HOP_MAX_ROWS:
        raise RuntimeError(
            f"sbi_b200: `{method}` was called with {rows} rows while the estimator's parameters are on "
            "the CPU; move it with `.to('cuda')` (only the reference's small shape probes are hopped "
            "to the device; there is no CPU fallback)")
    dev = hop_device()
    with torch.no_grad():
        tmp = copy.deepcopy(est).to(dev)
        out = getattr(tmp, method)(*[t.to(dev) for t in tensors], **kw)
    return out.cpu() if isinstance(out, torch.Tensor) else tuple(o.cpu() for o in out)
