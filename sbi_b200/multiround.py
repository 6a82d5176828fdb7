"""Multi-round losses on top of the sm_90a estimators (SURVEY 8f-2).

* `atomic_log_prob_proposal_posterior` -- NPE-C / APT atomic proposal correction
  (/root/reference/sbi/inference/trainers/npe/npe_c.py:356-440): every row of the batch is classified
  against `num_atoms - 1` contrastive thetas of the same batch under the current density estimator.
  The B x num_atoms evaluations are ONE launch of the flow's log-prob kernel (tensor-core kernel from
  256 rows) and, in training, one fused forward+backward launch with the soft-max weights as the
  per-row upstream gradient (`estimators._NsfLogProb`).
* `nre_a_loss`, `bnre_loss`, `nre_c_loss` -- the loss heads of NRE-A (AALR), BNRE and NRE-C on the
  classifier logits (/root/reference/sbi/inference/trainers/nre/nre_a.py:165-190, bnre.py:167-200,
  nre_c.py:168-243); the logits come from the ratio kernels (`ratio._RatioFn`).

The heads are a handful of element-wise torch ops on (B, num_atoms) device tensors; the work is in the
kernels they call.  `choices` (the contrastive indices) can be passed in so that a test can feed the
same draw to the reference and to this implementation.
"""
from __future__ import annotations

import math
import warnings
from typing import Optional

import torch
from torch import Tensor


def contrastive_choices(B: int, k: int, device, rows: Optional[tuple] = None) -> Tensor:
    """(n, k) indices j != i into a batch of B, distinct per row, uniform, for the batch rows
    i in [rows[0], rows[1]) (default: all B): same law as
    `torch.multinomial((1 - eye) / (B - 1), k, replacement=False)` (npe_c.py:379-381,
    nre_base.py:406-408) without the O(B^2) probability matrix: k draws without replacement from
    range(B-1), shifted past i."""
    lo, hi = rows if rows is not None else (0, B)
    n = hi - lo
    if B - 1 <= 4096:
        draws = torch.multinomial(torch.ones(n, B - 1, device=device), k, replacement=False)
    else:
        draws = torch.randint(0, B - 1, (n, k), device=device)
        while True:
            srt = draws.sort(dim=1).values
            dup = (srt[:, 1:] == srt[:, :-1]).any(dim=1)
            nd = int(dup.sum().item())
            if nd == 0:
                break
            draws[dup] = torch.randint(0, B - 1, (nd, k), device=device)
    own = torch.arange(lo, hi, device=device).unsqueeze(1)
    return draws + (draws >= own).long()


def clamp_num_atoms(num_atoms: int, batch_size: int) -> int:
    """`clamp_and_warn("num_atoms", ., 2, batch_size)` (sbiutils.py; npe_c.py:368-370)."""
    clamped = int(min(max(num_atoms, 2), batch_size))
    if clamped != num_atoms:
        warnings.warn(f"num_atoms={num_atoms} was clamped to {clamped} (batch size {batch_size}).", stacklevel=3)
    return clamped


def atomic_log_prob_proposal_posterior(net, prior, theta: Tensor, x: Tensor, masks: Tensor, num_atoms: int,
                                       use_combined_loss: bool = False,
                                       choices: Optional[Tensor] = None) -> Tensor:
    """log of the proposal posterior normalised over a discrete set of atoms (npe_c.py:356-440).

    theta (B, D), x (B, *) on the estimator's device; masks (B,) or (B, 1) is 1 for prior samples;
    returns (B,).  Gradients flow to the estimator's parameters through its log_prob."""
    B = theta.shape[0]
    num_atoms = clamp_num_atoms(num_atoms, B)
    if choices is None:
        choices = contrastive_choices(B, num_atoms - 1, theta.device)
    x2 = x.reshape(B, -1)
    repeated_x = x2.repeat_interleave(num_atoms, dim=0)                      # repeat_rows (npe_c.py:374)
    contrasting = theta[choices]                                             # (B, A-1, D)
    atomic_theta = torch.cat((theta[:, None, :], contrasting), dim=1).reshape(B * num_atoms, -1)
    log_prob_prior = prior.log_prob(atomic_theta).reshape(B, num_atoms)
    if not bool(torch.isfinite(log_prob_prior).all()):
        raise AssertionError("NaN/Inf present in prior eval.")
    cond = repeated_x.reshape(B * num_atoms, *net.condition_shape)
    log_prob_posterior = net.log_prob(atomic_theta.unsqueeze(0), cond).reshape(B, num_atoms)
    unnormalized = log_prob_posterior - log_prob_prior
    out = unnormalized[:, 0] - torch.logsumexp(unnormalized, dim=-1)
    if use_combined_loss:       # npe_c.py:426-438: maximum likelihood on the prior samples on top
        lp = net.log_prob(theta.unsqueeze(0), x.reshape(B, *net.condition_shape)).squeeze(0)
        out = masks.reshape(-1).to(lp.dtype) * lp + out
    return out


# ---------------------------------------------------------------------------------------- NRE heads
def nre_a_loss(logits: Tensor) -> Tensor:
    """Binary cross-entropy of NRE-A / AALR (nre_a.py:165-190).  logits (B, 2): column 0 the jointly
    drawn pair (label 1), column 1 the contrastive pair (label 0); the reference's flat vector alternates
    them, and BCELoss averages over all 2B entries."""
    flat = logits.reshape(-1)
    labels = torch.ones_like(flat)
    labels[1::2] = 0.0
    return torch.nn.BCELoss()(torch.sigmoid(flat), labels)


def bnre_loss(logits: Tensor, regularization_strength: float) -> Tensor:
    """NRE-A loss + balancing regulariser (bnre.py:167-200)."""
    flat = logits.reshape(-1)
    reg = (torch.sigmoid(flat[0::2]) + torch.sigmoid(flat[1::2]) - 1).mean().square()
    return nre_a_loss(logits) + regularization_strength * reg


def nre_c_loss(logits_marginal: Tensor, logits_joint: Tensor, gamma: float) -> Tensor:
    """Contrastive NRE loss (nre_c.py:168-243).  logits_marginal (B, K+1) and logits_joint (B, K) come
    from two independent contrastive draws; column 0 of each is the jointly drawn pair."""
    B, K = logits_joint.shape
    logits_marginal = logits_marginal[:, 1:]
    # (python floats instead of the reference's 0-d tensors: same fp32 values after the broadcast add, and no
    # host-to-device copy inside a CUDA-graph capture)
    loggamma = float(torch.tensor(gamma, dtype=logits_joint.dtype).log())
    logK = float(torch.tensor(K, dtype=logits_joint.dtype).log())
    col = torch.full((B, 1), logK, dtype=logits_joint.dtype, device=logits_joint.device)
    den_m = torch.concat([loggamma + logits_marginal, col], dim=-1)
    den_j = torch.concat([loggamma + logits_joint, col], dim=-1)
    log_prob_marginal = logK - torch.logsumexp(den_m, dim=-1)
    log_prob_joint = loggamma + logits_joint[:, 0] - torch.logsumexp(den_j, dim=-1)
    p_joint = gamma / (1 + gamma)
    p_marginal = 1 / (1 + gamma)
    return -torch.mean(p_marginal * log_prob_marginal + p_joint * log_prob_joint)


def assert_finite(t: Tensor, what: str):
    if not bool(torch.isfinite(t).all()):
        raise AssertionError(f"NaN/Inf present in {what}.")


def is_finite_number(v: float) -> bool:
    return math.isfinite(v)
