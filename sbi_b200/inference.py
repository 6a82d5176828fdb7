"""Device-resident trainers and posteriors mirroring the reference's public API for the path.

`NPE` / `NLE` mirror `sbi.inference.NPE` (NPE-C, first round) and `sbi.inference.NLE`
(/root/reference/sbi/inference/trainers/npe/npe_base.py:81-418,
 /root/reference/sbi/inference/trainers/nle/nle_base.py:190-272) and the shared loop of
/root/reference/sbi/inference/trainers/base.py:499-563 (get_dataloaders), :1060-1148
(_run_training_loop), :1150-1225 (_train_epoch/_validate_epoch), :1254-1284 (_converged):

* same `append_simulations(theta, x).train(...)` / `build_posterior()` call sequence,
  argument names, defaults and stopping rule (validation loss, `stop_after_epochs`);
* same loss, optimiser (Adam, lr 5e-4), gradient clipping (5.0), 90/10 split, per-epoch
  reshuffle with `drop_last`, epoch-granular early stopping restoring the best weights.

What is different is where the work happens: the (theta, x) set lives in HBM, an epoch is ONE
CUDA-graph launch (steps_per_epoch x [fused fwd+bwd kernel -> partial-gradient reduce ->
clip+Adam kernel] + the validation pass), and the host reads three scalars per epoch instead
of syncing twice per step.

Every trainer runs the same loop (`_Trainer._run`), the same device optimizer step (`_DeviceAdam`) and the
same graph capture (`_capture`); a trainer supplies the body of one epoch.
"""
from __future__ import annotations

import math
import time
import warnings
from copy import deepcopy
from typing import Any, Callable, Dict, Optional, Union

import torch
from torch import Tensor, nn

from . import _lib as L
from .estimators import FlowEstimator, NSFEstimator, Standardize
from .neural_nets import likelihood_nn, posterior_nn


def _process_device(device: str) -> str:
    """torchutils.py:54-103 (subset): only CUDA devices are valid here."""
    if device in ("gpu", "cuda"):
        device = "cuda:0"
    if not str(device).startswith("cuda"):
        raise RuntimeError(
            f"sbi_b200 trains on a CUDA (sm_90a) device only; got device={device!r}. "
            "There is no CPU fallback.")
    if not torch.cuda.is_available():
        raise RuntimeError("sbi_b200: no CUDA device available (no CPU fallback)")
    return str(device)


def _embedding_nets(net) -> list:
    """The torch embedding nets an estimator runs ahead of its kernels: the flows' and vector fields' condition
    embedding, the ratio estimator's theta and x embeddings ([] where every embedding is the identity)."""
    if hasattr(net, "embedding_nets"):
        return list(net.embedding_nets)
    return [] if getattr(net, "_embed_identity", True) else [net.embedding_net]


def _embedding_params(net) -> list:
    """The trainable parameters of an estimator's torch embedding nets ([] for identity embeddings)."""
    seen, out = set(), []
    for emb in _embedding_nets(net):
        for p in emb.parameters():
            if p.requires_grad and id(p) not in seen:
                seen.add(id(p))
                out.append(p)
    return out


def _embedding_buffers(embs: list) -> list:
    """The embedding nets' buffers that training can change (e.g. BatchNorm statistics).  The z-score
    (`Standardize`) is fixed at build time and is left alone: writing it would invalidate the kernel statistics
    that captured graphs read."""
    return [b for emb in embs for m in emb.modules() if not isinstance(m, Standardize) for b in m.buffers(recurse=False)]


def _weights(net) -> list:
    """The tensors a best-epoch snapshot covers: the kernel parameters and the embedding nets' parameters and
    buffers (the reference deep-copies the whole state_dict, trainers/base.py:1127, :1275)."""
    embs = _embedding_nets(net)
    return [net.flat.data] + [p.data for emb in embs for p in emb.parameters()] + _embedding_buffers(embs)


class _DeviceAdam:
    """Clip + Adam (`clip_grad_norm_` + `Adam.step`, trainers/base.py:1181-1187) on a network's flat
    parameters, in the kernels of csrc/optim.cu.  With several ranks the gradient is first summed over
    them: through our NVLink peer-memory kernel on one node (graph-capturable), else with an NCCL
    all-reduce (eager launches).  The clip norm is always taken on the summed gradient.

    A torch embedding net's parameters join the same update (one clip norm, one step count, one Adam state,
    like `Adam(neural_net.parameters())` in the reference): the flat kernel parameters and the embedding
    parameters become views of one vector `[flat | embedding]`, and each embedding parameter's `.grad` a view
    of the matching gradient slice, which autograd accumulates into in place."""

    def __init__(self, net, state: Tensor, step: Tensor, lr: float, clip_max_norm: Optional[float], world: int):
        self.flat, self.mask = net.flat, net.net._mask
        self.P = net.layout.n_params
        self.state, self.count = state, step
        self.emb = _embedding_params(net)
        self.emb_buffers = _embedding_buffers(_embedding_nets(net)) if self.emb else []
        self.n = self.P + sum(p.numel() for p in self.emb)
        self.lr = lr
        self.max_norm = float(clip_max_norm) if clip_max_norm is not None else 0.0
        self.world = world
        self.peer = None
        if world > 1:
            from .parallel import make_gradient_exchange
            self.peer = make_gradient_exchange(self.P)      # None -> NCCL all-reduce
        dev = state.device
        self.grad = torch.zeros(self.P, dtype=torch.float32, device=dev)
        # the peer exchange reads this rank's gradient from a buffer of its own
        self.grad_local = torch.zeros(self.P, dtype=torch.float32, device=dev) if self.peer is not None else self.grad
        n_sumsq = self.peer.n_sumsq if self.peer is not None else L.load().sbi_b200_sumsq_blocks(self.P)
        self.sumsq = torch.zeros(n_sumsq, dtype=torch.float32, device=dev)
        self.params = None           # the joint parameter vector, with an embedding net
        if self.emb:
            if world > 1:
                raise NotImplementedError("data-parallel training with an embedding net is not implemented")
            if any(p.dtype != torch.float32 for p in self.emb):
                raise TypeError("the fused trainers train float32 embedding nets (the optimizer state is float32)")
            self.params = torch.cat([self.flat.data.reshape(-1)] + [p.data.reshape(-1).float() for p in self.emb])
            self.grad = torch.zeros(self.n, dtype=torch.float32, device=dev)
            self.mask = torch.cat([self.mask, torch.ones(self.n - self.P, dtype=self.mask.dtype, device=dev)])
            self.flat.data = self.params[:self.P]
            o = self.P
            for p in self.emb:
                k = p.numel()
                p.data = self.params[o:o + k].view_as(p)
                p.grad = self.grad[o:o + k].view_as(p)
                o += k

    def zero_grad(self):
        """Clear the embedding gradients before the next backward accumulates into them."""
        if self.emb:
            self.grad[self.P:].zero_()

    @property
    def capturable(self) -> bool:
        """Whether a step can be captured in a CUDA graph (not with the NCCL all-reduce)."""
        return self.world == 1 or self.peer is not None

    def step(self, grad: Tensor):
        """One update from a gradient that is complete on this rank (autograd).  With an embedding net, `grad` is
        the flat parameters' gradient; the embedding gradients are the ones autograd accumulated since
        `zero_grad`."""
        if self.emb:
            self.grad[:self.P].copy_(grad)
            self._adam(self.grad, 0)
            return
        if self.peer is not None:     # summed over NVLink peer memory, with the sum(g^2) partials
            self.peer.sum(grad, self.grad, self.mask, self.sumsq)
            self._adam(self.grad, self.peer.n_sumsq)
            return
        if self.world > 1:
            torch.distributed.all_reduce(grad)
        self._adam(grad, 0)

    def step_partials(self, gpart: Tensor, n_part: int):
        """One update from the `n_part` per-CTA partial gradients of a fused loss kernel (and, with an
        embedding net, the embedding gradients autograd accumulated since `zero_grad`)."""
        if self.emb:                  # the clip+Adam kernel takes the norm over [flat | embedding] itself
            L.call("reduce_partials", gpart, n_part, self.P, self.grad)
            self._adam(self.grad, 0)
            return
        if self.world == 1:           # the reduction kernel also emits the sum(g^2) partials
            L.call("reduce_partials_norm", gpart, n_part, self.P, self.grad, self.mask, self.sumsq)
            self._adam(self.grad, self.sumsq.shape[0])
            return
        L.call("reduce_partials", gpart, n_part, self.P, self.grad_local)
        self.step(self.grad_local)

    def _adam(self, grad: Tensor, n_sumsq: int):
        """n_sumsq > 0: `sumsq` already holds that many sum(g^2) partials of `grad`."""
        if self.emb:
            L.call("adam_clip_step", self.params, grad, self.state, self.count, self.mask, self.n,
                   self.lr, 0.9, 0.999, 1e-8, self.max_norm, 1.0)
            return
        if n_sumsq:
            L.call("adam_clip_step_norm", self.flat.data, grad, self.state, self.count, self.mask, self.P,
                   self.lr, 0.9, 0.999, 1e-8, self.max_norm, 1.0, self.sumsq, n_sumsq)
        else:
            L.call("adam_clip_step", self.flat.data, grad, self.state, self.count, self.mask, self.P,
                   self.lr, 0.9, 0.999, 1e-8, self.max_norm, 1.0)

    def _tensors(self):
        params = self.flat.data if self.params is None else self.params
        return [params, self.state, self.count] + self.emb_buffers

    def snapshot(self):
        return [t.clone() for t in self._tensors()]

    def restore(self, snap):
        for t, s in zip(self._tensors(), snap):
            t.copy_(s)

    def close(self):
        if self.emb:      # after training the parameters own their storage again; gradients are released
            self.flat.data = self.flat.data.clone()
            for p in self.emb:
                p.data = p.data.clone()
                p.grad = None
        if self.peer is not None:
            timed_out = self.peer.error()
            self.peer.close()
            if timed_out:
                raise RuntimeError("peer-memory gradient exchange timed out (a rank fell behind or died)")


def _capture(opt: _DeviceAdam, warmup: Callable, *fns: Callable) -> list:
    """One CUDA graph per function of `fns`.  `warmup()` runs first on a side stream (allocations, kernel
    attributes); the parameters and the optimizer state are rewound after it and after the capture, so
    neither changes the run."""
    snap = opt.snapshot()
    dev = opt.flat.device
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        warmup()
    torch.cuda.current_stream(dev).wait_stream(side)
    opt.restore(snap)
    graphs = []
    for fn in fns:
        graphs.append(torch.cuda.CUDAGraph())
        with torch.cuda.graph(graphs[-1], stream=torch.cuda.Stream(device=dev)):
            fn()
    opt.restore(snap)
    return graphs


class _Trainer:
    """State and training loop shared by all trainers (trainers/base.py:1060-1284)."""

    def __init__(self, prior, build_neural_net: Callable, device: str, show_progress_bars: bool = False):
        self._prior = prior
        self._device = _process_device(device)
        self._build_neural_net = build_neural_net
        self._neural_net = None
        self._theta: Optional[Tensor] = None
        self._x: Optional[Tensor] = None
        self._show_progress_bars = show_progress_bars
        self._round = 0
        self.epoch = 0
        self._val_loss = float("Inf")
        self._summary: Dict[str, list] = dict(
            epochs_trained=[], best_validation_loss=[], validation_loss=[], training_loss=[],
            epoch_durations_sec=[])
        self._dist = None   # (rank, world) when data-parallel
        self._partition = "global"
        self.train_indices = self.val_indices = None
        self._opt_state = self._opt_step = None
        # multi-round bookkeeping (npe_base.py:188-299): round of every appended block and its proposal
        self._data_round_index: list = []
        self._proposal_roundwise: list = []
        self._round_rows: list = []          # rows of every appended block
        self._mr_opt = self._mr_split_n = None

    # ------------------------------------------------------------------ data
    def data_parallel(self, partition: str = "global"):
        """Train data-parallel over the initialised `torch.distributed` group (one process per
        GPU, SURVEY 8e).  Replicas are identical: rank 0's initial network and statistics are
        broadcast when `train()` starts, each step's flat gradients are summed over the ranks
        (NVLink peer-memory kernel on one node, NCCL otherwise) and every rank applies the same
        deterministic clip + Adam, so the replicas stay bit-identical.

        partition="global" (SURVEY 8e): every rank holds the SAME simulations; the split and every
            epoch permutation come from rank 0, and rank r differentiates rows
            [r*B/G, (r+1)*B/G) of each global batch of `training_batch_size` rows, so batch
            composition, loss and update equal the single-GPU run (strong scaling).
        partition="local": every rank appends ITS OWN simulations and draws its own batches of
            `training_batch_size` rows (global batch = G x that; weak scaling)."""
        from . import parallel
        if partition not in ("global", "local"):
            raise ValueError("partition must be 'global' or 'local'")
        self._dist = parallel.world()
        self._partition = partition
        return self

    # ---- data-parallel helpers (no-ops on one process) ---------------------------------------------
    def _dp(self):
        """(rank, world size, whether the ranks share one global batch: partition='global')."""
        rank, world = self._dist if self._dist is not None else (0, 1)
        return rank, world, world > 1 and self._partition == "global"

    def _dp_agree(self, value: int, what: str):
        """All ranks must see the same `value` (step counts, set sizes): a mismatch would leave a
        rank waiting in a collective forever."""
        rank, world, _ = self._dp()
        if world == 1:
            return
        t = torch.tensor([value, -value], dtype=torch.int64, device=self._device)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        if int(t[0]) != value or int(-t[1]) != value:
            raise RuntimeError(f"data-parallel training needs the same {what} on every rank "
                               f"(this rank: {value}, max {int(t[0])}, min {int(-t[1])})")

    def _dp_split(self, N: int, n_train: int):
        """90/10 split indices (base.py:525-539); with partition='global' rank 0's split is used."""
        perm = torch.randperm(N)
        if self._dp()[2]:
            p = perm.to(self._device)
            torch.distributed.broadcast(p, 0)
            perm = p.cpu()
        return perm[:n_train], perm[n_train:]

    def _dp_sync_net(self, net):
        """Replicas start identical: parameters AND standardisation statistics of rank 0."""
        _, world, _ = self._dp()
        if world > 1:
            for t in list(net.parameters()) + list(net.buffers()):
                torch.distributed.broadcast(t.data, 0)
            net._cache.clear()

    def _dp_sum(self, values):
        """Sum of per-rank epoch statistics (list of floats), identical on every rank."""
        _, world, _ = self._dp()
        if world == 1:
            return values
        t = torch.tensor(values, dtype=torch.float64, device=self._device)
        torch.distributed.all_reduce(t)
        return t.tolist()

    def append_simulations(self, theta: Tensor, x: Tensor, proposal=None,
                           exclude_invalid_x: Optional[bool] = None, data_device: Optional[str] = None):
        """Store simulations (npe_base.py:188-299): float32 only, rows with NaN/Inf in x are
        dropped (user_input_checks.py:708-765, sbiutils.py:491-525)."""
        # round of this block (npe_base.py:224-241): prior samples, and draws of a `RestrictedPrior` of the prior
        # (TSNPE), are round 0; anything else opens a new round
        from .restriction import is_restricted_prior
        restricted = is_restricted_prior(proposal)
        if proposal is None or proposal is self._prior or (restricted and proposal._prior is self._prior):
            current_round = 0
        elif not self._data_round_index:
            current_round = 1
        else:
            current_round = max(self._data_round_index) + 1
        if current_round > 0:
            if self._prior is None:
                raise ValueError("You did not pass a prior at initialization, but now you passed a proposal. "
                                 "Multi-round inference needs a prior.")
            if getattr(proposal, "default_x", "unset") is None:     # check_if_proposal_has_default_x
                raise ValueError("`proposal.default_x` is None: call `proposal.set_default_x(x_o)` first.")
            if getattr(proposal, "posterior_estimator", None) is not None \
                    and proposal.posterior_estimator is self._neural_net:
                raise ValueError("The proposal's posterior_estimator is the same object as the trainer's "
                                 "neural network; use trainer.build_posterior() or a deepcopy.")
            if restricted:     # npe_base.py:600-609
                warnings.warn("The proposal you passed is a `RestrictedPrior`, but the proposal distribution it "
                              "uses is not the prior (it can be accessed via `RestrictedPrior._prior`). We do not "
                              "recommend to mix the `RestrictedPrior` with multi-round NPE.", stacklevel=2)
        if exclude_invalid_x is None:
            exclude_invalid_x = current_round == 0
        if theta.dtype != torch.float32 or x.dtype != torch.float32:
            raise AssertionError("theta and x must be float32")
        if theta.shape[0] != x.shape[0]:
            raise AssertionError("Number of parameter sets must equal number of simulation outputs")
        xf = x.reshape(x.shape[0], -1)
        ok = ~torch.isnan(xf).any(1) & ~torch.isinf(xf).any(1)
        if not bool(ok.all()):
            if exclude_invalid_x:
                warnings.warn(f"Found {int((~ok).sum())} invalid simulations; they are excluded.",
                              stacklevel=2)
                theta, x = theta[ok], x[ok]
            else:
                warnings.warn(f"Found {int((~ok).sum())} simulations with NaN/Inf; they are kept "
                              "(multi-round losses normalise across the batch).", stacklevel=2)
        theta = theta.reshape(theta.shape[0], -1)
        self._data_round_index.append(current_round)
        self._proposal_roundwise.append(proposal)
        self._round_rows.append(int(theta.shape[0]))
        th = theta.to(self._device).contiguous()
        xx = x.to(self._device).contiguous()
        if self._theta is None:
            self._theta, self._x = th, xx
        else:
            self._theta = torch.cat([self._theta, th])
            self._x = torch.cat([self._x, xx])
        return self

    def get_simulations(self):
        return self._theta, self._x

    # ------------------------------------------------------------------ training
    def _prepare(self, validation_fraction: float, training_batch_size: int, resume_training: bool,
                 retrain_from_scratch: bool = False):
        """Set-up of a first-round run (base.py:499-563, npe_base.py:674-708): the 90/10 split on the CPU
        global generator, the network built from the CPU training split, rank 0's replica on every rank.
        Returns (network, B, Bv, steps, vsteps): training / validation batch rows and steps per epoch."""
        if self._theta is None:
            raise RuntimeError("call append_simulations() first")
        dev = self._device
        N = self._theta.shape[0]
        if self._dp()[2]:
            self._dp_agree(N, "number of simulations")
        n_train = int((1 - validation_fraction) * N)
        n_val = N - n_train
        if not resume_training or self.train_indices is None:
            self.train_indices, self.val_indices = self._dp_split(N, n_train)
        if self._neural_net is None or retrain_from_scratch:
            tr = self.train_indices.to(dev)
            self._neural_net = self._build_neural_net(self._theta[tr].cpu(), self._x[tr].cpu())
        net = self._neural_net.to(dev)
        self._neural_net = net
        if not resume_training:
            self._dp_sync_net(net)
        B, Bv = min(training_batch_size, n_train), min(training_batch_size, n_val)
        steps, vsteps = n_train // B, (n_val // Bv if Bv > 0 else 0)
        self._dp_agree(steps, "number of steps per epoch")
        return net, B, Bv, steps, vsteps

    def _reset_epochs(self):
        self.epoch, self._val_loss = 0, float("Inf")
        self._best_val_loss, self._best_flat, self._epochs_since_last_improvement = float("Inf"), None, 0

    def _optimizer(self, net, learning_rate: float, clip_max_norm: Optional[float],
                   resume_training: bool) -> _DeviceAdam:
        """The device optimizer of this run; its Adam state and the epoch count carry over with `resume_training`."""
        if not resume_training or self._opt_state is None:
            P = net.layout.n_params + sum(p.numel() for p in _embedding_params(net))
            self._opt_state = torch.zeros(2 * P, dtype=torch.float32, device=self._device)
            self._opt_step = torch.zeros(2, dtype=torch.int32, device=self._device)
            self._reset_epochs()
        return _DeviceAdam(net, self._opt_state, self._opt_step, learning_rate, clip_max_norm, self._dp()[1])

    def _rank_rows(self, B: int):
        """This rank's share of a global batch of `B` rows: (rows it handles, offset of its first row in the
        batch, rows behind one update).  With partition='global' the ranks split every batch; otherwise every
        rank draws whole batches of its own."""
        rank, world, glob = self._dp()
        if not glob:
            return B, 0, B * world
        if B % world:
            raise ValueError(f"partition='global' needs the batch size ({B}) divisible by the "
                             f"number of ranks ({world})")
        return B // world, rank * (B // world), B

    def _epoch_orders(self, B: int, steps: int, Bv: int, vsteps: int):
        """(perm_buf, vperm_buf, fill): static buffers for the rows of an epoch's `steps` training batches of `B`
        and `vsteps` validation batches of `Bv`, and `fill()`, which draws the next epoch's orders into them
        (base.py:499-563: reshuffled every epoch, `drop_last`).  With partition='global' every rank takes rank
        0's orders."""
        dev = self._device
        glob = self._dp()[2]
        train_idx, val_idx = self.train_indices.to(dev), self.val_indices.to(dev)
        perm_buf = torch.empty(steps * B, dtype=torch.int64, device=dev)
        vperm_buf = torch.empty(vsteps * Bv, dtype=torch.int64, device=dev)

        def fill():
            perm_buf.copy_(train_idx[torch.randperm(train_idx.shape[0], device=dev)[:steps * B]])
            if vsteps > 0:
                vperm_buf.copy_(val_idx[torch.randperm(val_idx.shape[0], device=dev)[:vsteps * Bv]])
            if glob:
                torch.distributed.broadcast(perm_buf, 0)
                if vsteps > 0:
                    torch.distributed.broadcast(vperm_buf, 0)
        return perm_buf, vperm_buf, fill

    def _step_epochs(self, opt: _DeviceAdam, B: int, Bv: int, steps: int, vsteps: int,
                     train_step: Callable, val_step: Callable, graphs: bool) -> Callable:
        """Epochs of per-step launches (NRE, NPSE).  `train_step(idx)` / `val_step(idx)` read the batch rows
        from a static index buffer, filled before each step, so that with `graphs` one CUDA graph per
        optimisation step and one per validation step are captured and replayed: a step is many small
        launches that the host cannot issue as fast as the GPU runs them at small batches.  Random draws
        inside a graph use torch's graph-safe Philox offsets.  Returns the function that runs one epoch."""
        dev = self._device
        perm_buf, vperm_buf, fill = self._epoch_orders(B, steps, Bv, vsteps)
        # the warm-up and capture run on the first rows of each split
        idx_buf = self.train_indices[:B].to(dev)
        vidx_buf = self.val_indices[:Bv].to(dev)
        run_train, run_val = (lambda: train_step(idx_buf)), (lambda: val_step(vidx_buf))
        if graphs and steps > 0 and opt.capturable:
            def warmup():
                for _ in range(3):
                    run_train()
                if vsteps > 0:
                    run_val()
            captured = _capture(opt, warmup, run_train, *([run_val] if vsteps > 0 else []))
            run_train = captured[0].replay
            if vsteps > 0:
                run_val = captured[1].replay

        def epoch():
            fill()
            for buf, order, n, run in ((idx_buf, perm_buf, steps, run_train), (vidx_buf, vperm_buf, vsteps, run_val)):
                b = buf.shape[0]
                for s in range(n):
                    buf.copy_(order[s * b:(s + 1) * b])
                    run()
        return epoch

    def _epoch_losses(self, stats: Tensor):
        """The epoch's one host sync: (training, validation) loss sums from the accumulators [train sum,
        train non-finite count, validation sum, validation non-finite count], summed over the ranks."""
        tl, tb, vl, vb = self._dp_sum(stats.tolist())
        if tb > 0 or vb > 0:
            raise AssertionError(self._nan_message)
        return tl, vl

    def _converged(self, net, stop_after_epochs: int) -> bool:
        """base.py:1254-1284."""
        if self.epoch == 0 or self._val_loss < self._best_val_loss:
            self._best_val_loss, self._epochs_since_last_improvement = self._val_loss, 0
            self._save_best(net)
        else:
            self._epochs_since_last_improvement += 1
        if self._epochs_since_last_improvement > stop_after_epochs - 1:
            self._load_best(net)
            return True
        return False

    def _save_best(self, net):
        self._best_flat = [t.clone() for t in _weights(net)]

    def _load_best(self, net):
        for t, s in zip(_weights(net), self._best_flat):
            t.copy_(s)

    def _record_epoch(self, train_loss: float, val_loss: float):
        self._val_loss = val_loss
        self._summary["training_loss"].append(train_loss)
        self._summary["validation_loss"].append(val_loss)

    def _run(self, net, epoch: Callable, max_num_epochs: int, stop_after_epochs: int,
             opt: Optional[_DeviceAdam] = None):
        """The training loop (base.py:1060-1138).  `epoch()` trains and validates one epoch and returns
        (training loss, validation loss) after the epoch's one host sync."""
        while self.epoch <= max_num_epochs and not self._converged(net, stop_after_epochs):
            t0 = time.time()
            self._record_epoch(*epoch())
            self._summary["epoch_durations_sec"].append(time.time() - t0)
            self.epoch += 1
        if self.epoch > max_num_epochs:   # base.py:1122-1129
            if self._val_loss < self._best_val_loss:
                self._best_val_loss = self._val_loss
                self._save_best(net)
            elif self._best_flat is not None:
                self._load_best(net)
            warnings.warn(f"Maximum number of epochs `max_num_epochs={max_num_epochs}` reached, "
                          "but network has not yet fully converged.", stacklevel=3)
        self._summary["epochs_trained"].append(self.epoch)
        self._summary["best_validation_loss"].append(self._best_val_loss)
        net.zero_grad(set_to_none=True)
        if opt is not None:
            opt.close()

    @property
    def summary(self):
        return self._summary


class _PotentialPosterior:
    """`build_posterior` of the trainers whose estimator gives a potential (NLE: likelihood, NRE: ratio)."""

    def build_posterior(self, density_estimator=None, prior=None, sample_with: str = "mcmc",
                        mcmc_method: str = "slice_np_vectorized", mcmc_parameters: Optional[dict] = None,
                        rejection_sampling_parameters: Optional[dict] = None,
                        importance_sampling_parameters: Optional[dict] = None, **kwargs):
        """nle_base.py:274-378, nre_base.py:311-394 (`sample_with` in {"mcmc", "rejection", "importance"})."""
        from .posteriors import ImportanceSamplingPosterior, MCMCPosterior, RejectionPosterior
        est = deepcopy(density_estimator if density_estimator is not None else self._neural_net)
        prior = prior if prior is not None else self._prior
        potential_fn, theta_transform = self._potential(est, prior)
        if sample_with == "mcmc":
            return MCMCPosterior(potential_fn, proposal=prior, theta_transform=theta_transform, method=mcmc_method,
                                 device=self._device, **(mcmc_parameters or {}))
        if sample_with == "rejection":
            return RejectionPosterior(potential_fn, proposal=prior, device=self._device,
                                      **(rejection_sampling_parameters or {}))
        if sample_with == "importance":   # trainers/base.py:1045-1053
            return ImportanceSamplingPosterior(potential_fn, proposal=prior, device=self._device,
                                               **(importance_sampling_parameters or {}))
        raise NotImplementedError(sample_with)


class _FlowTrainer(_Trainer):
    """Shared first-round trainer for density estimators (NPE: q(theta|x); NLE: q(x|theta))."""

    _swap = False   # NLE: estimator input = x, condition = theta
    _nan_message = "NaN/Inf present in NPE loss."

    def __init__(self, prior=None, density_estimator: Union[str, Callable] = "nsf",
                 device: str = "cuda", logging_level: Union[int, str] = "WARNING",
                 summary_writer=None, tracker=None, show_progress_bars: bool = False):
        if isinstance(density_estimator, str):
            factory = likelihood_nn if self._swap else posterior_nn
            density_estimator = factory(model=density_estimator)
        super().__init__(prior, density_estimator, device, show_progress_bars)

    def _inp_cond(self):
        """(estimator input set, condition set) as (N, .) device tensors."""
        th, xx = self._theta, self._x.reshape(self._x.shape[0], -1)
        return (xx, th) if self._swap else (th, xx)

    def train(self, training_batch_size: int = 200, learning_rate: float = 5e-4,
              validation_fraction: float = 0.1, stop_after_epochs: int = 20,
              max_num_epochs: int = 2 ** 31 - 1, clip_max_norm: Optional[float] = 5.0,
              calibration_kernel: Optional[Callable] = None, resume_training: bool = False,
              force_first_round_loss: bool = False, discard_prior_samples: bool = False,
              retrain_from_scratch: bool = False, show_train_summary: bool = False,
              dataloader_kwargs: Optional[dict] = None) -> NSFEstimator:
        if calibration_kernel is not None and self._swap:
            raise ValueError("calibration_kernel is an argument of the posterior-estimator trainers (NPE)")
        self._round = max(self._data_round_index) if self._data_round_index else 0
        if self._round > 0 and not self._swap and not force_first_round_loss:
            # later rounds of NPE: atomic proposal correction (npe_c.py), eager steps
            return self._train_multiround(
                training_batch_size=training_batch_size, learning_rate=learning_rate,
                validation_fraction=validation_fraction, stop_after_epochs=stop_after_epochs,
                max_num_epochs=max_num_epochs, clip_max_norm=clip_max_norm, calibration_kernel=calibration_kernel,
                resume_training=resume_training, discard_prior_samples=discard_prior_samples,
                retrain_from_scratch=retrain_from_scratch)
        if self._round > 0 and discard_prior_samples:
            raise NotImplementedError("discard_prior_samples with the first-round loss is not implemented "
                                      "(append only the rounds to train on)")
        dev = self._device
        rank, world, glob = self._dp()
        net, B, Bv, steps, vsteps = self._prepare(validation_fraction, training_batch_size, resume_training,
                                                  retrain_from_scratch)
        if not isinstance(net, FlowEstimator):
            raise TypeError(f"{type(self).__name__} needs an sbi_b200 flow estimator, "
                            f"got {type(net).__name__}")
        embed = not net._embed_identity
        if embed and self._dist is not None:
            raise NotImplementedError("data-parallel training with an embedding net is not implemented")
        # a parameter-free or frozen embedding only transforms the condition: no condition gradient is needed
        train_emb = bool(_embedding_params(net))
        Bl, o_t, Btot = self._rank_rows(B)
        # validation rows: every rank evaluates its contiguous share of the epoch's validation order
        from .parallel import shard_range
        v_lo, v_hi = shard_range(vsteps * Bv, rank, world) if glob else (0, vsteps * Bv)
        opt = self._optimizer(net, learning_rate, clip_max_norm, resume_training)

        inp_all, cond_all = self._inp_cond()
        if hasattr(net, "with_dummy"):     # `made`: the network's dummy first feature (nn_utils.py:166-167)
            inp_all = net.with_dummy(inp_all).contiguous()
        # embedding net: the condition rows in their event shape (e.g. (N, 1, 50) for a Conv1d) go through
        # Standardize + the user's module in torch; the VJP kernel returns the gradient of the embedded context
        cond_raw = (self._theta if self._swap else self._x) if embed else None
        emb = net.embedding_net
        perm_buf, vperm_buf, fill = self._epoch_orders(B, steps, Bv, vsteps)
        cond_tc = train_emb and net.vjp_cond_uses_tc(Bl)
        n_part = net.vjp_parts(Bl, param_grads_only=cond_tc or not train_emb)
        gpart = net._gpart(n_part)
        gcond = torch.empty(Bl, net.layout.C, dtype=torch.float32, device=dev) if train_emb else None
        loss_acc = torch.zeros(2, dtype=torch.float32, device=dev)
        val_lp = torch.empty(max(vsteps * Bv, 1), dtype=torch.float32, device=dev)
        stats = torch.zeros(4, dtype=torch.float32, device=dev)   # train nll sum, bad, val nll sum, val bad

        # calibration kernel (npe_base.py:373-378, :563-575): loss_r = K(x_r) * (-log q_r); the weights of
        # all simulations are evaluated once, a step's upstream gradient is -K(x_r) / B per row
        w_all = None
        if calibration_kernel is not None:
            w_all = torch.as_tensor(calibration_kernel(self._x), dtype=torch.float32).reshape(-1).to(dev).contiguous()
            if w_all.shape[0] != self._theta.shape[0]:
                raise ValueError("calibration_kernel(x) must return one weight per simulation")
            g_rows = torch.empty(Bl, dtype=torch.float32, device=dev)
            lp_rows = torch.empty(Bl, dtype=torch.float32, device=dev)

        def run_epoch():
            """All kernels of one epoch on the current stream (graph-capturable)."""
            m_tr = net._model(nbuf=3)
            loss_acc.zero_()
            if embed:
                emb.train()
            for s in range(steps):
                idx = perm_buf[s * B + o_t:s * B + o_t + Bl]
                if embed:
                    opt.zero_grad()
                    with torch.set_grad_enabled(train_emb):
                        ctx = net._embed(cond_raw[idx]).contiguous()
                    inp_b = inp_all[idx]
                    rows = L.rows(inp_b, ctx, n=Bl)
                else:
                    rows = L.rows(inp_all, cond_all, idx, Bl)
                if w_all is None:
                    net.vjp(m_tr, rows, Bl, None, -1.0 / Btot, None, gpart, None, gcond, loss_acc, cond_tc=cond_tc)
                else:
                    w = w_all[idx]
                    torch.mul(w, -1.0 / Btot, out=g_rows)
                    net.vjp(m_tr, rows, Bl, g_rows, 0.0, lp_rows, gpart, None, gcond, None, cond_tc=cond_tc)
                    fin = torch.isfinite(lp_rows)
                    loss_acc[0] -= (torch.where(fin, lp_rows, torch.zeros_like(lp_rows)) * w).sum()
                    loss_acc[1] += (~fin).sum()
                if train_emb:
                    ctx.backward(gcond)
                opt.step_partials(gpart, n_part)
            stats[0:2].copy_(loss_acc)
            stats[2:4].zero_()
            if v_hi > v_lo:
                vrows = vperm_buf[v_lo:v_hi]
                vlp = val_lp[:v_hi - v_lo]
                # the estimator's log-prob dispatch (wgmma kernel for bulk rows, its operands re-packed from the
                # just-updated parameters), written into the static buffer the captured graph reads
                if embed:
                    emb.eval()
                    with torch.no_grad():
                        vctx = net._embed(cond_raw[vrows]).contiguous()
                    net._logprob_raw(inp_all[vrows], vctx, False, out=vlp)
                else:
                    net._logprob_raw(inp_all, cond_all, False, index=vrows, n_rows=v_hi - v_lo, out=vlp)
                if w_all is None:
                    # -sum of the finite log-probs and the count of non-finite ones, one fused launch
                    L.call("nll_stats", vlp, v_hi - v_lo, stats[2:])
                else:
                    fin = torch.isfinite(vlp)
                    stats[2] = -(torch.where(fin, vlp, torch.zeros_like(vlp)) * w_all[vrows]).sum()
                    stats[3] = (~fin).sum().float()

        # warm-up (also sets kernel attributes) on a throw-away copy of the state, then capture
        run = run_epoch
        if opt.capturable:
            rng = torch.cuda.get_rng_state(dev)      # the warm-up's permutation draw leaves no trace:
            fill()                                   # a seed gives the same run with and without graphs
            torch.cuda.set_rng_state(rng, dev)
            run = _capture(opt, run_epoch, run_epoch)[0].replay

        def epoch():
            fill()
            run()
            tl, vl = self._epoch_losses(stats)
            return tl / (steps * Btot), (vl / (vsteps * Bv * (1 if glob else world)) if vsteps > 0 else float("nan"))

        self._run(net, epoch, max_num_epochs, stop_after_epochs, opt)
        return deepcopy(net)

    def _train_multiround(self, training_batch_size, learning_rate, validation_fraction, stop_after_epochs,
                          max_num_epochs, clip_max_norm, calibration_kernel, resume_training,
                          discard_prior_samples, retrain_from_scratch):
        """Rounds > 0 of NPE-C (npe_c.py:126-231 + the shared loop of trainers/base.py:1060-1284): the
        network of the previous round keeps training on the simulations of all rounds with the atomic
        proposal-posterior loss.  Steps are eager (log-prob kernel -> soft-max head in torch -> fused
        forward+backward kernel through autograd -> clip_grad_norm_ -> Adam), exactly the reference's
        operation sequence; the B x num_atoms evaluations per step are what the kernels are for."""
        from .multiround import atomic_log_prob_proposal_posterior, clamp_num_atoms
        from .posteriors import prior_to_device
        if self._dp()[1] > 1:
            raise NotImplementedError("multi-round training is single-process")
        dev = self._device
        num_atoms = int(self._num_atoms)
        combined = bool(self._use_combined_loss)
        start_round = int(bool(discard_prior_samples) and self._round > 0)        # base.py _get_start_index
        rounds = torch.repeat_interleave(torch.as_tensor(self._data_round_index),
                                         torch.as_tensor(self._round_rows)).to(dev)
        sel = torch.nonzero(rounds >= start_round).reshape(-1)
        theta_all, x_all = self._theta[sel], self._x[sel]
        masks_all = (rounds[sel] == 0).to(torch.float32)                         # mask_sims_from_prior
        N = theta_all.shape[0]
        n_train = int((1 - validation_fraction) * N)
        n_val = N - n_train
        if not resume_training or self._mr_split_n != N:
            perm = torch.randperm(N)
            self.train_indices, self.val_indices = perm[:n_train], perm[n_train:]
            self._mr_split_n = N
        if self._neural_net is None or retrain_from_scratch:
            tr = self.train_indices.to(dev)
            self._neural_net = self._build_neural_net(theta_all[tr].cpu(), x_all[tr].cpu())
        net = self._neural_net.to(dev)
        self._neural_net = net
        prior = prior_to_device(self._prior, dev)
        B, Bv = min(training_batch_size, n_train), min(training_batch_size, n_val)
        steps, vsteps = n_train // B, (n_val // Bv if Bv > 0 else 0)
        if not resume_training or self._mr_opt is None:
            self._mr_opt = torch.optim.Adam(list(net.parameters()), lr=learning_rate)
            self._reset_epochs()
        opt = self._mr_opt
        train_idx, val_idx = self.train_indices.to(dev), self.val_indices.to(dev)
        w_all = None
        if calibration_kernel is not None:
            w_all = torch.as_tensor(calibration_kernel(x_all), dtype=torch.float32).reshape(-1).to(dev)

        def losses_of(idx):
            th, xx, mk = theta_all[idx], x_all[idx], masks_all[idx]
            lp = atomic_log_prob_proposal_posterior(net, prior, th, xx, mk, num_atoms, combined)
            if not bool(torch.isfinite(lp).all()):
                raise AssertionError(self._nan_message)
            return -lp if w_all is None else -lp * w_all[idx]

        def epoch():
            with warnings.catch_warnings():
                warnings.filterwarnings("ignore", message="num_atoms=")
                net.train()
                perm = train_idx[torch.randperm(n_train, device=dev)]
                tsum = torch.zeros((), device=dev)
                for s_ in range(steps):
                    opt.zero_grad()
                    losses = losses_of(perm[s_ * B:(s_ + 1) * B])
                    losses.mean().backward()
                    tsum += losses.detach().sum()
                    if clip_max_norm is not None:
                        torch.nn.utils.clip_grad_norm_(net.parameters(), max_norm=clip_max_norm)
                    opt.step()
                net.eval()
                vsum = torch.zeros((), device=dev)
                with torch.no_grad():
                    vperm = val_idx[torch.randperm(n_val, device=dev)] if vsteps > 0 else None
                    for s_ in range(vsteps):
                        vsum += losses_of(vperm[s_ * Bv:(s_ + 1) * Bv]).sum()
            val_loss = float(vsum.item()) / (vsteps * Bv) if vsteps > 0 else float("nan")
            return float(tsum.item()) / (steps * B), val_loss

        clamp_num_atoms(num_atoms, min(B, Bv) if vsteps > 0 else B)      # warn once, like the reference does per call
        self._run(net, epoch, max_num_epochs, stop_after_epochs)
        net._cache.clear()
        return deepcopy(net)


class NPE(_FlowTrainer):
    """Neural posterior estimation, first round (reference: NPE_C, npe_c.py:91 / npe_base.py)."""
    _swap = False

    def train(self, num_atoms: int = 10, training_batch_size: int = 200, learning_rate: float = 5e-4,
              validation_fraction: float = 0.1, stop_after_epochs: int = 20, max_num_epochs: int = 2 ** 31 - 1,
              clip_max_norm: Optional[float] = 5.0, calibration_kernel: Optional[Callable] = None,
              resume_training: bool = False, force_first_round_loss: bool = False,
              discard_prior_samples: bool = False, use_combined_loss: bool = False,
              retrain_from_scratch: bool = False, show_train_summary: bool = False,
              dataloader_kwargs: Optional[dict] = None):
        """npe_c.py:126-231 (same argument order): `num_atoms` / `use_combined_loss` only matter from the
        second round on (atomic proposal correction, `_train_multiround`)."""
        self._num_atoms, self._use_combined_loss = num_atoms, use_combined_loss
        return super().train(training_batch_size=training_batch_size, learning_rate=learning_rate,
                             validation_fraction=validation_fraction, stop_after_epochs=stop_after_epochs,
                             max_num_epochs=max_num_epochs, clip_max_norm=clip_max_norm,
                             calibration_kernel=calibration_kernel, resume_training=resume_training,
                             force_first_round_loss=force_first_round_loss,
                             discard_prior_samples=discard_prior_samples,
                             retrain_from_scratch=retrain_from_scratch, show_train_summary=show_train_summary,
                             dataloader_kwargs=dataloader_kwargs)

    def build_posterior(self, density_estimator: Optional[nn.Module] = None, prior=None,
                        sample_with: str = "direct", importance_sampling_parameters: Optional[dict] = None,
                        **kwargs):
        """npe_base.py:425-509 (`sample_with` in {"direct", "importance"})."""
        from .posteriors import DirectPosterior, ImportanceSamplingPosterior
        if sample_with not in ("direct", "importance"):
            raise NotImplementedError("NPE.build_posterior supports sample_with='direct' and 'importance'")
        est = density_estimator if density_estimator is not None else self._neural_net
        prior = prior if prior is not None else self._prior
        if sample_with == "importance":
            from .potentials import posterior_estimator_based_potential
            potential_fn, _ = posterior_estimator_based_potential(deepcopy(est).to(self._device), prior)
            return ImportanceSamplingPosterior(potential_fn, proposal=prior, device=self._device,
                                               **(importance_sampling_parameters or {}))
        return DirectPosterior(deepcopy(est), prior, device=self._device)


NPE_C = NPE
SNPE = NPE


class NLE(_PotentialPosterior, _FlowTrainer):
    """Neural likelihood estimation (reference: NLE_A, nle_base.py:190-272, _loss :380-392)."""
    _swap = True

    @staticmethod
    def _potential(est, prior):
        from .potentials import likelihood_estimator_based_potential
        return likelihood_estimator_based_potential(est, prior, x_o=None)


NLE_A = NLE
SNLE = NLE


# =================================================================================================
class NRE_B(_PotentialPosterior, _Trainer):
    """Neural ratio estimation, NRE-B / SRE (reference: trainers/nre/nre_base.py:184-309 train,
    :396-415 `_classifier_logits`; trainers/nre/nre_b.py:157-182 `_loss`): 1-out-of-`num_atoms`
    classification of the jointly drawn (theta, x) pair against `num_atoms - 1` contrastive thetas
    from the same batch.  The classifier forward / backward run in the ratio kernels; the contrastive
    index draw and the softmax head are a handful of torch device ops."""

    _nan_message = "NaN/Inf present in NRE-B loss."

    def __init__(self, prior=None, classifier: Union[str, Callable] = "resnet", device: str = "cuda",
                 logging_level: Union[int, str] = "warning", summary_writer=None, tracker=None,
                 show_progress_bars: bool = False):
        from .ratio import classifier_nn
        super().__init__(prior, classifier_nn(classifier) if isinstance(classifier, str) else classifier, device,
                         show_progress_bars)

    @staticmethod
    def _potential(est, prior):
        from .potentials import ratio_estimator_based_potential
        return ratio_estimator_based_potential(est, prior, x_o=None)

    @staticmethod
    def _contrastive_choices(B: int, k: int, device, rows: Optional[tuple] = None) -> Tensor:
        """(n, k) indices j != i into a batch of B, distinct per row, uniform, for the batch rows
        i in [rows[0], rows[1]) (default: all B): same law as
        `torch.multinomial((1 - eye) / (B - 1), k, replacement=False)` (nre_base.py:406-408) without the
        O(B^2) probability matrix: k draws without replacement from range(B-1), shifted past i."""
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

    def _embed_batch(self, net, idx: Tensor):
        """(theta rows, x rows) of the batch `idx` through the estimator's embedding nets, each embedded once (the
        reference embeds its B x num_atoms repeated rows, nre_base.py:396-415): None for a side whose embedding
        is the identity (its rows are gathered raw by the kernels), None altogether when both are."""
        if net._embed_theta_identity and net._embed_x_identity:
            return None
        th = None if net._embed_theta_identity else net.embed_theta(self._theta[idx])
        xx = None if net._embed_x_identity else net.embed_x(self._x[idx])
        return th, xx

    def _logits_on(self, net, idx: Tensor, num_atoms: int, choices: Optional[Tensor] = None,
                   rows: Optional[tuple] = None, emb: Optional[tuple] = None) -> Tensor:
        """`_classifier_logits` (nre_base.py:396-415) of the batch rows [rows[0], rows[1]) (default: all)
        of the batch `idx`: (n, num_atoms) logits, column 0 the jointly drawn pair; the contrastive thetas
        of a row come from the WHOLE batch (SURVEY 8e: with the global batch on every rank the
        data-parallel loss keeps the single-GPU semantics).  `emb`: the batch's embedded rows
        (`_embed_batch`); an embedded side is paired by its batch-local index."""
        from .ratio import _RatioFn
        B = idx.shape[0]
        lo, hi = rows if rows is not None else (0, B)
        if choices is None:
            choices = self._contrastive_choices(B, num_atoms - 1, idx.device, (lo, hi))
        local = torch.cat([torch.arange(lo, hi, device=idx.device).unsqueeze(1), choices], dim=1)   # (n, A)
        if emb is None:
            ti = idx[local].reshape(-1).contiguous()
            xi = idx[lo:hi].repeat_interleave(num_atoms).contiguous()
            return _RatioFn.apply(net.net.flat, self._theta, self._x2d, net, ti, xi, False).reshape(hi - lo, num_atoms)
        th_e, x_e = emb
        th, ti = (self._theta, idx[local]) if th_e is None else (th_e, local)
        if x_e is None:
            xx, xi = self._x2d, idx[lo:hi].repeat_interleave(num_atoms)
        else:
            xx, xi = x_e, torch.arange(lo, hi, device=idx.device).repeat_interleave(num_atoms)
        return _RatioFn.apply(net.net.flat, th, xx, net, ti.reshape(-1).contiguous(), xi.contiguous(), False,
                              x_e is not None).reshape(hi - lo, num_atoms)

    def _loss_on(self, net, idx: Tensor, num_atoms: int, choices: Optional[Tensor] = None,
                 rows: Optional[tuple] = None) -> Tensor:
        """NRE-B loss (nre_b.py:157-182): 1-out-of-`num_atoms` cross-entropy."""
        logits = self._logits_on(net, idx, num_atoms, choices, rows, self._embed_batch(net, idx))
        log_prob = logits[:, 0] - torch.logsumexp(logits, dim=-1)
        return -torch.mean(log_prob)

    def train(self, num_atoms: int = 10, training_batch_size: int = 200, learning_rate: float = 5e-4,
              validation_fraction: float = 0.1, stop_after_epochs: int = 20, max_num_epochs: int = 2 ** 31 - 1,
              clip_max_norm: Optional[float] = 5.0, resume_training: bool = False,
              discard_prior_samples: bool = False, retrain_from_scratch: bool = False,
              show_train_summary: bool = False, dataloader_kwargs: Optional[dict] = None):
        dev = self._device
        world = self._dp()[1]
        net, B, Bv, steps, vsteps = self._prepare(validation_fraction, training_batch_size, resume_training,
                                                  retrain_from_scratch)
        embs = net.embedding_nets
        if embs and self._dist is not None:
            raise NotImplementedError("data-parallel training with an embedding net is not implemented")
        self._x2d = self._x.reshape(self._x.shape[0], -1).contiguous()
        num_atoms = int(min(max(num_atoms, 2), min(B, Bv)))     # nre_base.py:236-238 (clamp to batch size)
        self._dp_agree(vsteps, "number of validation steps per epoch")
        # rows of each (global) batch whose loss this rank differentiates / evaluates
        Bl, o_t, _ = self._rank_rows(B)
        Bvl, o_v, _ = self._rank_rows(Bv)
        t_rows, v_rows = (o_t, o_t + Bl), (o_v, o_v + Bvl)
        opt = self._optimizer(net, learning_rate, clip_max_norm, resume_training)
        train_sum = torch.zeros((), device=dev)
        val_sum = torch.zeros((), device=dev)

        def train_step(idx):
            net.net.flat.grad = None
            for e in embs:
                e.train()
            opt.zero_grad()
            # every rank's rows weigh 1/world of the update's batch mean; gradients are summed
            loss = self._loss_on(net, idx, num_atoms, rows=t_rows) / world
            loss.backward()
            train_sum.add_(loss.detach())
            opt.step(net.flat.grad)

        def val_step(idx):
            for e in embs:
                e.eval()
            with torch.no_grad():
                val_sum.add_(self._loss_on(net, idx, num_atoms, rows=v_rows) / world)

        graphs = B - 1 <= 4096      # larger batches draw their contrastive rows with host syncs
        run_steps = self._step_epochs(opt, B, Bv, steps, vsteps, train_step, val_step, graphs)

        def epoch():
            train_sum.zero_()
            val_sum.zero_()
            run_steps()
            tl, vl = self._dp_sum([float(train_sum.item()), float(val_sum.item())])
            if not (math.isfinite(tl) and math.isfinite(vl)):
                raise AssertionError(self._nan_message)
            # the reference divides the sum of per-batch MEAN losses by steps * batch_size (SURVEY a15 quirk)
            return tl / (steps * B), (vl / (vsteps * Bv) if vsteps > 0 else float("nan"))

        self._run(net, epoch, max_num_epochs, stop_after_epochs, opt)
        return deepcopy(net)


SNRE_B = NRE_B
SNRE = NRE_B


class NRE_A(NRE_B):
    """AALR / NRE-A (reference: trainers/nre/nre_a.py:103-190): binary classification of the jointly drawn
    pair against ONE contrastive pair; same trainer, two atoms, BCE head."""

    def train(self, training_batch_size: int = 200, learning_rate: float = 5e-4, validation_fraction: float = 0.1,
              stop_after_epochs: int = 20, max_num_epochs: int = 2 ** 31 - 1, clip_max_norm: Optional[float] = 5.0,
              resume_training: bool = False, discard_prior_samples: bool = False, retrain_from_scratch: bool = False,
              show_train_summary: bool = False, dataloader_kwargs: Optional[dict] = None):
        return NRE_B.train(self, num_atoms=2, training_batch_size=training_batch_size, learning_rate=learning_rate,
                           validation_fraction=validation_fraction, stop_after_epochs=stop_after_epochs,
                           max_num_epochs=max_num_epochs, clip_max_norm=clip_max_norm,
                           resume_training=resume_training, discard_prior_samples=discard_prior_samples,
                           retrain_from_scratch=retrain_from_scratch, show_train_summary=show_train_summary,
                           dataloader_kwargs=dataloader_kwargs)

    def _loss_on(self, net, idx, num_atoms, choices=None, rows=None):
        from .multiround import nre_a_loss
        return nre_a_loss(self._logits_on(net, idx, 2, choices, rows, self._embed_batch(net, idx)))


SNRE_A = NRE_A
AALR = NRE_A


class BNRE(NRE_A):
    """Balanced NRE (reference: trainers/nre/bnre.py:103-200): NRE-A plus the balancing regulariser
    `regularization_strength * (E[sigmoid(l_joint) + sigmoid(l_marginal) - 1])^2`."""

    def train(self, regularization_strength: float = 100.0, training_batch_size: int = 200, **kwargs):
        self._regularization_strength = float(regularization_strength)
        if self._dp()[1] > 1:
            raise NotImplementedError("the balancing regulariser is a function of the batch mean: BNRE trains "
                                      "on one process")
        return NRE_A.train(self, training_batch_size=training_batch_size, **kwargs)

    def _loss_on(self, net, idx, num_atoms, choices=None, rows=None):
        from .multiround import bnre_loss
        return bnre_loss(self._logits_on(net, idx, 2, choices, rows, self._embed_batch(net, idx)),
                         self._regularization_strength)


class NRE_C(NRE_B):
    """Contrastive NRE (reference: trainers/nre/nre_c.py:103-259): `num_classes` = K contrastive classes
    and the odds `gamma` of a jointly drawn pair; two independent contrastive draws per step (K + 1 and K
    atoms)."""

    def train(self, num_classes: int = 5, gamma: float = 1.0, training_batch_size: int = 200, **kwargs):
        self._gamma = float(gamma)
        return NRE_B.train(self, num_atoms=num_classes + 1, training_batch_size=training_batch_size, **kwargs)

    def _loss_on(self, net, idx, num_atoms, choices=None, rows=None):
        from .multiround import nre_c_loss
        K = num_atoms - 1
        if K < 1:
            raise AssertionError(f"num_classes = {K} must be greater than 1.")
        cm, cj = (choices if choices is not None else (None, None))
        emb = self._embed_batch(net, idx)       # both draws pair the same embedded rows
        logits_marginal = self._logits_on(net, idx, K + 1, cm, rows, emb)
        logits_joint = self._logits_on(net, idx, K, cj, rows, emb)
        return nre_c_loss(logits_marginal, logits_joint, self._gamma)


SNRE_C = NRE_C


# =================================================================================================
class FMPE(_Trainer):
    """Flow-matching posterior estimation (reference: trainers/vfpe/fmpe.py, base_vf_inference.py:
    train :206-350, validation at fixed times :524-543, EMA-smoothed summaries :589-636, z-score of
    the loss as stopping rule :352-420)."""

    _nan_message = "NaN/Inf present in FMPE loss."

    def __init__(self, prior=None, density_estimator: Union[str, Callable] = "mlp", device: str = "cuda",
                 logging_level: Union[int, str] = "WARNING", summary_writer=None, tracker=None,
                 show_progress_bars: bool = False):
        from .flowmatching import posterior_flow_nn
        if isinstance(density_estimator, str):
            density_estimator = posterior_flow_nn(model=density_estimator)
        super().__init__(prior, density_estimator, device, show_progress_bars)

    def train(self, training_batch_size: int = 200, learning_rate: float = 5e-4, validation_fraction: float = 0.1,
              stop_after_epochs: int = 20, max_num_epochs: int = 2 ** 31 - 1, clip_max_norm: Optional[float] = 5.0,
              calibration_kernel=None, ema_loss_decay: float = 0.1, validation_times: Union[Tensor, int] = 10,
              validation_times_nugget: float = 0.05, resume_training: bool = False, **kwargs):
        self._vf_check_rounds(kwargs)
        dev = self._device
        world, glob = self._dp()[1:]
        net, B, Bv, steps, vsteps = self._prepare(validation_fraction, training_batch_size, resume_training)
        x2d = self._x.reshape(self._x.shape[0], -1).contiguous()
        D = net.layout.D
        embed = not net._embed_identity
        if embed and self._dist is not None:
            raise NotImplementedError("data-parallel training with an embedding net is not implemented")
        train_emb = bool(_embedding_params(net))      # False: a parameter-free or frozen embedding
        emb = net.embedding_net
        self._dp_agree(vsteps, "number of validation steps per epoch")
        Bl, o_t, Btot = self._rank_rows(B)
        Bvl, o_v, _ = self._rank_rows(Bv)
        vt = self._validation_times(net, validation_times, validation_times_nugget)
        opt = self._optimizer(net, learning_rate, clip_max_norm, resume_training)
        self._ema_loss_decay = ema_loss_decay
        loss_acc = torch.zeros(2, dtype=torch.float32, device=dev)

        # One CUDA graph per epoch: every step is [t ~ U, theta_1 ~ N draws, fused loss fwd+bwd kernel,
        # reduce, clip+Adam].
        perm_buf, vperm_buf, fill = self._epoch_orders(B, steps, Bv, vsteps)
        stats = torch.zeros(4, dtype=torch.float32, device=dev)     # train loss sum, bad, val loss sum, bad

        # embedding net: the batch's x rows (event shape) go through Standardize + the user's module in torch; the
        # loss kernel returns the gradient of the embedded condition, which autograd takes back through the module
        gcond = torch.empty(Bl, net.layout.C, dtype=torch.float32, device=dev) if train_emb else None

        def run_epoch():
            loss_acc.zero_()
            if embed:
                emb.train()
            for s in range(steps):
                idx = perm_buf[s * B + o_t:s * B + o_t + Bl]
                tms = torch.rand(Bl, device=dev)
                eps = torch.randn(Bl, D, device=dev)
                if embed:
                    opt.zero_grad()
                    with torch.set_grad_enabled(train_emb):
                        ctx = net._embed(self._x[idx]).contiguous()
                    _, gpart, n_part = net.loss_raw(self._theta[idx], ctx, tms, eps, g_const=1.0 / Btot,
                                                    loss_acc=loss_acc, want_loss=False, gcond=gcond)
                    if train_emb:
                        ctx.backward(gcond)
                else:
                    _, gpart, n_part = net.loss_raw(self._theta, x2d, tms, eps, index=idx, g_const=1.0 / Btot,
                                                    loss_acc=loss_acc, want_loss=False)
                opt.step_partials(gpart, n_part)
            stats[0:2].copy_(loss_acc)
            # validation: every batch evaluated at all validation times (:524-543); g = 0 -> loss only
            loss_acc.zero_()
            if vsteps > 0:
                nt = vt.shape[0]
                if embed:
                    emb.eval()
                for s in range(vsteps):
                    vi = vperm_buf[s * Bv + o_v:s * Bv + o_v + Bvl]
                    idx = vi.repeat(nt).contiguous()
                    tms = vt.repeat_interleave(Bvl).contiguous()
                    eps = torch.randn(Bvl * nt, D, device=dev)
                    if embed:
                        with torch.no_grad():
                            vctx = net._embed(self._x[vi]).repeat(nt, 1).contiguous()
                        net.loss_raw(self._theta[idx], vctx, tms, eps, g_const=0.0, loss_acc=loss_acc,
                                     want_loss=False)
                    else:
                        net.loss_raw(self._theta, x2d, tms, eps, index=idx, g_const=0.0, loss_acc=loss_acc,
                                     want_loss=False)
            stats[2:4].copy_(loss_acc)

        run = run_epoch
        if opt.capturable and steps > 0:
            fill()
            run = _capture(opt, run_epoch, run_epoch)[0].replay

        def epoch():
            fill()
            run()
            tl, vl = self._epoch_losses(stats)
            val_loss = vl / (vsteps * Bv * (1 if glob else world) * vt.shape[0]) if vsteps > 0 else float("nan")
            # the reference normalises by len(loader) * loader.batch_size, i.e. WITHOUT the repeat over times
            val_loss *= vt.shape[0] if vsteps > 0 else 1.0
            return tl / (steps * Btot), val_loss

        self._run(net, epoch, max_num_epochs, stop_after_epochs, opt)
        return deepcopy(net)

    def _validation_times(self, net, validation_times: Union[Tensor, int], nugget: float) -> Tensor:
        """The fixed times every validation batch is evaluated at (base_vf_inference.py:524-543)."""
        if isinstance(validation_times, int):
            validation_times = torch.linspace(net.t_min + nugget, net.t_max - nugget, validation_times)
        return validation_times.to(self._device).float()

    def _vf_check_rounds(self, kwargs):
        """base_vf_inference.py:451-496: only the first-round loss exists for vector-field trainers."""
        rounds = getattr(self, "_data_round_index", None) or [0]
        if max(rounds) > 0 and not kwargs.get("force_first_round_loss", False):
            raise NotImplementedError(
                f"Multi-round {self.__class__.__name__} with arbitrary proposals is not implemented")

    def _converged(self, net, stop_after_epochs: int) -> bool:
        """base_vf_inference.py:352-420: an epoch counts as "no improvement" only if the validation loss sits more
        than two standard deviations (of the recent EMA-smoothed losses) above the best one."""
        if self.epoch == 0:
            self._best_val_loss, self._epochs_since_last_improvement, self._best_flat = float("inf"), 0, None
        if self._val_loss < self._best_val_loss:
            self._best_val_loss, self._epochs_since_last_improvement = self._val_loss, 0
            self._save_best(net)
        else:
            if len(self._summary["validation_loss"]) >= stop_after_epochs:
                recent = torch.tensor(self._summary["validation_loss"][-stop_after_epochs * 2:])
                z = (self._val_loss - self._best_val_loss) / recent.std().item()
                self._epochs_since_last_improvement = self._epochs_since_last_improvement + 1 if z > 2.0 else 0
            else:
                return False
        if self._epochs_since_last_improvement > stop_after_epochs - 1:
            if self._best_flat is not None:
                self._load_best(net)
            return True
        return False

    def _record_epoch(self, train_loss: float, val_loss: float):
        # base.py:1110 keeps the RAW validation loss in self._val_loss (what _converged compares
        # with the best loss); only the summaries hold the exponential moving averages
        # (base_vf_inference.py:589-636), whose spread normalises the stopping rule
        self._val_loss = val_loss
        if self._summary["training_loss"]:
            decay = self._ema_loss_decay
            train_loss = (1 - decay) * self._summary["training_loss"][-1] + decay * train_loss
            val_loss = (1 - decay) * self._summary["validation_loss"][-1] + decay * val_loss
        self._summary["training_loss"].append(train_loss)
        self._summary["validation_loss"].append(val_loss)

    def build_posterior(self, density_estimator=None, prior=None, sample_with: str = "ode", **kwargs):
        from .posteriors import VectorFieldPosterior
        if sample_with not in ("ode", "sde"):
            raise ValueError(f"sample_with must be 'ode' or 'sde', but is {sample_with}.")
        est = deepcopy(density_estimator if density_estimator is not None else self._neural_net)
        return VectorFieldPosterior(est, prior if prior is not None else self._prior, device=self._device,
                                    sample_with=sample_with)



class NPSE(FMPE):
    """Neural posterior score estimation (reference: trainers/vfpe/npse.py:69-268 on the shared loop of
    base_vf_inference.py): denoising score matching of a VE / VP / sub-VP score network (score.py).

    A step is [times + noise draws, noising and target arithmetic in torch, ONE launch of the network kernel over
    the noised inputs and the control-variate means, loss head in torch, ONE launch of the network's
    parameter-gradient kernel, clip + Adam kernel], captured once as a CUDA graph and replayed per batch; the
    validation step (all validation times at once, base_vf_inference.py:524-543) is a second graph."""

    _nan_message = "NaN/Inf present in NPSE loss."

    def __init__(self, prior=None, vf_estimator: Union[str, Callable, None] = None,
                 score_estimator: Union[str, Callable, None] = None, density_estimator: Optional[Callable] = None,
                 sde_type: Optional[str] = None, device: str = "cuda", logging_level: Union[int, str] = "WARNING",
                 summary_writer=None, tracker=None, show_progress_bars: bool = False):
        from .score import posterior_score_nn
        given = [e for e in (vf_estimator, score_estimator, density_estimator) if e is not None]
        if len(given) > 1:
            raise ValueError("pass only one of vf_estimator / score_estimator / density_estimator")
        est = given[0] if given else "mlp"
        if isinstance(est, str):
            est = posterior_score_nn(model=est, sde_type=sde_type or "ve")
        elif sde_type is not None:
            warnings.warn("sde_type is ignored when a build function is passed", stacklevel=2)
        _Trainer.__init__(self, prior, est, device, show_progress_bars)

    def train(self, training_batch_size: int = 200, learning_rate: float = 5e-4, validation_fraction: float = 0.1,
              stop_after_epochs: int = 20, max_num_epochs: int = 2 ** 31 - 1, clip_max_norm: Optional[float] = 5.0,
              calibration_kernel=None, ema_loss_decay: float = 0.1, validation_times: Union[Tensor, int] = 10,
              validation_times_nugget: float = 0.05, resume_training: bool = False, **kwargs):
        self._vf_check_rounds(kwargs)
        if self._dp()[1] > 1:
            raise NotImplementedError("NPSE training is single-process")
        dev = self._device
        net, B, Bv, steps, vsteps = self._prepare(validation_fraction, training_batch_size, resume_training)
        x2d = self._x.reshape(self._x.shape[0], -1).contiguous()
        vt = self._validation_times(net, validation_times, validation_times_nugget)
        nt = vt.shape[0]
        opt = self._optimizer(net, learning_rate, clip_max_norm, resume_training)
        self._ema_loss_decay = ema_loss_decay
        w_all = None
        if calibration_kernel is not None:
            w_all = torch.as_tensor(calibration_kernel(self._x), dtype=torch.float32).reshape(-1).to(dev)
        stats = torch.zeros(4, dtype=torch.float32, device=dev)     # train loss sum, bad, val loss sum, bad

        def losses_on(idx, times):
            losses = net.loss(self._theta[idx], x2d[idx], times=times)
            return losses if w_all is None else w_all[idx] * losses

        def train_step(idx):
            net.net.flat.grad = None
            losses = losses_on(idx, None)
            losses.mean().backward()
            ld = losses.detach()
            stats[0] += ld.sum()
            stats[1] += (~torch.isfinite(ld)).sum()
            opt.step(net.flat.grad)

        def val_step(idx):      # the batch repeated over all validation times (base_vf_inference.py:524-543)
            with torch.no_grad():
                ld = losses_on(idx.repeat(nt), vt.repeat_interleave(Bv))
                stats[2] += ld.sum()
                stats[3] += (~torch.isfinite(ld)).sum()

        run_steps = self._step_epochs(opt, B, Bv, steps, vsteps, train_step, val_step, True)

        def epoch():
            stats.zero_()
            run_steps()
            tl, vl = self._epoch_losses(stats)
            # the reference normalises the validation sum by len(loader) * batch_size, i.e. WITHOUT the repeat over times
            return tl / (steps * B), (vl / (vsteps * Bv) if vsteps > 0 else float("nan"))

        self._run(net, epoch, max_num_epochs, stop_after_epochs, opt)
        net._cache.clear()
        return deepcopy(net)

    def build_posterior(self, vector_field_estimator=None, prior=None, sample_with: str = "sde", **kwargs):
        """npse.py:219-261: same posterior as FMPE's, reverse-SDE sampling by default."""
        return super().build_posterior(density_estimator=vector_field_estimator, prior=prior, sample_with=sample_with,
                                       **kwargs)
