"""Data-parallel plumbing over `torch.distributed` (NCCL on the GPUs, gloo in the CPU tests).

SURVEY §8(e): the path shards over the simulation-batch axis.
* training: identical replicas; each rank differentiates its own batch with upstream gradient
  -1/(B * world) per row, ONE all-reduce(sum) of the flat gradient joins them, then every rank runs
  the same deterministic clip+Adam (the clip norm is taken on the reduced gradient, as
  `clip_grad_norm_` semantics require, trainers/base.py:1181-1187);
* log_prob / ODE / slice chains: contiguous row (chain) ranges per rank, no collective;
* rejection with a fixed proposal budget: every rank regenerates the SAME seeded candidate and
  uniform streams (cheap), evaluates the potential only on its own block (expensive), and one
  all-gather of (global index, row) pairs reassembles exactly the single-process accept set/order.
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import torch
import torch.distributed as dist
from torch import Tensor


def world() -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(n: int, rank: int, world_size: int) -> Tuple[int, int]:
    """Contiguous block [lo, hi) of n items for `rank` (first n % world ranks get one extra)."""
    base, extra = divmod(n, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def broadcast_parameters(flat: Tensor, src: int = 0) -> None:
    if world()[1] > 1:
        dist.broadcast(flat, src)


def allreduce_flat_gradient(grad: Tensor) -> Tensor:
    """Sum the per-rank flat gradients in place (rows were weighted 1/(B*world) upstream)."""
    if world()[1] > 1:
        dist.all_reduce(grad, op=dist.ReduceOp.SUM)
    return grad


def gather_accepted(rows: Tensor, global_index: Tensor) -> Tuple[Tensor, Tensor]:
    """All-gather variable-length accepted rows and their global proposal indices; returns them
    sorted by global index (identical on every rank, identical to the single-process order)."""
    rank, ws = world()
    if ws == 1:
        order = torch.argsort(global_index)
        return rows[order], global_index[order]
    n = torch.tensor([rows.shape[0]], dtype=torch.int64, device=rows.device)
    counts = [torch.zeros_like(n) for _ in range(ws)]
    dist.all_gather(counts, n)
    counts = [int(c.item()) for c in counts]
    m = max(max(counts), 1)
    pad_rows = torch.zeros(m, rows.shape[1], dtype=rows.dtype, device=rows.device)
    pad_idx = torch.full((m,), -1, dtype=torch.int64, device=rows.device)
    pad_rows[:rows.shape[0]] = rows
    pad_idx[:rows.shape[0]] = global_index
    all_rows = [torch.zeros_like(pad_rows) for _ in range(ws)]
    all_idx = [torch.zeros_like(pad_idx) for _ in range(ws)]
    dist.all_gather(all_rows, pad_rows)
    dist.all_gather(all_idx, pad_idx)
    rows_cat = torch.cat([r[:c] for r, c in zip(all_rows, counts)])
    idx_cat = torch.cat([i[:c] for i, c in zip(all_idx, counts)])
    order = torch.argsort(idx_cat)
    return rows_cat[order], idx_cat[order]


@torch.no_grad()
def rejection_fixed_budget(potential_fn: Callable[[Tensor], Tensor], proposal_sample: Callable[[int, torch.Generator], Tensor],
                           proposal_log_prob: Callable[[Tensor], Tensor], log_bound: float, num_proposals: int,
                           seed: int, device: str = "cpu") -> Tuple[Tensor, Tensor]:
    """Fixed-budget rejection sampling sharded over ranks (BASELINE configs[4]: 1M proposals).
    accept iff exp(potential - log q - log_bound) > u, candidates and u from generators seeded with
    `seed` (u on the CPU generator like the reference, rejection.py:178).  Returns (accepted rows,
    accepted global indices), identical on every rank and for every world size."""
    rank, ws = world()
    g = torch.Generator(device="cpu").manual_seed(seed)
    cands = proposal_sample(num_proposals, g)                      # same full stream on every rank
    u = torch.rand(num_proposals, generator=g)
    lo, hi = shard_range(num_proposals, rank, ws)
    mine = cands[lo:hi].to(device)
    ratio = torch.exp(potential_fn(mine) - proposal_log_prob(mine) - log_bound)
    keep = ratio > u[lo:hi].to(device)
    idx = torch.nonzero(keep).reshape(-1) + lo
    return gather_accepted(mine[keep], idx)


class PeerGradientSum:
    """Sum of the per-rank flat gradients over NVLink peer memory, fused with the Σg² partials the
    clip norm needs (kernel `peer_sum_kernel`, csrc/peer.cu) — the single-node replacement of
    `allreduce_flat_gradient` + norm pass.  All ranks must be processes on one node with P2P access
    between their GPUs; construction is collective (handles are exchanged with all_gather_object).

        ex = PeerGradientSum(n_params)                       # once, on every rank
        ex.sum(grad_local, grad_out, mask, sumsq)            # every step, graph-capturable
    The step number that tags the flags is the exchange's own device counter (it only grows: a
    warm-up pass whose optimizer state is rewound afterwards cannot leave matching flags); pass
    `opt_step` to tag with a caller-owned counter instead (all ranks must then agree on it).
    """

    def __init__(self, n_params: int):
        import ctypes as C
        from . import _lib as L
        self._L, self._C = L, C
        self.lib = L.load()
        self.rank, self.world = world()
        self.n = int(n_params)
        # Every collective below runs on every rank whatever happened locally; failures are
        # collected and agreed on at the end, so that either all ranks get a working exchange or
        # all ranks raise (and can fall back to NCCL together).
        ok = 1
        self.own = self.lib.sbi_b200_peer_alloc(self.n)
        h = C.create_string_buffer(64)
        if not self.own or self.lib.sbi_b200_peer_export(C.c_void_p(self.own), h) != 0:
            ok = 0
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(h.raw))
        self._imported = []
        ptrs = (C.c_void_p * self.world)()
        for r in range(self.world):
            if r == self.rank:
                ptrs[r] = self.own
            elif ok:
                p = self.lib.sbi_b200_peer_import(C.create_string_buffer(handles[r], 64))
                if not p:
                    ok = 0
                else:
                    self._imported.append(p)
                    ptrs[r] = p
        self._ptrs = ptrs
        self.n_sumsq = self.lib.sbi_b200_peer_blocks(self.n)
        flag = torch.tensor([ok], dtype=torch.int32, device="cuda")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            self.close()
            raise RuntimeError("peer-memory gradient exchange unavailable (allocation, IPC export or P2P "
                               "mapping failed on at least one rank)")

    def sum(self, grad_local: Tensor, grad_out: Tensor, mask: Optional[Tensor], sumsq: Optional[Tensor],
            opt_step: Optional[Tensor] = None) -> None:
        self._L.call("peer_sum", grad_local, self._ptrs, self.world, self.rank, self.n, grad_out, mask, sumsq,
                     opt_step)

    def error(self) -> bool:
        return self.lib.sbi_b200_peer_error(self._C.c_void_p(self.own), self.n) != 0

    def close(self) -> None:
        if getattr(self, "_closed", False):
            return
        self._closed = True
        torch.cuda.synchronize()
        dist.barrier()
        for p in self._imported:
            self.lib.sbi_b200_peer_close(self._C.c_void_p(p))
        self._imported = []
        dist.barrier()
        if self.own:
            self.lib.sbi_b200_peer_free(self._C.c_void_p(self.own))
        self.own = None


def make_gradient_exchange(n_params: int) -> Optional[PeerGradientSum]:
    """PeerGradientSum if the group has more than one rank, the ranks can map each other's memory and
    SBI_B200_NCCL != 1; otherwise None (callers then use `allreduce_flat_gradient`).  Collective."""
    import os
    if world()[1] <= 1 or os.environ.get("SBI_B200_NCCL", "") == "1":
        return None
    try:
        return PeerGradientSum(n_params)
    except RuntimeError:
        return None
