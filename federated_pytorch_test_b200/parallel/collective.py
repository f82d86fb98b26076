"""Block collectives: the three aggregation operators of the framework.

Logical collectives of the reference (SURVEY §2.9; Python loops over a dict on
one device):

* X1 FedAvg  ``z' = sum_k x_k / K``; ``dual = ||z - z'||``; write ``z'`` into every replica
  (/root/reference/src/federated_multi.py:204-217)
* X2 FedProx ``z' = mean``; ``dual``; ``primal = sum_k ||rho (x_k - z')||``; no write-back
  (fedprox_multi.py:211-232)
* X3 ADMM    ``z' = sum_k (y_k + rho x_k) / (K rho)``; ``dual``; ``y_k += rho (x_k - z')``;
  ``primal = sum_k ||rho (x_k - z')||`` (consensus_multi.py:281-297)
* X4 BB      per-worker dot products gathered from everyone (consensus_multi.py:248-278)

Each operator is ONE in-place call on flat block slices (views of the replicas'
parameter arenas).  :class:`TorchCollective` implements them with ATen (+ a
``torch.distributed`` all-reduce across processes: Gloo on CPU, NCCL on GPUs) —
this is the *baseline* and the test oracle.  :class:`FusedCollective`
(``parallel/fused.py``) implements the same interface with the hand-written
sm_90a kernels that reduce straight out of peer memory over NVLink.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from .topology import Topology


class TorchCollective:
    """ATen + torch.distributed implementation (baseline / oracle / CPU)."""

    name = "torch"
    fused = False

    def __init__(self, topo: Topology):
        self.topo = topo
        self.launches = 0  # number of framework-owned kernels launched (0 here: library path)

    # -- arena hooks ------------------------------------------------------
    def arena_allocator(self) -> Optional[Callable]:
        return None

    def register_arena(self, arena) -> None:
        return None

    def zeros_like_block(self, x: torch.Tensor, tag: str) -> torch.Tensor:
        """Zeroed companion vector of block slice ``x`` (ADMM duals).  The fused backend returns a slice of a
        symmetric arena so that peers can read it."""
        return torch.zeros_like(x)

    # -- primitives -------------------------------------------------------
    def _allreduce(self, t: torch.Tensor) -> torch.Tensor:
        if self.topo.is_distributed:
            dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.topo.group)
        return t

    def sum_blocks(self, contribs: Sequence[torch.Tensor]) -> torch.Tensor:
        """Sum over ALL K workers of one contribution per local worker (fresh tensor)."""
        acc = contribs[0].clone()
        for c in contribs[1:]:
            acc.add_(c)
        return self._allreduce(acc)

    def sum_scalars(self, t: torch.Tensor) -> torch.Tensor:
        return self._allreduce(t.clone())

    def gather_rows(self, local_rows: torch.Tensor) -> torch.Tensor:
        """``local_rows[i]`` belongs to ``topo.local_workers[i]``; returns ``[K, cols]`` by worker id."""
        K, cols = self.topo.K, local_rows.shape[1]
        full = torch.zeros(K, cols, dtype=local_rows.dtype, device=local_rows.device)
        for i, ck in enumerate(self.topo.local_workers):
            full[ck] = local_rows[i]
        return self._allreduce(full)

    def barrier(self) -> None:
        self.topo.barrier()

    # -- operators --------------------------------------------------------
    @torch.no_grad()
    def fedavg_(self, xs: List[torch.Tensor], z: torch.Tensor, write_back: bool = True) -> torch.Tensor:
        """In place: ``z <- mean_k x_k``, optionally ``x_k <- z``; returns ``||z_old - z_new||^2`` (0-dim)."""
        znew = self.sum_blocks(xs).div_(self.topo.K)
        diff = z - znew
        dual_sq = torch.dot(diff, diff)
        z.copy_(znew)
        if write_back:
            for x in xs:
                x.copy_(znew)
        return dual_sq

    @torch.no_grad()
    def fedprox_(self, xs: List[torch.Tensor], z: torch.Tensor, rho: float) -> Tuple[torch.Tensor, torch.Tensor]:
        """``z <- mean``; returns ``(dual_sq, sum_k ||rho (x_k - z)||)`` with the sum over ALL workers."""
        dual_sq = self.fedavg_(xs, z, write_back=False)
        local = z.new_zeros(())
        for x in xs:
            local = local + torch.norm(rho * (x - z))
        return dual_sq, self.sum_scalars(local.reshape(1))[0]

    @torch.no_grad()
    def admm_(self, xs: List[torch.Tensor], ys: List[torch.Tensor], z: torch.Tensor, rho: float,
              rho_dev: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """z-update, dual ascent on every local ``y_k``; returns ``(dual_sq, primal)`` as :meth:`fedprox_`."""
        if rho_dev is not None:
            rho = float(rho_dev)
        contribs = [y + rho * x for x, y in zip(xs, ys)]
        znew = self.sum_blocks(contribs).div_(self.topo.K * rho)
        diff = z - znew
        dual_sq = torch.dot(diff, diff)
        z.copy_(znew)
        local = z.new_zeros(())
        for x, y in zip(xs, ys):
            ydelta = rho * (x - z)
            local = local + torch.norm(ydelta)
            y.add_(ydelta)
        return dual_sq, self.sum_scalars(local.reshape(1))[0]

    @torch.no_grad()
    def bb_dots(self, xs, ys, yhat0s, x0s, z) -> torch.Tensor:
        """Six dots per worker, gathered: rows ``[a.a, a.b, b.b, a.c, b.c, c.c]`` with
        ``a = y - yhat0``, ``b = x - z``, ``c = x - x0`` (SURVEY §7.3(2))."""
        from ..ops import flatops

        rows = []
        for x, y, yh0, x0 in zip(xs, ys, yhat0s, x0s):
            a, b, c = y - yh0, x - z, x - x0
            rows.append(flatops.multi_dot([(a, a), (a, b), (b, b), (a, c), (b, c), (c, c)]))
        return self.gather_rows(torch.stack(rows))

    @torch.no_grad()
    def bb_seed_(self, xs, x0s) -> None:
        """Round 0 of a block visit: ``x0_k <- x_k`` (consensus_multi.py:244-246)."""
        for x, x0 in zip(xs, x0s):
            x0.copy_(x)

    @torch.no_grad()
    def bb_update_(self, xs, ys, yhat0s, x0s, z, rho: float, rho_dev: Optional[torch.Tensor], cfg) -> List[List[float]]:
        """Barzilai-Borwein penalty update (consensus_multi.py:248-278): returns one row per worker
        ``[d11, d12, d22, alpha, alphaSD, alphaMG, tested, rho after this worker's turn]``; ``yhat0``/``x0`` are carried
        forward in place and ``rho_dev`` (if given) receives the final rho.  ATen/NCCL baseline + oracle of the kernel."""
        import math

        rows = self.bb_dots(xs, ys, yhat0s, x0s, z).double().cpu()
        out, rho_at_turn = [], []
        for ck in range(self.topo.K):
            aa, ab, bb_, ac, bc, cc = (float(v) for v in rows[ck])
            rho_at_turn.append(rho)
            d11 = aa + 2.0 * rho * ab + rho * rho * bb_
            d12 = ac + rho * bc
            d22 = cc
            alpha = aSD = aMG = 0.0
            tested = 0.0
            if abs(d12) > cfg.epsilon and d11 > cfg.epsilon and d22 > cfg.epsilon:
                tested = 1.0
                alpha = d12 / math.sqrt(d11 * d22)
                aSD = d11 / d22
                aMG = d12 / d22
                ahat = aMG if 2.0 * aMG > aSD else aSD - 0.5 * aMG
                if alpha >= cfg.alphacorrmin and ahat < cfg.rhomax:
                    rho = ahat
            out.append([d11, d12, d22, alpha, aSD, aMG, tested, rho])
        # carry forward: yhat0_k <- y_k + rho_k (x_k - z) with the rho in force at worker k's turn
        for i, ck in enumerate(self.topo.local_workers):
            torch.add(ys[i], xs[i] - z, alpha=rho_at_turn[ck], out=yhat0s[i])
            x0s[i].copy_(xs[i])
        if rho_dev is not None:
            rho_dev.fill_(rho)
        return out


def make_collective(topo: Topology, kind: str = "auto"):
    """``kind``: 'torch' (baseline), 'fused' (sm_90a kernels; error if unavailable), 'auto'."""
    if kind == "torch":
        return TorchCollective(topo)
    want_fused = kind == "fused" or (kind == "auto" and topo.device.type == "cuda")
    if want_fused:
        from ..ops import functional as FX

        if kind == "auto" and not FX.fast_path_enabled():
            return TorchCollective(topo)
        from .fused import FusedCollective

        return FusedCollective(topo)
    return TorchCollective(topo)
