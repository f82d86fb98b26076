"""Simulated Byzantine workers, for studying robust aggregation (``federated_multi --byzantine b --attack ...``).

Workers ``K - b .. K - 1`` are attackers (worker 0, which prints the logs, stays honest).  Right before every aggregation,
after local training, each attacker's block slice is overwritten on its device, relative to the consensus vector ``z``
the round started from:

* ``signflip``:  ``x <- z - s (x - z)``   (the local update reversed and scaled)
* ``gaussian``:  ``x <- z + s xi``,  ``xi ~ N(0, 1)``
* ``nan``:       ``x <- NaN``

``xi`` is drawn from a generator seeded by ``(seed, worker id, aggregations done)``, so the draws do not depend on which
process hosts the worker, and ``--resume`` reproduces them (the aggregation count is part of the resume record).  This is
a simulation, not a hot path: a few ATen ops per attacker and round, outside the step graphs.
"""
from __future__ import annotations

import torch

from ..config import check_byzantine

_MASK64 = (1 << 64) - 1


def _mix(seed: int, ck: int, rnd: int) -> int:
    """A 63-bit generator seed from ``(seed, worker id, round)`` (splitmix64 finaliser over their combination)."""
    h = (seed * 0x9E3779B97F4A7C15 + ck * 0xBF58476D1CE4E5B9 + rnd * 0x94D049BB133111EB + 0x632BE59BD9B4E019) & _MASK64
    h = ((h ^ (h >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    h = ((h ^ (h >> 27)) * 0x94D049BB133111EB) & _MASK64
    return (h ^ (h >> 31)) & ((1 << 63) - 1)


class ByzantineAttack:
    """Called by the engine with itself right before each aggregation (``Engine.attack``)."""

    def __init__(self, K: int, byzantine: int, kind: str = "signflip", scale: float = 4.0, seed: int = 0):
        check_byzantine(byzantine, kind, scale, K)
        self.K, self.byzantine, self.kind, self.scale, self.seed = K, int(byzantine), kind, float(scale), int(seed)
        self.attackers = frozenset(range(K - self.byzantine, K))

    def noise(self, ck: int, rnd: int, like: torch.Tensor) -> torch.Tensor:
        """``xi`` of worker ``ck`` at aggregation ``rnd``: standard normal, shaped like the block slice ``like``."""
        g = torch.Generator(device=like.device)
        g.manual_seed(_mix(self.seed, ck, rnd))
        return torch.randn(like.shape, generator=g, device=like.device, dtype=like.dtype)

    @torch.no_grad()
    def apply(self, xs, cks, z: torch.Tensor, rnd: int) -> None:
        """Overwrite the attackers among the local block slices ``xs`` (of workers ``cks``) for aggregation ``rnd``."""
        for x, ck in zip(xs, cks):
            if ck not in self.attackers:
                continue
            if self.kind == "signflip":
                x.sub_(z).mul_(-self.scale).add_(z)
            elif self.kind == "gaussian":
                x.copy_(self.noise(ck, rnd, x).mul_(self.scale).add_(z))
            else:
                x.fill_(float("nan"))

    def __call__(self, engine) -> None:
        strat = engine.strategy
        rnd = engine.aggregations_done + (engine._pending_round is not None)   # the round being aggregated now
        self.apply(strat.xs, [rep.ck for rep in engine.replicas], strat.z, rnd)
