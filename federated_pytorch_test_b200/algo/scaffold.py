"""SCAFFOLD control variates for federated averaging with SGD client steps (Karimireddy et al., ICML 2020, Algorithm 1
with option II).  :class:`ControlVariates` owns the per-block state and the per-round launches; :func:`reference_round`
is the float64 oracle of one round.

For one block, with ``z`` the server model at the start of a round, ``x_i`` worker ``i``'s block after its ``tau_i``
local steps and ``lr`` the round's client learning rate:

* every local SGD step of worker ``i`` adds ``d_i = c - c_i`` to its data-loss gradient (after clipping, as a FedProx /
  ADMM term is added), so weight decay, momentum and Nesterov act on the corrected gradient;
* at the end of the round, before the model is aggregated:

  1. ``c_i <- (c_i - c) + s_i (z - x_i)`` with ``s_i = float32(1 / (tau_i lr))`` (computed in float64), for every worker
     with ``tau_i > 0``; a worker that sat out a sampled round keeps its ``c_i``;
  2. ``c <- (1/K) sum_k c_k`` over all K workers, unweighted.  Every ``c_k`` starts at 0 and a worker that sits out keeps
     its ``c_k``, so this is the paper's ``c + (|S| / N) mean_{k in S} (c_k^+ - c_k)``, with and without sampling;
  3. ``d_i <- c - c_i`` for every worker: the correction of the next round, written in place, so a captured SGD step
     keeps reading it at the same address.

``c`` and the ``c_i`` start at 0 at a block's first visit and persist across its later visits for the whole run.  With
momentum ``(z - x_i) / (tau_i lr)`` is not the mean gradient of the round but about ``1 / (1 - momentum)`` times it; like
most implementations this one uses the formula unchanged.

On the fused collective ``c`` and the ``c_i`` are slices of symmetric arenas, so step 2 is one launch of the existing
aggregation kernel (FedAvg without write-back), and two-shot ranks broadcast their share of ``c`` into every rank.  Steps
1 and 3 are one launch each for all local replicas (``csrc/flat_kernels.cu: scaffold_cv_kernel, scaffold_corr_kernel``).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..ops import flatops


def step_scale(tau: int, lr: float) -> float:
    """``s = float32(1 / (tau lr))``, computed in float64; 0 for a worker that took no step."""
    return float(np.float32(1.0 / (float(tau) * float(lr)))) if tau > 0 else 0.0


def reference_round(cis: Sequence[np.ndarray], xs: Sequence[np.ndarray], c: np.ndarray, z: np.ndarray,
                    taus: Sequence[int], lr: float) -> Tuple[List[np.ndarray], np.ndarray, List[np.ndarray]]:
    """Steps 1-3 of one round for all K workers in float64: ``(new c_i, new c, d_i)``.  ``cis``, ``xs`` and ``taus`` hold
    one entry per worker, by worker id."""
    c = np.asarray(c, dtype=np.float64)
    z = np.asarray(z, dtype=np.float64)
    new_cis = []
    for ci, x, tau in zip(cis, xs, taus):
        ci = np.asarray(ci, dtype=np.float64)
        if tau > 0:
            ci = (ci - c) + (z - np.asarray(x, dtype=np.float64)) / (float(tau) * float(lr))
        new_cis.append(ci)
    new_c = np.mean(np.stack(new_cis), axis=0)
    return new_cis, new_c, [new_c - ci for ci in new_cis]


class ControlVariates:
    """The server control variate ``c`` and this process' ``c_i`` / ``d_i`` of every visited block, and the launches of a
    round.  Per visit: :meth:`begin_block` (forms ``d_i``, one launch); per round: :meth:`note_local_steps`, then
    :meth:`end_round` (steps 1-3, three launches) before the model aggregation, and :meth:`corr_norm` once the round's
    record has been read."""

    def __init__(self, collective, topo):
        self.coll, self.topo = collective, topo
        self.c: Dict[int, torch.Tensor] = {}                  # block index -> c
        self.cis: Dict[int, List[torch.Tensor]] = {}          # block index -> c_i per local replica
        self.ds: Dict[int, List[torch.Tensor]] = {}           # block index -> d_i per local replica
        self._work: Dict[int, tuple] = {}                     # block index -> flatops.scaffold_workspace
        self._restored: Dict[int, Tuple[torch.Tensor, torch.Tensor]] = {}   # read from a resume record, installed at the visit
        self.ci: Optional[int] = None
        self._scales: Optional[List[float]] = None
        n_local = len(topo.local_workers)
        self._norm_host = torch.zeros(n_local, dtype=torch.float32, pin_memory=topo.device.type == "cuda")

    def begin_block(self, ci: int, xs: List[torch.Tensor]) -> None:
        if ci not in self.c:        # zeros_like_block zeroes on every call: only at the block's first visit
            self.c[ci] = self.coll.zeros_like_block(xs[0], "scaffold_c")
            self.cis[ci] = [self.coll.zeros_like_block(x, "scaffold_ci") for x in xs]
            self.ds[ci] = [torch.zeros_like(x) for x in xs]
            self._work[ci] = flatops.scaffold_workspace(xs[0].numel(), len(xs), xs[0].device)
            if ci in self._restored:
                self._install(ci, *self._restored.pop(ci))
        self.ci = ci
        self._correct()

    def correction(self, i: int) -> torch.Tensor:
        """``d_i`` of local replica ``i`` in the current block."""
        return self.ds[self.ci][i]

    def note_local_steps(self, steps: Sequence[int], lr: float) -> None:
        """The local steps each local replica took in the round that ends, and the round's client learning rate."""
        self._scales = [step_scale(t, lr) for t in steps]

    @torch.no_grad()
    def end_round(self, xs: List[torch.Tensor], z: torch.Tensor) -> None:
        """Steps 1-3, in stream order before the model aggregation (``z`` is still the round's starting model)."""
        if self._scales is None:
            raise RuntimeError("SCAFFOLD needs the round's local step counts (note_local_steps) before every aggregation")
        ci = self.ci
        flatops.scaffold_cv_(self.cis[ci], xs, self.c[ci], z, self._scales)
        self._scales = None
        self.coll.average_(self.cis[ci], self.c[ci])
        self._correct()

    def _correct(self) -> None:
        ci = self.ci
        norm_sq = flatops.scaffold_corr_(self.cis[ci], self.ds[ci], self.c[ci], self._work[ci])
        self._norm_host.copy_(norm_sq, non_blocking=True)     # read with the round's record, which waits for it

    def corr_norm(self) -> float:
        """Mean over the local replicas of ``||c - c_i||_2`` after the last round; valid once its record is read."""
        return float(self._norm_host.double().sqrt().mean())

    # -- resume ----------------------------------------------------------------------------------------------------
    def state(self) -> Dict[str, object]:
        """``c`` and this process' ``c_i`` of every block visited so far, including blocks restored from a resume record
        that this process has not visited yet."""
        cs = {ci: c for ci, (c, _) in self._restored.items()}
        cis = {ci: v for ci, (_, v) in self._restored.items()}
        cs.update(self.c)
        cis.update({ci: torch.stack(v) for ci, v in self.cis.items()})
        return {"scaffold_c": cs, "scaffold_ci": cis}

    def _install(self, ci: int, c: torch.Tensor, cis: torch.Tensor) -> None:
        self.c[ci].copy_(c.to(self.c[ci].device))
        for dst, src in zip(self.cis[ci], cis):
            dst.copy_(src.to(dst.device))

    def load_state(self, st: Dict[str, object]) -> None:
        cis = st.get("scaffold_ci") or {}
        for ci, c in (st.get("scaffold_c") or {}).items():
            if ci in self.c:
                self._install(ci, c, cis[ci])
            else:
                self._restored[ci] = (c, cis[ci])
        if self.ci in self.c:       # resumed inside a visit: the correction of the next step comes from the restored state
            self._correct()
