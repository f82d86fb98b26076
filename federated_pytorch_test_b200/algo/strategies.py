"""Aggregation strategies over one parameter block: FedAvg, FedProx, consensus
ADMM (with optional Barzilai-Borwein / spectral adaptive rho).

Mathematical spec: SURVEY §2.4; sources /root/reference/src/federated_multi.py:
203-217, fedprox_multi.py:183-234, consensus_multi.py:152-299.  In the reference
these are copy-pasted inline loops over Python dicts; here each is a small
object driven by the block-coordinate engine:

    strat.begin_block(ci, N, xs)      # xs: flat slices of the local replicas
    strat.penalty(i)                  # what the local optimizer must add to the loss
    strat.aggregate(nadmm)            # the collective + bookkeeping -> metrics

All vector work is delegated to a collective (``parallel.collective``), i.e. to
one fused NVLink kernel per aggregation on the GPU.

Preserved reference behaviour (SURVEY §2.12): ``z`` (and ``y``) start at 0 for
every block visit (Q6); FedProx/ADMM never write ``z`` back (Q7); ``rho`` is an
``[L,3]`` table of which only column 0 is used, shared by all workers and
updated sequentially over workers inside the BB step (Q8); the BB state
``yhat0`` is seeded with the parameter values (Q9).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch


@dataclass
class Penalty:
    """Terms the local objective gets on top of the data loss, on the block vector ``x``:
    ``y.(x-z) + rho/2 ||x-z||^2``."""

    z: Optional[torch.Tensor] = None
    y: Optional[torch.Tensor] = None
    rho: float = 0.0                            # host mirror (logs, L-BFGS closures)
    rho_dev: Optional[torch.Tensor] = None      # device-resident penalty read by the kernels (adaptive ADMM)


class Strategy:
    name = "base"
    write_back = False

    def __init__(self, collective, topo):
        self.coll = collective
        self.topo = topo
        self.xs: List[torch.Tensor] = []
        self.z: Optional[torch.Tensor] = None
        self.N = 0
        self.ci = 0

    def begin_block(self, ci: int, N: int, xs: List[torch.Tensor]) -> None:
        self.ci, self.N, self.xs = ci, int(N), xs
        # Q6: restart from the origin on every block visit.  The fused backend hands out a slice of a symmetric arena so
        # that peers can broadcast their part of the new consensus vector straight into it (two-shot aggregation).
        self.z = self.coll.zeros_like_block(xs[0], "z")

    def penalty(self, i: int) -> Penalty:
        return Penalty()

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        raise NotImplementedError

    # Split form used by the engine's deferred rounds: ``begin`` enqueues the aggregation, ``end`` reads its record.  The
    # default is synchronous (begin does everything); FedAvg / FedProx on the fused collective only LAUNCH in ``begin``, so
    # the host can queue the next minibatches before it waits for the residuals.
    def aggregate_begin(self, nadmm: int):
        return ("done", self.aggregate(nadmm))

    def aggregate_end(self, token) -> Dict[str, float]:
        return token[1]

    def rho_mean(self) -> float:
        return float("nan")

    # extra vectors a true-resume checkpoint must carry
    def state(self) -> Dict[str, object]:
        return {"z": self.z}


class NoConsensus(Strategy):
    """Stand-alone training: nothing is exchanged (no_consensus_multi.py)."""

    name = "none"

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        return {}


class FedAvg(Strategy):
    name = "fedavg"
    write_back = True

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        dual_sq = self.coll.fedavg_(self.xs, self.z, write_back=True)
        return {"dual": math.sqrt(max(float(dual_sq), 0.0)) / self.N}

    def aggregate_begin(self, nadmm: int):
        if getattr(self.coll, "supports_async", False):
            self.coll.launch_fedavg_(self.xs, self.z, True)
            return ("pending", self.N)
        return ("done", self.aggregate(nadmm))

    def aggregate_end(self, token) -> Dict[str, float]:
        if token[0] == "done":
            return token[1]
        return {"dual": math.sqrt(max(float(self.coll.read_record()[0]), 0.0)) / token[1]}

    def load_state(self, st: Dict[str, object]) -> None:
        self.z.copy_(st["z"].to(self.z.device))


class FedProx(Strategy):
    name = "fedprox"

    def __init__(self, collective, topo, num_blocks: int, rho0: float = 1.0):
        super().__init__(collective, topo)
        self.rho = torch.ones(num_blocks, 3) * rho0

    def penalty(self, i: int) -> Penalty:
        return Penalty(z=self.z, y=None, rho=float(self.rho[self.ci, 0]))

    def rho_mean(self) -> float:
        return float(self.rho.mean())

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        rho = float(self.rho[self.ci, 0])
        dual_sq, primal = self.coll.fedprox_(self.xs, self.z, rho)
        return {"dual": math.sqrt(max(float(dual_sq), 0.0)) / self.N, "primal": float(primal) / self.N}

    def aggregate_begin(self, nadmm: int):
        if getattr(self.coll, "supports_async", False):
            self.coll.launch_fedprox_(self.xs, self.z, float(self.rho[self.ci, 0]))
            return ("pending", self.N)
        return ("done", self.aggregate(nadmm))

    def aggregate_end(self, token) -> Dict[str, float]:
        if token[0] == "done":
            return token[1]
        v = self.coll.read_record()
        return {"dual": math.sqrt(max(float(v[0]), 0.0)) / token[1], "primal": float(v[1]) / token[1]}

    def state(self) -> Dict[str, object]:
        return {"z": self.z, "rho": self.rho}

    def load_state(self, st: Dict[str, object]) -> None:
        self.z.copy_(st["z"].to(self.z.device))
        self.rho.copy_(st["rho"])


@dataclass
class BBConfig:
    enabled: bool = False
    period_T: int = 2
    alphacorrmin: float = 0.2
    epsilon: float = 1e-3
    rhomax: float = 0.1
    seed_yhat0_with_x: bool = True   # Q9 (reference behaviour); False seeds with zeros


class ADMM(Strategy):
    name = "admm"

    def __init__(self, collective, topo, num_blocks: int, rho0: float = 0.1, bb: Optional[BBConfig] = None, log=print):
        super().__init__(collective, topo)
        self.rho = torch.ones(num_blocks, 3) * rho0          # host mirror of the reference's [L,3] table (column 0 used)
        self.bb = bb or BBConfig()
        self.ys: List[torch.Tensor] = []
        self.yhat0: List[torch.Tensor] = []
        self.x0: List[torch.Tensor] = []
        self.log = log
        # the penalty the kernels read: one float per block in device memory.  The BB kernel rewrites it in place, the
        # aggregation kernel and the fused Adam kernel read it — no host value is baked into a launch or a CUDA graph.
        self.rho_dev: Optional[torch.Tensor] = None
        if topo.device.type == "cuda":
            self.rho_dev = torch.full((num_blocks,), float(rho0), dtype=torch.float32, device=topo.device)

    def begin_block(self, ci: int, N: int, xs: List[torch.Tensor]) -> None:
        super().begin_block(ci, N, xs)
        self.ys = [self.coll.zeros_like_block(x, "y") for x in xs]
        if self.bb.enabled:
            self.yhat0 = [x.clone() if self.bb.seed_yhat0_with_x else torch.zeros_like(x) for x in xs]
            self.x0 = [torch.zeros_like(x) for x in xs]

    def _rho_slot(self) -> Optional[torch.Tensor]:
        return self.rho_dev[self.ci: self.ci + 1] if self.rho_dev is not None else None

    def penalty(self, i: int) -> Penalty:
        return Penalty(z=self.z, y=self.ys[i], rho=float(self.rho[self.ci, 0]), rho_dev=self._rho_slot())

    def rho_mean(self) -> float:
        return float(self.rho.mean())

    def state(self) -> Dict[str, object]:
        return {"z": self.z, "y": self.ys, "rho": self.rho, "yhat0": self.yhat0, "x0": self.x0}

    def load_state(self, st: Dict[str, object]) -> None:
        self.z.copy_(st["z"].to(self.z.device))
        self.rho.copy_(st["rho"])
        if self.rho_dev is not None:
            self.rho_dev.copy_(self.rho[:, 0].to(self.rho_dev.device))
        for dst, src in (("ys", "y"), ("yhat0", "yhat0"), ("x0", "x0")):
            for d, t in zip(getattr(self, dst), st.get(src) or []):
                d.copy_(t.to(d.device))

    # -- adaptive rho ---------------------------------------------------------
    def _bb_update(self, nadmm: int) -> None:
        """Spectral penalty selection, replayed identically on every rank.

        The reference loops over workers, each one reading and possibly
        overwriting the shared ``rho[ci,0]`` (consensus_multi.py:248-278).  With
        ``a=y-yhat0, b=x-z, c=x-x0`` the quantities it needs are
        ``d11 = a.a + 2 rho a.b + rho^2 b.b``, ``d12 = a.c + rho b.c``, ``d22 = c.c``,
        so six local dots per worker + one tiny gather reproduce the sequential
        rule without serialising the GPUs.  On the GPU all of it — dots, gather through
        the peer-mapped control pads, replay, ``yhat0``/``x0`` carry — is ONE kernel
        (``csrc/comm_kernels.cu: bb_update_kernel``) that leaves the new rho in
        device memory; the host only reads the log rows for the legacy print lines.
        """
        cfg = self.bb
        rho_in = float(self.rho[self.ci, 0])
        rows = self.coll.bb_update_(self.xs, self.ys, self.yhat0, self.x0, self.z, rho_in, self._rho_slot(), cfg)
        for ck in range(self.topo.K):
            d11, d12, d22, alpha, aSD, aMG, tested, rho_after = (float(v) for v in rows[ck])
            self.log("admm %d deltas=(%e,%e,%e)" % (nadmm, d11, d12, d22))
            if tested:
                self.log("admm %d alphas=(%e,%e,%e)" % (nadmm, alpha, aSD, aMG))
        self.rho[self.ci, 0] = float(rows[self.topo.K - 1][7])

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        if self.bb.enabled:
            if nadmm == 0:
                self.coll.bb_seed_(self.xs, self.x0)
            elif nadmm % self.bb.period_T == 0:
                self._bb_update(nadmm)
        rho = float(self.rho[self.ci, 0])
        dual_sq, primal = self.coll.admm_(self.xs, self.ys, self.z, rho, self._rho_slot())
        return {"dual": math.sqrt(max(float(dual_sq), 0.0)) / self.N, "primal": float(primal) / self.N}

    def aggregate_begin(self, nadmm: int):
        if not getattr(self.coll, "supports_async", False):
            return ("done", self.aggregate(nadmm))
        if self.bb.enabled:                      # the Barzilai-Borwein bookkeeping keeps its own (host-mirrored) log
            if nadmm == 0:
                self.coll.bb_seed_(self.xs, self.x0)
            elif nadmm % self.bb.period_T == 0:
                self._bb_update(nadmm)
        self.coll.launch_admm_(self.xs, self.ys, self.z, float(self.rho[self.ci, 0]), self._rho_slot())
        return ("pending", self.N)

    def aggregate_end(self, token) -> Dict[str, float]:
        if token[0] == "done":
            return token[1]
        v = self.coll.read_record()
        return {"dual": math.sqrt(max(float(v[0]), 0.0)) / token[1], "primal": float(v[1]) / token[1]}
