"""Block collectives: the three aggregation operators of the framework.

Logical collectives of the reference (SURVEY §2.9; Python loops over a dict on
one device):

* X1 FedAvg  ``z' = sum_k x_k / K``; ``dual = ||z - z'||``; write ``z'`` into every replica
  (/root/reference/src/federated_multi.py:204-217); with a server optimizer (``fedopt_``) ``z'`` is its step from ``z``
  along ``mean_k x_k - z`` instead of the plain mean; with a robust rule (``robust_``) ``z'`` is the coordinate-wise
  median or trimmed mean of the K workers instead of their mean; with DP (``dp_clip_`` first, then ``dp=`` on
  ``fedavg_`` / ``fedopt_``) the workers' updates are clipped and Gaussian noise is added to the mean (DP-FedAvg); with
  ``compress=`` on ``fedavg_`` / ``fedopt_`` every worker uploads its update ``x_k - z`` as stochastically rounded 8- or
  4-bit codes with one scale per group (``algo/compress.py``), and ``z' = z + mean_k q_k s_k``; with ``sample=`` on
  ``fedavg_`` / ``fedopt_`` only the round's ``S`` sampled workers are averaged, weighted by their sample counts
  (``z' = sum_{k in P} n_k x_k / sum_{k in P} n_k``, ``algo/sampling.py``), and every replica receives ``z'``; with
  ``secagg=`` on ``fedavg_`` / ``fedopt_`` every worker uploads its update ``x_k - z`` as int32 fixed-point codes masked
  with pairwise ChaCha20 keystreams that cancel in the sum (``algo/secagg.py``), and ``z' = z + decode(sum_k y_k)``; with
  ``topk=`` on ``fedavg_`` / ``fedopt_`` every worker uploads the ``k_sel`` largest-magnitude coordinates of its update
  (``algo/compress.py: topk_select``), and ``z' = z + mean_k s_k``
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

from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from .topology import Topology

# server optimizers of FedAvg (Hsu et al. 2019; Reddi et al. 2021), in the order of the kernel's codes 1..4
FEDOPT_KINDS = ("avgm", "adagrad", "adam", "yogi")
# Byzantine-robust aggregation rules (Yin et al. 2018), in the order of the kernel's codes 1..2 (0 is the mean)
ROBUST_AGGS = ("median", "trimmed_mean")


def check_robust(K: int, agg: str, trim_b: int) -> None:
    """Raise ``ValueError`` unless ``agg`` is a robust rule that can run over ``K`` workers with ``trim_b``."""
    if agg not in ROBUST_AGGS:
        raise ValueError("robust aggregation rule must be one of %s, got %r" % (", ".join(ROBUST_AGGS), agg))
    if agg == "trimmed_mean" and not 0 <= 2 * trim_b < K:
        raise ValueError("trimmed mean needs 0 <= 2 trim_b < K, got trim_b = %r at K = %d" % (trim_b, K))


@dataclass
class DPRound:
    """The noise of one DP-FedAvg round: ``std * xi(key, t, i)`` is added to the mean (``algo/privacy.py: dp_noise``).
    ``t`` is a one-element int64 tensor on the block's device: the round index over the run, advanced by the round.
    ``valid`` (uint8, on the block's device; None = every float is a parameter) holds, per 32-float chunk of the block,
    how many of its leading floats are parameters: the arena's alignment padding gets no noise and stays zero."""

    std: float
    key: int
    t: torch.Tensor
    valid: Optional[torch.Tensor] = None

    def mask(self, n: int) -> Optional[torch.Tensor]:
        """Boolean mask of the parameter coordinates of an ``n``-float block (None: all of them)."""
        if self.valid is None:
            return None
        i = torch.arange(n, device=self.valid.device)
        return (i % 32) < self.valid.long()[i // 32]


@dataclass
class QuantRound:
    """The compression of one round (``algo/compress.py``): ``bits`` (8 or 4), the key of the rounding stream and ``t``, a
    one-element int64 tensor on the block's device holding the index of the compressed round over the run (advanced by the
    round).  ``codes`` / ``scales`` are the local replicas' payload slices (:meth:`TorchCollective.payload_like_block`;
    on the fused collective peers read them), ``ef`` the local replicas' error-feedback vectors (in / out; None = off)."""

    bits: int
    key: int
    t: torch.Tensor
    codes: List[torch.Tensor]
    scales: List[torch.Tensor]
    ef: Optional[List[torch.Tensor]] = None


@dataclass
class SampleRound:
    """Client sampling of one round (``algo/sampling.py``): the ``S`` participants of sampled round ``t`` under ``key``
    are averaged with the weights ``n_k / sum_{j in P} n_j``.  ``t`` is a one-element int64 tensor on the block's device
    (the index of the sampled round over the run, advanced by the round), ``n`` the K workers' sample counts (int32, on
    the block's device)."""

    S: int
    key: int
    t: torch.Tensor
    n: torch.Tensor


@dataclass
class SecAggRound:
    """Secure aggregation of one round (``algo/secagg.py``): clip ``R``, fixed-point bits ``f``, the pair-key table
    ``keys`` (int32 ``[K (K - 1) / 2, 8]`` on the block's device, the uint32 words of :func:`secagg.pair_keys`) and ``t``,
    a one-element int64 tensor on the block's device holding the round index over the run (the nonce; advanced by the
    round).  ``payload`` holds the local replicas' payload slices (int32, 4 bytes per coordinate in whole segments of 16;
    :meth:`TorchCollective.payload32_like_block`; on the fused collective peers read them)."""

    clip: float
    f: int
    keys: torch.Tensor
    t: torch.Tensor
    payload: List[torch.Tensor]


@dataclass
class TopKRound:
    """Top-k sparsification of one round (``algo/compress.py: topk_select``): every worker sends the ``k`` coordinates of
    its update ``(x_k - z) + e_k`` with the largest magnitudes.  ``payload`` holds the local replicas' payload slices
    (:meth:`TorchCollective.sparse_payload_like_block`; on the fused collective peers read them), ``ef`` the local
    replicas' error-feedback vectors (in / out; None = off)."""

    k: int
    payload: List[torch.Tensor]
    ef: Optional[List[torch.Tensor]] = None


class TorchCollective:
    """ATen + torch.distributed implementation (baseline / oracle / CPU)."""

    name = "torch"
    fused = False

    def __init__(self, topo: Topology):
        self.topo = topo
        self.launches = 0  # number of framework-owned kernels launched (0 here: library path)
        self.last_dp = (0.0, 0.0)   # DP rounds: (#clipped workers, sum of their pre-clip update norms) over all K
        self.last_q = (0.0, 0.0)    # compressed / top-k rounds: (sum_k ||u_k - q_k s_k||^2, sum_k ||u_k||^2) over all K
        self.last_sa = (0, 0)       # secure-aggregation rounds: (#clipped, #non-finite coordinates) over all K

    # -- arena hooks ------------------------------------------------------
    def arena_allocator(self) -> Optional[Callable]:
        return None

    def register_arena(self, arena) -> None:
        return None

    def zeros_like_block(self, x: torch.Tensor, tag: str) -> torch.Tensor:
        """Zeroed companion vector of block slice ``x`` (ADMM duals).  The fused backend returns a slice of a
        symmetric arena so that peers can read it."""
        return torch.zeros_like(x)

    def payload_like_block(self, x: torch.Tensor, bits: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """Zeroed payload buffers of block slice ``x`` for ``bits``-bit codes: the codes (uint8, ``bits / 8`` bytes per
        coordinate, two 4-bit codes per byte with the even coordinate in the low nibble, whole segments of 16
        coordinates) and the scales (float32, one per group of ``compress.GROUP``).  The fused backend hands out slices of
        symmetric arenas so that peers can read them."""
        from ..algo.compress import GROUP

        n = x.numel()
        return (torch.zeros(-(-n // 16) * 2 * bits, dtype=torch.uint8, device=x.device),
                torch.zeros(-(-n // GROUP), dtype=torch.float32, device=x.device))

    def payload32_like_block(self, x: torch.Tensor) -> torch.Tensor:
        """Zeroed secure-aggregation payload of block slice ``x``: int32, one word per coordinate, whole segments of 16
        coordinates (one ChaCha20 block each).  The fused backend hands out slices of symmetric arenas."""
        return torch.zeros(-(-x.numel() // 16) * 16, dtype=torch.int32, device=x.device)

    def sparse_payload_like_block(self, x: torch.Tensor, k_sel: int) -> torch.Tensor:
        """Zeroed top-k payload of block slice ``x`` with ``k_sel`` entries: int32 words, layout
        ``algo/compress.py: topk_layout``.  The fused backend hands out slices of symmetric arenas."""
        from ..algo.compress import topk_layout

        return torch.zeros(topk_layout(x.numel(), k_sel)[3], dtype=torch.int32, device=x.device)

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

    def gather_blocks(self, xs: Sequence[torch.Tensor]) -> torch.Tensor:
        """``[K, n]``: the block slices of ALL K workers, row ``ck`` = worker ``ck`` (local replica ``j`` of rank ``r`` is
        worker ``r + j * world``)."""
        local = torch.stack(list(xs))
        W = self.topo.world_size
        if not self.topo.is_distributed:
            parts = [local]
        else:
            parts = [torch.empty_like(local) for _ in range(W)]
            dist.all_gather(parts, local, group=self.topo.group)
        full = torch.empty((self.topo.K,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        for r, part in enumerate(parts):
            for j in range(part.shape[0]):
                full[r + j * W] = part[j]
        return full

    def robust_aggregate(self, xs: Sequence[torch.Tensor], agg: str, trim_b: int) -> torch.Tensor:
        """Coordinate-wise order statistic over all K workers (fresh tensor).  NaN orders as +inf, +-inf keep their sign.
        'median': the middle value for odd K, ``(lo + hi) * 0.5`` of the two middle values for even K (``np.median``).
        'trimmed_mean': drop ``trim_b`` values at each end and average the rest, summed in ascending order
        (``scipy.stats.trim_mean``)."""
        K = self.topo.K
        check_robust(K, agg, trim_b)
        full = self.gather_blocks(xs)
        full = torch.where(torch.isnan(full), torch.full_like(full, float("inf")), full)
        srt = torch.sort(full, dim=0).values
        if agg == "median":
            hi = srt[K // 2]
            return hi.clone() if K % 2 else (srt[K // 2 - 1] + hi) * 0.5
        acc = srt[trim_b].clone()
        for j in range(trim_b + 1, K - trim_b):
            acc.add_(srt[j])
        return acc.div_(K - 2 * trim_b)

    def barrier(self) -> None:
        self.topo.barrier()

    # -- operators --------------------------------------------------------
    @torch.no_grad()
    def dp_clip_(self, xs: List[torch.Tensor], z: torch.Tensor, bound: float) -> None:
        """DP-FedAvg update clipping, in place: every local ``x_k`` with ``||x_k - z|| > bound`` becomes
        ``z + (bound / ||x_k - z||) (x_k - z)``; the others are not written (nor are non-finite norms).  The number of
        clipped workers and the sum of the pre-clip norms over all K go to :attr:`last_dp`."""
        stats = torch.zeros(2, dtype=torch.float64, device=z.device)
        z64 = z.double()
        for x in xs:                                  # in double: no finite float32 update overflows the norm
            d = x.double() - z64
            norm = torch.linalg.vector_norm(d)
            stats[1] += norm
            if bool(torch.isfinite(norm)) and bool(norm > bound):
                stats[0] += 1.0
                x.copy_(z64 + (bound / norm) * d)
        c, s = self.sum_scalars(stats).tolist()
        self.last_dp = (c, s)

    @staticmethod
    def _add_dp_noise_(mean: torch.Tensor, dp: DPRound) -> None:
        """``mean += std * xi(key, t)`` (the same draw on every rank), then ``t += 1``."""
        from ..algo.privacy import dp_noise

        t = int(dp.t.item())
        if dp.std != 0.0:
            xi = torch.from_numpy(dp_noise(dp.key, t, mean.numel())).to(device=mean.device, dtype=mean.dtype)
            mask = dp.mask(mean.numel())
            if mask is not None:
                xi.mul_(mask)
            mean.add_(xi.mul_(dp.std))
        dp.t.add_(1)

    @staticmethod
    def quantize_(u: torch.Tensor, bits: int, key: int, k: int, t: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """Codes (int8) and scales (float32) of update ``u`` of worker ``k`` in compressed round ``t``
        (``algo/compress.py: quantize``), on ``u``'s device."""
        from ..algo.compress import quantize

        codes, scales = quantize(u.detach().float().cpu().numpy(), bits, key, k, t)
        return torch.from_numpy(codes).to(u.device), torch.from_numpy(scales).to(u.device)

    @staticmethod
    def dequantize(codes: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
        """``q s`` per coordinate (float32)."""
        from ..algo.compress import GROUP

        return codes.float() * scales.repeat_interleave(GROUP)[: codes.numel()]

    @torch.no_grad()
    def _compressed_update(self, xs: List[torch.Tensor], z: torch.Tensor, q: QuantRound) -> torch.Tensor:
        """``d = (1/K) sum_k q_k s_k`` of a compressed round, summed in float32 in worker order ``k = 0 .. K-1``: every
        local replica is quantized (updating its error feedback and its payload slices), then the K dequantized updates
        are gathered.  Advances ``q.t``; the statistics go to :attr:`last_q`."""
        from ..algo.compress import pack4

        t = int(q.t.item())
        deqs, stats = [], torch.zeros(2, dtype=torch.float64, device=z.device)
        for j, (x, ck) in enumerate(zip(xs, self.topo.local_workers)):
            u = x - z
            if q.ef is not None:
                u = u + q.ef[j]
            codes, scales = self.quantize_(u, q.bits, q.key, ck, t)
            deq = self.dequantize(codes, scales)
            e = u - deq
            if q.ef is not None:
                q.ef[j].copy_(e)
            stats[0] += e.double().square().sum()
            stats[1] += u.double().square().sum()
            raw = codes.view(torch.uint8) if q.bits == 8 else torch.from_numpy(pack4(codes.cpu().numpy())).to(z.device)
            q.codes[j][: raw.numel()].copy_(raw)
            q.scales[j][: scales.numel()].copy_(scales)
            deqs.append(deq)
        full = self.gather_blocks(deqs)
        acc = full[0].clone()
        for k in range(1, self.topo.K):
            acc.add_(full[k])
        self.last_q = tuple(self.sum_scalars(stats).tolist())
        q.t.add_(1)
        return acc.mul_(1.0 / self.topo.K)

    @torch.no_grad()
    def _topk_update(self, xs: List[torch.Tensor], z: torch.Tensor, tk: TopKRound) -> torch.Tensor:
        """``d = (1/K) sum_k s_k`` of a top-k round, summed in float32 in worker order ``k = 0 .. K-1``: every local
        replica's update is selected with the oracle (updating its error feedback and its payload slice), then the K
        sparse updates are gathered densely.  The statistics go to :attr:`last_q`."""
        from ..algo.compress import topk_indices, topk_pack, topk_select

        sparse, stats = [], torch.zeros(2, dtype=torch.float64, device=z.device)
        for j, x in enumerate(xs):
            u = x - z
            if tk.ef is not None:
                u = u + tk.ef[j]
            pay = topk_select(u.detach().cpu().numpy(), tk.k)
            sel = torch.from_numpy(topk_indices(pay[0], pay[1])).to(z.device)
            s = torch.zeros_like(u)
            s[sel] = u[sel]
            e = u.clone()
            e[sel] = 0.0
            if tk.ef is not None:
                tk.ef[j].copy_(e)
            stats[0] += e.double().square().sum()
            stats[1] += u.double().square().sum()
            words = torch.from_numpy(topk_pack(pay, u.numel()))
            tk.payload[j][: words.numel()].copy_(words)
            sparse.append(s)
        full = self.gather_blocks(sparse)
        acc = full[0].clone()
        for k in range(1, self.topo.K):
            acc.add_(full[k])
        self.last_q = tuple(self.sum_scalars(stats).tolist())
        return acc.mul_(1.0 / self.topo.K)

    @torch.no_grad()
    def _secagg_update(self, xs: List[torch.Tensor], z: torch.Tensor, sa: SecAggRound) -> torch.Tensor:
        """``d = decode(sum_k y_k)`` of a secure-aggregation round: every local replica's update is encoded and masked with
        the oracle (into its payload slice), the K payloads are gathered and summed as integers mod 2^32, then decoded.
        Advances ``sa.t``; the counts go to :attr:`last_sa`."""
        from ..algo import secagg

        K, t, n = self.topo.K, int(sa.t.item()), z.numel()
        keys = sa.keys.cpu().numpy().view(np.uint32)
        zn = z.detach().float().cpu().numpy()
        pays, counts = [], torch.zeros(2, dtype=torch.int64)
        for j, (x, ck) in enumerate(zip(xs, self.topo.local_workers)):
            q, clipped, nonfinite = secagg.encode(x.detach().float().cpu().numpy() - zn, sa.clip, sa.f)
            y = torch.from_numpy(secagg.payload(q, keys, K, ck, t).view(np.int32))
            sa.payload[j][:n].copy_(y)
            pays.append((y.long() & 0xFFFFFFFF).to(z.device))
            counts += torch.tensor([clipped, nonfinite])
        S = self.gather_blocks(pays).sum(dim=0).remainder_(1 << 32).cpu().numpy().astype(np.uint32).view(np.int32)
        self.last_sa = tuple(int(v) for v in self.sum_scalars(counts.to(z.device)).tolist())
        sa.t.add_(1)
        return torch.from_numpy(secagg.decode(S, sa.f, K)).to(z.device)

    @torch.no_grad()
    def _sampled_mean(self, xs: List[torch.Tensor], s: SampleRound) -> torch.Tensor:
        """``sum_{k in P} w_k x_k`` of sampled round ``t = s.t`` (``algo/sampling.py``), summed in float32 in worker order,
        each term rounded before it is added; the K blocks are gathered, only the participants' rows are used.
        Advances ``s.t``."""
        from ..algo import sampling

        K = self.topo.K
        m = sampling.mask(s.key, int(s.t.item()), K, s.S)
        w = sampling.weights(s.n.cpu().numpy(), m)
        full = self.gather_blocks(xs)
        acc = torch.zeros_like(full[0])
        for k in range(K):
            if m[k]:
                acc = acc + full[k] * torch.tensor(w[k], dtype=full.dtype, device=full.device)
        s.t.add_(1)
        return acc

    @torch.no_grad()
    def average_(self, xs: List[torch.Tensor], z: torch.Tensor) -> None:
        """In place ``z <- mean_k x_k`` over all K workers, nothing written back and no residual read by the host (the
        SCAFFOLD server control variate)."""
        self.fedavg_(xs, z, write_back=False)

    @torch.no_grad()
    def fedavg_(self, xs: List[torch.Tensor], z: torch.Tensor, write_back: bool = True,
                dp: Optional[DPRound] = None, compress: Optional[QuantRound] = None,
                sample: Optional[SampleRound] = None, secagg: Optional[SecAggRound] = None,
                topk: Optional[TopKRound] = None) -> torch.Tensor:
        """In place: ``z <- mean_k x_k``, optionally ``x_k <- z``; returns ``||z_old - z_new||^2`` (0-dim).  With ``dp``
        the mean is noised (:class:`DPRound`; clip the replicas with :meth:`dp_clip_` first).  With ``compress``
        (:class:`QuantRound`) ``z <- z + (1/K) sum_k q_k s_k``, the workers' updates as uploaded.  With ``sample``
        (:class:`SampleRound`) ``z <-`` the sample-weighted mean of the round's participants; every replica receives it.
        With ``secagg`` (:class:`SecAggRound`) ``z <- z + d``, ``d`` decoded from the sum of the masked payloads.  With
        ``topk`` (:class:`TopKRound`) ``z <- z + (1/K) sum_k s_k``, the workers' sparse updates as uploaded."""
        if topk is not None:
            znew = z + self._topk_update(xs, z, topk)
        elif secagg is not None:
            znew = z + self._secagg_update(xs, z, secagg)
        elif sample is not None:
            znew = self._sampled_mean(xs, sample)
        elif compress is not None:
            znew = z + self._compressed_update(xs, z, compress)
        else:
            znew = self.sum_blocks(xs).div_(self.topo.K)
        if dp is not None:
            self._add_dp_noise_(znew, dp)
        diff = z - znew
        dual_sq = torch.dot(diff, diff)
        z.copy_(znew)
        if write_back:
            for x in xs:
                x.copy_(znew)
        return dual_sq

    @torch.no_grad()
    def robust_(self, xs: List[torch.Tensor], z: torch.Tensor, agg: str, trim_b: int = 0,
                write_back: bool = True) -> torch.Tensor:
        """:meth:`fedavg_` with a robust rule (:meth:`robust_aggregate`) in place of the mean: ``z <-`` the aggregate,
        optionally ``x_k <- z``; returns ``||z_old - z_new||^2`` (0-dim)."""
        znew = self.robust_aggregate(xs, agg, trim_b)
        diff = z - znew
        dual_sq = torch.dot(diff, diff)
        z.copy_(znew)
        if write_back:
            for x in xs:
                x.copy_(znew)
        return dual_sq

    @torch.no_grad()
    def fedopt_(self, xs: List[torch.Tensor], z: torch.Tensor, m: torch.Tensor, v: Optional[torch.Tensor], kind: str,
                lr: float, beta1: float, beta2: float, tau: float, agg: str = "mean", trim_b: int = 0,
                dp: Optional[DPRound] = None, compress: Optional[QuantRound] = None,
                sample: Optional[SampleRound] = None, secagg: Optional[SecAggRound] = None,
                topk: Optional[TopKRound] = None) -> torch.Tensor:
        """FedAvg with a server optimizer, in place: ``d = mean_k x_k - z`` is the pseudo-gradient of server optimizer
        ``kind`` (one of :data:`FEDOPT_KINDS`; ``beta1`` is the momentum of 'avgm'), whose state ``m`` (and ``v``, unused
        by 'avgm') it updates; ``z`` and every replica receive the new server model.  Returns ``||z_old - z_new||^2``.
        With a robust rule ``agg`` (one of :data:`ROBUST_AGGS`) its aggregate replaces the mean in ``d``; with ``dp`` the
        noised mean does (DP-FedOpt: post-processing); with ``compress`` ``d`` is the dequantized mean update itself
        (FedPAQ with a server optimizer); with ``sample`` the sample-weighted mean of the round's participants does; with
        ``secagg`` ``d`` is the decoded sum of the masked payloads; with ``topk`` ``d`` is the mean sparse update itself."""
        mean = None
        if topk is not None:
            d = self._topk_update(xs, z, topk)
        elif secagg is not None:
            d = self._secagg_update(xs, z, secagg)
        elif sample is not None:
            mean = self._sampled_mean(xs, sample)
        elif compress is not None:
            d = self._compressed_update(xs, z, compress)
        elif agg == "mean":
            mean = self.sum_blocks(xs).div_(self.topo.K)
            if dp is not None:
                self._add_dp_noise_(mean, dp)
        else:
            mean = self.robust_aggregate(xs, agg, trim_b)
        if mean is not None:
            d = mean - z
        if kind == "avgm":
            m.mul_(beta1).add_(d)
            # = z + lr m; from the mean exactly the mean when beta = 0 and lr = 1 (FedAvg)
            znew = z + lr * m if mean is None else mean + (lr * m - d)
        else:
            m.mul_(beta1).add_(d, alpha=1.0 - beta1)
            d2 = d * d
            if kind == "adagrad":
                v.add_(d2)
            elif kind == "adam":
                v.mul_(beta2).add_(d2, alpha=1.0 - beta2)
            elif kind == "yogi":
                v.sub_((1.0 - beta2) * d2 * torch.sign(v - d2))
            else:
                raise ValueError("unknown server optimizer %r" % (kind,))
            znew = z + lr * m / (v.sqrt() + tau)
        diff = z - znew
        dual_sq = torch.dot(diff, diff)
        z.copy_(znew)
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
