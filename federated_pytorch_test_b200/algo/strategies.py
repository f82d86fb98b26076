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

With client sampling (``FedAvg`` / ``FedOpt`` with ``client_n``) only the round's
participants train: the engine asks ``strat.participates(i)`` before the round's
steps and skips the others.

Preserved reference behaviour (SURVEY §2.12): ``z`` (and ``y``) start at 0 for
every block visit (Q6); FedProx/ADMM never write ``z`` back (Q7); ``rho`` is an
``[L,3]`` table of which only column 0 is used, shared by all workers and
updated sequentially over workers inside the BB step (Q8); the BB state
``yhat0`` is seeded with the parameter values (Q9).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence

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

    def participates(self, i: int) -> bool:
        """Whether local replica ``i`` trains in the current round (every replica, unless the strategy samples clients)."""
        return True

    def note_local_steps(self, steps: Sequence[int], lr: Optional[float]) -> None:
        """Called by the engine before every aggregation: the local steps each local replica took since the last one
        (0 for a replica that sat out) and the round's client learning rate.  Only SCAFFOLD uses them."""

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
    """FedAvg: ``z <-`` the mean of the K replicas, written back into every replica.  ``aggregator`` 'median' or
    'trimmed_mean' (Yin et al. 2018) replaces the mean by a coordinate-wise order statistic over the K replicas that a
    minority of diverging or malicious workers cannot move arbitrarily far (``trimmed_mean`` drops
    ``floor(trim_fraction K)`` values at each end); the round is otherwise the same.

    ``dp_clip > 0`` makes it DP-FedAvg (client-level differential privacy, McMahan et al. 2018; ``algo/privacy.py``).
    With ``z`` the server model the round started from, every worker's update ``x_k - z`` is clipped to
    ``C = dp_clip sqrt(N)`` (a worker within the bound is not written at all), and ``z <- mean_k x_k + (sigma C / K) xi``
    with ``sigma = dp_noise`` and ``xi`` the counter-based draw of DP round ``t`` (``t`` counts the DP rounds of the run and
    lives in device memory).  Each round is two launches on the fused collective (clip, aggregate).  ``z`` starts each
    block visit as the server model, i.e. the replicas' common value, instead of 0 (Q6), so the ``dual`` of the first round
    of a visit differs from plain FedAvg.  The round metrics gain ``dp_clipped`` (workers clipped), ``dp_update_norm``
    (mean pre-clip update norm over the K workers), ``dp_clip_norm`` (``C``) and ``dp_epsilon`` (spent so far at
    ``dp_delta``).

    ``compress_bits`` 8 or 4 compresses the workers' uploads (QSGD / FedPAQ; ``algo/compress.py``): with ``z`` the server
    model the round started from, worker ``k`` sends ``u_k = x_k - z`` (``+ e_k`` with ``compress_ef``) as stochastically
    rounded codes with one scale per 128 coordinates, and ``z <- z + (1/K) sum_k q_k s_k``, written back into every
    replica in fp32.  With error feedback ``e_k <- u_k - q_k s_k`` belongs to the worker and the block and persists across
    the block's visits for the whole run.  The rounding of compressed round ``t`` (``t`` counts the compressed rounds of
    the run and lives in device memory) is keyed by ``(seed, k, t, coordinate)``.  A round is one launch on the fused
    collective.  As with DP, ``z`` starts each block visit as the replicas' common value instead of 0 (Q6), so the
    ``dual`` of the first round of a visit differs from plain FedAvg.  The round metrics gain ``q_bits``, ``q_bytes``
    (payload bytes per worker: ``N bits / 8 + 4 ceil(N / 128)``) and ``q_rel_err``
    (``sqrt(sum_k ||u_k - q_k s_k||^2 / sum_k ||u_k||^2)``).

    ``client_n`` (the K workers' sample counts) makes it sample-weighted FedAvg with client sampling (McMahan et al.
    2017, Algorithm 1; ``algo/sampling.py``): sampled round ``t`` (``t`` counts the sampled rounds of the run and lives in
    device memory) trains only its ``clients_per_round`` participants (0 = all K), drawn uniformly from ``(seed, t)``, and
    ``z <- sum_{k in P} w_k x_k`` with ``w_k = n_k / sum_{j in P} n_j``, written back into every replica, participant or
    not.  Workers that sit out are never read.  A round is one launch on the fused collective.  The round metrics gain
    ``participants`` (the worker ids) and ``participant_samples`` (``sum_{k in P} n_k``).

    ``secagg`` makes it secure aggregation (SecAgg, Bonawitz et al. 2017; ``algo/secagg.py``): with ``z`` the server model
    the round started from, worker ``k`` uploads ``u_k = x_k - z`` as int32 fixed-point codes ``rint(clamp(u, -R, R) 2^f)``
    (``R = secagg_clip``) plus pairwise ChaCha20 masks keyed by pair keys derived from ``seed`` (or ``secagg_keys``) and
    the run's secure-aggregation round ``t`` (in device memory), which cancel in the sum; ``z <- z + (sum_k q_k) 2^-f / K``,
    written back into every replica.  Integer sums are exact, so the new model does not depend on the process layout.  A
    round is one launch on the fused collective.  As with DP, ``z`` starts each block visit as the replicas' common value
    instead of 0 (Q6), so the ``dual`` of the first round of a visit differs from plain FedAvg.  The round metrics gain
    ``sa_frac_bits`` (``f``) and ``sa_clipped`` (coordinates clipped, over all K); a non-finite update coordinate codes to
    0 and is reported as ``nonfinite``, so the NaN guard fires.

    ``compress_topk`` ``r`` in (0, 1) sparsifies the workers' uploads (top-k with optional error feedback, Stich et al.
    2018; ``algo/compress.py: topk_select``): with ``z`` the server model the round started from, worker ``k`` sends the
    ``k_sel = max(1, ceil(r N))`` coordinates of ``u_k = x_k - z`` (``+ e_k`` with ``compress_ef``) with the largest
    magnitudes, unchanged, and ``z <- z + (1/K) sum_k s_k``, written back into every replica.  With error feedback
    ``e_k <- u_k - s_k`` persists per worker and block for the whole run, as for ``compress_bits``.  A round is two launches
    on the fused collective (select, aggregate), and its sum does not depend on the process layout.  As with DP, ``z``
    starts each block visit as the replicas' common value instead of 0 (Q6).  The round metrics gain ``topk_k``,
    ``q_bytes`` (payload bytes per worker: ``6 k_sel + 4 (ceil(N / 8192) + 1)``) and ``q_rel_err``
    (``sqrt(sum_k ||u_k - s_k||^2 / sum_k ||u_k||^2)``).

    ``scaffold`` adds SCAFFOLD control variates (Karimireddy et al. 2020, option II; ``algo/scaffold.py``) to SGD client
    steps: every local step of worker ``i`` adds ``d_i = c - c_i`` to its gradient (``penalty(i).y``), and every round
    first updates the ``c_i`` of the workers that trained from their model change, averages ``c`` over all K and forms the
    next ``d_i`` (three launches), then aggregates the model as without it (mean, sample-weighted mean or server
    optimizer).  ``c`` and ``c_i`` persist per block for the whole run.  As with DP, ``z`` starts each block visit as the
    replicas' common value instead of 0 (Q6), so the ``dual`` of the first round of a visit differs from plain FedAvg.  The
    round metrics gain ``scaffold_corr``, the mean over this process' replicas of ``||c - c_i||``."""

    name = "fedavg"
    write_back = True
    forms_server_model = False      # FedOpt averages the replicas into z at the start of a visit itself

    def __init__(self, collective, topo, aggregator: str = "mean", trim_fraction: float = 0.1, dp_clip: float = 0.0,
                 dp_noise: float = 1.0, dp_delta: float = 1e-5, seed: int = 0, compress_bits: int = 0,
                 compress_ef: bool = False, clients_per_round: int = 0, client_n: Optional[Sequence[int]] = None,
                 secagg: bool = False, secagg_clip: float = 1.0, secagg_keys=None, scaffold: bool = False,
                 compress_topk: float = 0.0):
        from ..config import (check_aggregator, check_compress, check_dp, check_sampling, check_scaffold, check_secagg,
                              trim_count)

        super().__init__(collective, topo)
        check_aggregator(aggregator, trim_fraction, topo.K)
        check_dp(dp_clip, dp_noise, dp_delta, aggregator)
        check_compress(compress_bits, compress_ef, dp_clip, aggregator, compress_topk)
        self.aggregator = aggregator
        self.trim_b = trim_count(trim_fraction, topo.K) if aggregator == "trimmed_mean" else 0
        if aggregator != "mean" and hasattr(collective, "warm_robust"):
            collective.warm_robust = True
        self.dp = dp_clip > 0.0
        self.dp_clip, self.dp_noise, self.dp_delta = float(dp_clip), float(dp_noise), float(dp_delta)
        self.dp_rounds = 0                     # host mirror of the device round counter dp_t
        if self.dp:
            from .privacy import noise_key

            self.dp_key = noise_key(seed)
            self.dp_t = torch.zeros(1, dtype=torch.int64, device=topo.device)
            self.dp_layouts: Dict[int, torch.Tensor] = {}     # block index -> parameter layout (DPRound.valid)
            if hasattr(collective, "warm_dp"):
                collective.warm_dp = True
        self.q_bits, self.q_ef_on = int(compress_bits), bool(compress_ef)
        self.topk_r = float(compress_topk)
        self.q_rounds = 0                      # host mirror of the device round counter q_t
        self.q_ef: Dict[int, List[torch.Tensor]] = {}      # block index -> error feedback per local replica
        self._q_restored: Dict[int, torch.Tensor] = {}     # error feedback read from a resume record, installed at the visit
        if self.q_bits:
            from .compress import compress_key

            self.q_key = compress_key(seed)
            self.q_t = torch.zeros(1, dtype=torch.int64, device=topo.device)
            self.q_payload: List = []                          # (codes, scales) per local replica, current block
            if hasattr(collective, "warm_compress"):
                collective.warm_compress = self.q_bits
        if self.topk_r:
            self.topk_k = 0                                    # k_sel of the current block
            self.topk_payload: List[torch.Tensor] = []         # per local replica, current block
            if hasattr(collective, "warm_topk"):
                collective.warm_topk = True
        self.sampled = client_n is not None
        self.samp_rounds = 0                   # host mirror of the device round counter samp_t
        if self.sampled:
            from .sampling import sample_key

            check_sampling(clients_per_round, topo.K, "dirichlet", aggregator, dp_clip, compress_bits, compress_topk)
            if len(client_n) != topo.K or min(client_n) < 1:
                raise ValueError("client_n needs one sample count >= 1 per worker, got %r" % (list(client_n),))
            self.samp_S = int(clients_per_round) or topo.K
            self.samp_key = sample_key(seed)
            self.client_n = [int(v) for v in client_n]
            self.samp_t = torch.zeros(1, dtype=torch.int64, device=topo.device)
            self.samp_n = torch.tensor(self.client_n, dtype=torch.int32, device=topo.device)
            self._round_ids = (-1, None)                          # (t, participants of sampled round t)
            self._last_ids: List[int] = []
            if hasattr(collective, "warm_sample"):
                collective.warm_sample = True
        self.sa = bool(secagg)
        self.sa_rounds = 0                     # host mirror of the device round counter sa_t (the masks' nonce)
        if self.sa:
            import numpy as np

            from . import secagg as sa

            check_secagg(True, secagg_clip, topo.K, aggregator, dp_clip, compress_bits, clients_per_round,
                         "dirichlet" if client_n is not None else "iid", compress_topk)
            self.sa_clip = float(np.float32(secagg_clip))
            self.sa_f = sa.frac_bits(secagg_clip, topo.K)
            keys = sa.pair_keys(seed, topo.K) if secagg_keys is None else np.asarray(secagg_keys, dtype=np.uint32)
            if keys.shape != (topo.K * (topo.K - 1) // 2, 8):
                raise ValueError("secagg_keys needs one row of 8 words per worker pair, got shape %r" % (keys.shape,))
            self.sa_digest = sa.key_digest(keys)
            self.sa_keys = torch.from_numpy(keys.view(np.int32).copy()).to(topo.device)
            self.sa_t = torch.zeros(1, dtype=torch.int64, device=topo.device)
            self.sa_payload: List[torch.Tensor] = []                 # per local replica, current block
            if hasattr(collective, "warm_secagg"):
                collective.warm_secagg = True
        check_scaffold(scaffold, aggregator, dp_clip, compress_bits, secagg, compress_topk=compress_topk)
        self.scaffold = None
        if scaffold:
            from .scaffold import ControlVariates

            self.scaffold = ControlVariates(collective, topo)

    def begin_block(self, ci: int, N: int, xs: List[torch.Tensor]) -> None:
        super().begin_block(ci, N, xs)
        # the server model: the replicas are equal here, so a local copy suffices
        if (self.dp or self.q_bits or self.topk_r or self.sa
                or (self.scaffold is not None and not self.forms_server_model)):
            self.z.copy_(xs[0])
        if self.scaffold is not None:
            self.scaffold.begin_block(ci, xs)
        if self.sa:
            self.sa_payload = [self.coll.payload32_like_block(x) for x in xs]
        if self.q_bits:
            self.q_payload = [self.coll.payload_like_block(x, self.q_bits) for x in xs]
        if self.topk_r:
            from .compress import topk_count

            self.topk_k = topk_count(N, self.topk_r)
            self.topk_payload = [self.coll.sparse_payload_like_block(x, self.topk_k) for x in xs]
        if (self.q_bits or self.topk_r) and self.q_ef_on and ci not in self.q_ef:
            self.q_ef[ci] = [torch.zeros_like(x) for x in xs]
            if ci in self._q_restored:
                self._install_ef(ci, self._q_restored.pop(ci))

    # -- SCAFFOLD --------------------------------------------------------------------------------------------------------
    def penalty(self, i: int) -> Penalty:
        return Penalty(y=self.scaffold.correction(i)) if self.scaffold is not None else Penalty()

    def note_local_steps(self, steps: Sequence[int], lr: Optional[float]) -> None:
        if self.scaffold is not None:
            self.scaffold.note_local_steps(steps, lr)

    def _scaffold_round(self) -> None:
        """Steps 1-3 of the control variates, launched before the model aggregation (which overwrites ``z``)."""
        if self.scaffold is not None:
            self.scaffold.end_round(self.xs, self.z)

    def _with_scaffold(self, metrics: Dict[str, float]) -> Dict[str, float]:
        if self.scaffold is not None:
            metrics["scaffold_corr"] = self.scaffold.corr_norm()
        return metrics

    def _scaffold_state(self) -> Dict[str, object]:
        if self.scaffold is None:
            return {}
        return {"scaffold": True, **self.scaffold.state()}

    def _check_scaffold_state(self, st: Dict[str, object]) -> None:
        got, want = bool(st.get("scaffold", False)), self.scaffold is not None
        if got != want:
            raise ValueError("resume record was written with scaffold %r, this run uses scaffold %r" % (got, want))
        if self.scaffold is not None:
            self.scaffold.load_state(st)

    # -- client sampling -------------------------------------------------------------------------------------------------
    def round_participants(self) -> List[int]:
        """The workers of the round in progress (all K without sampling)."""
        if not self.sampled:
            return list(range(self.topo.K))
        if self._round_ids[0] != self.samp_rounds:
            from .sampling import participants

            self._round_ids = (self.samp_rounds, [int(k) for k in participants(self.samp_key, self.samp_rounds,
                                                                                self.topo.K, self.samp_S)])
        return self._round_ids[1]

    def participates(self, i: int) -> bool:
        return not self.sampled or self.topo.local_workers[i] in self.round_participants()

    def _samp_kw(self) -> Dict[str, object]:
        """The sampling argument of the aggregation (which advances the round counter)."""
        if not self.sampled:
            return {}
        from ..parallel.collective import SampleRound

        self._last_ids = self.round_participants()
        self.samp_rounds += 1
        return {"sample": SampleRound(self.samp_S, self.samp_key, self.samp_t, self.samp_n)}

    def _with_samp(self, metrics: Dict[str, float]) -> Dict[str, float]:
        if self.sampled:
            metrics.update(participants=list(self._last_ids),
                           participant_samples=float(sum(self.client_n[k] for k in self._last_ids)))
        return metrics

    def _samp_state(self) -> Dict[str, object]:
        if not self.sampled:
            return {}
        return {"sample": (self.samp_S, self.samp_key, tuple(self.client_n)), "samp_t": self.samp_rounds}

    def _check_samp_state(self, st: Dict[str, object]) -> None:
        got = tuple(st["sample"]) if st.get("sample") is not None else None
        want = self._samp_state().get("sample")
        if got != want:
            raise ValueError("resume record holds client-sampling settings (clients_per_round, key, shard sizes) %r, this "
                             "run uses %r" % (got, want))
        if self.sampled:
            self.samp_rounds = int(st["samp_t"])
            self.samp_t.fill_(self.samp_rounds)

    # -- secure aggregation ---------------------------------------------------------------------------------------------
    def _sa_kw(self) -> Dict[str, object]:
        """The secure-aggregation argument of the aggregation (which advances the round counter)."""
        if not self.sa:
            return {}
        from ..parallel.collective import SecAggRound

        self.sa_rounds += 1
        return {"secagg": SecAggRound(self.sa_clip, self.sa_f, self.sa_keys, self.sa_t, self.sa_payload)}

    def _with_sa(self, metrics: Dict[str, float]) -> Dict[str, float]:
        if self.sa:
            clipped, nonfinite = self.coll.last_sa
            metrics.update(sa_frac_bits=float(self.sa_f), sa_clipped=float(clipped))
            if nonfinite:
                metrics["nonfinite"] = float(nonfinite)
        return metrics

    def _sa_state(self) -> Dict[str, object]:
        if not self.sa:
            return {}
        return {"secagg": (self.sa_clip, self.sa_f, self.sa_digest), "sa_t": self.sa_rounds}

    def _check_sa_state(self, st: Dict[str, object]) -> None:
        got = tuple(st["secagg"]) if st.get("secagg") is not None else None
        want = self._sa_state().get("secagg")
        if got != want:
            raise ValueError("resume record holds secure-aggregation settings (secagg_clip, f, SHA-256 of the pair keys) %r, "
                             "this run uses %r" % (got, want))
        if self.sa:
            self.sa_rounds = int(st["sa_t"])
            self.sa_t.fill_(self.sa_rounds)

    # -- compressed updates -------------------------------------------------------------------------------------------
    def _q_kw(self) -> Dict[str, object]:
        """The compression argument of the aggregation."""
        if not self.q_bits:
            return {}
        from ..parallel.collective import QuantRound

        self.q_rounds += 1
        return {"compress": QuantRound(self.q_bits, self.q_key, self.q_t, [c for c, _ in self.q_payload],
                                       [s for _, s in self.q_payload], self.q_ef.get(self.ci))}

    def _with_q(self, metrics: Dict[str, float]) -> Dict[str, float]:
        if self.q_bits:
            from .compress import payload_bytes, relative_error

            err, nrm = self.coll.last_q
            metrics.update(q_bits=float(self.q_bits), q_bytes=float(payload_bytes(self.N, self.q_bits)),
                           q_rel_err=relative_error(float(err), float(nrm)))
        return metrics

    def _install_ef(self, ci: int, ef: torch.Tensor) -> None:
        for dst, src in zip(self.q_ef[ci], ef):
            dst.copy_(src.to(dst.device))

    def _ef_state(self) -> Dict[str, object]:
        """The error feedback of this process' workers; blocks restored but not visited yet keep their record."""
        if not self.q_ef_on:
            return {}
        ef = dict(self._q_restored)
        ef.update({ci: torch.stack(v) for ci, v in self.q_ef.items()})
        return {"q_ef": ef}

    def _load_ef(self, st: Dict[str, object]) -> None:
        for ci, ef in (st.get("q_ef") or {}).items():
            if ci in self.q_ef:
                self._install_ef(ci, ef)
            else:
                self._q_restored[ci] = ef

    def _q_state(self) -> Dict[str, object]:
        if not self.q_bits:
            return {}
        return {"compress": (self.q_bits, self.q_ef_on, self.q_key), "q_t": self.q_rounds, **self._ef_state()}

    def _check_q_state(self, st: Dict[str, object]) -> None:
        got = tuple(st["compress"]) if st.get("compress") is not None else None
        want = self._q_state().get("compress")
        if got != want:
            raise ValueError("resume record holds compression settings (compress_bits, compress_ef, key) %r, this run uses "
                             "%r" % (got, want))
        if self.q_bits:
            self.q_rounds = int(st["q_t"])
            self.q_t.fill_(self.q_rounds)
            self._load_ef(st)

    # -- top-k sparsified updates ------------------------------------------------------------------------------------
    def _topk_kw(self) -> Dict[str, object]:
        """The top-k argument of the aggregation."""
        if not self.topk_r:
            return {}
        from ..parallel.collective import TopKRound

        return {"topk": TopKRound(self.topk_k, self.topk_payload, self.q_ef.get(self.ci))}

    def _with_topk(self, metrics: Dict[str, float]) -> Dict[str, float]:
        if self.topk_r:
            from .compress import relative_error, topk_payload_bytes

            err, nrm = self.coll.last_q
            metrics.update(topk_k=float(self.topk_k), q_bytes=float(topk_payload_bytes(self.N, self.topk_k)),
                           q_rel_err=relative_error(float(err), float(nrm)))
        return metrics

    def _topk_state(self) -> Dict[str, object]:
        if not self.topk_r:
            return {}
        return {"topk": (self.topk_r, self.q_ef_on), **self._ef_state()}

    def _check_topk_state(self, st: Dict[str, object]) -> None:
        got = tuple(st["topk"]) if st.get("topk") is not None else None
        want = self._topk_state().get("topk")
        if got != want:
            raise ValueError("resume record holds top-k settings (compress_topk, compress_ef) %r, this run uses %r"
                             % (got, want))
        if self.topk_r:
            self._load_ef(st)

    # -- DP -------------------------------------------------------------------------------------------------------
    def set_param_layout(self, ci: int, chunk_counts: List[int]) -> None:
        """The parameter layout of block ``ci`` (``FlatArena.chunk_counts``): the noise skips the alignment padding.
        Without it every float of the block slice is noised."""
        if ci not in self.dp_layouts:
            self.dp_layouts[ci] = torch.tensor(chunk_counts, dtype=torch.uint8, device=self.topo.device)

    def dp_bound(self) -> float:
        """``C`` of the current block."""
        return self.dp_clip * math.sqrt(self.N)

    def _dp_kw(self) -> Dict[str, object]:
        """Clip the local replicas (first launch of a DP round) and return the noise argument of the aggregation."""
        if not self.dp:
            return {}
        from ..parallel.collective import DPRound

        C = self.dp_bound()
        self.coll.dp_clip_(self.xs, self.z, C)
        self.dp_rounds += 1
        return {"dp": DPRound(self.dp_noise * C / self.topo.K, self.dp_key, self.dp_t, self.dp_layouts.get(self.ci))}

    def dp_epsilon(self, rounds: Optional[int] = None) -> float:
        from .privacy import gaussian_epsilon

        return gaussian_epsilon(self.dp_noise, self.dp_rounds if rounds is None else rounds, self.dp_delta)

    def _with_dp(self, metrics: Dict[str, float]) -> Dict[str, float]:
        if self.dp:
            clipped, norms = self.coll.last_dp
            metrics.update(dp_clipped=float(clipped), dp_update_norm=float(norms) / self.topo.K,
                           dp_clip_norm=self.dp_bound(), dp_epsilon=self.dp_epsilon())
        return metrics

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        self._scaffold_round()
        if self.aggregator == "mean":
            dual_sq = self.coll.fedavg_(self.xs, self.z, write_back=True, **self._dp_kw(), **self._q_kw(),
                                        **self._samp_kw(), **self._sa_kw(), **self._topk_kw())
        else:
            dual_sq = self.coll.robust_(self.xs, self.z, self.aggregator, self.trim_b)
        return self._with_topk(self._with_scaffold(self._with_sa(self._with_samp(self._with_q(self._with_dp(
            {"dual": math.sqrt(max(float(dual_sq), 0.0)) / self.N}))))))

    def aggregate_begin(self, nadmm: int):
        if getattr(self.coll, "supports_async", False):
            self._scaffold_round()
            if self.aggregator == "mean":
                self.coll.launch_fedavg_(self.xs, self.z, True, **self._dp_kw(), **self._q_kw(), **self._samp_kw(),
                                         **self._sa_kw(), **self._topk_kw())
            else:
                self.coll.launch_robust_(self.xs, self.z, self.aggregator, self.trim_b)
            return ("pending", self.N)
        return ("done", self.aggregate(nadmm))

    def aggregate_end(self, token) -> Dict[str, float]:
        if token[0] == "done":
            return token[1]
        return self._with_topk(self._with_scaffold(self._with_sa(self._with_samp(self._with_q(self._with_dp(
            {"dual": math.sqrt(max(float(self.coll.read_record()[0]), 0.0)) / token[1]}))))))

    def _robust_state(self) -> Dict[str, object]:
        return {} if self.aggregator == "mean" else {"aggregator": self.aggregator, "trim_b": self.trim_b}

    def _check_robust_state(self, st: Dict[str, object]) -> None:
        got = (st.get("aggregator", "mean"), int(st.get("trim_b", 0)))
        if got != (self.aggregator, self.trim_b):
            raise ValueError("resume record holds aggregator %r (trim_b %d), this run uses %r (trim_b %d)"
                             % (got + (self.aggregator, self.trim_b)))

    def _dp_state(self) -> Dict[str, object]:
        if not self.dp:
            return {}
        return {"dp": (self.dp_clip, self.dp_noise, self.dp_delta, self.dp_key), "dp_t": self.dp_rounds}

    def _check_dp_state(self, st: Dict[str, object]) -> None:
        got = tuple(st["dp"]) if st.get("dp") is not None else None
        want = self._dp_state().get("dp")
        if got != want:
            raise ValueError("resume record holds DP settings (dp_clip, dp_noise, dp_delta, key) %r, this run uses %r"
                             % (got, want))
        if self.dp:
            self.dp_rounds = int(st["dp_t"])
            self.dp_t.fill_(self.dp_rounds)

    def state(self) -> Dict[str, object]:
        return {"z": self.z, **self._robust_state(), **self._dp_state(), **self._q_state(), **self._samp_state(),
                **self._sa_state(), **self._scaffold_state(), **self._topk_state()}

    def load_state(self, st: Dict[str, object]) -> None:
        self._check_robust_state(st)
        self._check_dp_state(st)
        self._check_q_state(st)
        self._check_topk_state(st)
        self._check_samp_state(st)
        self._check_sa_state(st)
        self._check_scaffold_state(st)
        self.z.copy_(st["z"].to(self.z.device))


class FedOpt(FedAvg):
    """FedAvg with a server optimizer (FedAvgM, Hsu et al. 2019; FedAdagrad / FedAdam / FedYogi, Reddi et al. 2021,
    Algorithm 2 without bias correction).  The round's mean change ``d = mean_k x_k - z`` is a pseudo-gradient:

    * avgm:     ``m <- beta m + d``;                                          ``z <- z + lr m``
    * adagrad:  ``m <- beta1 m + (1 - beta1) d``;  ``v <- v + d^2``;          ``z <- z + lr m / (sqrt(v) + tau)``
    * adam:     same ``m``;  ``v <- beta2 v + (1 - beta2) d^2``;              same ``z``
    * yogi:     same ``m``;  ``v <- v - (1 - beta2) d^2 sign(v - d^2)``;      same ``z``

    and the new ``z`` is written into every replica, as FedAvg does.  ``z`` is the server model: the mean of the replicas
    at the start of a block visit (one extra aggregation launch per visit).  ``m`` / ``v`` belong to a block and persist
    across its visits for the whole run (``m = 0``, ``v = tau^2`` at its first visit); on the fused collective they are
    slices of symmetric arenas, so two-shot ranks broadcast their slice of both into every rank and every rank ends each
    round with the same ``z``, ``m`` and ``v``.  With a robust ``aggregator`` its aggregate replaces the mean in ``d``
    (e.g. robust FedAdam); the server model at the start of a visit stays the mean (the replicas are equal then).  With DP
    (``dp_clip > 0``) the noised mean of the clipped workers replaces the mean in ``d`` (DP-FedAdam etc.: post-processing),
    and the server model at the start of a visit is the replicas' common value, copied locally (no launch).  With
    compressed updates (``compress_bits``) ``d`` is the dequantized mean update itself (FedPAQ with a server optimizer),
    and the server model at the start of a visit is again the replicas' common value.  With client sampling
    (``client_n``) the participants' sample-weighted mean replaces the mean in ``d``; the server model at the start of a
    visit stays the unsampled mean of the (equal) replicas and does not advance the sampling counter.  With secure
    aggregation (``secagg``) ``d`` is the decoded sum of the masked updates, and the server model at the start of a visit
    is the replicas' common value.  With SCAFFOLD (``scaffold``) the control variates are updated before the server step,
    exactly as for FedAvg; ``avgm`` with ``momentum 0`` and ``lr eta_g`` is the paper's global step size ``eta_g``."""

    name = "fedopt"
    forms_server_model = True

    def __init__(self, collective, topo, kind: str = "adam", lr: float = 0.0, momentum: float = 0.9, beta1: float = 0.9,
                 beta2: float = 0.99, tau: float = 1e-3, aggregator: str = "mean", trim_fraction: float = 0.1,
                 dp_clip: float = 0.0, dp_noise: float = 1.0, dp_delta: float = 1e-5, seed: int = 0, compress_bits: int = 0,
                 compress_ef: bool = False, clients_per_round: int = 0, client_n: Optional[Sequence[int]] = None,
                 secagg: bool = False, secagg_clip: float = 1.0, secagg_keys=None, scaffold: bool = False,
                 compress_topk: float = 0.0):
        from ..config import check_server_opt
        from ..parallel.collective import FEDOPT_KINDS

        super().__init__(collective, topo, aggregator, trim_fraction, dp_clip, dp_noise, dp_delta, seed, compress_bits,
                         compress_ef, clients_per_round, client_n, secagg, secagg_clip, secagg_keys, scaffold,
                         compress_topk)
        if kind not in FEDOPT_KINDS:
            raise ValueError("server optimizer must be one of %s, got %r" % (", ".join(FEDOPT_KINDS), kind))
        check_server_opt(kind, lr, momentum, beta1, beta2, tau)
        self.kind = kind
        self.adaptive = kind != "avgm"
        self.lr = float(lr) or (1e-2 if self.adaptive else 1.0)
        self.beta1 = float(beta1 if self.adaptive else momentum)
        self.beta2, self.tau = float(beta2), float(tau)
        self.m: Optional[torch.Tensor] = None
        self.v: Optional[torch.Tensor] = None
        self.ms: Dict[int, torch.Tensor] = {}              # block index -> server state slice, for the whole run
        self.vs: Dict[int, torch.Tensor] = {}
        self._restored: Dict[int, tuple] = {}              # state of blocks read from a resume record, installed at their visit
        if hasattr(collective, "warm_fedopt"):
            collective.warm_fedopt = True

    def begin_block(self, ci: int, N: int, xs: List[torch.Tensor]) -> None:
        super().begin_block(ci, N, xs)
        if ci not in self.ms:
            self.ms[ci] = self.coll.zeros_like_block(xs[0], "srv_m")
            if self.adaptive:
                self.vs[ci] = self.coll.zeros_like_block(xs[0], "srv_v").fill_(self.tau * self.tau)
            if ci in self._restored:
                self._install(ci, *self._restored.pop(ci))
        self.m, self.v = self.ms[ci], self.vs.get(ci)
        if not (self.dp or self.q_bits or self.topk_r or self.sa):   # (else FedAvg.begin_block copied the replicas' value)
            self.coll.fedavg_(xs, self.z, write_back=False)      # the server model: the replicas' mean, no write-back

    def _hyper(self):
        return self.kind, self.lr, self.beta1, self.beta2, self.tau

    def _agg_kw(self) -> Dict[str, object]:
        return {} if self.aggregator == "mean" else {"agg": self.aggregator, "trim_b": self.trim_b}

    def aggregate(self, nadmm: int) -> Dict[str, float]:
        self._scaffold_round()
        dual_sq = self.coll.fedopt_(self.xs, self.z, self.m, self.v, *self._hyper(), **self._agg_kw(), **self._dp_kw(),
                                    **self._q_kw(), **self._samp_kw(), **self._sa_kw(), **self._topk_kw())
        return self._with_topk(self._with_scaffold(self._with_sa(self._with_samp(self._with_q(self._with_dp(
            {"dual": math.sqrt(max(float(dual_sq), 0.0)) / self.N}))))))

    def aggregate_begin(self, nadmm: int):
        if getattr(self.coll, "supports_async", False):
            self._scaffold_round()
            self.coll.launch_fedopt_(self.xs, self.z, self.m, self.v, *self._hyper(), **self._agg_kw(), **self._dp_kw(),
                                     **self._q_kw(), **self._samp_kw(), **self._sa_kw(), **self._topk_kw())
            return ("pending", self.N)
        return ("done", self.aggregate(nadmm))

    def state(self) -> Dict[str, object]:
        """``z`` and the state of every block visited so far in the run, including blocks restored from a resume record
        that this process has not visited yet (their state is still the recorded one)."""
        ms = {ci: m for ci, (m, _) in self._restored.items()}
        vs = {ci: v for ci, (_, v) in self._restored.items() if v is not None}
        ms.update(self.ms)
        vs.update(self.vs)
        return {"z": self.z, "server_opt": self.kind, "m": ms, "v": vs, **self._robust_state(), **self._dp_state(),
                **self._q_state(), **self._samp_state(), **self._sa_state(), **self._scaffold_state(), **self._topk_state()}

    def _install(self, ci: int, m: torch.Tensor, v: Optional[torch.Tensor]) -> None:
        self.ms[ci].copy_(m.to(self.ms[ci].device))
        if self.adaptive:
            self.vs[ci].copy_(v.to(self.vs[ci].device))

    def load_state(self, st: Dict[str, object]) -> None:
        if st.get("server_opt") != self.kind:
            raise ValueError("resume record holds server optimizer %r, this run uses %r" % (st.get("server_opt"), self.kind))
        self._check_robust_state(st)
        self._check_dp_state(st)
        self._check_q_state(st)
        self._check_topk_state(st)
        self._check_samp_state(st)
        self._check_sa_state(st)
        self._check_scaffold_state(st)
        self.z.copy_(st["z"].to(self.z.device))
        vs = st.get("v") or {}
        for ci, m in (st.get("m") or {}).items():
            if ci in self.ms:
                self._install(ci, m, vs.get(ci))
            else:                                                 # buffers are made at the block's next visit
                self._restored[ci] = (m, vs.get(ci))


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
