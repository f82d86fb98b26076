"""``federated_multi`` — federated averaging over one parameter block at a time.

Reference: /root/reference/src/federated_multi.py (mean over K then write-back into every
replica, ``dual = ||z - z_new|| / N``; CE + gated elastic net; Adam 1e-3 per block visit).
On the GPU the aggregation is one fused NVLink kernel on the block slice of the replicas'
parameter arenas (``csrc/comm_kernels.cu``), no NCCL on the path.

``--server_opt avgm|adagrad|adam|yogi`` replaces the plain mean by a server optimizer step (``FedOpt``), fused into
the same kernel; the default ``none`` is the reference's FedAvg.

``--aggregator median|trimmed_mean`` (``--trim_fraction``) replaces the mean of the K replicas by a coordinate-wise order
statistic (Byzantine-robust aggregation), with or without a server optimizer; ``--byzantine b --attack
signflip|gaussian|nan --attack_scale s`` turns the last b workers into simulated attackers (``algo/byzantine.py``).

``--dp_clip c --dp_noise sigma --dp_delta delta`` makes the mean DP-FedAvg (client-level differential privacy, with or
without a server optimizer): every worker's block update is clipped to ``c sqrt(N)`` and Gaussian noise is added to the
mean (``algo/privacy.py``).  The root logs ``dp: ...`` lines with the planned and the spent epsilon.

``--compress_bits 8|4 [--compress_ef]`` compresses what every worker uploads (QSGD / FedPAQ, with or without a server
optimizer): its block update ``x_k - z`` as stochastically rounded codes with one scale per 128 coordinates, optionally
with error feedback (``algo/compress.py``); the new model is still broadcast in fp32.  Round metrics gain ``q_bits``,
``q_bytes`` and ``q_rel_err``.

``--compress_topk r [--compress_ef]`` sparsifies what every worker uploads (top-k, with or without a server optimizer and
error feedback): the ``max(1, ceil(r N))`` largest-magnitude coordinates of its block update ``x_k - z``, unchanged, with
their indices (``algo/compress.py: topk_select``); the new model is still broadcast in fp32.  Round metrics gain
``topk_k``, ``q_bytes`` and ``q_rel_err``.

``--clients_per_round S`` trains and averages a uniform random subset of S of the K workers in every round (FedAvg's
partial participation, with or without a server optimizer); ``--partition dirichlet --dirichlet_alpha a`` splits the
training set with Dirichlet label skew into unequal shards.  Either one makes the aggregate the sample-weighted mean
``sum_{k in P} n_k x_k / sum_{k in P} n_k`` of the round's participants P (all K without ``--clients_per_round``), one
fused launch that reads only the participants (``algo/sampling.py``); workers that sit out take no step and receive the
new model.  Round metrics gain ``participants`` and ``participant_samples``; the root writes a ``partition`` row with the
shard sizes and per-worker class counts.

``--secagg [--secagg_clip R]`` makes every round secure aggregation (SecAgg, with or without a server optimizer): each
worker uploads its block update ``x_k - z`` as int32 fixed-point codes of ``clamp(u, -R, R)`` masked with pairwise
ChaCha20 keystreams that cancel in the sum (``algo/secagg.py``), so the server learns only the sum.  The pair keys are
derived from ``--seed`` in place of a key agreement: whoever knows the seed can unmask.  Round metrics gain
``sa_frac_bits`` and ``sa_clipped``.

``--scaffold`` (with ``--optimizer sgd``) adds SCAFFOLD control variates (Karimireddy et al. 2020, option II) against
client drift on skewed shards, with or without a server optimizer, client sampling or a Dirichlet partition: every local
SGD step adds ``c - c_i`` to the gradient, and every round updates the workers' ``c_i`` from their model change
``(z - x_i) / (tau_i lr)``, averages ``c`` over all K workers, then aggregates the model as without it
(``algo/scaffold.py``).  With momentum that model change is about ``1 / (1 - momentum)`` times the mean gradient; it is
used unchanged, as in most implementations.  Simulated Byzantine workers (``--byzantine``) attack before the control
variates are updated, so an attacker's ``c_i`` comes from its attacked model.  Round metrics gain ``scaffold_corr``
(mean ``||c - c_i||`` over the process' workers).
"""
from __future__ import annotations

from ..algo.byzantine import ByzantineAttack
from ..algo.privacy import dp_line
from ..algo.strategies import FedAvg, FedOpt
from ..config import FederatedConfig, parse_config, sampled_rounds
from . import common

Config = FederatedConfig


def make_strategy(cfg: Config, coll, topo, client_n=None):
    """The run's strategy.  ``client_n``: the workers' sample counts, which weight sampled rounds (default: equal)."""
    robust = {} if cfg.aggregator == "mean" else dict(aggregator=cfg.aggregator, trim_fraction=cfg.trim_fraction)
    if cfg.dp_clip > 0.0:
        robust.update(dp_clip=cfg.dp_clip, dp_noise=cfg.dp_noise, dp_delta=cfg.dp_delta, seed=cfg.seed)
    if cfg.compress_bits:
        robust.update(compress_bits=cfg.compress_bits, compress_ef=cfg.compress_ef, seed=cfg.seed)
    if cfg.compress_topk:
        robust.update(compress_topk=cfg.compress_topk, compress_ef=cfg.compress_ef)
    if sampled_rounds(cfg.clients_per_round, cfg.K, cfg.partition):
        robust.update(clients_per_round=cfg.clients_per_round, client_n=client_n or [1] * cfg.K, seed=cfg.seed)
    if cfg.secagg:
        robust.update(secagg=True, secagg_clip=cfg.secagg_clip, seed=cfg.seed)
    if cfg.scaffold:
        robust.update(scaffold=True)
    if cfg.server_opt == "none":
        return FedAvg(coll, topo, **robust)
    return FedOpt(coll, topo, cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_beta1, cfg.server_beta2,
                  cfg.server_tau, **robust)


def make_attack(cfg: Config):
    """The simulated Byzantine workers of the run, or None (``byzantine = 0``)."""
    if cfg.byzantine == 0:
        return None
    return ByzantineAttack(cfg.K, cfg.byzantine, cfg.attack, cfg.attack_scale, cfg.seed)


def run(cfg: Config, log=print):
    topo, coll = common.setup_runtime(cfg)
    task = common.ClassifierTask(cfg, topo, cfg.lambda1, cfg.lambda2)
    strategy = make_strategy(cfg, coll, topo, task.shard_sizes())
    dp_log = strategy.dp and topo.is_root
    if dp_log:
        planned = cfg.Nloop * len(list(task.visits(0))) * cfg.Nadmm * cfg.Nepoch
        log(dp_line(cfg.dp_noise, cfg.dp_clip, cfg.dp_delta, planned, planned=True))
    engine = common.run_engine(cfg, task, topo, coll, strategy, None, log, attack=make_attack(cfg))
    if dp_log:
        log(dp_line(cfg.dp_noise, cfg.dp_clip, cfg.dp_delta, strategy.dp_rounds, planned=False))
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="federated_multi"))


if __name__ == "__main__":
    main()
