"""``federated_multi`` — federated averaging over one parameter block at a time.

Reference: /root/reference/src/federated_multi.py (mean over K then write-back into every
replica, ``dual = ||z - z_new|| / N``; CE + gated elastic net; Adam 1e-3 per block visit).
On the GPU the aggregation is one fused NVLink kernel on the block slice of the replicas'
parameter arenas (``csrc/comm_kernels.cu``), no NCCL on the path.

``--server_opt avgm|adagrad|adam|yogi`` replaces the plain mean by a server optimizer step (``FedOpt``), fused into
the same kernel; the default ``none`` is the reference's FedAvg.
"""
from __future__ import annotations

from ..algo.strategies import FedAvg, FedOpt
from ..config import FederatedConfig, parse_config
from . import common

Config = FederatedConfig


def make_strategy(cfg: Config, coll, topo):
    if cfg.server_opt == "none":
        return FedAvg(coll, topo)
    return FedOpt(coll, topo, cfg.server_opt, cfg.server_lr, cfg.server_momentum, cfg.server_beta1, cfg.server_beta2,
                  cfg.server_tau)


def run(cfg: Config, log=print):
    topo, coll = common.setup_runtime(cfg)
    task = common.ClassifierTask(cfg, topo, cfg.lambda1, cfg.lambda2)
    engine = common.run_engine(cfg, task, topo, coll, make_strategy(cfg, coll, topo), None, log)
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="federated_multi"))


if __name__ == "__main__":
    main()
