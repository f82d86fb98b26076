"""``federated_multi`` — federated averaging over one parameter block at a time.

Reference: /root/reference/src/federated_multi.py (mean over K then write-back into every
replica, ``dual = ||z - z_new|| / N``; CE + gated elastic net; Adam 1e-3 per block visit).
On the GPU the aggregation is one fused NVLink kernel on the block slice of the replicas'
parameter arenas (``csrc/comm_kernels.cu``), no NCCL on the path.
"""
from __future__ import annotations

from ..algo.strategies import FedAvg
from ..config import FederatedConfig, parse_config
from . import common

Config = FederatedConfig


def run(cfg: Config, log=print):
    topo, coll = common.setup_runtime(cfg)
    task = common.ClassifierTask(cfg, topo, cfg.lambda1, cfg.lambda2)
    engine = common.run_engine(cfg, task, topo, coll, FedAvg(coll, topo), None, log)
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="federated_multi"))


if __name__ == "__main__":
    main()
