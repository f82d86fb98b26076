"""``fedprox_multi`` — FedProx over one parameter block at a time.

Reference: /root/reference/src/fedprox_multi.py (local loss + mu/2 ||x - z||^2 with
mu = ``admm_rho0`` = 1.0, z = mean, no write-back, primal/dual residuals).  The proximal
gradient is closed-form inside the optimizer kernel; the aggregation kernel also returns
both residual norms.

``--partition dirichlet`` gives the workers label-skewed shards of unequal size; z stays the unweighted mean of the K
workers, as in the reference (sample-count weights and client sampling are ``federated_multi``'s).
"""
from __future__ import annotations

from ..algo.strategies import FedProx
from ..config import FedProxConfig, parse_config
from . import common

Config = FedProxConfig


def run(cfg: Config, log=print):
    topo, coll = common.setup_runtime(cfg)
    task = common.ClassifierTask(cfg, topo, cfg.lambda1, cfg.lambda2)
    strat = FedProx(coll, topo, len(task.blocks), cfg.admm_rho0)
    engine = common.run_engine(cfg, task, topo, coll, strat, None, log)
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="fedprox_multi"))


if __name__ == "__main__":
    main()
