"""``consensus_multi`` — consensus ADMM per block, optional Barzilai-Borwein adaptive rho.

Reference: /root/reference/src/consensus_multi.py (x/z/y updates, spectral penalty every
``bb_period_T`` rounds, primal/dual residuals).  z-update + dual ascent + both residuals
are one fused kernel; the BB rule is replayed deterministically on every rank from six
dot products per worker (SURVEY §7.3(2)).

``--partition dirichlet`` gives the workers label-skewed shards of unequal size; the z-update stays the unweighted
average of the K workers, as in the reference (sample-count weights and client sampling are ``federated_multi``'s).
"""
from __future__ import annotations

from ..algo.strategies import ADMM, BBConfig
from ..config import ConsensusConfig, parse_config
from . import common

Config = ConsensusConfig


def run(cfg: Config, log=print):
    topo, coll = common.setup_runtime(cfg)
    task = common.ClassifierTask(cfg, topo, cfg.lambda1, cfg.lambda2)
    bb = BBConfig(cfg.bb_update, cfg.bb_period_T, cfg.bb_alphacorrmin, cfg.bb_epsilon, cfg.bb_rhomax,
                  seed_yhat0_with_x=not cfg.bb_seed_yhat0_zero)
    root_log = (lambda m: log(m)) if topo.is_root else (lambda m: None)
    strat = ADMM(coll, topo, len(task.blocks), cfg.admm_rho0, bb, log=root_log)
    engine = common.run_engine(cfg, task, topo, coll, strat, None, log)
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="consensus_multi"))


if __name__ == "__main__":
    main()
