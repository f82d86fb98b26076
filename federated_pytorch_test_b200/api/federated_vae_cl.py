"""``federated_vae_cl`` — FedAvg for the variational-clustering VAE.

Reference: /root/reference/src/federated_vae_cl.py: three blocks (encoder, decoder,
latent); LBFGSNew(history 10, max_iter 4, stochastic) for encoder/decoder, Adam(1e-4) for the
latent block; loss = sum over clusters of c1 + 10 (c2 + c3) + c21, plus lambda2 ||x||^2 on the
trainable vector (always on).  The four costs are one vectorised expression here instead of
Python loops over the batch; per-cluster costs are still logged per minibatch when verbose.
"""
from __future__ import annotations

import torch

from .. import models
from ..algo.engine import Replica, Visit
from ..algo.strategies import FedAvg
from ..config import VAECLConfig, parse_config
from ..ops import losses
from ..utils import legacy_log
from . import common, federated_vae

Config = VAECLConfig


class VAECLTask(federated_vae.VAETask):
    def __init__(self, cfg, topo):
        super().__init__(cfg, topo)
        self.factory = lambda: models.AutoEncoderCNNCL(K=cfg.Kc, L=cfg.Lc, batched_clusters=cfg.batched_clusters)
        probe = self.factory()
        self.blocks = probe.train_order_block_ids()
        self.n_params = sum(1 for _ in probe.parameters())

    def visits(self, nloop: int):
        for ci, (lo, hi) in enumerate(self.blocks):
            if ci == 2:  # latent space: Adam 1e-4, reparametrisation explicitly enabled
                yield Visit("net", lo, hi, ci, (lo, hi), "adam", dict(lr=1e-4), lambda2=self.cfg.lambda2, tag={"repr": True})
            else:
                yield Visit("net", lo, hi, ci, (lo, hi), "lbfgs",
                            dict(history_size=10, max_iter=4, line_search_fn=True, batch_mode=True),
                            lambda2=self.cfg.lambda2, tag={"repr": False})

    def batches(self, rep: Replica, visit: Visit, epoch: int):
        net = rep.nets["net"]
        if visit.tag.get("repr"):
            net.enable_repr()
        else:
            net.disable_repr()  # NB: leaves it enabled, as in the reference (Q11)
        return iter(self.loader(rep.ck))

    def loss(self, rep: Replica, batch) -> torch.Tensor:
        x, _ = batch
        out = rep.nets["net"](x)
        return losses.vae_cl_loss(*out, x)

    def after_minibatch(self, rep, visit, batch, i, epoch, nloop, N, loss1, engine) -> None:
        if not self.cfg.be_verbose:
            return
        x, _ = batch
        with torch.no_grad():
            c1, c2, c21, c3 = losses.vae_cl_costs(*rep.nets["net"](x), x)
        for k in range(c1.shape[0]):
            engine.log(legacy_log.cluster_costs_line(k, float(c1[k]), float(c2[k]), float(c21[k]), float(c3[k])))
        engine.log(legacy_log.minibatch_line(rep.ck, visit.label, nloop, N, i, epoch, float(loss1)))


def run(cfg: Config, log=print):
    common.require_iid(cfg, "federated_vae_cl")
    common.require_batch_norm(cfg, "federated_vae_cl")
    common.require_default_client_opt(cfg, "federated_vae_cl")
    topo, coll = common.setup_runtime(cfg)
    task = VAECLTask(cfg, topo)
    engine = common.run_engine(cfg, task, topo, coll, FedAvg(coll, topo), None, log)
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="federated_vae_cl"))


if __name__ == "__main__":
    main()
