"""``federated_vae`` — FedAvg for a convolutional VAE, one *layer* (weight+bias pair) at a time.

Reference: /root/reference/src/federated_vae.py.  Layers are trained in natural order
(``unfreeze_one_layer(net, ci)`` for ci in 0..11) while the reference's log lines print
``train_order_block_ids()[ci]`` — a different order (SURVEY Q10).  The training order is
preserved; ``label_mode='reference'`` reproduces the mislabelled log, ``'true'`` prints the
parameter indices actually trained.
"""
from __future__ import annotations

from typing import Iterator, List

import torch

from .. import models
from ..algo.engine import Replica, Visit
from ..algo.strategies import FedAvg
from ..config import VAEConfig, parse_config
from ..ops import losses
from ..utils import legacy_log
from ..utils.simple_utils import init_weights
from . import common

Config = VAEConfig


class VAETask(common.ClassifierTask):
    label_mode = "reference"

    def __init__(self, cfg, topo):
        if cfg.augment:     # the loader would crop and flip the VAE's reconstruction targets too
            raise ValueError("augment is supported by the classifier drivers only, not by %s" % type(self).__name__)
        common.require_no_mix(cfg, type(self).__name__)
        cfg_model, cfg_optimizer = cfg.model, cfg.optimizer
        # placeholders for the base-class probe and checks; replaced below (this task fixes its own optimizer)
        cfg.model, cfg.optimizer = "Net", "adam"
        try:
            super().__init__(cfg, topo)
        finally:
            cfg.model, cfg.optimizer = cfg_model, cfg_optimizer
        self.factory = models.AutoEncoderCNN
        probe = self.factory()
        self.blocks = probe.train_order_block_ids()
        self.n_params = sum(1 for _ in probe.parameters())
        self.channels_last = False

    def visits(self, nloop: int):
        for ci in range(len(self.blocks)):
            lo, hi = 2 * ci, 2 * ci + 1
            label = tuple(self.blocks[ci]) if self.label_mode == "reference" else (lo, hi)
            yield Visit("net", lo, hi, ci, label, "adam", dict(lr=1e-3))

    def loss(self, rep: Replica, batch) -> torch.Tensor:
        x, _ = batch
        recon, mu, logvar = rep.nets["net"](x)
        return losses.vae_loss(recon, x, mu, logvar)

    def after_minibatch(self, rep, visit, batch, i, epoch, nloop, N, loss1, engine) -> None:
        if self.cfg.be_verbose:  # unconditional in the reference (federated_vae.py:173)
            engine.log(legacy_log.minibatch_line(rep.ck, visit.label, nloop, N, i, epoch, float(loss1)))

    def evaluate(self, reps, engine):
        return None


def run(cfg: Config, log=print):
    common.require_iid(cfg, "federated_vae")
    common.require_batch_norm(cfg, "federated_vae")
    common.require_default_client_opt(cfg, "federated_vae")
    topo, coll = common.setup_runtime(cfg)
    task = VAETask(cfg, topo)
    engine = common.run_engine(cfg, task, topo, coll, FedAvg(coll, topo), None, log)
    common.save_legacy(cfg, engine)
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="federated_vae"))


if __name__ == "__main__":
    main()
