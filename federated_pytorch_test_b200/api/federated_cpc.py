"""``federated_cpc`` — FedAvg for Contrastive Predictive Coding on LOFAR patches.

Reference: /root/reference/src/federated_cpc.py: three sub-models per worker (encoder,
context generator, predictor) trained one after the other, block by block, with
LBFGSNew(history 7, max_iter 2, stochastic); ``Niter`` random minibatches per worker per
round; InfoNCE over the patch grid; FedAvg of the active block.

Fixes relative to the shipped script (SURVEY Q12/Q13): the block *index* is passed to
``unfreeze_one_block`` (the reference passes a list and raises TypeError); data come from an
in-memory LOFAR-shaped source (synthetic by default); rows are batch-major so the later
``view(batch, px, py, -1)`` is consistent (``--patch_layout reference`` restores the
original order); checkpoints follow the reference's naming (loads ``./encoder.model``...,
saves ``encoder{ck}.model``...).
"""
from __future__ import annotations

import os
from typing import Iterator

import torch

from .. import models
from ..algo.engine import Replica, Task, Visit
from ..algo.strategies import FedAvg
from ..config import CPCConfig, parse_config
from ..data.lofar import LofarSource, get_data_minibatch
from ..ops import losses
from ..utils import ckpt, legacy_log
from ..utils.simple_utils import init_weights
from . import common

Config = CPCConfig
_MODELS = ("encoder", "contextgen", "predictor")


class CPCTask(Task):
    def __init__(self, cfg: Config, topo):
        if cfg.augment:
            raise ValueError("augment is supported by the classifier drivers only, not by CPCTask")
        common.require_no_mix(cfg, "CPCTask")
        self.cfg, self.topo = cfg, topo
        files = [f for f in cfg.file_list.split(",") if f]
        saps = [s for s in cfg.sap_list.split(",") if s]
        if files:
            assert len(files) == cfg.K and len(saps) == cfg.K, "file_list and sap_list need K entries"
        self.sources = {}
        for ck in topo.local_workers:
            if files:
                src = LofarSource.from_h5(files[ck], saps[ck])
            else:
                src = LofarSource.synthetic(cfg.nbase, cfg.ntime, cfg.nfreq, seed=cfg.data_seed + ck)
            self.sources[ck] = src.to(topo.device)
        self.gens = {ck: torch.Generator().manual_seed(cfg.seed + 17 * ck) for ck in topo.local_workers}
        self.grid = {}

    def build_replica(self, ck: int, device, allocator) -> Replica:
        cfg = self.cfg
        nets = {
            "encoder": models.EncoderCNN(latent_dim=cfg.Lc),
            "contextgen": models.ContextgenCNN(latent_dim=cfg.Lc),
            "predictor": models.PredictorCNN(latent_dim=cfg.Lc, reduced_dim=cfg.Rc),
        }
        rep = Replica(ck, nets, device, allocator=allocator)
        if cfg.load_model:
            for key in _MODELS:
                path = os.path.join(cfg.ckpt_dir, key + ".model")
                if os.path.exists(path):
                    ckpt.load_model_only(path, nets[key], device)
        if cfg.init_model:
            torch.manual_seed(0)
            for key in _MODELS:
                nets[key].apply(init_weights)
        return rep

    def visits(self, nloop: int):
        probe = {"encoder": models.EncoderCNN(latent_dim=8), "contextgen": models.ContextgenCNN(latent_dim=8),
                 "predictor": models.PredictorCNN(latent_dim=8, reduced_dim=4)}
        opt = dict(history_size=7, max_iter=2, line_search_fn=True, batch_mode=True)
        for mdl, key in enumerate(_MODELS):
            for ci, (lo, hi) in enumerate(probe[key].train_order_block_ids()):
                yield Visit(key, lo, hi, ci, (lo, hi), "lbfgs", dict(opt), tag={"mdl": mdl})

    def batches(self, rep: Replica, visit: Visit, epoch: int) -> Iterator:
        cfg = self.cfg
        for _ in range(cfg.Niter):
            px, py, y = get_data_minibatch(self.sources[rep.ck], cfg.batch_size, 32, self.gens[rep.ck], cfg.patch_layout)
            yield (y, px, py)

    def batch_size_of(self, batch) -> int:
        return self.cfg.batch_size

    def loss(self, rep: Replica, batch) -> torch.Tensor:
        y, px, py = batch
        B = self.cfg.batch_size
        lat = rep.nets["encoder"](y).reshape(B, px, py, -1).permute(0, 3, 1, 2).contiguous()
        ctx = rep.nets["contextgen"](lat)
        reduced, pred = rep.nets["predictor"](lat, ctx)
        return losses.info_nce(reduced, pred)

    def after_minibatch(self, rep, visit, batch, i, epoch, nloop, N, loss1, engine) -> None:
        if self.cfg.be_verbose:
            engine.log("%d %d %d %f" % (0, rep.ck, i, float(loss1)))

    def aggregate_log(self, visit, metrics, ctx, engine) -> None:
        engine.log(legacy_log.cpc_dual_line(ctx["N"], self.cfg.Niter - 1, ctx["nloop"], visit.tag["mdl"], visit.ci,
                                            ctx["nadmm"], metrics["dual"]), root_only=True)


def run(cfg: Config, log=print):
    common.require_iid(cfg, "federated_cpc")
    common.require_batch_norm(cfg, "federated_cpc")
    common.require_default_client_opt(cfg, "federated_cpc")
    topo, coll = common.setup_runtime(cfg)
    task = CPCTask(cfg, topo)
    ecfg = common.engine_config(cfg, Nepoch=1, diagnostics="pre")  # the reference has no diagnostics forward here
    engine = common.run_engine(cfg, task, topo, coll, FedAvg(coll, topo), ecfg, log)
    if cfg.save_model:
        for rep in engine.replicas:
            for key in _MODELS:
                ckpt.save_model_only(os.path.join(cfg.ckpt_dir, "%s%d.model" % (key, rep.ck)), rep.nets[key])
    return engine


def main(argv=None):
    return run(parse_config(Config, argv, prog="federated_cpc"))


if __name__ == "__main__":
    main()
