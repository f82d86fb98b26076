"""Shared plumbing of the seven entry points: runtime set-up, the CIFAR
classifier task, evaluation, legacy checkpoints.

Reference call stack being re-implemented: SURVEY §3.1 (module-level script
``federated_multi.py`` and siblings): shard construction and per-worker normalisation
``src/federated_multi.py:55-71``, model construction / identical initialisation ``:127-150``, evaluation with
batch-statistics BatchNorm ``:108-121`` (Q4, Q5), end-of-run checkpoints ``:226-233`` and warm start ``:100-103``.
"""
from __future__ import annotations

import functools
import os
from typing import Callable, Dict, Iterator, List, Optional, Tuple

import torch
import torch.nn as nn

from .. import models
from ..algo.engine import Engine, EngineConfig, Replica, Task, Visit
from ..config import (ADAM_LR, CLIENT_RECIPE_DEFAULTS, MIX_DEFAULTS, CommonConfig, check_client_opt, check_mix, check_norm,
                      check_partition)
from ..data.cifar import (CifarData, ShardLoader, augment_key, class_histogram, dirichlet_shards, mix_key, shard_ranges,
                          worker_norm)
from ..ops import functional as FX
from ..ops import losses
from ..parallel.collective import make_collective
from ..parallel.topology import Topology
from ..utils import ckpt, legacy_log
from ..utils.metrics import MetricsLog
from ..utils.simple_utils import init_weights

_MODEL_FACTORIES = {
    "Net": models.Net, "Net1": models.Net1, "Net2": models.Net2,
    "ResNet18": models.ResNet18, "ResNet9": models.ResNet9,
}


def require_batch_norm(cfg: CommonConfig, driver: str) -> None:
    """The VAE, VAE-CL and CPC networks have no GroupNorm variant and accept only the default ``norm``."""
    if getattr(cfg, "norm", "batch") != "batch":
        raise ValueError("%s supports only norm 'batch', got norm %r" % (driver, cfg.norm))


def require_default_client_opt(cfg: CommonConfig, driver: str) -> None:
    """The VAE, VAE-CL and CPC drivers fix their own optimizers (as the reference does) and accept none of the client-optimizer
    flags of the classifier drivers."""
    for name, default in (("lr", 0.0), ("momentum", 0.0), ("nesterov", False), ("weight_decay", 0.0)) + CLIENT_RECIPE_DEFAULTS:
        if getattr(cfg, name, default) != default:
            raise ValueError("%s fixes its own optimizer and does not take %s, got %s %r"
                             % (driver, name, name, getattr(cfg, name)))
    if getattr(cfg, "optimizer", "adam") == "adamw":
        raise ValueError("%s fixes its own optimizer and does not take optimizer 'adamw'" % driver)


def require_no_mix(cfg: CommonConfig, task: str) -> None:
    """Label smoothing, mixup and CutMix belong to the classifier drivers' cross-entropy (and mixup / CutMix would blend the
    VAE's reconstruction targets too)."""
    for name, default in MIX_DEFAULTS:
        if getattr(cfg, name, default) != default:
            raise ValueError("%s is supported by the classifier drivers only, not by %s" % (name, task))


def require_iid(cfg: CommonConfig, driver: str) -> None:
    """The unsupervised drivers (VAE, VAE-CL, CPC) train without labels and accept only the default split."""
    if getattr(cfg, "partition", "iid") != "iid":
        raise ValueError("%s supports only partition 'iid', got partition %r" % (driver, cfg.partition))


def setup_runtime(cfg: CommonConfig) -> Tuple[Topology, object]:
    """Seed, fast-path switch, topology and collective for a run."""
    torch.manual_seed(cfg.seed)
    FX.set_fast_path(bool(cfg.fast))
    use_cuda = cfg.use_cuda and torch.cuda.is_available()
    if cfg.distributed and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        topo = Topology.from_env(cfg.K, use_cuda=use_cuda)
    else:
        topo = Topology.single_process(cfg.K, torch.device("cuda", torch.cuda.current_device()) if use_cuda else torch.device("cpu"))
    coll = make_collective(topo, cfg.collective)
    return topo, coll


def engine_config(cfg: CommonConfig, **kw) -> EngineConfig:
    base = dict(Nloop=cfg.Nloop, Nadmm=cfg.Nadmm, Nepoch=cfg.Nepoch, check_results=cfg.check_results,
                be_verbose=cfg.be_verbose, diagnostics=cfg.diagnostics, graphs=cfg.graphs,
                max_minibatches=cfg.max_minibatches or None, nan_guard=getattr(cfg, "nan_guard", "raise"),
                resume_path=getattr(cfg, "resume_out", ""), streams=getattr(cfg, "streams", True),
                lr_schedule=cfg.lr_schedule, lr_warmup=cfg.lr_warmup, lr_gamma=cfg.lr_gamma,
                lr_step_rounds=cfg.lr_step_rounds, lr_min=cfg.lr_min, label_smoothing=cfg.label_smoothing,
                mixup_alpha=cfg.mixup_alpha, cutmix_alpha=cfg.cutmix_alpha)
    base.update(kw)
    return EngineConfig(**base)


def load_cifar(cfg: CommonConfig, device: torch.device) -> CifarData:
    if cfg.data == "torchvision":
        data = CifarData.from_torchvision()
    else:
        data = CifarData.synthetic(cfg.data_seed, cfg.train_size, cfg.test_size, getattr(cfg, "data_noise", 0.6))
    if cfg.data_on_device or device.type != "cuda":
        return data.to(device)
    return data.to(device, pin=True)  # pinned host memory; batches go through the native assembler


class ClassifierTask(Task):
    """CIFAR10 classification with CE (+ gated elastic net) — C4..C7 of SURVEY §2.1."""

    def __init__(self, cfg: CommonConfig, topo: Topology, lambda1: float = 0.0, lambda2: float = 0.0,
                 whole_model: bool = False):
        self.cfg, self.topo = cfg, topo
        self.lambda1, self.lambda2 = lambda1, lambda2
        self.whole_model = whole_model  # no_consensus: all parameters trainable, no block schedule
        if cfg.eval_bn not in ("batch", "running"):
            raise ValueError("eval_bn must be 'batch' or 'running', got %r" % (cfg.eval_bn,))
        name = cfg.model or ("ResNet18" if cfg.use_resnet else "Net")
        self.model_name = name
        norm = getattr(cfg, "norm", "batch")
        check_norm(norm, getattr(cfg, "norm_groups", 32), name)
        check_client_opt(cfg.optimizer, cfg.lr, cfg.momentum, cfg.nesterov, cfg.weight_decay, cfg.lr_schedule, cfg.lr_warmup,
                         cfg.lr_gamma, cfg.lr_step_rounds, cfg.lr_min, cfg.clip_norm)
        check_mix(cfg.label_smoothing, cfg.mixup_alpha, cfg.cutmix_alpha)
        self.factory = _MODEL_FACTORIES[name]
        if norm != "batch":
            self.factory = functools.partial(self.factory, norm=norm, groups=cfg.norm_groups)
        self.data = load_cifar(cfg, topo.device)
        partition = getattr(cfg, "partition", "iid")
        check_partition(partition, getattr(cfg, "dirichlet_alpha", 0.5))
        self.partition_row = None              # the metrics row describing a non-default split
        if partition == "dirichlet":
            self.shards = [torch.from_numpy(s) for s in dirichlet_shards(
                self.data.train_labels, cfg.K, cfg.dirichlet_alpha, cfg.data_seed, cfg.default_batch)]
            self.partition_row = dict(kind="partition", partition=partition, alpha=float(cfg.dirichlet_alpha),
                                      shard_sizes=self.shard_sizes(),
                                      class_histogram=class_histogram(self.data.train_labels, self.shards))
        else:
            self.shards = shard_ranges(cfg.K, self.data.train_images.shape[0], drop_last_sample=not cfg.fix_shard_off_by_one)
        self.channels_last = bool(cfg.fast and topo.device.type == "cuda" and name.startswith("ResNet"))
        self._loaders: Dict[int, ShardLoader] = {}
        self._test_loaders: Dict[int, ShardLoader] = {}
        self._eval_graphs: Dict = {}
        self._eval_counters: Dict[int, torch.Tensor] = {}
        probe = self.factory()
        self.blocks = probe.train_order_block_ids()
        self.linear_ids = probe.linear_layer_ids()
        self.n_params = sum(1 for _ in probe.parameters())
        self.dense_param_ids = set()
        if cfg.intended_elastic_net_gate:
            for idx, (pname, p) in enumerate(probe.named_parameters()):
                if p.dim() == 2:
                    self.dense_param_ids.update((idx, idx + 1))

    def shard_sizes(self) -> List[int]:
        """``n_k``: the number of training samples of every worker's shard."""
        return [len(s) for s in self.shards]

    # -- replicas -------------------------------------------------------------
    def build_replica(self, ck: int, device: torch.device, allocator) -> Replica:
        net = self.factory()
        rep = Replica(ck, {"net": net}, device, allocator=allocator, channels_last_weights=self.channels_last)
        if self.cfg.load_model:
            ckpt.load_worker(self.cfg.ckpt_dir, ck, net, device)
        if self.cfg.init_model:
            torch.manual_seed(0)  # identical initialisation for every worker (federated_multi.py:124-128)
            net.apply(init_weights)
        return rep

    # -- schedule -------------------------------------------------------------
    def _gate(self, ci: int, lo: int, hi: int) -> bool:
        if self.cfg.intended_elastic_net_gate:
            return any(i in self.dense_param_ids for i in range(lo, hi + 1))
        return ci in self.linear_ids  # Q2: block index tested against parameter indices

    def visits(self, nloop: int):
        cfg = self.cfg
        if cfg.optimizer == "adam":
            opt_kwargs = dict(lr=cfg.lr or ADAM_LR)
        elif cfg.optimizer == "adamw":
            opt_kwargs = dict(lr=cfg.lr or ADAM_LR, weight_decay=cfg.weight_decay)
        elif cfg.optimizer == "sgd":
            opt_kwargs = dict(lr=cfg.lr, momentum=cfg.momentum, nesterov=cfg.nesterov, weight_decay=cfg.weight_decay)
        else:
            opt_kwargs = dict(history_size=10, max_iter=4, line_search_fn=True, batch_mode=True)
        if cfg.clip_norm > 0.0:
            opt_kwargs["clip_norm"] = cfg.clip_norm
        if self.whole_model:
            yield Visit("net", 0, self.n_params - 1, 0, (0, self.n_params - 1), self.cfg.optimizer, opt_kwargs)
            return
        for ci, (lo, hi) in enumerate(self.blocks):
            gated = self._gate(ci, lo, hi)
            yield Visit("net", lo, hi, ci, (lo, hi), self.cfg.optimizer, opt_kwargs,
                        lambda1=self.lambda1 if gated else 0.0, lambda2=self.lambda2 if gated else 0.0)

    # -- data -----------------------------------------------------------------
    def loader(self, ck: int) -> ShardLoader:
        ld = self._loaders.get(ck)
        if ld is None:
            mean, std = worker_norm(ck, self.cfg.biased_input)
            ld = ShardLoader(self.data.train_images, self.data.train_labels, self.shards[ck], self.cfg.default_batch,
                             self.topo.device, mean, std, shuffle=True, seed=self.cfg.seed + 1000 * ck,
                             channels_last=self.channels_last, augment=self.cfg.augment,
                             aug_key=augment_key(self.cfg.seed, ck), mixup_alpha=self.cfg.mixup_alpha,
                             cutmix_alpha=self.cfg.cutmix_alpha, mix_key=mix_key(self.cfg.seed, ck))
            self._loaders[ck] = ld
        return ld

    def test_loader(self, ck: int) -> ShardLoader:
        ld = self._test_loaders.get(ck)
        if ld is None:
            mean, std = worker_norm(ck, self.cfg.biased_input)  # the test set gets the worker's biased transform too
            n = self.data.test_images.shape[0]
            ld = ShardLoader(self.data.test_images, self.data.test_labels, range(n), self.cfg.default_batch,
                             self.topo.device, mean, std, shuffle=False, channels_last=self.channels_last)
            self._test_loaders[ck] = ld
        return ld

    def batches(self, rep: Replica, visit: Visit, epoch: int) -> Iterator:
        return iter(self.loader(rep.ck))

    def loss(self, rep: Replica, batch) -> torch.Tensor:
        x, y = batch[0], batch[1]
        lam = batch[2] if len(batch) == 3 else None        # a mixed batch carries its lam_eff
        return losses.cross_entropy(rep.nets["net"](x), y, self.cfg.label_smoothing, lam)

    # -- logging / evaluation ----------------------------------------------------
    def after_minibatch(self, rep, visit, batch, i, epoch, nloop, N, loss1, engine) -> None:
        if self.cfg.be_verbose:
            if self.whole_model:
                engine.log(legacy_log.minibatch_line_noblock(rep.ck, i, epoch, float(loss1)))
            else:
                engine.log(legacy_log.minibatch_line(rep.ck, visit.label, nloop, N, i, epoch, float(loss1)))

    def aggregate_log(self, visit, metrics, ctx, engine) -> None:
        if "primal" in metrics:
            engine.log(legacy_log.admm_line(visit.label, ctx["N"], ctx["rho_mean"], ctx["nadmm"], ctx["nloop"],
                                            metrics["primal"], metrics["dual"]), root_only=True)
        elif "dual" in metrics:
            engine.log(legacy_log.dual_line(ctx["epoch"], ctx["nloop"], visit.label, ctx["nadmm"], metrics["dual"]),
                       root_only=True)

    @torch.no_grad()
    def evaluate(self, reps: List[Replica], engine: Engine) -> List[float]:
        """Test-set accuracy of every local replica (verification_error_check, federated_multi.py:108-121).

        By default networks stay in training mode as in the reference (Q4): BatchNorm
        uses batch statistics and keeps updating its running statistics on test data.
        With ``eval_bn='running'`` each network is evaluated in eval mode (running
        statistics, left unchanged) and put back into training mode afterwards.  A
        GroupNorm network computes the same in either mode.  Runs
        under ``no_grad`` (no numerical effect).  Counting stays on the device; one
        read per replica.
        """
        fused = self.topo.device.type == "cuda" and FX.fast_path_enabled()
        graphed = fused and bool(getattr(self.cfg, "graphs", False))
        running = self.cfg.eval_bn == "running"
        counters = []
        for rep in reps:
            net = rep.nets["net"]
            counter = self._eval_counters.setdefault(rep.ck, torch.zeros(2, dtype=torch.int64, device=rep.device))
            counter.zero_()                                                      # [#correct, #seen], stays on the device
            if running:
                net.eval()
            try:
                for x, y in self.test_loader(rep.ck):
                    if graphed:
                        from ..algo.graphs import GraphedEval

                        key = (rep.ck, tuple(x.shape), net.training)             # a graph bakes in the BatchNorm mode
                        ge = self._eval_graphs.get(key)
                        if ge is None:
                            ge = self._eval_graphs[key] = GraphedEval(net, (x, y), counter, rep.device)
                        ge.run((x, y))                                           # forward + argmax/compare/count: one graph launch
                        continue
                    logits = net(x)
                    if fused:
                        from ..ops import cuda_ops

                        cuda_ops.argmax_count(logits, y, counter)                # argmax + compare + count: one kernel (G21)
                    else:
                        counter[0] += (logits.argmax(dim=1) == y).sum()
                        counter[1] += y.shape[0]
            finally:
                if running:
                    net.train()
            counters.append(counter)
        accs = []
        for rep, counter in zip(reps, counters):                                 # ONE read per replica, after all forwards are queued
            c, total = (int(v) for v in counter.tolist())
            engine.log(legacy_log.accuracy_line(rep.ck, total, c))
            accs.append(legacy_log.accuracy_exact(c, total))
        return accs


def save_legacy(cfg: CommonConfig, engine: Engine, model_key: str = "net") -> None:
    if not cfg.save_model:
        return
    for rep, opt in zip(engine.replicas, engine.optimizers or [None] * len(engine.replicas)):
        ckpt.save_worker(cfg.ckpt_dir, rep.ck, rep.nets[model_key], engine.last_epoch, opt, rep.running_loss)


def run_engine(cfg: CommonConfig, task: Task, topo: Topology, coll, strategy, ecfg: Optional[EngineConfig] = None,
               log: Callable[[str], None] = print, attack: Optional[Callable[[Engine], None]] = None) -> Engine:
    metrics = MetricsLog(cfg.metrics_path or None)
    engine = Engine(task, topo, strategy, coll, ecfg or engine_config(cfg), log=log, metrics=metrics)
    engine.attack = attack
    if getattr(task, "partition_row", None) and topo.is_root:
        metrics.write(task.partition_row)
    if cfg.resume:
        ckpt.load_resume(cfg.resume, engine)
    engine.run()
    metrics.close()
    return engine
