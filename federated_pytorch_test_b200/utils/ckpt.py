"""Checkpoints: the reference's per-worker files + a true resume record.

Legacy schema (SURVEY §5.4; /root/reference/src/federated_multi.py:226-233,
100-103): ``./s{ck}.model`` = ``{'model_state_dict', 'epoch',
'optimizer_state_dict', 'running_loss'}``, loading restores the model weights
only.  CPC writes ``encoder{ck}.model`` / ``contextgen{ck}.model`` /
``predictor{ck}.model`` with only ``model_state_dict`` and loads the un-suffixed
``./encoder.model`` … into every worker (federated_cpc.py:125-134,308-318).

Files written here are readable by the reference scripts and vice versa: tensors
are detached from the flat arena and made dense before saving.

The resume record (new) additionally stores the schedule position, the
consensus variables (z, y_k, rho, BB state), optimizer state and RNG states.
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import torch
import torch.nn as nn


def dense_state_dict(net: nn.Module) -> Dict[str, torch.Tensor]:
    """``state_dict`` with every tensor cloned out of the arena into standalone contiguous storage."""
    return {k: v.detach().clone(memory_format=torch.contiguous_format) for k, v in net.state_dict().items()}


def load_into(net: nn.Module, state: Dict[str, torch.Tensor]) -> None:
    """``load_state_dict`` that keeps arena views intact (copies element-wise into the existing storage)."""
    own = net.state_dict()
    missing = [k for k in own if k not in state]
    unexpected = [k for k in state if k not in own]
    if missing or unexpected:
        raise KeyError("state_dict mismatch: missing=%s unexpected=%s" % (missing, unexpected))
    with torch.no_grad():
        for k, v in own.items():
            v.copy_(state[k].to(v.device))
    if any(v.is_cuda for v in own.values()):
        from ..ops import cuda_ops

        cuda_ops.clear_caches()   # derived tensors (e.g. flipped dgrad filters) of frozen layers are now stale


def worker_path(ckpt_dir: str, ck: int, stem: str = "s") -> str:
    return os.path.join(ckpt_dir, "%s%d.model" % (stem, ck))


def save_worker(ckpt_dir: str, ck: int, net: nn.Module, epoch: int, optimizer, running_loss: float, stem: str = "s") -> str:
    path = worker_path(ckpt_dir, ck, stem)
    torch.save({
        "model_state_dict": dense_state_dict(net),
        "epoch": epoch,
        "optimizer_state_dict": optimizer.state_dict() if optimizer is not None else {},
        "running_loss": running_loss,
    }, path)
    return path


def load_worker(ckpt_dir: str, ck: int, net: nn.Module, device, stem: str = "s") -> None:
    ckpt = torch.load(worker_path(ckpt_dir, ck, stem), map_location=device, weights_only=False)
    load_into(net, ckpt["model_state_dict"])
    net.train()


def save_model_only(path: str, net: nn.Module) -> str:
    torch.save({"model_state_dict": dense_state_dict(net)}, path)
    return path


def load_model_only(path: str, net: nn.Module, device) -> None:
    ckpt = torch.load(path, map_location=device, weights_only=False)
    load_into(net, ckpt["model_state_dict"])
    net.train()


# ----------------------------------------------------------------------------
def save_resume(path: str, engine, position: Dict) -> str:
    """True resume record (SURVEY §5.4), written by the engine after every aggregation round when
    ``EngineConfig.resume_path`` is set: schedule position ``(nloop, visit, round)`` = where to RE-ENTER, consensus
    state of the open block visit (z, y_k, rho table, BB vectors), per-replica weights + BatchNorm buffers, the
    optimizers' flat state (Adam moments + step / SGD momentum buffer + settings / L-BFGS history, direction, Welford
    statistics), the optimizer's name and the learning-rate schedule and clipping settings in the position, loader RNG
    streams and
    augmentation counters,
    global RNG states and the run counters.  Written atomically (tmp + rename); one file per rank."""
    strat_state = {}
    for k, v in engine.strategy.state().items():
        if torch.is_tensor(v):
            strat_state[k] = v.detach().cpu().clone()
        elif isinstance(v, list):
            strat_state[k] = [t.detach().cpu().clone() for t in v]
        elif isinstance(v, dict):                  # per-block state, e.g. a server optimizer's moments by block index
            strat_state[k] = {i: t.detach().cpu().clone() for i, t in v.items()}
        else:
            strat_state[k] = v
    opts = {}
    for rep, opt in zip(engine.replicas, engine.optimizers or []):
        opts[rep.ck] = opt.flat_state() if hasattr(opt, "flat_state") else None
    loaders = {}
    for ck, ld in getattr(engine.task, "_loaders", {}).items():
        if hasattr(ld, "gen"):
            nxt = getattr(ld, "_next_order", None)        # the next epoch's permutation may already have been drawn (prefetch)
            loaders[ck] = {"gen": ld.gen.get_state(), "next_order": None if nxt is None else nxt.detach().cpu().clone(),
                           "aug_counter": int(getattr(ld, "aug_counter", 0))}
    rec = {
        "position": dict(position),
        "strategy": engine.strategy.name,
        "strategy_state": strat_state,
        "local_workers": list(engine.topo.local_workers),
        "replicas": {
            rep.ck: {key: dense_state_dict(net) for key, net in rep.nets.items()} for rep in engine.replicas
        },
        "optimizers": opts,
        "loader_rng": loaders,
        "counters": {"images_seen": engine.images_seen, "steps_done": engine.steps_done,
                     "aggregations_done": getattr(engine, "aggregations_done", 0)},
        "rng": {"torch": torch.get_rng_state(),
                "cuda": torch.cuda.get_rng_state_all() if torch.cuda.is_available() else None},
    }
    if engine.topo.is_distributed:
        path = "%s.rank%d" % (path, engine.topo.rank)
    tmp = path + ".tmp"
    torch.save(rec, tmp)
    os.replace(tmp, path)
    return path


def load_resume(path: str, engine) -> Dict:
    """Restore a record written by :func:`save_resume` and arm the engine to re-enter the schedule at the recorded
    position: weights now; consensus / optimizer state when the engine reaches the recorded block visit (the buffers
    only exist then)."""
    if engine.topo.is_distributed:
        path = "%s.rank%d" % (path, engine.topo.rank)
    rec = torch.load(path, map_location="cpu", weights_only=False)
    if rec.get("strategy") not in (None, engine.strategy.name):
        raise ValueError("resume record was written by strategy %r, this run uses %r" % (rec.get("strategy"), engine.strategy.name))
    for rep in engine.replicas:
        for key, net in rep.nets.items():
            load_into(net, rec["replicas"][rep.ck][key])
    torch.set_rng_state(rec["rng"]["torch"])
    if rec["rng"]["cuda"] is not None and torch.cuda.is_available():
        try:
            torch.cuda.set_rng_state_all(rec["rng"]["cuda"])
        except Exception:
            pass
    for ck, state in (rec.get("loader_rng") or {}).items():
        ld = engine.task.loader(ck) if hasattr(engine.task, "loader") else None
        if ld is not None and hasattr(ld, "gen"):
            ld.gen.set_state(state["gen"])
            nxt = state.get("next_order")
            ld._next_order = None if nxt is None else nxt.to(ld.images.device)
            ld.aug_counter = int(state.get("aug_counter", 0))      # augmentation draws continue where the record left off
    cnt = rec.get("counters") or {}
    engine.images_seen = int(cnt.get("images_seen", 0))
    engine.steps_done = int(cnt.get("steps_done", 0))
    engine.aggregations_done = int(cnt.get("aggregations_done", 0))
    engine._resume_pos = dict(rec["position"])
    engine._resume_state = {"strategy_state": rec.get("strategy_state"), "optimizers": rec.get("optimizers")}
    return rec
