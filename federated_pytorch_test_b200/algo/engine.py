"""Block-coordinate federated training engine.

One engine replaces the seven copy-pasted driver loops of the reference
(/root/reference/src/federated_multi.py:143-220 and siblings; SURVEY §2.4):

    for nloop:  for block visit:  unfreeze block in every replica; z=0; new optimizer state
        for nadmm:  for epoch:
            for local replica:  for minibatch:  opt.step(closure); diagnostics loss
            strategy.aggregate()          <- ONE fused collective on the block slice
            (optional) evaluate all replicas on the test set

What differs from the reference by construction:

* replicas live where the :class:`~..parallel.topology.Topology` puts them (one
  per GPU under torchrun); only *local* replicas are stepped, all ranks run the
  same schedule and meet in the collective;
* a block is a zero-copy slice of each replica's flat arena — no pack/unpack, no
  ``torch.cat`` inside closures; penalty gradients are closed-form inside the
  optimizer kernel;
* the per-minibatch step of the Adam and SGD drivers can be captured once per
  (replica, block) as a CUDA graph and replayed (``graphs=True``), which removes
  the ~400 eager launches and the per-step host sync of the reference;
* the diagnostics loss is accumulated on the device; it is read back once per
  round (or per minibatch only when ``be_verbose``);
* with client sampling, replicas outside the round's participant set
  (``Strategy.participates``) take no step: their loaders, optimizer state and
  ``images_seen`` do not move, and the aggregation writes the new model into them.

A *task* (``api/*.py``) supplies models, data, loss, schedule and evaluation.
"""
from __future__ import annotations

import math
import os
import time
from dataclasses import dataclass, field
from typing import Callable, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from ..ops import flatops
from ..optim.block_adam import BlockAdam
from ..optim.block_sgd import BlockSGD
from ..optim.lbfgsnew import LBFGSNew
from ..optim.schedule import round_lr, schedule_active
from ..parallel.topology import Topology
from ..utils.flat import FlatArena
from ..utils.metrics import MetricsLog, PhaseTimers, nvtx_range
from .compress import payload_bytes, topk_payload_bytes
from .strategies import Penalty, Strategy

BLOCK_OPTIMIZERS = (BlockAdam, BlockSGD)   # fused block update: penalty in the kernel, the step graphed


@dataclass
class Visit:
    """One entry of the block schedule."""

    model: str                 # key of the sub-model being trained ('net', 'encoder', ...)
    lo: int                    # first trainable parameter index (inclusive)
    hi: int                    # last trainable parameter index (inclusive)
    ci: int                    # block index: selects rho[ci], the elastic-net gate, log labels
    label: Tuple[int, int]     # what the legacy log lines print as block=[a,b]
    optimizer: str = "adam"    # 'adam' | 'adamw' | 'sgd' | 'lbfgs'
    opt_kwargs: Dict = field(default_factory=dict)
    lambda1: float = 0.0       # elastic net on the block vector (already gated by the task)
    lambda2: float = 0.0
    tag: Dict = field(default_factory=dict)



def _grad_sink():
    """Weight-gradient kernels may accumulate straight into the arena's gradient views during these backward calls."""
    from ..ops import functional as FX

    if torch.cuda.is_available() and FX.fast_path_enabled():
        from ..ops import cuda_ops

        return cuda_ops.accumulate_into_grad()
    import contextlib

    return contextlib.nullcontext()


class Replica:
    """One logical worker: its models, arenas and data."""

    def __init__(self, ck: int, nets: Dict[str, nn.Module], device: torch.device, allocator=None,
                 channels_last_weights: bool = False):
        self.ck = ck
        self.nets = nets
        self.device = device
        self.arenas: Dict[str, FlatArena] = {}
        for key, net in nets.items():
            net.to(device)
            self.arenas[key] = FlatArena(net, device=device, allocator=allocator,
                                         channels_last_weights=channels_last_weights)
        self._running = 0.0             # running loss of the last pass: a device scalar until somebody asks (no sync per round)
        self.extra: Dict = {}

    @property
    def running_loss(self) -> float:
        return float(self._running) if self._running is not None else 0.0

    @running_loss.setter
    def running_loss(self, v) -> None:
        self._running = v

    def set_trainable(self, visit: Visit) -> None:
        for key, net in self.nets.items():
            active = key == visit.model
            for idx, p in enumerate(net.parameters()):
                p.requires_grad = active and visit.lo <= idx <= visit.hi
            self.arenas[key].attach_grads()

    def block(self, visit: Visit) -> torch.Tensor:
        return self.arenas[visit.model].block(visit.lo, visit.hi)

    def block_grad(self, visit: Visit) -> torch.Tensor:
        return self.arenas[visit.model].block_grad(visit.lo, visit.hi)


class Task:
    """What a driver must provide.  See ``api/`` for the seven concrete tasks."""

    def build_replica(self, ck: int, device: torch.device, allocator) -> Replica:
        raise NotImplementedError

    def visits(self, nloop: int) -> Iterable[Visit]:
        raise NotImplementedError

    def batches(self, rep: Replica, visit: Visit, epoch: int) -> Iterator:
        raise NotImplementedError

    def loss(self, rep: Replica, batch) -> torch.Tensor:
        raise NotImplementedError

    def batch_size_of(self, batch) -> int:
        return int(batch[0].shape[0])

    def evaluate(self, reps: List[Replica], engine: "Engine") -> Optional[List[float]]:
        return None

    def on_epoch_start(self, epoch: int, engine: "Engine") -> None:
        """Hook at the top of every epoch (``no_consensus`` prints ``Epoch %d``)."""

    def after_minibatch(self, rep: Replica, visit: Visit, batch, i: int, epoch: int, nloop: int, N: int,
                        loss1: torch.Tensor, engine: "Engine") -> None:
        """Per-minibatch logging hook (verbose drivers)."""

    def aggregate_log(self, visit: Visit, metrics: Dict[str, float], ctx: Dict, engine: "Engine") -> None:
        """Print the legacy per-round line."""


@dataclass
class EngineConfig:
    Nloop: int = 1
    Nadmm: int = 1
    Nepoch: int = 1
    check_results: bool = False
    be_verbose: bool = False
    diagnostics: str = "post"        # 'post' = reference (extra forward after the step, Q17) | 'pre' = reuse closure loss
    graphs: bool = False             # CUDA-graph the Adam / SGD minibatch step
    deferred_rounds: bool = True     # enqueue the next round's first minibatch BEFORE reading the aggregation's record (FedAvg / FedProx
                                     # on the fused collective; not with per-round evaluation, verbose logs or resume records)
    graph_closures: bool = True      # ... and (with graphs=True) the L-BFGS closure: one graph for gradient evaluations, one for probes
    max_minibatches: Optional[int] = None   # cap per round (benchmarks / smoke tests)
    aggregate_in_epoch_loop: bool = True    # reference: aggregation sits inside the epoch loop
    reset_optimizer_each_epoch: bool = False  # no_consensus_multi.py:129-132 recreates Adam every epoch (Q18)
    nan_guard: str = "raise"         # non-finite aggregation residual: 'raise' | 'warn' | 'off' (SURVEY §5.3)
    resume_path: str = ""            # write a true-resume record here after every aggregation round ('' = never)
    streams: bool = True             # co-resident replicas (K > #GPUs) step concurrently on their own CUDA streams
    round_metrics: bool = True       # per-round JSONL: images/s, step / aggregate / eval device ms, bus GB/s
    # client learning-rate schedule over the run's rounds (optim/schedule.py); the base rate is the visit's opt_kwargs lr
    lr_schedule: str = "const"
    lr_warmup: int = 0
    lr_gamma: float = 0.1
    lr_step_rounds: int = 0
    lr_min: float = 0.0
    # training-loss regularisers of the classifier drivers (label smoothing, mixup, CutMix): part of the resume recipe
    label_smoothing: float = 0.0
    mixup_alpha: float = 0.0
    cutmix_alpha: float = 0.0

    def recipe(self, clip_norm: float = 0.0) -> Dict:
        """The schedule, clipping and mixing settings a resume record must match."""
        return dict(lr_schedule=self.lr_schedule, lr_warmup=self.lr_warmup, lr_gamma=self.lr_gamma,
                    lr_step_rounds=self.lr_step_rounds, lr_min=self.lr_min, clip_norm=clip_norm,
                    label_smoothing=self.label_smoothing, mixup_alpha=self.mixup_alpha, cutmix_alpha=self.cutmix_alpha)


class Engine:
    def __init__(self, task: Task, topo: Topology, strategy: Strategy, collective, cfg: EngineConfig,
                 log: Callable[[str], None] = print, metrics: Optional[MetricsLog] = None):
        self.task, self.topo, self.strategy, self.coll, self.cfg = task, topo, strategy, collective, cfg
        self._log = log
        self.metrics = metrics or MetricsLog(None)
        self.timers = PhaseTimers(topo.device)
        alloc = collective.arena_allocator()
        self.replicas: List[Replica] = [task.build_replica(ck, topo.device, alloc) for ck in topo.local_workers]
        for rep in self.replicas:
            for arena in rep.arenas.values():
                collective.register_arena(arena)
        if hasattr(collective, "warmup"):
            collective.warmup()          # lazy CUDA initialisation of the aggregation kernels belongs here, not in round 0
        self.optimizers: List = []
        self.images_seen = 0
        self.steps_done = 0
        self.last_epoch = 0
        self._graphs: Dict = {}
        self._block_opt_cache: Dict = {}
        self.stop_requested = False
        self.step_hook: Optional[Callable[["Engine"], None]] = None
        self.attack: Optional[Callable[["Engine"], None]] = None   # simulated Byzantine workers, before every aggregation
        self.last_loss1: Optional[torch.Tensor] = None
        self.graph_replays = 0
        self._pending_round = None
        self.graph_kernel_launches = 0
        self.aggregations_done = 0
        self._resume_pos: Optional[Dict] = None       # set by ckpt.load_resume: schedule position to re-enter at
        self._resume_state: Optional[Dict] = None
        self._round_mark = {"images": 0, "t": time.perf_counter(), "ms": {}}
        self._streams: Dict[int, "torch.cuda.Stream"] = {}
        self._round_extra: Dict = {}
        self._round_steps: Dict[int, int] = {}       # worker id -> local steps since the last aggregation
        # client learning-rate schedule: round r of T (a pure function of the schedule position)
        self.scheduled = schedule_active(cfg.lr_schedule, cfg.lr_warmup)
        self.total_rounds = 0
        self._visit_base: List[int] = []      # rounds before each nloop's first visit, in visits
        if self.scheduled:
            counts = [sum(1 for _ in task.visits(n)) for n in range(cfg.Nloop)]
            self._visit_base = [sum(counts[:n]) for n in range(cfg.Nloop)]
            self.total_rounds = sum(counts) * cfg.Nadmm * cfg.Nepoch
            if cfg.lr_warmup >= self.total_rounds:
                raise ValueError("lr_warmup must be smaller than the run's number of rounds T = %d (Nloop x block visits x "
                                 "Nadmm x Nepoch), got lr_warmup %d" % (self.total_rounds, cfg.lr_warmup))

    # ------------------------------------------------------------------
    def log(self, msg: str, root_only: bool = False) -> None:
        if root_only and not self.topo.is_root:
            return
        self._log(msg)

    # ------------------------------------------------------------------
    def _make_optimizer(self, rep: Replica, visit: Visit):
        arena = rep.arenas[visit.model]
        if visit.optimizer in ("adam", "adamw"):
            key = (rep.ck, visit.model, visit.lo, visit.hi) if visit.optimizer == "adam" else \
                ("adamw", rep.ck, visit.model, visit.lo, visit.hi)
            opt = self._block_opt_cache.get(key)
            kw = dict(visit.opt_kwargs)
            lr = kw.pop("lr", 1e-3)
            if opt is None:
                opt = BlockAdam(arena, visit.lo, visit.hi, lr=lr, adamw=visit.optimizer == "adamw",
                                device_lr=self.scheduled, **kw)
                self._block_opt_cache[key] = opt
            else:
                opt.reset(lr=lr)  # same as a freshly constructed Adam (Q18), but buffers/graphs persist
            return opt
        if visit.optimizer == "sgd":
            key = ("sgd", rep.ck, visit.model, visit.lo, visit.hi)
            opt = self._block_opt_cache.get(key)
            if opt is None:
                opt = BlockSGD(arena, visit.lo, visit.hi, device_lr=self.scheduled, **visit.opt_kwargs)
                self._block_opt_cache[key] = opt
            else:
                opt.reset(lr=visit.opt_kwargs["lr"])  # a zero momentum buffer, as a fresh SGD (Q18); buffers/graphs persist
            return opt
        if visit.optimizer == "lbfgs":
            return LBFGSNew(arena.params[visit.lo: visit.hi + 1], **visit.opt_kwargs)
        raise ValueError("unknown optimizer %r" % visit.optimizer)

    # ------------------------------------------------------------------
    def _train_step(self, rep: Replica, opt, visit: Visit, batch, pen: Penalty) -> torch.Tensor:
        """One ``opt.step(closure)`` + diagnostics; returns the diagnostics loss (0-dim, on device)."""
        task, cfg = self.task, self.cfg
        pre_loss = [None]
        if isinstance(opt, BLOCK_OPTIMIZERS):
            opt.set_penalty(pen.z, pen.y, pen.rho, visit.lambda1, visit.lambda2, pen.rho_dev)

            def closure():
                opt.zero_grad()
                loss = task.loss(rep, batch)
                with _grad_sink():
                    loss.backward()
                pre_loss[0] = loss.detach()
                return loss

            opt.step(closure)
        elif cfg.graphs and cfg.graph_closures and rep.device.type == "cuda" and isinstance(opt, LBFGSNew):
            gc_ = self._graphed_closure(rep, opt, visit, batch)
            gc_.bind(batch, pen)
            opt.step(gc_)
            if cfg.diagnostics == "post":
                return gc_.evaluate(False)[1]
            return gc_.first
        else:
            x = rep.block(visit)
            g = rep.block_grad(visit)
            has_pen = pen.z is not None or visit.lambda1 != 0.0 or visit.lambda2 != 0.0

            def closure():
                if torch.is_grad_enabled():
                    opt.zero_grad()
                loss = task.loss(rep, batch)
                if loss.requires_grad:
                    with _grad_sink():
                        loss.backward()
                    if has_pen:
                        flatops.add_penalty_grad_(g, x, pen.z, pen.y, pen.rho, visit.lambda1, visit.lambda2)
                total = loss.detach()
                if pre_loss[0] is None:
                    pre_loss[0] = total
                if has_pen:
                    total = total + flatops.penalty_value(x, pen.z, pen.y, pen.rho, visit.lambda1, visit.lambda2)
                return total

            opt.step(closure)
        if cfg.diagnostics == "post":
            with torch.no_grad():
                return task.loss(rep, batch).detach()
        return pre_loss[0]

    # ------------------------------------------------------------------
    def run(self) -> Dict:
        cfg, task, strat = self.cfg, self.task, self.strategy
        t0 = time.time()
        pos = self._resume_pos or {}
        for nloop in range(int(pos.get("nloop", 0)), cfg.Nloop):
            for vi, visit in enumerate(task.visits(nloop)):
                if self.stop_requested:
                    break
                if self._resume_pos is not None and nloop == pos.get("nloop", 0) and vi < pos.get("visit", 0):
                    continue                      # block visits completed before the checkpoint
                self._run_visit(nloop, vi, visit)
            if self.stop_requested:
                break
        self.log("Finished Training", root_only=True)
        return {"images_seen": self.images_seen, "steps": self.steps_done, "wall_s": time.time() - t0}

    def _refresh_derived(self) -> None:
        """Derived filters cached by the kernels' autograd glue must follow the weights (ADVICE r1, high): weights of a
        block change during ITS visit (Adam, FedAvg write-back) and are frozen again afterwards."""
        if self.topo.device.type != "cuda":
            return
        from ..ops import functional as FX

        if FX.fast_path_enabled():
            from ..ops import cuda_ops

            cuda_ops.refresh_caches()

    def _run_visit(self, nloop: int, vi: int, visit: Visit) -> None:
        cfg, task, strat = self.cfg, self.task, self.strategy
        for rep in self.replicas:
            rep.set_trainable(visit)
        self._refresh_derived()
        xs = [rep.block(visit) for rep in self.replicas]
        arena0 = self.replicas[0].arenas[visit.model]
        N = arena0.count(visit.lo, visit.hi)
        if getattr(strat, "dp", False):            # DP noise goes to parameters only, not to the arena's alignment padding
            strat.set_param_layout(visit.ci, arena0.chunk_counts(visit.lo, visit.hi))
        strat.begin_block(visit.ci, N, xs)
        self.optimizers = [self._make_optimizer(rep, visit) for rep in self.replicas]
        first_round = 0
        if self._resume_pos is not None:          # re-enter the schedule inside this visit (true resume, SURVEY §5.4)
            held = self._resume_pos.get("optimizer", visit.optimizer)     # records written before SGD did not store it
            if held != visit.optimizer:
                raise ValueError("resume record was written with optimizer %r, this run uses optimizer %r"
                                 % (held, visit.optimizer))
            want = cfg.recipe(visit.opt_kwargs.get("clip_norm", 0.0))
            # records written before schedules (or before mixing) lack the fields: they were run with the defaults
            held = dict(EngineConfig().recipe(), **self._resume_pos.get("recipe", {}))
            for name, val in want.items():
                if held[name] != val:
                    raise ValueError("resume record was written with %s %r, this run uses %s %r"
                                     % (name, held[name], name, val))
            first_round = int(self._resume_pos.get("round", 0))
            self._restore_visit_state()
            self._resume_pos = None
        rounds = [(nadmm, epoch) for nadmm in range(cfg.Nadmm) for epoch in range(cfg.Nepoch)]
        clip = visit.opt_kwargs.get("clip_norm", 0.0) > 0.0
        try:
            for ri, (nadmm, epoch) in enumerate(rounds):
                if ri < first_round:
                    continue
                self.last_epoch = epoch
                if cfg.reset_optimizer_each_epoch and epoch > 0:
                    self.optimizers = [self._make_optimizer(rep, visit) for rep in self.replicas]
                extra: Dict = {}
                if self.scheduled:
                    # round r of the whole run; written on the current stream, which the replicas' streams wait on
                    r = (self._visit_base[nloop] + vi) * len(rounds) + ri
                    extra["lr"] = round_lr(visit.opt_kwargs["lr"], r, self.total_rounds, cfg.lr_schedule, cfg.lr_warmup,
                                           cfg.lr_gamma, cfg.lr_step_rounds, cfg.lr_min)
                    for opt in self.optimizers:
                        opt.set_lr(extra["lr"])
                task.on_epoch_start(epoch, self)
                with nvtx_range("fedb200:steps"):
                    self._run_replicas(visit, nloop, epoch, N)
                if self.stop_requested:
                    return
                last_epoch_of_round = epoch == cfg.Nepoch - 1
                if cfg.aggregate_in_epoch_loop or last_epoch_of_round:
                    if clip:
                        extra["clip"] = self._take_clip_stats()
                    self._round_extra = extra          # the round row's lr / clip fields, carried with the pending round
                    self._aggregate(visit, nloop, nadmm, epoch if cfg.aggregate_in_epoch_loop else cfg.Nepoch - 1, N)
                    if cfg.resume_path:
                        from ..utils import ckpt

                        ckpt.save_resume(cfg.resume_path, self, dict(nloop=nloop, visit=vi, round=ri + 1, nadmm=nadmm, epoch=epoch,
                                                                    optimizer=visit.optimizer,
                                                                    recipe=cfg.recipe(visit.opt_kwargs.get("clip_norm", 0.0))))
        finally:
            if self._pending_round is not None:      # the last round of the visit (or a stop request): nothing left to overlap with
                self._finish_round()

    def _take_clip_stats(self) -> torch.Tensor:
        """``[sum of pre-clip norms, clipped steps, steps]`` over the local optimizers since the last call, and zero their
        accumulators; in stream order, so a minibatch queued behind a deferred aggregation counts toward the next round."""
        stats = [opt.clip_stats for opt in self.optimizers]
        snap = torch.stack(stats).sum(0)
        for st in stats:
            st.zero_()
        return snap

    def _restore_visit_state(self) -> None:
        st = self._resume_state or {}
        if st.get("strategy_state") and hasattr(self.strategy, "load_state"):
            self.strategy.load_state(st["strategy_state"])
        for rep, opt in zip(self.replicas, self.optimizers):
            osd = (st.get("optimizers") or {}).get(rep.ck)
            if osd is not None and hasattr(opt, "load_flat_state"):
                opt.load_flat_state(osd)
        self._resume_state = None

    # ------------------------------------------------------------------
    def _stream_of(self, i_rep: int):
        stx = self._streams.get(i_rep)
        if stx is None:
            stx = torch.cuda.Stream(device=self.topo.device)
            self._streams[i_rep] = stx
        return stx

    def _run_replicas(self, visit: Visit, nloop: int, epoch: int, N: int) -> None:
        """One pass over the local replicas' shards.  One replica: plain loop.  Several co-resident replicas (K > #GPUs;
        the reference's default K = 10): minibatch-major order with every replica on its own CUDA stream, so replica
        j+1's kernels are queued while replica j's run and small layers of different replicas overlap on the SMs
        (SURVEY §2.8).  Replicas are independent between aggregations, so the order does not change any result.
        Replicas that sit out the round (client sampling) are skipped: their loaders are not even iterated."""
        cfg = self.cfg
        reps = self.replicas
        active = [i for i in range(len(reps)) if self.strategy.participates(i)]
        multi = (cfg.streams and len(reps) > 1 and self.topo.device.type == "cuda" and not cfg.be_verbose)
        if not multi:
            for i_rep in active:
                self._run_shard(reps[i_rep], self.optimizers[i_rep], visit, self.strategy.penalty(i_rep), nloop, epoch, N)
                if self.stop_requested:
                    return
            return
        cur = torch.cuda.current_stream(self.topo.device)
        iters = {i: iter(enumerate(self.task.batches(reps[i], visit, epoch))) for i in active}
        pens = [self.strategy.penalty(i) for i in range(len(reps))]
        running = [None] * len(reps)
        live = list(active)               # unequal shards: a replica leaves the list when its shard is exhausted
        for i in live:
            self._stream_of(i).wait_stream(cur)
        while live and not self.stop_requested:
            nxt = []
            for i in live:
                with torch.cuda.stream(self._stream_of(i)):       # the batch gather / H2D belongs to the replica's stream too
                    try:
                        bi, batch = next(iters[i])
                    except StopIteration:
                        continue
                    if cfg.max_minibatches is not None and bi >= cfg.max_minibatches:
                        continue
                    running[i] = self._one_step(reps[i], self.optimizers[i], visit, batch, pens[i], running[i], bi, epoch, nloop, N)
                nxt.append(i)
                if self.stop_requested:
                    break
            live = nxt
        for i in active:
            cur.wait_stream(self._stream_of(i))
            reps[i].running_loss = running[i]

    def _one_step(self, rep: Replica, opt, visit: Visit, batch, pen: Penalty, running, i: int, epoch: int, nloop: int, N: int):
        cfg, task = self.cfg, self.task
        with self.timers.phase("step"):
            if cfg.graphs and isinstance(opt, BLOCK_OPTIMIZERS) and rep.device.type == "cuda":
                loss1 = self._graphed_step(rep, opt, visit, batch, pen)
            else:
                loss1 = self._train_step(rep, opt, visit, batch, pen)
        if self._pending_round is not None:
            self._finish_round()          # the GPU already has this minibatch queued behind the aggregation
        running = loss1 if running is None else running + loss1
        self.last_loss1 = loss1
        self.images_seen += task.batch_size_of(batch)
        self.steps_done += 1
        self._round_steps[rep.ck] = self._round_steps.get(rep.ck, 0) + 1
        task.after_minibatch(rep, visit, batch, i, epoch, nloop, N, loss1, self)
        if self.step_hook is not None:
            self.step_hook(self)
        return running

    def _run_shard(self, rep: Replica, opt, visit: Visit, pen: Penalty, nloop: int, epoch: int, N: int) -> None:
        cfg, task = self.cfg, self.task
        running = None
        for i, batch in enumerate(task.batches(rep, visit, epoch)):
            if cfg.max_minibatches is not None and i >= cfg.max_minibatches:
                break
            running = self._one_step(rep, opt, visit, batch, pen, running, i, epoch, nloop, N)
            if self.stop_requested:
                break
        rep.running_loss = running

    def _aggregate(self, visit: Visit, nloop: int, nadmm: int, epoch: int, N: int) -> None:
        """End of a round.  The aggregation is ONE kernel in stream order (write-back included), so the next minibatch can
        be queued right behind it; what the host wants from it (residuals, non-finite count, time-out status) is a record in
        pinned memory.  With ``deferred_rounds`` the record is read after the next minibatch has been enqueued instead of
        draining the GPU first, so the step that contains the round boundary does not wait for the host's read."""
        cfg = self.cfg
        # On by default up to 4 ranks only: with more ranks the first deferred aggregation of a run and adaptive-ADMM runs were not
        # shown to gain from it.  FEDB200_DEFERRED_ROUNDS=1 forces it on.
        env = os.environ.get("FEDB200_DEFERRED_ROUNDS", "auto")
        # (only a collective with asynchronous entry points actually defers: FusedCollective; the others answer "done")
        defer = (cfg.deferred_rounds and not cfg.check_results and not cfg.be_verbose
                 and not cfg.resume_path and env != "0" and (env == "1" or self.topo.world_size <= 4))
        if self._pending_round is not None:
            # the previous round is still deferred when no local replica took a step since (all of them sat out a sampled
            # round): finish it here, before its record is overwritten
            self._finish_round()
        if self.attack is not None:
            self.attack(self)
        # the round's local step counts (0 for replicas that sat out) and client learning rate, known on the host
        self.strategy.note_local_steps([self._round_steps.get(rep.ck, 0) for rep in self.replicas],
                                       self._round_extra.get("lr", visit.opt_kwargs.get("lr")))
        self._round_steps = {}
        with nvtx_range("fedb200:aggregate"), self.timers.phase("aggregate"):
            token = self.strategy.aggregate_begin(nadmm) if defer else ("done", self.strategy.aggregate(nadmm))
        self._pending_round = (token, visit, nloop, nadmm, epoch, N, self._round_extra)
        self._round_extra = {}
        if token[0] == "done":
            self._finish_round()

    def _finish_round(self) -> None:
        token, visit, nloop, nadmm, epoch, N, extra = self._pending_round
        self._pending_round = None
        metrics = self.strategy.aggregate_end(token)
        self.aggregations_done += 1
        ctx = {"nloop": nloop, "nadmm": nadmm, "epoch": epoch, "N": N, "rho_mean": self.strategy.rho_mean()}
        if metrics is not None and getattr(self.coll, "last_nonfinite", 0.0):
            metrics["nonfinite"] = float(self.coll.last_nonfinite)      # counted inside the aggregation kernel
        self._check_finite(visit, metrics, ctx)
        acc = None
        if self.cfg.check_results:
            with nvtx_range("fedb200:eval"), self.timers.phase("eval"):
                acc = self.task.evaluate(self.replicas, self)
        if metrics:
            self.task.aggregate_log(visit, metrics, ctx, self)
            row = dict(kind="round", block=visit.ci, label=list(visit.label), model=visit.model, **ctx, **metrics)
            if "lr" in extra:
                row["lr"] = extra["lr"]
            if "clip" in extra:                    # mean pre-clip gradient norm of the round's local steps, clipped share
                norm_sum, clipped, steps = (float(v) for v in extra["clip"].tolist())
                row["grad_norm"] = norm_sum / steps if steps else float("nan")
                row["clip_frac"] = clipped / steps if steps else float("nan")
            if self.cfg.round_metrics:
                row.update(self._round_perf(N))
            self.metrics.write(row)
        if acc is not None:
            self.metrics.write(dict(kind="eval", block=visit.ci, **ctx, accuracy=acc))

    def _round_perf(self, N: int) -> Dict[str, float]:
        """Throughput and device-time fields of the round that just ended (SURVEY §5.5): images/s of this process,
        device ms per phase (CUDA events, resolved lazily: the round's own host read has already synchronised),
        aggregation latency and NVLink bus bandwidth (nccl-tests convention: 2 (W-1)/W * bytes / time)."""
        now = time.perf_counter()
        mark = self._round_mark
        # only the (few) aggregate / eval events are resolved here — the GPU is idle while the host is in this function
        summ = self.timers.summary(reduce_max=False, names=("aggregate", "eval"))
        out: Dict[str, float] = {}
        dt = max(now - mark["t"], 1e-9)
        out["images_per_s"] = (self.images_seen - mark["images"]) / dt
        for k, v in summ.items():
            prev = mark["ms"].get(k, {"ms": 0.0, "count": 0})
            d_ms, d_n = v["ms"] - prev["ms"], v["count"] - prev["count"]
            if d_n > 0:
                out[k + "_ms"] = d_ms
                out[k + "_count"] = d_n
        agg_ms = out.get("aggregate_ms")
        if agg_ms:
            out["aggregate_us"] = 1e3 * agg_ms / max(out.get("aggregate_count", 1), 1)
            W = max(self.topo.world_size, 1)
            if W > 1:                          # compressed rounds move their payload instead of 4 bytes per coordinate
                bits = getattr(self.strategy, "q_bits", 0)
                nbytes = payload_bytes(N, bits) if bits else 4.0 * N
                if getattr(self.strategy, "topk_r", 0.0):
                    nbytes = topk_payload_bytes(N, self.strategy.topk_k)
                out["bus_GBs"] = 2.0 * (W - 1) / W * nbytes / (out["aggregate_us"] * 1e-6) / 1e9
        out["two_shot"] = bool(getattr(self.coll, "last_two_shot", False))
        self._round_mark = {"images": self.images_seen, "t": now, "ms": {k: dict(v) for k, v in summ.items()}}
        return out

    def _check_finite(self, visit: Visit, metrics: Optional[Dict[str, float]], ctx: Dict) -> None:
        """Failure detection (SURVEY §5.3): the residuals are norms over the REDUCED vector of every worker, so one
        NaN/Inf anywhere in any replica's block shows up here, one round after it appeared, on every rank."""
        if not metrics or self.cfg.nan_guard == "off":
            return
        bad = [k for k in ("dual", "primal") if k in metrics and not math.isfinite(float(metrics[k]))]
        if not bad and metrics.get("nonfinite"):
            bad = ["reduced vector (%d non-finite entries)" % int(metrics["nonfinite"])]
        if not bad:
            return
        msg = ("non-finite %s residual after aggregating block %s (ids %s) at loop %d, round %d, epoch %d on rank %d: "
               "a replica diverged (NaN/Inf in its parameters, duals or consensus vector)"
               % ("/".join(bad), visit.ci, list(visit.label), ctx["nloop"], ctx["nadmm"], ctx["epoch"], self.topo.rank))
        self.metrics.write(dict(kind="fault", block=visit.ci, **ctx, nonfinite=bad))
        if self.cfg.nan_guard == "raise":
            raise FloatingPointError(msg)
        self.log("WARNING: " + msg)

    # ------------------------------------------------------------------
    # CUDA-graphed block-optimizer step (Adam / SGD)
    # ------------------------------------------------------------------
    def _graphed_closure(self, rep: Replica, opt, visit: Visit, batch):
        """One graphed closure per replica: the graphs of the previous block visit are dropped (their activations pools are
        as large as the network's; an L-BFGS visit re-creates its optimizer anyway, Q18)."""
        from .graphs import GraphedClosure

        slot = ("lbfgs", rep.ck)
        ident = (visit.model, visit.lo, visit.hi, tuple(tuple(t.shape) for t in batch if torch.is_tensor(t)))
        cur = self._graphs.get(slot)
        if cur is None or cur[0] != ident or cur[1].opt is not opt:
            cur = (ident, GraphedClosure(self, rep, opt, visit, batch))
            self._graphs[slot] = cur
        return cur[1]

    def _graphed_step(self, rep: Replica, opt, visit: Visit, batch, pen: Penalty) -> torch.Tensor:
        from .graphs import GraphedAdamStep

        key = (rep.ck, visit.model, visit.lo, visit.hi, tuple(tuple(t.shape) for t in batch if torch.is_tensor(t)))
        gs = self._graphs.get(key)
        if gs is None:
            gs = GraphedAdamStep(self, rep, opt, visit, batch, pen)
            self._graphs[key] = gs
        return gs.run(batch, pen)
