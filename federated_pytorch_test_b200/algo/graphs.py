"""CUDA-graph capture of the per-minibatch block-optimizer step, Adam or SGD (SURVEY §7.1 ``sched/``, G-launch-bound).

The reference's hot loop issues ~400 eager kernel launches per minibatch (forward,
backward, foreach-Adam, a second diagnostics forward) plus a ``.item()`` host sync
(/root/reference/src/federated_multi.py:178-197).  Here the whole step

    zero block gradient -> forward -> loss -> backward -> fused Adam / SGD (+penalty) -> diagnostics forward

is captured ONCE per (replica, block, batch shape) into a ``torch.cuda.CUDAGraph`` on
static input buffers and replayed with one launch per minibatch.  Everything that
varies between minibatches lives in device memory (inputs, Adam step counter,
consensus vectors), so the graph never needs re-capture inside a block visit; across
visits the optimizer buffers persist (``BlockAdam.reset`` / ``BlockSGD.reset``) and so do the graphs.

No tracing compiler is involved: the graph is just the recorded launch sequence of
the hand-written kernels (and the few ATen ops that remain).
"""
from __future__ import annotations

from typing import List, Optional

import torch

from ..ops import cuda_ops



def _grad_sink():
    """Weight-gradient kernels may accumulate straight into the arena's gradient views during these backward calls."""
    from ..ops import functional as FX

    if torch.cuda.is_available() and FX.fast_path_enabled():
        from ..ops import cuda_ops

        return cuda_ops.accumulate_into_grad()
    import contextlib

    return contextlib.nullcontext()


def capture_graph(stream, body, pool=None):
    """Capture ``body()`` into a new CUDA graph on ``stream``; returns ``(graph, body's return value)``.  ``pool``: the
    memory pool of another graph that never runs concurrently with this one (its private memory is shared).

    A CUDAGraph that is garbage (e.g. the graphs of a previous Engine, kept alive by a reference cycle) must not be
    finalised while a capture is in progress: cudaGraphExecDestroy is "not permitted when stream is capturing" and
    invalidates the capture.  torch.cuda.graph no longer collects by itself, so: collect
    first, keep the cyclic collector off during the capture."""
    import gc

    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    gc.collect()
    was_enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(g, stream=stream, pool=pool):
            out = body()
    finally:
        if was_enabled:
            gc.enable()
    return g, out


class GraphedEval:
    """Evaluation forward of one replica at one batch shape as a CUDA graph (SURVEY G21, X6): the reference evaluates all K
    models on 10 000 test images after EVERY aggregation round (79 batches x K x 360 rounds for ResNet18,
    /root/reference/src/federated_multi.py:108-121) with ~70 eager launches per batch.  Captured here: forward (train-mode
    BatchNorm statistics included, Q4, or eval-mode BatchNorm with ``eval_bn='running'``: the network's mode at capture time is
    baked in, so callers key graphs by it) + the fused argmax / compare / count kernel; the counter lives on the device."""

    WARMUP = 2

    def __init__(self, net, batch, counter: torch.Tensor, device):
        self.net, self.counter = net, counter
        self.static = [t.clone() for t in batch]
        self.graph = None
        self.calls = 0
        self.stream = torch.cuda.Stream(device=device)

    def _body(self):
        logits = self.net(self.static[0])
        cuda_ops.argmax_count(logits, self.static[1], self.counter)
        return None

    @torch.no_grad()
    def run(self, batch) -> None:
        for dst, src in zip(self.static, batch):
            dst.copy_(src, non_blocking=True)
        self.calls += 1
        if self.graph is None:
            if self.calls <= self.WARMUP:
                self._body()
                return
            self.graph, _ = capture_graph(self.stream, self._body)
        self.graph.replay()


class GraphedAdamStep:
    """The minibatch step of a block optimizer (``BlockAdam`` or ``BlockSGD``: it only calls ``zero_grad``,
    ``apply_update`` and ``set_penalty``).  The graph is captured once per (replica, block, batch shape) and a change of
    learning rate does not invalidate it: with a schedule the optimizer passes its device ``lr_dev``, which the engine
    rewrites in stream order at the start of every round, and without one the host rate is constant over the run.
    With clipping the captured update is two kernels, the gradient norm and the step."""

    WARMUP = 3

    def __init__(self, engine, rep, opt, visit, batch, pen):
        self.engine, self.rep, self.opt, self.visit = engine, rep, opt, visit
        self.static = [t.clone() if torch.is_tensor(t) else t for t in batch]
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.loss_out: Optional[torch.Tensor] = None
        self.calls = 0
        self.kernels_per_replay = 0
        self.pen_key = None
        self.stream = torch.cuda.Stream(device=rep.device)

    # the step body; must not touch the host
    def _body(self) -> torch.Tensor:
        task, rep, opt = self.engine.task, self.rep, self.opt
        opt.zero_grad()
        loss = task.loss(rep, self.static)
        with _grad_sink():
            loss.backward()
        opt.apply_update()
        if self.engine.cfg.diagnostics == "post":
            with torch.no_grad():
                return task.loss(rep, self.static).detach()
        return loss.detach()

    def _pen_key(self, pen):
        # a device-resident rho (adaptive ADMM) never invalidates the graph; a host-side one is baked into the launch
        rho_key = ("dev", pen.rho_dev.data_ptr()) if pen.rho_dev is not None else ("host", float(pen.rho))
        return (pen.z.data_ptr() if pen.z is not None else 0, pen.y.data_ptr() if pen.y is not None else 0,
                rho_key, self.visit.lambda1, self.visit.lambda2)

    def _capture(self) -> None:
        before = cuda_ops.launch_count()
        self.graph, self.loss_out = capture_graph(self.stream, self._body)
        self.kernels_per_replay = cuda_ops.launch_count() - before

    def run(self, batch, pen) -> torch.Tensor:
        opt = self.opt
        key = self._pen_key(pen)
        if key != self.pen_key:          # consensus buffers changed (new block visit): the graph bakes their addresses
            self.pen_key = key
            self.graph = None
            self.calls = 0
        opt.set_penalty(pen.z, pen.y, pen.rho, self.visit.lambda1, self.visit.lambda2, pen.rho_dev)
        for dst, src in zip(self.static, batch):
            if torch.is_tensor(dst):
                if dst.shape != src.shape:
                    raise RuntimeError("graphed step called with a different batch shape")
                dst.copy_(src, non_blocking=True)
        self.calls += 1
        if self.graph is None:
            if self.calls <= self.WARMUP:
                return self._body().clone()   # eager warm-up (lazy inits, cudaFuncSetAttribute, autotune)
            self._capture()
            # the capture itself does not execute: replay once for this minibatch
        self.graph.replay()
        self.engine.graph_replays += 1
        self.engine.graph_kernel_launches += self.kernels_per_replay
        return self.loss_out.clone()


class GraphedClosure:
    """The L-BFGS closure as two CUDA graphs per (replica, block visit, batch shape).

    ``LBFGSNew.step`` evaluates its closure 5-20 times per minibatch (/root/reference/src/lbfgsnew.py:590-659: gradient
    evaluations with autograd on, line-search probes under ``no_grad``); for the small VAE-CL / CPC networks every one of
    those evaluations is ~100-300 launches of microsecond kernels, i.e. host-bound (SURVEY §7.3(5)).  Captured here:

    * ``grad``: zero the block gradient, forward, loss, backward (weight-gradient kernels accumulate straight into the arena's
      gradient slice), closed-form FedProx / ADMM / elastic-net gradient, total loss;
    * ``eval``: no-grad forward + penalty value.

    Both read the minibatch from static buffers and the parameters from the arena (the line search moves ``x`` in place), and
    write ``[total, data-loss]`` into a static pair; the two graphs share one memory pool.  Nothing inside touches the host."""

    WARMUP = 2

    def __init__(self, engine, rep, opt, visit, batch):
        self.engine, self.rep, self.opt, self.visit = engine, rep, opt, visit
        self.static = [t.clone() if torch.is_tensor(t) else t for t in batch]
        self.stream = torch.cuda.Stream(device=rep.device)
        self.graph = {True: None, False: None}
        self.out = {True: None, False: None}
        self.kernels = {True: 0, False: 0}
        self.calls = {True: 0, False: 0}
        self.pen = None
        self.pen_key = None
        self.first = None

    def _key(self, pen):
        rho_key = ("dev", pen.rho_dev.data_ptr()) if pen.rho_dev is not None else ("host", float(pen.rho))
        return (pen.z.data_ptr() if pen.z is not None else 0, pen.y.data_ptr() if pen.y is not None else 0, rho_key)

    def bind(self, batch, pen) -> None:
        """Start of one ``opt.step``: new minibatch into the static buffers; a changed consensus buffer invalidates the graphs."""
        key = self._key(pen)
        if key != self.pen_key:
            self.pen_key = key
            self.graph = {True: None, False: None}
            self.calls = {True: 0, False: 0}
        self.pen = pen
        for dst, src in zip(self.static, batch):
            if torch.is_tensor(dst):
                if dst.shape != src.shape:
                    raise RuntimeError("graphed closure called with a different batch shape")
                dst.copy_(src, non_blocking=True)
        self.first = None

    def _body(self, with_grad: bool) -> torch.Tensor:
        from ..ops import flatops

        task, rep, visit, pen = self.engine.task, self.rep, self.visit, self.pen
        x = rep.block(visit)
        has_pen = pen.z is not None or visit.lambda1 != 0.0 or visit.lambda2 != 0.0
        if with_grad:
            self.opt.zero_grad()
            loss = task.loss(rep, self.static)
            with _grad_sink():
                loss.backward()
            if has_pen:
                flatops.add_penalty_grad_(rep.block_grad(visit), x, pen.z, pen.y, pen.rho, visit.lambda1, visit.lambda2)
        else:
            with torch.no_grad():
                loss = task.loss(rep, self.static)
        base = loss.detach()
        total = base + flatops.penalty_value(x, pen.z, pen.y, pen.rho, visit.lambda1, visit.lambda2) if has_pen else base
        return torch.stack([total.reshape(()), base.reshape(())])

    def evaluate(self, with_grad: bool) -> torch.Tensor:
        """``[total, data loss]`` (device) at the current parameters."""
        self.calls[with_grad] += 1
        if self.graph[with_grad] is None:
            if self.calls[with_grad] <= self.WARMUP:
                with torch.enable_grad() if with_grad else torch.no_grad():
                    out = self._body(with_grad)
                if self.first is None:
                    self.first = out[1]
                return out
            other = self.graph[not with_grad]
            before = cuda_ops.launch_count()
            with torch.enable_grad() if with_grad else torch.no_grad():
                self.graph[with_grad], self.out[with_grad] = capture_graph(
                    self.stream, lambda: self._body(with_grad), pool=other.pool() if other is not None else None)
            self.kernels[with_grad] = cuda_ops.launch_count() - before
        self.graph[with_grad].replay()
        self.engine.graph_replays += 1
        self.engine.graph_kernel_launches += self.kernels[with_grad]
        out = self.out[with_grad].clone()
        if self.first is None:
            self.first = out[1]
        return out

    def __call__(self) -> torch.Tensor:
        return self.evaluate(torch.is_grad_enabled())[0]
