"""``BlockAdam`` — Adam over ONE contiguous block of a flat arena, with the
FedProx / augmented-Lagrangian / elastic-net gradients folded into the update.

The reference creates ``torch.optim.Adam(lr=1e-3)`` over the trainable tensors
for every block visit (/root/reference/src/federated_multi.py:156-159, SURVEY
Q18) and builds the penalty terms through autograd on a ``torch.cat`` of the
block inside every closure (consensus_multi.py:214-220).  Here:

* moments ``m``/``v`` are two flat buffers the size of the block slice;
* one kernel (``flat_kernels.cu: adam_prox_kernel``) reads ``x, g, m, v`` (+ ``z``,
  ``y``) once and writes ``x, m, v`` — the penalty gradient
  ``y + rho (x - z) + lambda1 sign(x) + 2 lambda2 x`` is computed in registers
  (SURVEY G14/G15);
* numerics are ``torch.optim.Adam`` defaults (betas 0.9/0.999, eps 1e-8, bias
  correction, no amsgrad, no weight decay), or ``torch.optim.AdamW`` with
  ``adamw=True`` (decoupled decay ``x *= 1 - lr weight_decay`` before the step);
* ``device_lr=True`` keeps the learning rate in a 1-element device tensor that
  :meth:`set_lr` rewrites between rounds (a schedule), so the graphed step is
  replayed, not re-captured;
* ``clip_norm > 0`` adds one kernel before the update
  (``flat_kernels.cu: grad_norm_kernel``) that writes the block gradient's norm;
  the update scales the data-loss gradient by
  ``min(1, clip_norm / (norm + 1e-6))`` as ``clip_grad_norm_`` does.  Each step
  adds ``[norm, norm > clip_norm, 1]`` to :attr:`clip_stats` on the device.

It subclasses ``torch.optim.Optimizer`` so ``state_dict()`` has the stock Adam
layout (``step`` / ``exp_avg`` / ``exp_avg_sq`` per parameter) for the legacy
checkpoint schema.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
from torch.optim.optimizer import Optimizer

from ..ops import flatops
from ..utils.flat import FlatArena


class BlockAdam(Optimizer):
    def __init__(self, arena: FlatArena, lo: int, hi: int, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 adamw: bool = False, weight_decay: float = 0.0, clip_norm: float = 0.0, device_lr: bool = False):
        if weight_decay != 0.0 and not adamw:
            raise ValueError("weight_decay needs adamw=True (decoupled decay), got weight_decay %r" % (weight_decay,))
        if not weight_decay >= 0.0:
            raise ValueError("weight_decay must be >= 0, got %r" % (weight_decay,))
        if not clip_norm >= 0.0:
            raise ValueError("clip_norm must be >= 0, got %r" % (clip_norm,))
        params = arena.params[lo: hi + 1]
        if adamw:           # torch.optim.AdamW's param-group keys, so state_dict() loads into it
            defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                            foreach=None, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=True)
        else:
            defaults = dict(lr=lr, betas=betas, eps=eps)
        super().__init__(params, defaults)
        self.arena, self.lo, self.hi = arena, lo, hi
        self.adamw, self.weight_decay, self.clip_norm = bool(adamw), float(weight_decay), float(clip_norm)
        a, b = arena.span(lo, hi)
        self._span = (a, b)
        self.m = torch.zeros(b - a, dtype=torch.float32, device=arena.data.device)
        self.v = torch.zeros_like(self.m)
        self.lr_dev: Optional[torch.Tensor] = (torch.full((1,), lr, dtype=torch.float32, device=arena.data.device)
                                               if device_lr else None)
        self.clip_ws = flatops.clip_workspace(self.m) if clip_norm > 0.0 else None
        self.t = 0
        # device-resident step counter: lets the update be replayed from a CUDA graph (no host-side scalars)
        self.t_dev = torch.zeros(1, dtype=torch.int32, device=arena.data.device) if arena.data.is_cuda else None
        # penalty configuration (set by the aggregation strategy for the current block visit)
        self.z: Optional[torch.Tensor] = None
        self.y: Optional[torch.Tensor] = None
        self.rho = 0.0
        self.rho_dev: Optional[torch.Tensor] = None   # device-resident penalty (adaptive ADMM); wins over ``rho``
        self.lambda1 = 0.0
        self.lambda2 = 0.0

    # -- views --------------------------------------------------------------
    @property
    def x(self) -> torch.Tensor:
        return self.arena.data[self._span[0]: self._span[1]]

    @property
    def g(self) -> torch.Tensor:
        return self.arena.grad[self._span[0]: self._span[1]]

    def set_penalty(self, z=None, y=None, rho: float = 0.0, lambda1: float = 0.0, lambda2: float = 0.0, rho_dev=None) -> None:
        self.z, self.y, self.rho, self.lambda1, self.lambda2 = z, y, float(rho), float(lambda1), float(lambda2)
        self.rho_dev = rho_dev

    def reset(self, lr: Optional[float] = None) -> None:
        """Back to the state of a freshly constructed optimizer (zero moments, step 0)."""
        self.m.zero_()
        self.v.zero_()
        self.t = 0
        if self.t_dev is not None:
            self.t_dev.zero_()
        if lr is not None:
            self.set_lr(lr)

    def set_lr(self, lr: float) -> None:
        """The learning rate of the following steps; with ``device_lr`` written in stream order, no host sync."""
        self.param_groups[0]["lr"] = lr
        if self.lr_dev is not None:
            self.lr_dev.fill_(lr)

    @property
    def clip_stats(self) -> Optional[torch.Tensor]:
        """``[sum of pre-clip norms, clipped steps, steps]`` since the last zeroing (device; ``None`` without clipping)."""
        return self.clip_ws[0][1:4] if self.clip_ws is not None else None

    def zero_grad(self, set_to_none: bool = False) -> None:
        self.g.zero_()

    @torch.no_grad()
    def apply_update(self) -> None:
        """The update alone (gradients already in the arena); CUDA-graph friendly: no host reads."""
        self.t += 1
        grp = self.param_groups[0]
        step = self.t
        if self.t_dev is not None and flatops._cuda(self.x):
            from ..ops import cuda_ops

            cuda_ops.bump_step(self.t_dev)
            step = self.t_dev
        flatops.adam_prox_step(self.x, self.g, self.m, self.v, step, self.lr_dev if self.lr_dev is not None else grp["lr"],
                               grp["betas"][0], grp["betas"][1], grp["eps"], self.z, self.y, self.rho, self.lambda1,
                               self.lambda2, self.rho_dev, weight_decay=self.weight_decay, clip_norm=self.clip_norm,
                               clip_ws=self.clip_ws)

    def step(self, closure: Optional[Callable] = None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.apply_update()
        return loss

    # -- true resume (utils/ckpt.py) ----------------------------------------------
    def flat_state(self) -> dict:
        t = int(self.t_dev.item()) if self.t_dev is not None else self.t
        rec = {"m": self.m.detach().cpu().clone(), "v": self.v.detach().cpu().clone(), "t": max(t, self.t),
               "lr": self.param_groups[0]["lr"]}
        if self.adamw:
            rec.update(optimizer="adamw", weight_decay=self.weight_decay)
        return rec

    def load_flat_state(self, rec: dict) -> None:
        held = rec.get("optimizer", "adam")
        if held != ("adamw" if self.adamw else "adam"):
            raise ValueError("resume record holds the state of optimizer %r, this run uses optimizer %r"
                             % (held, "adamw" if self.adamw else "adam"))
        if self.adamw and rec["weight_decay"] != self.weight_decay:
            raise ValueError("resume record holds AdamW weight_decay %r, this run uses weight_decay %r"
                             % (rec["weight_decay"], self.weight_decay))
        self.m.copy_(rec["m"].to(self.m.device))
        self.v.copy_(rec["v"].to(self.v.device))
        self.t = int(rec["t"])
        if self.t_dev is not None:
            self.t_dev.fill_(self.t)
        self.set_lr(rec.get("lr", self.param_groups[0]["lr"]))

    # -- stock-Adam (AdamW) compatible state ------------------------------------
    def state_dict(self):
        base = self._span[0]
        if self.t_dev is not None:      # graph replays only advance the device counter (ADVICE r1)
            self.t = max(self.t, int(self.t_dev.item()))
        for i in range(self.lo, self.hi + 1):
            p = self.arena.params[i]
            o = self.arena.offsets[i] - base
            n = self.arena.numels[i]
            self.state[p] = {
                "step": torch.tensor(float(self.t)),
                "exp_avg": self.m[o: o + n].view(p.shape).clone(),
                "exp_avg_sq": self.v[o: o + n].view(p.shape).clone(),
            }
        sd = super().state_dict()
        for p in list(self.state.keys()):
            del self.state[p]
        return sd
