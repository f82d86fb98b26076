"""``BlockSGD`` — SGD (momentum, Nesterov, weight decay) over ONE contiguous block of a flat arena, with the FedProx /
augmented-Lagrangian / elastic-net gradients folded into the update; the sibling of :class:`~.block_adam.BlockAdam`.

* the momentum buffer is one flat buffer the size of the block slice, and does not exist when ``momentum == 0``;
* one kernel (``flat_kernels.cu: sgd_prox_kernel``) reads ``x, g, buf`` (+ ``z``, ``y``) once and writes ``x, buf``;
* numerics are ``torch.optim.SGD`` with ``dampening = 0`` and ``maximize = False``.  A zeroed buffer gives torch's first
  step (``buf = g``), so there is no step counter and the update has no host-side state that changes between steps:
  it replays from a CUDA graph as it is;
* ``device_lr`` and ``clip_norm`` work as for :class:`~.block_adam.BlockAdam` (a device learning rate that a schedule
  rewrites between rounds; the gradient-norm kernel before the update).

It subclasses ``torch.optim.Optimizer`` so ``state_dict()`` has the stock SGD layout (``momentum_buffer`` per parameter,
SGD's param-group keys) for the legacy checkpoint schema.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch
from torch.optim.optimizer import Optimizer

from ..ops import flatops
from ..utils.flat import FlatArena


class BlockSGD(Optimizer):
    def __init__(self, arena: FlatArena, lo: int, hi: int, lr: float, momentum: float = 0.0, nesterov: bool = False,
                 weight_decay: float = 0.0, clip_norm: float = 0.0, device_lr: bool = False):
        if not lr > 0.0:
            raise ValueError("lr must be > 0 for SGD, got %r" % (lr,))
        if not 0.0 <= momentum < 1.0:
            raise ValueError("momentum must lie in [0, 1), got %r" % (momentum,))
        if nesterov and momentum == 0.0:
            raise ValueError("nesterov needs momentum > 0")
        if not weight_decay >= 0.0:
            raise ValueError("weight_decay must be >= 0, got %r" % (weight_decay,))
        if not clip_norm >= 0.0:
            raise ValueError("clip_norm must be >= 0, got %r" % (clip_norm,))
        params = arena.params[lo: hi + 1]
        super().__init__(params, dict(lr=lr, momentum=momentum, dampening=0, weight_decay=weight_decay,
                                      nesterov=bool(nesterov), maximize=False, foreach=None, differentiable=False,
                                      fused=None))
        self.arena, self.lo, self.hi = arena, lo, hi
        a, b = arena.span(lo, hi)
        self._span = (a, b)
        self.buf: Optional[torch.Tensor] = (torch.zeros(b - a, dtype=torch.float32, device=arena.data.device)
                                            if momentum != 0.0 else None)
        self.clip_norm = float(clip_norm)
        self.lr_dev: Optional[torch.Tensor] = (torch.full((1,), lr, dtype=torch.float32, device=arena.data.device)
                                               if device_lr else None)
        self.clip_ws = flatops.clip_workspace(self.x) if clip_norm > 0.0 else None
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
        """Back to the state of a freshly constructed optimizer (zero momentum buffer)."""
        if self.buf is not None:
            self.buf.zero_()
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
        grp = self.param_groups[0]
        flatops.sgd_prox_step(self.x, self.g, self.buf, self.lr_dev if self.lr_dev is not None else grp["lr"],
                              grp["momentum"], grp["nesterov"], grp["weight_decay"], self.z, self.y, self.rho,
                              self.lambda1, self.lambda2, self.rho_dev, clip_norm=self.clip_norm, clip_ws=self.clip_ws)

    def step(self, closure: Optional[Callable] = None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.apply_update()
        return loss

    # -- true resume (utils/ckpt.py) ----------------------------------------------
    def flat_state(self) -> dict:
        grp = self.param_groups[0]
        return {"optimizer": "sgd", "buf": None if self.buf is None else self.buf.detach().cpu().clone(),
                "lr": grp["lr"], "momentum": grp["momentum"], "nesterov": grp["nesterov"],
                "weight_decay": grp["weight_decay"]}

    def load_flat_state(self, rec: dict) -> None:
        if rec.get("optimizer") != "sgd":
            raise ValueError("resume record holds the state of another optimizer (keys %s), this run uses optimizer 'sgd'"
                             % sorted(rec))
        grp = self.param_groups[0]
        held = (rec["momentum"], rec["nesterov"], rec["weight_decay"])
        if held != (grp["momentum"], grp["nesterov"], grp["weight_decay"]):
            raise ValueError("resume record holds SGD settings (momentum, nesterov, weight_decay) %r, this run uses %r"
                             % (held, (grp["momentum"], grp["nesterov"], grp["weight_decay"])))
        if self.buf is not None:
            self.buf.copy_(rec["buf"].to(self.buf.device))
        self.set_lr(rec["lr"])

    # -- stock-SGD compatible state -------------------------------------------
    def state_dict(self):
        base = self._span[0]
        for i in range(self.lo, self.hi + 1):
            p = self.arena.params[i]
            o = self.arena.offsets[i] - base
            n = self.arena.numels[i]
            # the buffer slice has the parameter's memory layout (channels-last conv weights included)
            self.state[p] = {"momentum_buffer": None if self.buf is None
                             else self.buf[o: o + n].as_strided(p.shape, p.stride()).clone()}
        sd = super().state_dict()
        for p in list(self.state.keys()):
            del self.state[p]
        return sd
