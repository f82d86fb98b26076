"""Client learning-rate schedule over communication rounds.

A *round* is one entry of the engine's ``(nloop, visit, nadmm, epoch)`` loop; ``r`` counts rounds from 0 over the whole
run and ``T`` is the run's number of rounds.  ``r`` is a function of the schedule position alone, so a resumed run, any
process layout and a worker that sat out a sampled round all train round ``r`` at the same learning rate.

With base ``lr``, warmup ``W``, ``d = max(0, r - W)`` and ``D = T - W``::

    warm(r)  = (r + 1) / (W + 1) for r < W, else 1        torch LinearLR(start_factor=1/(W+1), total_iters=W)
    const    : 1
    step     : gamma ** (d // S)                           torch StepLR(step_size=S, gamma) after d steps
    cosine   : m + (1 - m) (1 + cos(pi d / D)) / 2         torch CosineAnnealingLR(T_max=D, eta_min=m lr) after d steps
    lr_r     = lr * warm(r) * decay(d)

computed in float64 and rounded to float32, the precision the update kernels read it in.
"""
from __future__ import annotations

import math

import numpy as np

from ..config import LR_SCHEDULES


def schedule_active(lr_schedule: str = "const", lr_warmup: int = 0) -> bool:
    """Whether the client learning rate changes between rounds (anything but a constant rate without warmup)."""
    return lr_schedule != "const" or lr_warmup > 0


def round_lr(lr: float, r: int, T: int, lr_schedule: str = "const", lr_warmup: int = 0, lr_gamma: float = 0.1,
             lr_step_rounds: int = 0, lr_min: float = 0.0) -> float:
    """The client learning rate of round ``r`` of ``T`` (module docstring), as the float32 value the kernels use."""
    if lr_schedule not in LR_SCHEDULES:
        raise ValueError("lr_schedule must be one of %s, got %r" % (", ".join(LR_SCHEDULES), lr_schedule))
    if not 0 <= lr_warmup < T:
        raise ValueError("lr_warmup must lie in [0, T) where T = %d is the run's number of rounds, got lr_warmup %r"
                         % (T, lr_warmup))
    if not 0 <= r < T:
        raise ValueError("round %r outside the run's %d rounds" % (r, T))
    W = lr_warmup
    warm = (r + 1) / (W + 1) if r < W else 1.0
    d, D = max(0, r - W), T - W
    if lr_schedule == "step":
        if lr_step_rounds < 1:
            raise ValueError("lr_schedule 'step' needs lr_step_rounds >= 1, got %r" % (lr_step_rounds,))
        decay = lr_gamma ** (d // lr_step_rounds)
    elif lr_schedule == "cosine":
        decay = lr_min + (1.0 - lr_min) * (1.0 + math.cos(math.pi * d / D)) / 2.0
    else:
        decay = 1.0
    return float(np.float32(lr * warm * decay))
