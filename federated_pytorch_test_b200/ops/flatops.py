"""Level-1 algebra on flat parameter vectors (SURVEY G14-G16, G20).

Every routine has the sm_90a implementation in ``csrc/flat_kernels.cu``
(reached through :mod:`.cuda_ops` for CUDA tensors) and the ATen composition
below, which is also the oracle the kernels are tested against.

The point of the CUDA versions is launch/sync count, not FLOPs: the reference
issues one ATen kernel + one ``.item()`` host sync per dot/axpy/norm
(lbfgsnew.py:590-659 — 15-25 syncs per ``step``); here one inner L-BFGS
iteration costs three kernel launches and one batched scalar read.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch


def _cuda(t: torch.Tensor) -> bool:
    if not t.is_cuda:
        return False
    from . import functional

    return functional.fast_path_enabled()


# ----------------------------------------------------------------------------
def l1_l2(g: torch.Tensor) -> Tuple[float, float]:
    """``(sum|g|, ||g||_2)`` with a single device->host read."""
    if _cuda(g):
        from . import cuda_ops

        return cuda_ops.l1_l2(g)
    return float(g.abs().sum()), float(g.norm())


def dir_stats(g: torch.Tensor, d: torch.Tensor) -> Tuple[float, float]:
    """``(g.d, sum|d|)`` of a search direction — ONE device->host read on CUDA (the reference does ``float(dot)`` and
    ``float(abs().sum())`` separately, lbfgsnew.py:679-681, :741; on CUDA the dot used to be a cuBLAS call)."""
    if _cuda(g):
        from . import cuda_ops

        gtd = cuda_ops.ext().multi_dot([g.contiguous()], [d.contiguous()])
        l1 = cuda_ops.ext().l1_l2(d)
        a, b, _ = torch.cat([gtd, l1]).tolist()
        return float(a), float(b)
    return float(torch.dot(g, d)), float(d.abs().sum())


def loss_and_l1(loss, g: torch.Tensor) -> Tuple[float, float]:
    """``(float(loss), sum|g|)`` with one device->host read when ``loss`` is a CUDA tensor."""
    if torch.is_tensor(loss) and loss.is_cuda and _cuda(g):
        from . import cuda_ops

        a, b, _ = torch.cat([loss.detach().reshape(1).float(), cuda_ops.ext().l1_l2(g)]).tolist()
        return float(a), float(b)
    lv = float(loss)
    return lv, l1_l2(g)[0]


def make_pair(g: torch.Tensor, g_prev: torch.Tensor, d: torch.Tensor, t: float, trust: float):
    """Curvature pair of one L-BFGS iteration.

    ``s = t*d``; ``y = g - g_prev + trust*s``; returns ``(y, s, y.s, ||s||, y.y)``
    (lbfgsnew.py:590-598, :630).  One pass over the four vectors on CUDA.
    """
    if _cuda(g):
        from . import cuda_ops

        return cuda_ops.make_pair(g, g_prev, d, t, trust)
    y = g.sub(g_prev)
    s = d.mul(t)
    if trust != 0.0:
        y.add_(s, alpha=trust)
    return y, s, float(y.dot(s)), float(s.norm()), float(y.dot(y))


def welford_update(g: torch.Tensor, mean: torch.Tensor, m2: torch.Tensor, n: int) -> float:
    """Online inter-batch mean / second-moment update (lbfgsnew.py:601-613).

    ``delta=g-mean; mean+=delta/n; m2+=(g-mean)*delta``; returns ``sum(m2)``.
    """
    if _cuda(g):
        from . import cuda_ops

        return cuda_ops.welford_update(g, mean, m2, n)
    delta = g - mean
    mean.add_(delta, alpha=1.0 / n)
    m2.addcmul_(g - mean, delta, value=1)
    return float(m2.sum())


class PairHistory:
    """FIFO of at most ``m`` curvature pairs stored as rows of two ``[m, n]`` buffers."""

    def __init__(self, m: int, like: torch.Tensor):
        self.m = int(m)
        self.n = like.numel()
        self.Y = torch.zeros(self.m, self.n, dtype=like.dtype, device=like.device)
        self.S = torch.zeros(self.m, self.n, dtype=like.dtype, device=like.device)
        self.order: List[int] = []          # row indices, oldest first
        self._free = list(range(self.m))
        self._ro: List[Optional[torch.Tensor]] = [None] * self.m
        self._al: List[Optional[torch.Tensor]] = [None] * self.m

    def __len__(self) -> int:
        return len(self.order)

    def push(self, y: torch.Tensor, s: torch.Tensor) -> None:
        if len(self.order) == self.m:
            row = self.order.pop(0)
        else:
            row = self._free.pop(0)
        self.Y[row].copy_(y)
        self.S[row].copy_(s)
        self.order.append(row)

    def dirs(self) -> List[torch.Tensor]:
        return [self.Y[r] for r in self.order]

    def steps(self) -> List[torch.Tensor]:
        return [self.S[r] for r in self.order]

    def ro_list(self):
        return list(self._ro)

    def al_list(self):
        return list(self._al)

    def two_loop(self, g: torch.Tensor, H_diag) -> torch.Tensor:
        """``d = -H g`` by the two-loop recursion (lbfgsnew.py:645-659)."""
        k = len(self.order)
        if _cuda(g) and k > 0:
            from . import cuda_ops

            return cuda_ops.lbfgs_two_loop(self.Y, self.S, self.order, g, float(H_diag))
        ys, ss = self.dirs(), self.steps()
        ro, al = self._ro, self._al
        for i in range(k):
            ro[i] = 1.0 / ys[i].dot(ss[i])
        q = g.neg()
        for i in range(k - 1, -1, -1):
            al[i] = ss[i].dot(q) * ro[i]
            q.add_(ys[i], alpha=-float(al[i]))
        r = q.mul_(H_diag) if not torch.is_tensor(H_diag) else q.mul_(float(H_diag))
        for i in range(k):
            be = ys[i].dot(r) * ro[i]
            r.add_(ss[i], alpha=float(al[i] - be))
        return r


# ----------------------------------------------------------------------------
# Fused Adam (+ closed-form penalty gradients) over a flat slice — SURVEY G14/G15
# ----------------------------------------------------------------------------
def adam_prox_step(
    x: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int,
    lr: float, beta1: float, beta2: float, eps: float,
    z: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None, rho: float = 0.0,
    lambda1: float = 0.0, lambda2: float = 0.0, rho_dev: Optional[torch.Tensor] = None,
) -> None:
    """One Adam update of ``x`` with the penalty gradients added in closed form:

    ``g_total = g + y + rho*(x - z) + lambda1*sign(x) + 2*lambda2*x``

    (the reference builds these terms through autograd on a ``torch.cat`` of the
    block inside every closure, consensus_multi.py:214-220).  Adam follows
    ``torch.optim.Adam`` defaults semantics (no amsgrad, no weight decay).
    """
    if _cuda(x):
        from . import cuda_ops

        cuda_ops.adam_prox_step(x, g, m, v, step, lr, beta1, beta2, eps, z, y, rho, lambda1, lambda2, rho_dev)
        return
    if rho_dev is not None:
        rho = float(rho_dev)
    gt = penalty_grad(x, g, z, y, rho, lambda1, lambda2)
    m.mul_(beta1).add_(gt, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(gt, gt, value=1 - beta2)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = (v.sqrt() / (bc2 ** 0.5)).add_(eps)
    x.addcdiv_(m, denom, value=-lr / bc1)


def penalty_grad(x, g, z=None, y=None, rho: float = 0.0, lambda1: float = 0.0, lambda2: float = 0.0) -> torch.Tensor:
    gt = g.clone()
    if z is not None and rho != 0.0:
        gt.add_(x - z, alpha=rho)
    if y is not None:
        gt.add_(y)
    if lambda1 != 0.0:
        gt.add_(torch.sign(x), alpha=lambda1)
    if lambda2 != 0.0:
        gt.add_(x, alpha=2.0 * lambda2)
    return gt


def add_penalty_grad_(g, x, z=None, y=None, rho: float = 0.0, lambda1: float = 0.0, lambda2: float = 0.0) -> None:
    """In place ``g += y + rho (x - z) + lambda1 sign(x) + 2 lambda2 x`` (one kernel on CUDA)."""
    if _cuda(g):
        from . import cuda_ops

        cuda_ops.penalty_grad_(g, x, z, y, rho, lambda1, lambda2)
        return
    g.copy_(penalty_grad(x, g, z, y, rho, lambda1, lambda2))


def penalty_value(x, z=None, y=None, rho: float = 0.0, lambda1: float = 0.0, lambda2: float = 0.0) -> torch.Tensor:
    """``y.(x-z) + rho/2 ||x-z||^2 + lambda1 ||x||_1 + lambda2 ||x||_2^2`` as a 0-dim tensor."""
    if _cuda(x):
        from . import cuda_ops

        return cuda_ops.penalty_value(x, z, y, rho, lambda1, lambda2)
    val = x.new_zeros(())
    if z is not None:
        dx = x - z
        if y is not None:
            val = val + torch.dot(y, dx)
        if rho != 0.0:
            val = val + 0.5 * rho * torch.dot(dx, dx)
    if lambda1 != 0.0:
        val = val + lambda1 * x.abs().sum()
    if lambda2 != 0.0:
        val = val + lambda2 * torch.dot(x, x)
    return val


def multi_dot(pairs) -> torch.Tensor:
    """Several dot products of equal-length vectors in one pass -> 1-D tensor (SURVEY G20)."""
    if pairs and _cuda(pairs[0][0]):
        from . import cuda_ops

        return cuda_ops.multi_dot(pairs)
    return torch.stack([torch.dot(a, b) for a, b in pairs])
