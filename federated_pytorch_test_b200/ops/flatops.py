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
    """The kernels take float32 CUDA tensors; every other tensor (float64 on a GPU included) takes the ATen path."""
    if not t.is_cuda or t.dtype != torch.float32:
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
        """``d = -H g`` by the two-loop recursion (lbfgsnew.py:645-659).  One cooperative kernel on CUDA for up to
        ``cuda_ops.TWO_LOOP_MAX_HIST`` pairs; longer histories run the ATen recursion below."""
        k = len(self.order)
        if _cuda(g) and k > 0:
            from . import cuda_ops

            if k <= cuda_ops.TWO_LOOP_MAX_HIST:
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
def clip_workspace(x: torch.Tensor) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """``(ws, ticket)`` for gradient-norm clipping of a block like ``x``: ``ws = [norm, sum of norms, clipped steps, steps,
    per-CTA partials of the CUDA norm kernel]`` and one int32 ticket (``None`` on the ATen path).  ``ws[1:4]`` accumulates over
    the steps until the caller zeroes it."""
    if _cuda(x):
        from . import cuda_ops

        n = cuda_ops.GRAD_NORM_HEADER + cuda_ops.grad_norm_blocks(x.numel())
        return (torch.zeros(n, dtype=torch.float32, device=x.device),
                torch.zeros(1, dtype=torch.int32, device=x.device))
    return torch.zeros(4, dtype=torch.float32, device=x.device), None


def grad_norm_(g: torch.Tensor, ws: torch.Tensor, ticket: Optional[torch.Tensor], clip_norm: float) -> torch.Tensor:
    """``ws[0] = ||g||_2`` and ``ws[1:4] += [norm, norm > clip_norm, 1]``; returns ``ws[0:1]``.  The ATen norm is summed
    in float64, so on the CPU it does not depend on how many threads reduce it."""
    if _cuda(g):
        from . import cuda_ops

        cuda_ops.grad_norm(g, ws, ticket, clip_norm)
        return ws[0:1]
    norm = g.double().square().sum().sqrt().float()
    ws[0] = norm
    ws[1:4] += torch.stack([norm, (norm > clip_norm).float(), torch.ones((), dtype=torch.float32, device=g.device)])
    return ws[0:1]


def _clip_scale(norm: torch.Tensor, clip_norm: float) -> torch.Tensor:
    """``torch.nn.utils.clip_grad_norm_``'s factor ``min(1, c / (norm + 1e-6))``; a NaN norm gives a NaN factor."""
    return (clip_norm / (norm + 1e-6)).clamp(max=1.0)


def _lr_value(lr) -> float:
    return float(lr) if torch.is_tensor(lr) else lr


def _clipped_grad(x, g, clip_norm: float, clip_ws):
    """``(g, norm_dev)``: on the CPU the clipped gradient itself, on CUDA the unclipped one and the device norm the update
    kernel scales it by."""
    if clip_norm <= 0.0:
        return g, None
    ws, ticket = clip_ws if clip_ws is not None else clip_workspace(x)
    norm = grad_norm_(g, ws, ticket, clip_norm)
    if _cuda(x):
        return g, norm
    return g * _clip_scale(norm, clip_norm), None


def adam_prox_step(
    x: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int,
    lr, beta1: float, beta2: float, eps: float,
    z: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None, rho: float = 0.0,
    lambda1: float = 0.0, lambda2: float = 0.0, rho_dev: Optional[torch.Tensor] = None,
    weight_decay: float = 0.0, clip_norm: float = 0.0, clip_ws=None,
) -> None:
    """One Adam update of ``x`` with the penalty gradients added in closed form:

    ``g_total = g + y + rho*(x - z) + lambda1*sign(x) + 2*lambda2*x``

    (the reference builds these terms through autograd on a ``torch.cat`` of the
    block inside every closure, consensus_multi.py:214-220).  Adam follows
    ``torch.optim.Adam`` defaults semantics (no amsgrad, no weight decay).

    ``lr`` is a float or a 1-element tensor (read on the device by the CUDA kernel, so a schedule can change it between
    graph replays).  ``weight_decay`` makes it ``torch.optim.AdamW``: ``x *= 1 - lr*weight_decay`` before the moment
    update.  ``clip_norm > 0`` first scales ``g`` (the data-loss gradient only, not the penalty gradient) as
    ``torch.nn.utils.clip_grad_norm_(block, clip_norm)`` does; ``clip_ws`` is the :func:`clip_workspace` whose
    accumulator counts the step.
    """
    if _cuda(x):
        from . import cuda_ops

        g, norm_dev = _clipped_grad(x, g, clip_norm, clip_ws)
        lr_dev = lr if torch.is_tensor(lr) else None
        cuda_ops.adam_prox_step(x, g, m, v, step, 0.0 if lr_dev is not None else lr, beta1, beta2, eps, z, y, rho, lambda1,
                                lambda2, rho_dev, lr_dev=lr_dev, weight_decay=weight_decay, norm_dev=norm_dev,
                                clip_norm=clip_norm)
        return
    if rho_dev is not None:
        rho = float(rho_dev)
    lr = _lr_value(lr)
    g, _ = _clipped_grad(x, g, clip_norm, clip_ws)
    gt = penalty_grad(x, g, z, y, rho, lambda1, lambda2)
    if weight_decay != 0.0:
        x.mul_(1 - lr * weight_decay)
    m.mul_(beta1).add_(gt, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(gt, gt, value=1 - beta2)
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = (v.sqrt() / (bc2 ** 0.5)).add_(eps)
    x.addcdiv_(m, denom, value=-lr / bc1)


def sgd_prox_step(
    x: torch.Tensor, g: torch.Tensor, buf: Optional[torch.Tensor], lr, momentum: float = 0.0,
    nesterov: bool = False, weight_decay: float = 0.0,
    z: Optional[torch.Tensor] = None, y: Optional[torch.Tensor] = None, rho: float = 0.0,
    lambda1: float = 0.0, lambda2: float = 0.0, rho_dev: Optional[torch.Tensor] = None,
    clip_norm: float = 0.0, clip_ws=None,
) -> None:
    """One ``torch.optim.SGD`` update (dampening 0) of ``x`` with the penalty gradients of :func:`adam_prox_step`:

    ``gt = penalty_grad(...) + weight_decay*x``; ``buf = momentum*buf + gt``;
    ``x -= lr * (gt + momentum*buf if nesterov else buf)``.

    ``buf`` starts at zero (which gives torch's first step, ``buf = gt``) and is ``None`` exactly when ``momentum == 0``.
    ``lr``, ``clip_norm`` and ``clip_ws`` as for :func:`adam_prox_step`.
    """
    if (buf is None) != (momentum == 0.0):
        raise ValueError("sgd_prox_step: pass a momentum buffer exactly when momentum != 0, got momentum %r" % (momentum,))
    if _cuda(x):
        from . import cuda_ops

        g, norm_dev = _clipped_grad(x, g, clip_norm, clip_ws)
        lr_dev = lr if torch.is_tensor(lr) else None
        cuda_ops.sgd_prox_step(x, g, buf, 0.0 if lr_dev is not None else lr, momentum, nesterov, weight_decay, z, y, rho,
                               lambda1, lambda2, rho_dev, lr_dev=lr_dev, norm_dev=norm_dev, clip_norm=clip_norm)
        return
    if rho_dev is not None:
        rho = float(rho_dev)
    lr = _lr_value(lr)
    g, _ = _clipped_grad(x, g, clip_norm, clip_ws)
    gt = penalty_grad(x, g, z, y, rho, lambda1, lambda2)
    if weight_decay != 0.0:
        gt.add_(x, alpha=weight_decay)
    if buf is not None:
        buf.mul_(momentum).add_(gt)
        d = gt.add_(buf, alpha=momentum) if nesterov else buf
    else:
        d = gt
    x.add_(d, alpha=-lr)


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


# ----------------------------------------------------------------------------
# SCAFFOLD control variates (algo/scaffold.py), all local replicas per call
# ----------------------------------------------------------------------------
def scaffold_workspace(n: int, n_local: int, device) -> Tuple[torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor]]:
    """``(norm_sq, ws, tickets)`` of :func:`scaffold_corr_`: one squared norm per replica, and on CUDA the per-CTA partials
    and the replicas' tickets (``None`` on the ATen path)."""
    norm_sq = torch.zeros(n_local, dtype=torch.float32, device=device)
    if torch.device(device).type == "cuda" and _cuda(norm_sq):
        from . import cuda_ops

        return (norm_sq, torch.zeros(n_local * cuda_ops.scaffold_corr_blocks(n), dtype=torch.float32, device=device),
                torch.zeros(n_local, dtype=torch.int32, device=device))
    return norm_sq, None, None


def scaffold_cv_(cs: List[torch.Tensor], xs: List[torch.Tensor], c: torch.Tensor, z: torch.Tensor,
                 scales: List[float]) -> None:
    """SCAFFOLD step 1, in place: ``c_j <- (c_j - c) + s_j (z - x_j)`` for every ``j`` with ``s_j != 0``; the others are
    not written.  Each operation is rounded to float32, so the CUDA kernel gives the same bits."""
    if _cuda(c):
        from . import cuda_ops

        cuda_ops.scaffold_cv(cs, xs, c, z, scales)
        return
    for ci, x, s in zip(cs, xs, scales):
        if s != 0.0:
            ci.copy_((ci - c) + torch.tensor(s, dtype=torch.float32) * (z - x))


def scaffold_corr_(cs: List[torch.Tensor], ds: List[torch.Tensor], c: torch.Tensor, work) -> torch.Tensor:
    """SCAFFOLD step 3, in place: ``d_j <- c - c_j`` for every ``j``; returns ``norm_sq`` of ``work``
    (:func:`scaffold_workspace`) holding ``||d_j||^2`` (summed in float64 on the ATen path)."""
    norm_sq, ws, tickets = work
    if _cuda(c):
        from . import cuda_ops

        cuda_ops.scaffold_corr(cs, ds, c, norm_sq, ws, tickets)
        return norm_sq
    for j, (ci, d) in enumerate(zip(cs, ds)):
        torch.sub(c, ci, out=d)
        norm_sq[j] = d.double().square().sum().float()
    return norm_sq


def multi_dot(pairs) -> torch.Tensor:
    """Several dot products of equal-length vectors in one pass -> 1-D tensor (SURVEY G20)."""
    if pairs and _cuda(pairs[0][0]):
        from . import cuda_ops

        return cuda_ops.multi_dot(pairs)
    return torch.stack([torch.dot(a, b) for a, b in pairs])
