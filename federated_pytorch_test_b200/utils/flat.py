"""Flat parameter arena: every parameter of a replica is a *view* into one
contiguous fp32 buffer, and every gradient a view into a twin buffer.

Why (SURVEY G13, §7.3(3)): the reference packs the trainable block into a fresh
vector (``get_trainable_values``), ``torch.cat``s it again inside every closure
call for FedProx/ADMM, and scatters the average back tensor by tensor
(/root/reference/src/simple_utils.py:47-77, consensus_multi.py:214-215).  All
block tables are inclusive *index ranges* in registration order, so with this
layout a block IS a contiguous slice: aggregation kernels read/write parameter
storage directly, the fused optimizers walk one pointer range, L-BFGS' flat
gradient is free, and the same buffer can be allocated from NVLink-registered
symmetric memory so peers reduce straight out of each other's weights.

Layout: parameters in ``net.parameters()`` order, each start aligned to
``align`` floats (default 32 = 128 B, which satisfies TMA's 16 B global-address
rule and vectorised/multimem accesses).  Alignment gaps hold zeros forever
(they belong to no parameter, their gradient slots stay zero) so reductions,
norms and dot products over a padded slice equal those over the compact vector.
"""
from __future__ import annotations

from typing import Callable, Iterable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

Allocator = Callable[[int, torch.device], torch.Tensor]


def _default_alloc(numel: int, device: torch.device) -> torch.Tensor:
    return torch.zeros(numel, dtype=torch.float32, device=device)


class FlatArena:
    def __init__(
        self,
        module: nn.Module,
        device: Optional[torch.device] = None,
        allocator: Optional[Allocator] = None,
        grad_allocator: Optional[Allocator] = None,
        align: int = 32,
        channels_last_weights: bool = False,
    ):
        params = list(module.parameters())
        if not params:
            raise ValueError("module has no parameters")
        if any(p.dtype != torch.float32 for p in params):
            raise TypeError("FlatArena stores fp32 master parameters only")
        device = torch.device(device) if device is not None else params[0].device
        self.module = module
        self.device = device
        self.align = int(align)
        self.channels_last_weights = bool(channels_last_weights)
        self.params: List[nn.Parameter] = params
        self.numels = [p.numel() for p in params]
        self.offsets: List[int] = []
        off = 0
        for n in self.numels:
            self.offsets.append(off)
            off += -(-n // self.align) * self.align
        self.total = off
        self.total_params = sum(self.numels)

        self.data = (allocator or _default_alloc)(self.total, device)
        self.grad = (grad_allocator or _default_alloc)(self.total, device)
        if self.data.numel() < self.total or self.grad.numel() < self.total:
            raise ValueError("allocator returned a buffer that is too small")
        self.data = self.data[: self.total]
        self.grad = self.grad[: self.total]
        with torch.no_grad():
            self.data.zero_()
            self.grad.zero_()
            for i, p in enumerate(params):
                v = self._view(self.data, i, p)
                v.copy_(p.detach().to(device))
                p.data = v
                p.grad = None
                p._arena_owner = self
        self._grad_views: List[Optional[torch.Tensor]] = [None] * len(params)
        module._flat_arena = self  # discoverable from simple_utils / optimizers

    # ------------------------------------------------------------------
    def _view(self, buf: torch.Tensor, i: int, p: torch.Tensor) -> torch.Tensor:
        flat = buf[self.offsets[i]: self.offsets[i] + self.numels[i]]
        if self.channels_last_weights and p.dim() == 4:
            o, c, h, w = p.shape
            return flat.view(o, h, w, c).permute(0, 3, 1, 2)
        return flat.view(p.shape)

    def grad_view(self, i: int) -> torch.Tensor:
        g = self._grad_views[i]
        if g is None:
            g = self._view(self.grad, i, self.params[i])
            self._grad_views[i] = g
        return g

    # ------------------------------------------------------------------
    def span(self, lo: int, hi: int) -> Tuple[int, int]:
        """Float offsets ``[start, stop)`` of parameters ``lo..hi`` inclusive."""
        if not (0 <= lo <= hi < len(self.params)):
            raise IndexError("bad parameter range [%d,%d]" % (lo, hi))
        return self.offsets[lo], self.offsets[hi] + self.numels[hi]

    def count(self, lo: int, hi: int) -> int:
        """Number of real parameters in ``lo..hi`` (the reference's ``N``)."""
        return sum(self.numels[lo: hi + 1])

    def block(self, lo: int, hi: int) -> torch.Tensor:
        a, b = self.span(lo, hi)
        return self.data[a:b]

    def chunk_counts(self, lo: int, hi: int, chunk: int = 32) -> List[int]:
        """Per ``chunk``-float chunk of :meth:`block` ``(lo, hi)``, how many of its leading floats are parameters (the
        rest is alignment padding).  Needs ``align`` to be a multiple of ``chunk``, so no chunk spans two parameters."""
        if self.align % chunk:
            raise ValueError("chunk_counts needs align (%d) to be a multiple of %d" % (self.align, chunk))
        a, b = self.span(lo, hi)
        counts = [0] * (-(-(b - a) // chunk))
        for i in range(lo, hi + 1):
            rel = self.offsets[i] - a
            for c in range(rel // chunk, -(-(rel + self.numels[i]) // chunk)):
                counts[c] = min(chunk, rel + self.numels[i] - c * chunk)
        return counts

    def block_grad(self, lo: int, hi: int) -> torch.Tensor:
        a, b = self.span(lo, hi)
        return self.grad[a:b]

    def trainable_range(self) -> Optional[Tuple[int, int]]:
        """``(lo, hi)`` if the trainable parameters form one contiguous index range."""
        idx = [i for i, p in enumerate(self.params) if p.requires_grad]
        if not idx:
            return None
        lo, hi = idx[0], idx[-1]
        return (lo, hi) if len(idx) == hi - lo + 1 else None

    def attach_grads(self) -> None:
        """Point ``.grad`` of trainable parameters at the gradient arena (frozen → None)."""
        for i, p in enumerate(self.params):
            p.grad = self.grad_view(i) if p.requires_grad else None

    def zero_grads(self, lo: Optional[int] = None, hi: Optional[int] = None) -> None:
        if lo is None:
            self.grad.zero_()
        else:
            a, b = self.span(lo, hi)
            self.grad[a:b].zero_()

    # ------------------------------------------------------------------
    def compact(self, lo: int, hi: int, out: Optional[torch.Tensor] = None, src: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Gap-free copy of a block (length ``count(lo,hi)``), reference ordering."""
        src = self.data if src is None else src
        n = self.count(lo, hi)
        if out is None:
            out = torch.empty(n, dtype=torch.float32, device=src.device)
        pos = 0
        for i in range(lo, hi + 1):
            k = self.numels[i]
            seg = src[self.offsets[i]: self.offsets[i] + k]
            if self.channels_last_weights and self.params[i].dim() == 4:
                o, c, h, w = self.params[i].shape
                seg = seg.view(o, h, w, c).permute(0, 3, 1, 2).reshape(-1)
            out[pos: pos + k].copy_(seg)
            pos += k
        return out

    def scatter(self, lo: int, hi: int, vec: torch.Tensor) -> None:
        """Inverse of :meth:`compact` into the parameter arena."""
        pos = 0
        with torch.no_grad():
            for i in range(lo, hi + 1):
                k = self.numels[i]
                self.params[i].data.copy_(vec[pos: pos + k].view(self.params[i].shape))
                pos += k

    def check_views(self) -> bool:
        """True iff every parameter still aliases the arena (``.to()``/``.data=`` can break this)."""
        base = self.data.untyped_storage().data_ptr()
        return all(p.data.untyped_storage().data_ptr() == base for p in self.params)


def arena_of(module: nn.Module) -> Optional[FlatArena]:
    arena = getattr(module, "_flat_arena", None)
    if arena is not None and not arena.check_views():
        return None
    return arena


def flatten_module(module: nn.Module, **kw) -> FlatArena:
    """Create (or return the existing) arena of ``module``."""
    arena = arena_of(module)
    return arena if arena is not None else FlatArena(module, **kw)
