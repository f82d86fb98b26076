"""Loopback world: W *virtual ranks* of the fused collectives inside ONE process on ONE GPU.

Purpose (SURVEY §4 "distributed without a cluster"): the cross-rank code of ``csrc/comm_kernels.cu`` — per-CTA flag
barriers in peer pads, two-shot slice ownership + broadcast stores, payload exchange of the residual scalars, the
Barzilai-Borwein row gather — can only be exercised with more than one rank.  Here every virtual rank owns its own
arenas, control pad, epoch counter and CUDA stream; "peer pointers" are simply the other ranks' device pointers (valid
in-process), so the kernels run their P2P path unchanged (no multicast object on one device).  The W kernels of one
aggregation are launched on W streams and meet at their barriers while co-resident: their grids are capped
(``max_blocks``) so that all of them fit on the chip at once, and the barrier timeout is short, so a scheduling
accident surfaces as ``CollectiveTimeout`` instead of a hang.

Used by ``tests/test_gpu_loopback.py``, which runs the fused collectives on a single GPU.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch

from .fused import FusedCollective
from .topology import Topology


class _SharedRegistry:
    def __init__(self, world: int, device: torch.device):
        self.world, self.device = world, device
        self.groups: List[Dict] = []          # allocation i: {tensors[W], ptrs[W], nbytes}
        self.cursor = [0] * world

    def alloc(self, rank: int, numel: int, dtype) -> torch.Tensor:
        i = self.cursor[rank]
        self.cursor[rank] += 1
        if i == len(self.groups):
            ts = [torch.zeros(numel, dtype=dtype, device=self.device) for _ in range(self.world)]
            self.groups.append(dict(tensors=ts, ptrs=[t.data_ptr() for t in ts], nbytes=numel * ts[0].element_size()))
        g = self.groups[i]
        if g["nbytes"] != numel * g["tensors"][0].element_size():
            raise RuntimeError("loopback ranks must allocate in the same order with the same sizes")
        return g["tensors"][rank]


class LoopbackHeap:
    """Heap view of virtual rank ``rank``: same interface as :class:`..parallel.fused.SymmetricHeap`."""

    transport = "loopback"

    def __init__(self, shared: _SharedRegistry, rank: int):
        self.shared, self.rank = shared, rank

    def alloc(self, numel: int, dtype=torch.float32) -> torch.Tensor:
        return self.shared.alloc(self.rank, numel, dtype)

    def locate(self, t: torch.Tensor) -> Tuple[Dict, int]:
        p = t.data_ptr()
        for g in self.shared.groups:
            base = g["ptrs"][self.rank]
            if base <= p < base + g["nbytes"]:
                return dict(base=base, nbytes=g["nbytes"], peer_ptrs=g["ptrs"], mc_ptr=0), p - base
        raise KeyError("tensor does not live in the loopback heap")

    def contains(self, t: torch.Tensor) -> bool:
        try:
            self.locate(t)
            return True
        except KeyError:
            return False


class LoopbackWorld:
    def __init__(self, world: int, device=None, max_blocks: int = 16, timeout_s: float = 5.0, K: int = 0):
        device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.world, self.device = world, device
        self.shared = _SharedRegistry(world, device)
        self.colls: List[FusedCollective] = []
        self.streams = [torch.cuda.Stream(device=device) for _ in range(world)]
        for r in range(world):
            topo = Topology(K=K or world, world_size=world, rank=r, device=device)
            self.colls.append(FusedCollective(topo, heap=LoopbackHeap(self.shared, r), max_blocks=max_blocks, timeout_s=timeout_s))

    def alloc(self, numel: int) -> List[torch.Tensor]:
        """One symmetric allocation: the W per-rank tensors."""
        return [c.heap.alloc(numel) for c in self.colls]

    def run(self, fn) -> List:
        """``fn(rank, coll)`` launches rank's part of a collective (no host reads!) on that rank's stream; returns after
        all ranks' kernels have finished."""
        cur = torch.cuda.current_stream(self.device)
        out = []
        for r, (c, st) in enumerate(zip(self.colls, self.streams)):
            st.wait_stream(cur)
            with torch.cuda.stream(st):
                out.append(fn(r, c))
        for st in self.streams:
            cur.wait_stream(st)
        torch.cuda.synchronize(self.device)
        return out
