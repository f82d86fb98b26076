"""``FusedCollective`` — the block collectives as ONE sm_90a kernel each, reducing
straight out of peer memory over NVLink (``csrc/comm_kernels.cu``).  No NCCL on this path.

Reference loops being replaced (Python loops over a dict of K modules): FedAvg mean + write-back + dual residual
``src/federated_multi.py:204-214``, FedProx mean + primal/dual residuals ``src/fedprox_multi.py:205-234``, ADMM z/y
updates + residuals ``src/consensus_multi.py:226-299``, Barzilai-Borwein penalty update ``:242-278``.

Memory model (SURVEY §5.8, §7.3(3)): every replica's flat parameter arena (and same-shaped arenas for the
consensus vector ``z`` and the ADMM duals ``y``) is allocated from a :class:`SymmetricHeap`:

* ``world == 1``  — ordinary device memory (all K replicas are co-resident; the kernel
  just gets K local pointers — the reference's topology, but one launch instead of
  K+2 ATen kernels and K·#tensors copies);
* ``world > 1``   — ``torch.distributed._symmetric_memory`` (CUDA VMM allocations
  mapped into every process, bound to an NVSwitch multicast object when the fabric
  supports it); if that is unavailable, plain allocations exported with CUDA IPC.
  ``torch.distributed`` is used for the handle exchange only.

A block is a slice at the same offset of every arena, so the kernel needs nothing but
K base pointers + one offset.  Cross-rank synchronisation is a per-CTA flag barrier in a
peer-mapped control pad (release/acquire at system scope, epoch counted in device
memory); the penalty ``rho`` of adaptive ADMM, the epoch and all accumulators live in device
memory, so an aggregation round is host-free and CUDA-graph capturable: one cooperative launch
(+ one more for the Barzilai-Borwein update).  The host reads ONE 32-byte record per round.

Small blocks are reduced ONE-SHOT (every rank pulls the whole vector: ``multimem.ld_reduce`` in the
switch, or K P2P loads); blocks of 256 KB and more TWO-SHOT: rank r reduces slice r and broadcasts
it with ``multimem.st`` (or P2P stores) into every rank's weights / consensus vector.
"""
from __future__ import annotations

import os
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from ..ops import cuda_ops
from .collective import TorchCollective
from .topology import Topology

_MAX_LOCAL = 16
_OUT_FLOATS = 8
_SCRATCH_FLOATS = 4 + _MAX_LOCAL
_BB_SCRATCH_FLOATS = 8 * _MAX_LOCAL + 8 + _MAX_LOCAL
_PAD_WORDS = 8192
OUT_DUAL_SQ, OUT_PRIMAL, OUT_NONFINITE, OUT_STATUS, OUT_RHO, OUT_EPOCH, OUT_TWO_SHOT = range(7)

TWO_SHOT_MIN_BYTES = int(os.environ.get("FEDB200_TWO_SHOT_BYTES", str(256 * 1024)))
TWO_SHOT_MODE = os.environ.get("FEDB200_TWO_SHOT", "auto")          # 'auto' | '0' (never) | '1' (whenever legal)
BARRIER_TIMEOUT_S = float(os.environ.get("FEDB200_BARRIER_TIMEOUT_S", "120"))


class CollectiveTimeout(RuntimeError):
    """A rank did not reach a cross-rank barrier of the aggregation kernel in time (SURVEY §5.3)."""


class SymmetricHeap:
    """Allocates fp32/int32 buffers addressable by every rank; remembers peer base pointers."""

    def __init__(self, topo: Topology):
        self.topo = topo
        self.allocs: List[Dict] = []     # {tensor, base, nbytes, peer_ptrs[world], mc_ptr}
        self.transport = "local"
        self._symm = None
        if topo.is_distributed:
            try:
                import torch.distributed._symmetric_memory as symm_mem

                self._symm = symm_mem
                self.transport = "symm_mem"
            except Exception:  # pragma: no cover
                self.transport = "ipc"

    # -- allocation ---------------------------------------------------------
    def alloc(self, numel: int, dtype=torch.float32) -> torch.Tensor:
        dev = self.topo.device
        if not self.topo.is_distributed:
            t = torch.zeros(numel, dtype=dtype, device=dev)
            self._record(t, [t.data_ptr()], 0)
            return t
        if self.transport == "symm_mem":
            try:
                t = self._symm.empty(numel, dtype=dtype, device=dev)
                hdl = self._symm.rendezvous(t, group=dist.group.WORLD)
                t.zero_()
                ptrs = [int(p) for p in hdl.buffer_ptrs]
                mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
                self._record(t, ptrs, mc, handle=hdl)
                return t
            except Exception as exc:  # fall back once, loudly
                if self.allocs:
                    raise
                print("[fedb200] torch symmetric memory unavailable (%s); using CUDA IPC" % (exc,), flush=True)
                self.transport = "ipc"
        return self._alloc_ipc(numel, dtype)

    def _alloc_ipc(self, numel: int, dtype) -> torch.Tensor:
        e = cuda_ops.ext()
        t = torch.zeros(numel, dtype=dtype, device=self.topo.device)
        torch.cuda.synchronize()
        share = t.untyped_storage()._share_cuda_()
        handle, offset = share[1], share[3]
        gathered: List = [None] * self.topo.world_size
        dist.all_gather_object(gathered, (bytes(handle), int(offset)))
        ptrs = []
        for r, (h, off) in enumerate(gathered):
            if r == self.topo.rank:
                ptrs.append(t.data_ptr())
            else:
                ptrs.append(int(e.ipc_open_handle(h)) + off)
        self._record(t, ptrs, 0, keep=share)
        return t

    def _record(self, t: torch.Tensor, ptrs: List[int], mc: int, **keep) -> None:
        self.allocs.append(dict(tensor=t, base=t.data_ptr(), nbytes=t.numel() * t.element_size(), peer_ptrs=ptrs, mc_ptr=mc, **keep))

    # -- lookup -----------------------------------------------------------------
    def locate(self, t: torch.Tensor) -> Tuple[Dict, int]:
        p = t.data_ptr()
        for a in self.allocs:
            if a["base"] <= p < a["base"] + a["nbytes"]:
                return a, p - a["base"]
        raise KeyError("tensor does not live in the symmetric heap")

    def contains(self, t: torch.Tensor) -> bool:
        try:
            self.locate(t)
            return True
        except KeyError:
            return False


class FusedCollective(TorchCollective):
    name = "fused"
    fused = True

    def __init__(self, topo: Topology, heap=None, max_blocks: int = 0, timeout_s: Optional[float] = None):
        super().__init__(topo)
        if topo.device.type != "cuda":
            raise RuntimeError("FusedCollective needs a CUDA device")
        if topo.is_distributed and topo.K % topo.world_size != 0:
            raise RuntimeError("fused collectives need K to be a multiple of the number of ranks")
        self.ext = cuda_ops.ext()
        self.heap = heap if heap is not None else SymmetricHeap(topo)
        dev = topo.device
        self.out = torch.zeros(_OUT_FLOATS, dtype=torch.float32, device=dev)
        self.scratch = torch.zeros(_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
        self.bb_scratch = torch.zeros(_BB_SCRATCH_FLOATS, dtype=torch.float32, device=dev)
        self.bb_log = torch.zeros(8 * max(topo.K, 1), dtype=torch.float32, device=dev)
        self.sync = torch.zeros(4, dtype=torch.int32, device=dev)
        self._host_out = torch.zeros(self.out.numel(), dtype=torch.float32).pin_memory()
        self._out_event = torch.cuda.Event()
        self._out_pending = False
        self.ctrl = self.heap.alloc(_PAD_WORDS, dtype=torch.int32)
        self.ctrl_ptrs = list(self.heap.locate(self.ctrl)[0]["peer_ptrs"])
        self._aux: Dict[Tuple[int, str], torch.Tensor] = {}
        # in-switch reduction pays from 4 peers on; between 2 GPUs there is nothing to reduce in the switch and the P2P variant of
        # the same kernel is used.  FEDB200_MULTIMEM=0|1 forces either.
        mm = os.environ.get("FEDB200_MULTIMEM", "auto")
        self.default_multimem = (topo.world_size > 2) if mm == "auto" else (mm != "0")
        self.use_multimem = self.default_multimem
        self.two_shot_mode = TWO_SHOT_MODE
        self.max_blocks = int(max_blocks)
        self.timeout_s = BARRIER_TIMEOUT_S if timeout_s is None else float(timeout_s)
        self.last_nonfinite = 0.0
        self.last_two_shot = False
        self.last_rho = float("nan")

    def warmup(self) -> None:
        """One tiny aggregation of every kind on scratch buffers: CUDA module loading, occupancy queries and the first
        cross-rank handshake happen here, at engine construction, not inside the first training round (the first launch
        is far slower than the ones after it).  Collective: every rank calls it at the same point."""
        if getattr(self, "_warm", False):
            return
        self._warm = True
        n = 256
        xs = [self.heap.alloc(n) for _ in range(len(self.topo.local_workers))]
        ys = [self.zeros_like_block(x, "y") for x in xs]
        z = self.zeros_like_block(xs[0], "z")
        rho = torch.full((1,), 0.5, dtype=torch.float32, device=self.topo.device)
        keep = self.two_shot_mode
        for mode_2shot in ("0", "1"):
            self.two_shot_mode = mode_2shot
            self._launch(0, xs, None, z, 0.0)
            self._launch(1, xs, None, z, 0.5)
            self._launch(2, xs, ys, z, 0.5, rho)
        self.two_shot_mode = keep
        x0 = [torch.zeros_like(x) for x in xs]
        yh = [torch.zeros_like(x) for x in xs]
        self.bb_seed_(xs, x0)
        self._bb_launch(xs, ys, yh, x0, z, rho, None, False)
        self.read_record()

    # -- arena hooks ------------------------------------------------------------
    def arena_allocator(self) -> Callable:
        def alloc(numel: int, device) -> torch.Tensor:
            return self.heap.alloc(numel)
        return alloc

    def register_arena(self, arena) -> None:
        self.heap.locate(arena.data)  # raises if the arena was not allocated from the heap

    def zeros_like_block(self, x: torch.Tensor, tag: str) -> torch.Tensor:
        """A zeroed buffer that mirrors block slice ``x`` (same offset in a same-sized symmetric arena)."""
        a, off = self.heap.locate(x)
        key = (a["base"], tag)
        buf = self._aux.get(key)
        if buf is None:
            buf = self.heap.alloc(a["nbytes"] // 4)
            self._aux[key] = buf
        sl = buf[off // 4: off // 4 + x.numel()]
        sl.zero_()
        return sl

    # -- pointer tables -------------------------------------------------------------
    def _tables(self, slices: List[torch.Tensor]):
        """Pointers of ALL K workers' slices (worker ck = rank + j*world for local replica j), local indices, multicast."""
        W, rank, K = self.topo.world_size, self.topo.rank, self.topo.K
        ptrs = [0] * K
        mc = 0
        for j, t in enumerate(slices):
            a, off = self.heap.locate(t)
            for r in range(W):
                ptrs[r + j * W] = a["peer_ptrs"][r] + off
            if len(slices) == 1 and a["mc_ptr"] and self.use_multimem and W > 1:
                mc = a["mc_ptr"] + off
        local_idx = [rank + j * W for j in range(len(slices))]
        return ptrs, local_idx, mc

    def _want_two_shot(self, mode: int, xs, z: torch.Tensor, n: int) -> bool:
        W = self.topo.world_size
        if W <= 1 or len(xs) != 1 or self.topo.K != W or self.two_shot_mode == "0":
            return False
        if mode != 0 and not self.heap.contains(z):
            return False
        return self.two_shot_mode == "1" or n * 4 >= TWO_SHOT_MIN_BYTES

    def _launch(self, mode: int, xs, ys, z, rho: float, rho_dev=None) -> None:
        n = xs[0].numel()
        if any(t.numel() != n for t in xs) or z.numel() != n:
            raise ValueError("block slices must have equal length")
        W = self.topo.world_size
        xp, local_idx, mcx = self._tables(xs)
        yp, mcy = [], 0
        if ys is not None:
            yp, _, mcy = self._tables(ys)
        if mode == 2 and not (mcx and mcy):
            mcx = mcy = 0
        two = self._want_two_shot(mode, xs, z, n)
        mcz, xw, zw = 0, [], []
        if two:
            xw = [xp[r] for r in range(W)]
            if mode != 0:
                za, zoff = self.heap.locate(z)
                zw = [za["peer_ptrs"][r] + zoff for r in range(W)]
                if za["mc_ptr"] and self.use_multimem:
                    mcz = za["mc_ptr"] + zoff
        self.ext.block_reduce(mode, xp, yp, local_idx, z, n, float(rho), rho_dev, self.out, self.scratch, self.ctrl_ptrs,
                              self.sync, W, self.topo.rank, mcx, mcy, mcz, xw, zw, bool(two), self.max_blocks,
                              self.timeout_s)
        self.launches += 1
        self.last_two_shot = bool(two)

    supports_async = True

    def _record_async(self) -> None:
        """Deferred rounds only: the round's record follows the kernel into pinned host memory on the same stream, so the host can
        enqueue the next minibatches first and pick the record up later without draining the GPU.  (The synchronous operators
        below read ``self.out`` directly, exactly as before.)"""
        if not torch.cuda.is_current_stream_capturing():
            self._host_out.copy_(self.out, non_blocking=True)
            self._out_event.record()
            self._out_pending = True

    def launch_fedavg_(self, xs, z, write_back: bool = True) -> None:
        self._launch(0 if write_back else 1, xs, None, z, 0.0)
        self._record_async()

    def launch_fedprox_(self, xs, z, rho: float) -> None:
        self._launch(1, xs, None, z, rho)
        self._record_async()

    def launch_admm_(self, xs, ys, z, rho: float, rho_dev=None) -> None:
        self._launch(2, xs, ys, z, rho, rho_dev)
        self._record_async()

    def read_record(self) -> List[float]:
        """The ONE device->host read of a round: dual^2, primal, #non-finite, status, rho, epoch, two-shot flag."""
        if self._out_pending:
            self._out_event.synchronize()
            self._out_pending = False
            vals = self._host_out.tolist()
        else:
            vals = self.out.tolist()
        if vals[OUT_STATUS] != 0.0:
            raise CollectiveTimeout("fedb200: rank %d timed out (%.0f s) waiting for rank %d in aggregation %d"
                                    % (self.topo.rank, self.timeout_s, int(vals[OUT_STATUS]) - 100, int(vals[OUT_EPOCH])))
        self.last_nonfinite = vals[OUT_NONFINITE]
        self.last_rho = vals[OUT_RHO]
        return vals

    # -- operators ----------------------------------------------------------------------
    @torch.no_grad()
    def fedavg_(self, xs, z, write_back: bool = True):
        self._launch(0 if write_back else 1, xs, None, z, 0.0)
        return self.read_record()[OUT_DUAL_SQ]

    @torch.no_grad()
    def fedprox_(self, xs, z, rho: float):
        self._launch(1, xs, None, z, rho)
        v = self.read_record()
        return v[OUT_DUAL_SQ], v[OUT_PRIMAL]

    @torch.no_grad()
    def admm_(self, xs, ys, z, rho: float, rho_dev=None):
        self._launch(2, xs, ys, z, rho, rho_dev)
        v = self.read_record()
        return v[OUT_DUAL_SQ], v[OUT_PRIMAL]

    # -- Barzilai-Borwein ---------------------------------------------------------------------
    def _bb_launch(self, xs, ys, yhat0s, x0s, z, rho_dev, cfg, seed_only: bool) -> None:
        W = self.topo.world_size
        workers = [self.topo.rank + j * W for j in range(len(xs))]
        self.ext.bb_update(list(xs), list(ys), list(yhat0s), list(x0s), z, workers, self.topo.K, rho_dev, self.bb_log,
                           self.bb_scratch, self.out, self.ctrl_ptrs, self.sync, W, self.topo.rank,
                           float(getattr(cfg, "epsilon", 1e-3)), float(getattr(cfg, "alphacorrmin", 0.2)),
                           float(getattr(cfg, "rhomax", 0.1)), bool(seed_only), self.max_blocks, self.timeout_s)
        self.launches += 1

    @torch.no_grad()
    def bb_seed_(self, xs, x0s) -> None:
        dummy = xs[0]
        rho = torch.zeros(1, dtype=torch.float32, device=dummy.device)
        self._bb_launch(xs, [], [], x0s, dummy, rho, None, True)

    @torch.no_grad()
    def bb_update_(self, xs, ys, yhat0s, x0s, z, rho: float, rho_dev, cfg):
        if rho_dev is None:
            rho_dev = torch.full((1,), float(rho), dtype=torch.float32, device=z.device)
        self._bb_launch(xs, ys, yhat0s, x0s, z, rho_dev, cfg, False)
        # one read: the legacy log lines need the rows.  A barrier timeout is sticky in out[OUT_STATUS] and raised by the
        # read_record() of the aggregation that always follows.
        return self.bb_log[: 8 * self.topo.K].view(self.topo.K, 8).tolist()
