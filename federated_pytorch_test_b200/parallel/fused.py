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

The robust rules (coordinate-wise median / trimmed mean) run in separate instantiations of the same kernel: every
coordinate's K values are loaded over P2P (there is no in-switch order statistic; the two-shot broadcast may still use
``multimem.st``) and sorted in registers, so K <= 16.

DP-FedAvg (client-level differential privacy) is two launches per round, in stream order and host-free: a cooperative
clip kernel on each rank's own replicas (no peer memory), then DP instantiations of the aggregation kernel, which add
the counter-based Gaussian noise to the mean and advance the device-resident round counter, so a graph-captured round
draws fresh noise on every replay.

Compressed rounds (stochastic 8- / 4-bit codes with one scale per group, optional error feedback) are one launch of the
compressed instantiations: before barrier A every rank encodes its own replicas' updates into symmetric payload arenas
(:meth:`FusedCollective.payload_like_block`), and pass 1 reads the K workers' codes and scales over P2P (there is no
in-switch reduction of codes with per-group scales; the two-shot broadcast may still use ``multimem.st``), so a rank pulls
about 4x (8-bit) or 7.5x (4-bit) fewer bytes from its peers.  The rounding counter lives in device memory as the DP one.

Sampled rounds (client sampling with sample-count weights) are one launch of the sampled instantiations: every CTA
selects the round's participants from the device-resident round counter, and pass 1 forms their weighted sum with P2P
loads of the participants only (``multimem.ld_reduce`` sums every bound device with weight 1; the two-shot broadcast may
still use ``multimem.st``).  A worker that sits out is never read, and receives the new model in pass 2.

Secure-aggregation rounds (pairwise-masked fixed-point updates) are one launch of the SecAgg instantiations, on the
compressed rounds' tiling: before barrier A every rank encodes its own replicas' updates as int32 codes and adds or
subtracts the K - 1 ChaCha20 keystreams of its pairs, computed in registers, into 32-bit symmetric payload arenas
(:meth:`FusedCollective.payload32_like_block`); pass 1 sums the K payloads over P2P as integers mod 2^32, where the masks
cancel, and decodes.  The sum is exact, so the new model does not depend on the process layout or on one-shot versus
two-shot.  The nonce counter lives in device memory as the DP one.

Top-k rounds (sparsified updates, optional error feedback) are two launches: a cooperative selection kernel on each rank's
own replicas (no peer memory) writes every replica's sparse payload (tile offsets, then its entries in index order) into
symmetric payload arenas (:meth:`FusedCollective.sparse_payload_like_block`), then the top-k instantiations of the
aggregation kernel scatter-add the K workers' entries of each tile into shared memory in worker order, over P2P.  Adding
zeros is exact, so the new model does not depend on the process layout or on one-shot versus two-shot.
"""
from __future__ import annotations

import os
import struct
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from ..ops import cuda_ops
from .collective import (FEDOPT_KINDS, ROBUST_AGGS, DPRound, QuantRound, SampleRound, SecAggRound, TopKRound,
                         TorchCollective, check_robust)
from .topology import Topology

_MAX_LOCAL = 16
_OUT_FLOATS = 14
_SCRATCH_FLOATS = 4 + _MAX_LOCAL
_MAX_BLOCKS = 160                                         # csrc/fedb200.h: COMM_MAX_BLOCKS
_DP_STATS_FLOATS = 2 * _MAX_LOCAL * _MAX_BLOCKS + 2 * _MAX_LOCAL      # DP_STATS_FLOATS: double partials, norms, flags
_BB_SCRATCH_FLOATS = 8 * _MAX_LOCAL + 8 + _MAX_LOCAL
_Q_PART_FLOATS = 2 * _MAX_BLOCKS + 2                      # TOPK_STATS_FLOATS (>= Q_PART_FLOATS): per-CTA partials
_Q_GROUP = 128                                            # Q_GROUP (algo/compress.py: GROUP)
_PAD_WORDS = 8192
OUT_DUAL_SQ, OUT_PRIMAL, OUT_NONFINITE, OUT_STATUS, OUT_RHO, OUT_EPOCH, OUT_TWO_SHOT = range(7)
OUT_DP_CLIPPED, OUT_DP_NORM_SUM = 8, 9
OUT_Q_ERR_SQ, OUT_Q_NORM_SQ = 10, 11
OUT_SA_CLIPPED, OUT_SA_NONFINITE = 12, 13              # uint32 bit patterns

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
        self.dp_stats = torch.zeros(_DP_STATS_FLOATS, dtype=torch.float32, device=dev)
        self.q_part = torch.zeros(_Q_PART_FLOATS, dtype=torch.float32, device=dev)
        self.bb_log = torch.zeros(8 * max(topo.K, 1), dtype=torch.float32, device=dev)
        self.sync = torch.zeros(4, dtype=torch.int32, device=dev)
        self._host_out = torch.zeros(self.out.numel(), dtype=torch.float32).pin_memory()
        self._out_event = torch.cuda.Event()
        self._out_pending = False
        self.ctrl = self.heap.alloc(_PAD_WORDS, dtype=torch.int32)
        self.ctrl_ptrs = list(self.heap.locate(self.ctrl)[0]["peer_ptrs"])
        self._aux: Dict[Tuple[int, str], torch.Tensor] = {}
        self._payload: Dict[Tuple[int, int], Tuple[torch.Tensor, torch.Tensor]] = {}   # (arena base, bits) -> code / scale arenas
        self._sparse: Dict[int, torch.Tensor] = {}      # arena base -> top-k payload arena
        self._topk_ws: Dict[Tuple[int, int, bool], Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}
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
        self.warm_fedopt = False          # set by the FedOpt strategy: warm the server-optimizer instantiation too
        self.warm_robust = False          # set by robust strategies: warm the robust instantiation(s) for this K too
        self.warm_dp = False              # set by DP strategies: warm the clip kernel and the DP instantiation(s) too
        self.warm_compress = 0            # set by compressing strategies to their bit width: warm those instantiations too
        self.warm_sample = False          # set by sampling strategies: warm the sampled instantiation(s) too
        self.warm_secagg = False          # set by secure-aggregation strategies: warm the SecAgg instantiation(s) too
        self.warm_topk = False            # set by top-k strategies: warm the selection kernel and top-k instantiation(s) too

    def warmup(self) -> None:
        """One tiny aggregation of every kind on scratch buffers: CUDA module loading, occupancy queries and the first
        cross-rank handshake happen here, at engine construction, not inside the first training round (the first launch
        is far slower than the ones after it).  The server-optimizer kernel is warmed only when ``warm_fedopt`` is set, the
        robust kernels (of this K; with the server optimizer if both are set) only when ``warm_robust`` is set, the DP
        kernels (likewise) only when ``warm_dp`` is set, the compressed ones of ``warm_compress`` bits (likewise) only when
        that is set, the sampled ones (likewise) only when ``warm_sample`` is set, the SecAgg ones (likewise) only when
        ``warm_secagg`` is set, the top-k ones (likewise) only when ``warm_topk`` is set; their round counters are throwaway tensors, so warm-up advances no counter of the run.
        Collective: every rank calls it at the same point."""
        if getattr(self, "_warm", False):
            return
        self._warm = True
        n = 256
        xs = [self.heap.alloc(n) for _ in range(len(self.topo.local_workers))]
        ys = [self.zeros_like_block(x, "y") for x in xs]
        z = self.zeros_like_block(xs[0], "z")
        rho = torch.full((1,), 0.5, dtype=torch.float32, device=self.topo.device)
        if self.warm_fedopt:
            m, v = self.zeros_like_block(xs[0], "srv_m"), self.zeros_like_block(xs[0], "srv_v")
        if self.warm_compress:
            pay = [self.payload_like_block(x, self.warm_compress) for x in xs]
            qr = QuantRound(self.warm_compress, 0, torch.zeros(1, dtype=torch.int64, device=self.topo.device),
                            [c for c, _ in pay], [sc for _, sc in pay])
        if self.warm_sample:
            sr = SampleRound(1, 0, torch.zeros(1, dtype=torch.int64, device=self.topo.device),
                             torch.ones(self.topo.K, dtype=torch.int32, device=self.topo.device))
        if self.warm_secagg:
            K = self.topo.K
            sa = SecAggRound(1.0, 0, torch.zeros(K * (K - 1) // 2, 8, dtype=torch.int32, device=self.topo.device),
                             torch.zeros(1, dtype=torch.int64, device=self.topo.device),
                             [self.payload32_like_block(x) for x in xs])
        if self.warm_topk:
            tk = TopKRound(8, [self.sparse_payload_like_block(x, 8) for x in xs])
        keep = self.two_shot_mode
        for mode_2shot in ("0", "1"):
            self.two_shot_mode = mode_2shot
            self._launch(0, xs, None, z, 0.0)
            self._launch(1, xs, None, z, 0.5)
            self._launch(2, xs, ys, z, 0.5, rho)
            if self.warm_fedopt:
                self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3)
            if self.warm_robust:
                self._launch(0, xs, None, z, 0.0, agg="median")
                if self.warm_fedopt:
                    self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, agg="median")
            if self.warm_dp:
                dp = DPRound(1e-3, 0, torch.zeros(1, dtype=torch.int64, device=self.topo.device))
                self.dp_clip_(xs, z, 1.0)
                self._launch(0, xs, None, z, 0.0, dp=dp)
                if self.warm_fedopt:
                    self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, dp=dp)
            if self.warm_compress:
                self._launch(0, xs, None, z, 0.0, compress=qr)
                if self.warm_fedopt:
                    self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, compress=qr)
            if self.warm_sample:
                self._launch(0, xs, None, z, 0.0, sample=sr)
                if self.warm_fedopt:
                    self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, sample=sr)
            if self.warm_secagg:
                self._launch(0, xs, None, z, 0.0, secagg=sa)
                if self.warm_fedopt:
                    self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, secagg=sa)
            if self.warm_topk:
                self._launch(0, xs, None, z, 0.0, topk=tk)
                if self.warm_fedopt:
                    self._launch_fedopt(xs, z, m, v, "adam", 1e-2, 0.9, 0.99, 1e-3, topk=tk)
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

    def payload_like_block(self, x: torch.Tensor, bits: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """The payload slices of block slice ``x`` for ``bits``-bit codes (layout: :meth:`TorchCollective.payload_like_block`)
        in symmetric arenas that mirror ``x``'s arena: the codes of the arena's float ``i`` at byte ``i bits / 8``, the
        scale of a group starting at float ``i`` at float ``i / 32`` of a scale arena.  So every block slice has its own
        payload at the same offset in every rank.  ``x`` must start at a multiple of 32 floats (the arenas' alignment)."""
        a, off = self.heap.locate(x)
        i0 = off // 4
        if i0 % 32:
            raise ValueError("compressed rounds need block slices that start at a multiple of 32 floats, got %d" % i0)
        key = (a["base"], int(bits))
        bufs = self._payload.get(key)
        if bufs is None:
            nf = a["nbytes"] // 4
            bufs = (self.heap.alloc(nf * bits // 8 + 64, dtype=torch.uint8), self.heap.alloc(nf // 32 + 2))
            self._payload[key] = bufs
        n = x.numel()
        codes = bufs[0][i0 * bits // 8: i0 * bits // 8 + -(-n // 16) * 2 * bits]
        scales = bufs[1][i0 // 32: i0 // 32 + -(-n // _Q_GROUP)]
        codes.zero_()
        scales.zero_()
        return codes, scales

    def payload32_like_block(self, x: torch.Tensor) -> torch.Tensor:
        """The secure-aggregation payload slice of block slice ``x`` (layout: :meth:`TorchCollective.payload32_like_block`):
        the codes arena of :meth:`payload_like_block` for 32-bit codes, viewed as int32, so the arena's float ``i`` has its
        word at word ``i`` and every block slice its own payload at the same offset in every rank."""
        return self.payload_like_block(x, 32)[0].view(torch.int32)

    def sparse_payload_like_block(self, x: torch.Tensor, k_sel: int) -> torch.Tensor:
        """The top-k payload slice of block slice ``x`` with ``k_sel`` entries (layout:
        :meth:`TorchCollective.sparse_payload_like_block`) in a symmetric arena that mirrors ``x``'s arena: two words per
        float of the arena, the block starting at float ``i`` at word ``2 i``.  A payload takes at most
        ``1.5 n + n / 8192 + 9`` words and blocks start at multiples of 32 floats, so every block slice has its own payload
        at the same offset in every rank."""
        from ..algo.compress import topk_layout

        a, off = self.heap.locate(x)
        i0 = off // 4
        if i0 % 32:
            raise ValueError("top-k rounds need block slices that start at a multiple of 32 floats, got %d" % i0)
        buf = self._sparse.get(a["base"])
        if buf is None:
            buf = self.heap.alloc(2 * (a["nbytes"] // 4) + 64, dtype=torch.int32)
            self._sparse[a["base"]] = buf
        pay = buf[2 * i0: 2 * i0 + topk_layout(x.numel(), k_sel)[3]]
        pay.zero_()
        return pay

    def _topk_scratch(self, n: int, n_local: int, ef: bool):
        """The selection kernel's workspace (its histograms are zero between launches) and, without error feedback, its
        ``u`` scratch: one pair per block length, kept for the collective's lifetime (graphs capture their addresses)."""
        key = (n, n_local, ef)
        got = self._topk_ws.get(key)
        if got is None:
            dev = self.topo.device
            ws = torch.zeros(self.ext.topk_ws_ints(n, n_local), dtype=torch.int32, device=dev)
            u = None if ef else torch.empty(n_local, -(-n // 4) * 4, dtype=torch.float32, device=dev)
            got = self._topk_ws[key] = (ws, u)
        return got

    def _select_topk(self, xs, z, tk: TopKRound) -> None:
        """The first launch of a top-k round: every local replica's payload, error feedback and statistics."""
        ef = list(tk.ef) if tk.ef is not None else []
        ws, u = self._topk_scratch(z.numel(), len(xs), bool(ef))
        self.ext.topk_select(list(xs), z, int(tk.k), list(tk.payload), ef, u, ws, self.q_part, self.max_blocks)
        self.launches += 1

    def _topk_args(self, tk: Optional[TopKRound]):
        """The top-k arguments of the aggregation bindings: k_sel, the K workers' payload pointers, the statistics buffer."""
        if tk is None:
            return 0, [], None
        pp, _, _ = self._tables(tk.payload)
        return int(tk.k), pp, self.q_part

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

    def _agg_code(self, agg: str, trim_b: int) -> int:
        """Kernel code of aggregation rule ``agg`` (0 = the mean); raises ``ValueError`` for a rule the kernel cannot run."""
        if agg == "mean":
            return 0
        check_robust(self.topo.K, agg, trim_b)
        if self.topo.K > 16:
            raise ValueError("robust aggregation supports at most 16 workers, got K = %d" % self.topo.K)
        return ROBUST_AGGS.index(agg) + 1

    def _dp_args(self, dp: Optional[DPRound]):
        """The DP arguments of the aggregation bindings: noise std, key (as a signed 64-bit int), counter, clip stats,
        parameter layout."""
        if dp is None:
            return 0.0, 0, None, None, None
        key = int(dp.key) & ((1 << 64) - 1)
        return float(dp.std), key - (1 << 64) if key >= 1 << 63 else key, dp.t, self.dp_stats, dp.valid

    def _q_args(self, q: Optional[QuantRound]):
        """The compression arguments of the aggregation bindings: bits, group size, key (as a signed 64-bit int), counter,
        the K workers' code and scale pointers, the local error-feedback slices, the statistics buffer."""
        if q is None:
            return 0, _Q_GROUP, 0, None, [], [], [], None
        key = int(q.key) & ((1 << 64) - 1)
        cp, _, _ = self._tables(q.codes)
        sp, _, _ = self._tables(q.scales)
        return (int(q.bits), _Q_GROUP, key - (1 << 64) if key >= 1 << 63 else key, q.t, cp, sp,
                list(q.ef) if q.ef is not None else [], self.q_part)

    def _samp_args(self, s: Optional[SampleRound]):
        """The sampling arguments of the aggregation bindings: participants per round, key (as a signed 64-bit int),
        counter, sample counts."""
        if s is None:
            return 0, 0, None, None
        key = int(s.key) & ((1 << 64) - 1)
        return int(s.S), key - (1 << 64) if key >= 1 << 63 else key, s.t, s.n

    def _sa_args(self, sa: Optional[SecAggRound]):
        """The secure-aggregation arguments of the aggregation bindings: f, clip, pair keys, counter, the K workers' payload
        pointers, the statistics buffer."""
        if sa is None:
            return 0, 0.0, None, None, [], None
        pp, _, _ = self._tables(sa.payload)
        return int(sa.f), float(sa.clip), sa.keys, sa.t, pp, self.q_part

    def _launch(self, mode: int, xs, ys, z, rho: float, rho_dev=None, agg: str = "mean", trim_b: int = 0,
                dp: Optional[DPRound] = None, compress: Optional[QuantRound] = None,
                sample: Optional[SampleRound] = None, secagg: Optional[SecAggRound] = None,
                topk: Optional[TopKRound] = None) -> None:
        """Modes 0 / 1 take a robust rule ``agg`` (:data:`ROBUST_AGGS`) in place of the mean; mode 0 with the mean takes
        the noise of a DP round (``dp``; after :meth:`dp_clip_`), compresses the workers' updates (``compress``),
        averages the sampled participants of the round (``sample``), sums their masked updates (``secagg``) or sums
        their top-k updates (``topk``; the selection is a launch of its own)."""
        if dp is not None and (mode != 0 or agg != "mean"):
            raise ValueError("DP aggregation needs FedAvg with the mean")
        if compress is not None and (mode != 0 or agg != "mean" or dp is not None):
            raise ValueError("compressed aggregation needs FedAvg with the mean, without DP")
        if sample is not None and (mode != 0 or agg != "mean" or dp is not None or compress is not None):
            raise ValueError("sampled aggregation needs FedAvg with the mean, without DP or compression")
        if secagg is not None and (mode != 0 or agg != "mean" or dp is not None or compress is not None or sample is not None):
            raise ValueError("secure aggregation needs FedAvg with the mean, without DP, compression or sampling")
        if topk is not None and (mode != 0 or agg != "mean" or dp is not None or compress is not None or sample is not None
                                 or secagg is not None):
            raise ValueError("top-k aggregation needs FedAvg with the mean, without DP, compression, sampling or secure "
                             "aggregation")
        code = self._agg_code(agg, trim_b)
        n = xs[0].numel()
        if any(t.numel() != n for t in xs) or z.numel() != n:
            raise ValueError("block slices must have equal length")
        if topk is not None:
            self._select_topk(xs, z, topk)
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
                              self.timeout_s, code, int(trim_b), *self._dp_args(dp), *self._q_args(compress),
                              *self._samp_args(sample), *self._sa_args(secagg), *self._topk_args(topk))
        self.launches += 1
        self.last_two_shot = bool(two)

    def _launch_fedopt(self, xs, z, m, v, kind: str, lr: float, beta1: float, beta2: float, tau: float, agg: str = "mean",
                       trim_b: int = 0, dp: Optional[DPRound] = None, compress: Optional[QuantRound] = None,
                       sample: Optional[SampleRound] = None, secagg: Optional[SecAggRound] = None,
                       topk: Optional[TopKRound] = None) -> None:
        """FedAvg with a server optimizer: mode 0 of the kernel's FedOpt instantiation.  Two-shot, rank r broadcasts slice r
        of the new weights, of ``m`` and of ``v`` into every rank, so ``m`` / ``v`` must be symmetric slices then
        (:meth:`zeros_like_block`).  A robust rule ``agg`` replaces the mean as the aggregate the step is taken towards; a
        DP round (``dp``, mean only) noises the mean first; a compressed round (``compress``, mean only) steps along the
        dequantized mean update; a sampled round (``sample``, mean only) steps towards the participants' weighted mean; a
        SecAgg round (``secagg``, mean only) steps along the decoded sum of the masked updates; a top-k round (``topk``,
        mean only) steps along the mean sparse update."""
        code = self._agg_code(agg, trim_b)
        if dp is not None and agg != "mean":
            raise ValueError("DP aggregation needs the mean")
        if compress is not None and (agg != "mean" or dp is not None):
            raise ValueError("compressed aggregation needs the mean, without DP")
        if sample is not None and (agg != "mean" or dp is not None or compress is not None):
            raise ValueError("sampled aggregation needs the mean, without DP or compression")
        if secagg is not None and (agg != "mean" or dp is not None or compress is not None or sample is not None):
            raise ValueError("secure aggregation needs the mean, without DP, compression or sampling")
        if topk is not None and (agg != "mean" or dp is not None or compress is not None or sample is not None
                                 or secagg is not None):
            raise ValueError("top-k aggregation needs the mean, without DP, compression, sampling or secure aggregation")
        n = xs[0].numel()
        adaptive = kind != "avgm"
        if any(t.numel() != n for t in xs) or z.numel() != n or m.numel() != n or (adaptive and v.numel() != n):
            raise ValueError("block slices must have equal length")
        if topk is not None:
            self._select_topk(xs, z, topk)
        W = self.topo.world_size
        xp, local_idx, mcx = self._tables(xs)
        two = self._want_two_shot(0, xs, z, n) and self.heap.contains(m) and (not adaptive or self.heap.contains(v))
        mcm = mcv = 0
        xw, mw, vw = [], [], []
        if two:
            xw = [xp[r] for r in range(W)]
            mw, _, mcm = self._tables([m])
            if adaptive:
                vw, _, mcv = self._tables([v])
        self.ext.block_reduce_fedopt(FEDOPT_KINDS.index(kind) + 1, float(lr), float(beta1), float(beta2), float(tau), m,
                                     v if adaptive else None, xp, local_idx, z, n, self.out, self.scratch, self.ctrl_ptrs,
                                     self.sync, W, self.topo.rank, mcx, mcm, mcv, xw, mw, vw, bool(two), self.max_blocks,
                                     self.timeout_s, code, int(trim_b), *self._dp_args(dp), *self._q_args(compress),
                                     *self._samp_args(sample), *self._sa_args(secagg), *self._topk_args(topk))
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

    def launch_fedavg_(self, xs, z, write_back: bool = True, dp: Optional[DPRound] = None,
                       compress: Optional[QuantRound] = None, sample: Optional[SampleRound] = None,
                       secagg: Optional[SecAggRound] = None, topk: Optional[TopKRound] = None) -> None:
        self._launch(0 if write_back else 1, xs, None, z, 0.0, dp=dp, compress=compress, sample=sample, secagg=secagg,
                     topk=topk)
        self._record_async()

    def launch_fedopt_(self, xs, z, m, v, kind: str, lr: float, beta1: float, beta2: float, tau: float, agg: str = "mean",
                       trim_b: int = 0, dp: Optional[DPRound] = None, compress: Optional[QuantRound] = None,
                       sample: Optional[SampleRound] = None, secagg: Optional[SecAggRound] = None,
                       topk: Optional[TopKRound] = None) -> None:
        self._launch_fedopt(xs, z, m, v, kind, lr, beta1, beta2, tau, agg, trim_b, dp, compress, sample, secagg, topk)
        self._record_async()

    @torch.no_grad()
    def dp_clip_(self, xs, z, bound: float) -> None:
        """DP-FedAvg update clipping of the local replicas (one cooperative launch, no peer memory, no host work).  Its
        statistics reach :attr:`last_dp` through the record of the DP aggregation that must follow."""
        if any(t.numel() != z.numel() for t in xs):
            raise ValueError("block slices must have equal length")
        self.ext.dp_clip(list(xs), z, float(bound), self.dp_stats, self.max_blocks)
        self.launches += 1

    launch_dp_clip_ = dp_clip_

    def launch_robust_(self, xs, z, agg: str, trim_b: int = 0, write_back: bool = True) -> None:
        self._launch(0 if write_back else 1, xs, None, z, 0.0, agg=agg, trim_b=trim_b)
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
        self.last_dp = (vals[OUT_DP_CLIPPED], vals[OUT_DP_NORM_SUM])
        self.last_q = (vals[OUT_Q_ERR_SQ], vals[OUT_Q_NORM_SQ])
        self.last_sa = struct.unpack("<2I", struct.pack("<2f", vals[OUT_SA_CLIPPED], vals[OUT_SA_NONFINITE]))
        return vals

    # -- operators ----------------------------------------------------------------------
    @torch.no_grad()
    def average_(self, xs, z) -> None:
        """``z <- mean_k x_k``: one launch of FedAvg without write-back whose record nobody reads, so it must not set
        ``_out_pending`` (a following synchronous round would read this launch's pinned copy instead of its own).  A
        time-out is still raised: ``OUT_STATUS`` is sticky, and the next round's record reports it."""
        self._launch(1, xs, None, z, 0.0)

    @torch.no_grad()
    def fedavg_(self, xs, z, write_back: bool = True, dp: Optional[DPRound] = None,
                compress: Optional[QuantRound] = None, sample: Optional[SampleRound] = None,
                secagg: Optional[SecAggRound] = None, topk: Optional[TopKRound] = None):
        self._launch(0 if write_back else 1, xs, None, z, 0.0, dp=dp, compress=compress, sample=sample, secagg=secagg,
                     topk=topk)
        return self.read_record()[OUT_DUAL_SQ]

    @torch.no_grad()
    def robust_(self, xs, z, agg: str, trim_b: int = 0, write_back: bool = True):
        self._launch(0 if write_back else 1, xs, None, z, 0.0, agg=agg, trim_b=trim_b)
        return self.read_record()[OUT_DUAL_SQ]

    @torch.no_grad()
    def fedopt_(self, xs, z, m, v, kind: str, lr: float, beta1: float, beta2: float, tau: float, agg: str = "mean",
                trim_b: int = 0, dp: Optional[DPRound] = None, compress: Optional[QuantRound] = None,
                sample: Optional[SampleRound] = None, secagg: Optional[SecAggRound] = None,
                topk: Optional[TopKRound] = None):
        self._launch_fedopt(xs, z, m, v, kind, lr, beta1, beta2, tau, agg, trim_b, dp, compress, sample, secagg, topk)
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
