"""Compressed client updates for federated averaging: stochastic 8- and 4-bit quantization with one scale per group of
coordinates (QSGD, Alistarh et al. 2017; FedPAQ, Reisizadeh et al. 2020), optionally with error feedback (Seide et al.
2014; Karimireddy et al. 2019).  This module is the float32 numpy oracle of the CUDA encoder
(``csrc/comm_kernels.cu: q_encode``) and the payload arithmetic.

In a compressed round worker ``k`` uploads its block update ``u_k = x_k - z`` (``+ e_k`` with error feedback) as codes:

* ``u`` is cut into groups of :data:`GROUP` consecutive coordinates, counted from the block start;
* a group's scale is ``s = max|u| / L`` with ``L = 127`` (8 bits) or ``7`` (4 bits);
* a coordinate's code is ``q = clamp(floor(u / s + U), -L, L)``, ``U`` in ``[0, 1)`` the counter-based uniform of
  ``(key, k, t, i)`` (:func:`uniforms`), so ``E[q s] = u`` (unbiased stochastic rounding);
* an all-zero group gets ``s = 0`` and codes 0; a group holding a NaN or an infinity gets ``s = NaN`` and codes 0, so
  its dequantized values are NaN and the run's NaN guard fires instead of the coordinate being silently zeroed;
* with error feedback ``e_k <- u_k - q_k s_k``.

Every step is a correctly rounded float32 operation, so the device codes and scales equal these bit for bit.

Top-k sparsification (:func:`topk_select`) is the other kind of compressed update: worker ``k`` sends the ``k_sel``
largest-magnitude coordinates of ``u_k`` unchanged, with error feedback ``e_k <- u_k - s_k``.
"""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np

from .privacy import _GAMMA, _MASK64, _splitmix64_finaliser

GROUP = 128                            # coordinates per scale (csrc/fedb200.h: Q_GROUP)
BITS = (8, 4)
_Q_TAG = 0x5153474446455051            # separates the rounding key from the other streams seeded by the run's seed


def levels(bits: int) -> int:
    """``L``: the largest code magnitude of a ``bits``-bit code."""
    if bits not in BITS:
        raise ValueError("compress_bits must be 0 (off), 8 or 4, got %r" % (bits,))
    return (1 << (bits - 1)) - 1


def payload_bytes(n: int, bits: int) -> int:
    """Bytes one worker uploads for an ``n``-coordinate block: the codes plus one float32 scale per group."""
    return -(-int(n) * bits // 8) + 4 * -(-int(n) // GROUP)


def compress_key(seed: int) -> int:
    """64-bit key of the stochastic-rounding stream of a run seeded with ``seed``."""
    z = np.array([(int(seed) ^ _Q_TAG) & _MASK64], dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(_splitmix64_finaliser(z)[0])


def uniforms(key: int, k: int, t: int, n: int) -> np.ndarray:
    """``U`` of worker ``k`` (global id) in compressed round ``t`` for coordinates ``0 .. n - 1`` (float32, in [0, 1)).

    Coordinates ``2p`` and ``2p + 1`` share the 64-bit word ``w = F(F(F(key + (t + 1) G) + (k + 1) G) + (p + 1) G)``,
    arithmetic mod ``2**64``, with ``F`` the splitmix64 finaliser and ``G = 0x9E3779B97F4A7C15`` (the construction of the
    DP noise, ``privacy.dp_noise``): ``U_2p = w[63:40] 2**-24``, ``U_2p+1 = w[23:0] 2**-24``.  A pure function of
    ``(key, k, t, i)``: the process layout and the one-shot / two-shot split do not change it."""
    npair = (int(n) + 1) // 2
    with np.errstate(over="ignore"):
        r = _splitmix64_finaliser(np.array([(int(key) + (int(t) + 1) * _GAMMA) & _MASK64], dtype=np.uint64))[0]
        wk = _splitmix64_finaliser(np.array([(int(r) + (int(k) + 1) * _GAMMA) & _MASK64], dtype=np.uint64))[0]
        p = np.arange(npair, dtype=np.uint64) + np.uint64(1)
        w = _splitmix64_finaliser(wk + p * np.uint64(_GAMMA))
    out = np.empty(2 * npair, dtype=np.float32)
    out[0::2] = (w >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
    out[1::2] = (w & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(2.0 ** -24)
    return out[: int(n)]


def quantize(u: np.ndarray, bits: int, key: int, k: int, t: int) -> Tuple[np.ndarray, np.ndarray]:
    """Codes (int8, one per coordinate) and scales (float32, one per group) of update ``u`` (float32) of worker ``k`` in
    compressed round ``t``."""
    L = levels(bits)
    u = np.asarray(u, dtype=np.float32)
    n = u.size
    ng = -(-n // GROUP)
    ug = np.zeros(ng * GROUP, dtype=np.float32)
    ug[:n] = u
    ug = ug.reshape(ng, GROUP)
    finite = np.isfinite(ug).all(axis=1)
    amax = np.where(finite[:, None], np.abs(ug), np.float32(0)).max(axis=1)
    scales = np.where(finite, amax / np.float32(L), np.float32(np.nan)).astype(np.float32)
    coded = finite & (scales > 0)
    U = uniforms(key, k, t, ng * GROUP).reshape(ng, GROUP)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.floor(ug / scales[:, None] + U)
    q = np.where(coded[:, None], np.clip(r, -L, L), np.float32(0))
    return q.astype(np.int8).reshape(-1)[:n], scales


def dequantize(codes: np.ndarray, scales: np.ndarray) -> np.ndarray:
    """``q s`` per coordinate (float32)."""
    codes = np.asarray(codes)
    return codes.astype(np.float32) * np.repeat(np.asarray(scales, dtype=np.float32), GROUP)[: codes.size]


def pack4(codes: np.ndarray) -> np.ndarray:
    """The payload bytes of 4-bit codes: two per byte, the even coordinate in the low nibble (two's complement)."""
    c = np.asarray(codes, dtype=np.int8).astype(np.uint8) & np.uint8(0xF)
    if c.size % 2:
        c = np.append(c, np.uint8(0))
    return c[0::2] | (c[1::2] << np.uint8(4))


def unpack4(payload: np.ndarray, n: int) -> np.ndarray:
    """Inverse of :func:`pack4` for ``n`` codes."""
    b = np.asarray(payload, dtype=np.uint8)
    out = np.empty(2 * b.size, dtype=np.int8)
    out[0::2] = ((b & np.uint8(0xF)) << np.uint8(4)).astype(np.int8) >> 4
    out[1::2] = (b & np.uint8(0xF0)).astype(np.int8) >> 4
    return out[:n]


def relative_error(err_sq: float, norm_sq: float) -> float:
    """``sqrt(sum_k ||u_k - q_k s_k||^2 / sum_k ||u_k||^2)`` (0 for an all-zero update)."""
    return math.sqrt(err_sq / norm_sq) if norm_sq > 0.0 else (0.0 if err_sq == 0.0 else math.inf)


# ---- top-k sparsification (Stich et al. 2018; Lin et al. 2018, Deep Gradient Compression) ---------------------------
# Worker k sends the k_sel coordinates of u = (x_k - z) + e_k with the largest sort key bits(u) & 0x7fffffff (read as
# uint32: the magnitude order for finite values, then +-inf, then NaN), ties broken by the lower index.  The values are
# sent unchanged; with error feedback e_k <- u - s_k (0 on the selected coordinates, u elsewhere).  The oracle of
# csrc/comm_kernels.cu: topk_select_kernel.

TOPK_TILE = 8192                       # coordinates per tile of the sparse payload (csrc: Q_TILE = COMM_THREADS * Q_SEG)


def topk_count(n: int, r: float) -> int:
    """``k_sel = max(1, ceil(r n))``, in float64: the coordinates one worker sends of an ``n``-coordinate block."""
    return max(1, int(math.ceil(float(r) * float(n))))


def topk_keys(u: np.ndarray) -> np.ndarray:
    """The sort key of every coordinate: ``bits(u) & 0x7fffffff`` as uint32."""
    return np.ascontiguousarray(u, dtype=np.float32).view(np.uint32) & np.uint32(0x7FFFFFFF)


def topk_select(u: np.ndarray, k: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The sparse payload of update ``u`` (float32) with ``k`` coordinates: ``tile_offsets`` (uint32, one per tile of
    :data:`TOPK_TILE` coordinates counted from the block start, plus the total), then per selected coordinate in ascending
    index order its offset within its tile (``in_tile_idx``, uint16) and its value (``values``, float32, exactly ``u_i``)."""
    u = np.ascontiguousarray(u, dtype=np.float32).reshape(-1)
    n = u.size
    if not 1 <= k <= n:
        raise ValueError("top-k needs 1 <= k <= n, got k = %d at n = %d" % (k, n))
    key = topk_keys(u)
    thr = np.partition(key, n - k)[n - k]               # the k-th largest key
    mask = key > thr
    mask[np.flatnonzero(key == thr)[: k - int(mask.sum())]] = True     # ties: the lowest indices
    sel = np.flatnonzero(mask)
    ntiles = -(-n // TOPK_TILE)
    counts = np.bincount(sel // TOPK_TILE, minlength=ntiles)
    offsets = np.zeros(ntiles + 1, dtype=np.uint32)
    offsets[1:] = np.cumsum(counts)
    return offsets, (sel % TOPK_TILE).astype(np.uint16), u[sel].copy()


def topk_indices(tile_offsets: np.ndarray, in_tile_idx: np.ndarray) -> np.ndarray:
    """The block coordinates of a payload's entries."""
    tiles = np.repeat(np.arange(tile_offsets.size - 1), np.diff(tile_offsets.astype(np.int64)))
    return tiles * TOPK_TILE + in_tile_idx.astype(np.int64)


def topk_payload_bytes(n: int, k: int) -> int:
    """Bytes one worker sends for an ``n``-coordinate block with ``k`` entries: ``6 k + 4 (ceil(n / 8192) + 1)``."""
    return 6 * int(k) + 4 * (-(-int(n) // TOPK_TILE) + 1)


def topk_layout(n: int, k: int) -> Tuple[int, int, int, int]:
    """``(tiles, val, idx, words)`` of the payload buffer (int32 words, ``csrc/fedb200.h: topk_layout``): the ``tiles + 1``
    offsets from word 0, the ``k`` values from word ``val``, the ``k`` uint16 in-tile offsets (two per word, the lower
    index in the low half) from word ``idx``; sections start at 16-byte boundaries."""
    T = -(-int(n) // TOPK_TILE)
    val = (T + 1 + 3) & ~3
    idx = val + ((int(k) + 3) & ~3)
    return T, val, idx, idx + (((int(k) + 1) // 2 + 3) & ~3)


def topk_pack(payload: Tuple[np.ndarray, np.ndarray, np.ndarray], n: int) -> np.ndarray:
    """The buffer words (int32) of a payload ``(tile_offsets, in_tile_idx, values)`` of an ``n``-coordinate block."""
    offsets, idx, vals = payload
    k = vals.size
    T, v0, i0, words = topk_layout(n, k)
    out = np.zeros(words, dtype=np.int32)
    out[: T + 1] = offsets.astype(np.uint32).view(np.int32)
    out[v0: v0 + k] = vals.astype(np.float32).view(np.int32)
    out[i0: words].view(np.uint16)[:k] = idx
    return out


def topk_unpack(words: np.ndarray, n: int, k: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Inverse of :func:`topk_pack`."""
    w = np.ascontiguousarray(words, dtype=np.int32)
    T, v0, i0, n_words = topk_layout(n, k)
    return (w[: T + 1].view(np.uint32).copy(), w[i0: n_words].view(np.uint16)[:k].copy(),
            w[v0: v0 + k].view(np.float32).copy())
