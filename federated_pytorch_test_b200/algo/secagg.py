"""Secure aggregation for federated averaging: pairwise-masked fixed-point updates (SecAgg, Bonawitz et al. 2017).  This
module is the numpy oracle of the CUDA encoder and decoder (``csrc/comm_kernels.cu: sa_encode, sa_gather``) and the
payload arithmetic.

In a secure-aggregation round with ``K`` workers and server model ``z``:

* **scale**: ``R = float32(clip)``; ``f`` is the largest integer with ``K rint(R 2^f) <= 2^31 - 1``, so K clipped codes
  cannot overflow an int32 sum (:func:`frac_bits`);
* **encode** worker ``k``: ``u = x_k - z`` (float32); a non-finite ``u`` codes to 0 and is counted, any other to
  ``q = rint(clamp(u, -R, R) 2^f)`` (int32, round half to even; the product is exact), counted as clipped when
  ``|u| > R`` (:func:`encode`);
* **pair keys**: for ``i < j``, ``key_ij = SHA-256(b"secagg-pair-key" || seed (8 bytes LE) || i (4 bytes LE) || j (4 bytes
  LE))`` read as 8 little-endian uint32 words (:func:`pair_keys`).  It stands in for the Diffie-Hellman key agreement of
  Bonawitz et al.: whoever knows the seed can unmask every update;
* **mask**: ``m_ij[c]`` is word ``c mod 16`` of the ChaCha20 block function (RFC 8439 §2.3) with key ``key_ij``, block
  counter ``c div 16`` and nonce words ``(t mod 2^32, t div 2^32, 0)``, ``t`` the secure-aggregation round index of the
  run, which never repeats (a reused key and nonce would reveal the difference of two updates);
* worker ``k`` uploads ``y_k = q_k + sum_{j>k} m_kj - sum_{j<k} m_jk (mod 2^32)``, 4 bytes per coordinate (:func:`payload`);
* **decode**: ``S = int32(sum_k y_k mod 2^32) = sum_k q_k`` exactly; ``d = (float32(S) 2^-f) (1 / K)``, each product
  correctly rounded, with ``1 / K`` the correctly rounded float32 reciprocal (:func:`decode`).

Integer sums do not depend on order, so the new model is the same bit for bit for every process layout.
"""
from __future__ import annotations

import hashlib
import struct
from typing import Tuple

import numpy as np

MAX_FRAC_BITS = 126                    # 2^f and 2^-f stay normal floats (csrc/fedb200.h: SA_MAX_FRAC_BITS)
_SIGMA = np.array([0x61707865, 0x3320646E, 0x79622D32, 0x6B206574], dtype=np.uint32)
_INT32_MAX = 2 ** 31 - 1


def frac_bits(clip: float, K: int) -> int:
    """``f``: the largest integer with ``K rint(float32(clip) 2^f) <= 2^31 - 1``.  Raises ``ValueError`` when the clip is
    not finite and positive or when ``f`` would fall outside ``[0, 126]``."""
    R = float(np.float32(clip))
    if not (np.isfinite(R) and R > 0.0):
        raise ValueError("secagg_clip must be finite and > 0, got %r" % (clip,))
    for f in range(MAX_FRAC_BITS + 1, -1, -1):          # R 2^f is exact in float64; round() rounds half to even
        if int(K) * round(R * 2.0 ** f) <= _INT32_MAX:
            if f > MAX_FRAC_BITS:
                break
            return f
    raise ValueError("secagg_clip %r gives no fixed-point scale 2^f with 0 <= f <= %d at K = %d (K rint(R 2^f) must "
                     "fit an int32)" % (clip, MAX_FRAC_BITS, K))


def encode(u: np.ndarray, clip: float, f: int) -> Tuple[np.ndarray, int, int]:
    """Fixed-point codes (int32) of update ``u`` (float32), the number of clipped and of non-finite coordinates."""
    u = np.asarray(u, dtype=np.float32)
    R = np.float32(clip)
    finite = np.isfinite(u)
    with np.errstate(invalid="ignore"):
        clipped = int(np.count_nonzero(finite & (np.abs(u) > R)))
        c = np.where(finite, np.clip(u, -R, R), np.float32(0)) * np.float32(2.0 ** f)
    return np.rint(c).astype(np.int32), clipped, int(u.size - np.count_nonzero(finite))


def pair_keys(seed: int, K: int) -> np.ndarray:
    """``[K (K - 1) / 2, 8]`` uint32: the key of every pair ``i < j``, in lexicographic order."""
    rows = []
    for i in range(K):
        for j in range(i + 1, K):
            h = hashlib.sha256(b"secagg-pair-key" + struct.pack("<qII", int(seed), i, j)).digest()
            rows.append(np.frombuffer(h, dtype="<u4"))
    return np.array(rows, dtype=np.uint32).reshape(-1, 8)


def pair_row(i: int, j: int, K: int) -> int:
    """Row of pair ``(i, j)``, ``i < j``, in :func:`pair_keys`."""
    return i * (2 * K - i - 1) // 2 + (j - i - 1)


def _rotl(x: np.ndarray, n: int) -> np.ndarray:
    return (x << np.uint32(n)) | (x >> np.uint32(32 - n))


def _quarter(s, a, b, c, d):
    s[a] += s[b]; s[d] ^= s[a]; s[d] = _rotl(s[d], 16)      # noqa: E702
    s[c] += s[d]; s[b] ^= s[c]; s[b] = _rotl(s[b], 12)      # noqa: E702
    s[a] += s[b]; s[d] ^= s[a]; s[d] = _rotl(s[d], 8)       # noqa: E702
    s[c] += s[d]; s[b] ^= s[c]; s[b] = _rotl(s[b], 7)       # noqa: E702


def chacha20_blocks(key: np.ndarray, counters: np.ndarray, nonce: Tuple[int, int, int]) -> np.ndarray:
    """The ChaCha20 block function (RFC 8439 §2.3) for every block counter in ``counters``: uint32 ``[len(counters) * 16]``,
    block after block (the keystream)."""
    counters = np.asarray(counters, dtype=np.uint32)
    st = np.empty((16, counters.size), dtype=np.uint32)
    st[0:4] = _SIGMA[:, None]
    st[4:12] = np.asarray(key, dtype=np.uint32).reshape(8, 1)
    st[12] = counters
    st[13:16] = np.array(nonce, dtype=np.uint32)[:, None]
    s = st.copy()
    for _ in range(10):
        _quarter(s, 0, 4, 8, 12); _quarter(s, 1, 5, 9, 13); _quarter(s, 2, 6, 10, 14); _quarter(s, 3, 7, 11, 15)  # noqa: E702
        _quarter(s, 0, 5, 10, 15); _quarter(s, 1, 6, 11, 12); _quarter(s, 2, 7, 8, 13); _quarter(s, 3, 4, 9, 14)  # noqa: E702
    s += st
    return np.ascontiguousarray(s.T).reshape(-1)


def nonce(t: int) -> Tuple[int, int, int]:
    """The nonce words of secure-aggregation round ``t``."""
    t = int(t) & ((1 << 64) - 1)
    return t & 0xFFFFFFFF, t >> 32, 0


def mask(keys: np.ndarray, K: int, k: int, t: int, n: int) -> np.ndarray:
    """``sum_{j>k} m_kj - sum_{j<k} m_jk (mod 2^32)`` of worker ``k`` in round ``t`` at coordinates ``0 .. n - 1`` (uint32)."""
    nb = -(-int(n) // 16)
    ctr = np.arange(nb, dtype=np.uint32)
    acc = np.zeros(nb * 16, dtype=np.uint32)
    for j in range(K):
        if j == k:
            continue
        m = chacha20_blocks(keys[pair_row(min(j, k), max(j, k), K)], ctr, nonce(t))
        if j > k:
            acc += m
        else:
            acc -= m
    return acc[:n]


def payload(q: np.ndarray, keys: np.ndarray, K: int, k: int, t: int) -> np.ndarray:
    """``y_k = q_k + mask (mod 2^32)`` (uint32) of worker ``k`` in round ``t``."""
    q = np.asarray(q, dtype=np.int32)
    return q.view(np.uint32) + mask(keys, K, k, t, q.size)


def unmask_sum(payloads: np.ndarray) -> np.ndarray:
    """``S = int32(sum_k y_k mod 2^32)`` over the rows of ``payloads`` (``[K, n]`` uint32)."""
    return np.asarray(payloads, dtype=np.uint32).sum(axis=0, dtype=np.uint32).view(np.int32)


def decode(S: np.ndarray, f: int, K: int) -> np.ndarray:
    """The mean update ``d = (float32(S) 2^-f) (1 / K)`` (float32, each product correctly rounded)."""
    return (np.asarray(S, dtype=np.int32).astype(np.float32) * np.float32(2.0 ** -f)) * (np.float32(1) / np.float32(K))


def key_digest(keys: np.ndarray) -> str:
    """SHA-256 (hex) of a pair-key table: identifies the keys in a resume record without storing them."""
    return hashlib.sha256(np.ascontiguousarray(keys, dtype="<u4").tobytes()).hexdigest()
