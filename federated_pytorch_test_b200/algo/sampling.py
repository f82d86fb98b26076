"""Client sampling for federated averaging (partial participation, McMahan et al. 2017, Algorithm 1) and the
sample-count weights of the aggregate: the numpy oracle of the selection the aggregation kernel makes on the device.

Sampled round ``t`` (``t`` counts the sampled rounds of the run) gives worker ``k`` the 64-bit word
``h_k = F(F(key + (t + 1) G) + (k + 1) G)``, arithmetic mod ``2**64``, with ``F`` the splitmix64 finaliser and
``G = 0x9E3779B97F4A7C15`` (as for the DP noise, ``algo/privacy.py``).  The round's participants are the ``S`` workers
with the smallest ``(h_k, k)``: a uniform ``S``-subset of the K workers that depends on ``(key, t)`` only, not on the
process layout, so every rank (and every CTA of the kernel) selects the same set without communicating.

The new model is ``z = sum_{k in P} w_k x_k`` with ``w_k = n_k / sum_{j in P} n_j`` in float32 (``n_k`` the sample count of
worker ``k``'s shard), summed in worker order.  Workers outside ``P`` take no step in the round and are never read.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np

_MASK64 = (1 << 64) - 1
_GAMMA = 0x9E3779B97F4A7C15
_SAMPLE_TAG = 0x53414D504C45434C        # separates the sampling key from the other streams seeded by the run's seed


def _splitmix64_finaliser(z: np.ndarray) -> np.ndarray:
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def sample_key(seed: int) -> int:
    """64-bit key of the client-sampling stream of a run seeded with ``seed``."""
    z = np.array([(int(seed) ^ _SAMPLE_TAG) & _MASK64], dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(_splitmix64_finaliser(z)[0])


def words(key: int, t: int, K: int) -> np.ndarray:
    """``h_k`` of sampled round ``t`` for the K workers (uint64)."""
    with np.errstate(over="ignore"):
        rk = _splitmix64_finaliser(np.array([(int(key) + (int(t) + 1) * _GAMMA) & _MASK64], dtype=np.uint64))[0]
        k = np.arange(int(K), dtype=np.uint64) + np.uint64(1)
        return _splitmix64_finaliser(rk + k * np.uint64(_GAMMA))


def participants(key: int, t: int, K: int, S: int) -> np.ndarray:
    """The ``S`` workers of sampled round ``t``, in ascending worker order (int64)."""
    if not 1 <= int(S) <= int(K):
        raise ValueError("clients per round must lie in 1..K = 1..%d, got %r" % (K, S))
    h = words(key, t, K)
    order = np.lexsort((np.arange(int(K)), h))           # by h_k, ties by k
    return np.sort(order[: int(S)]).astype(np.int64)


def mask(key: int, t: int, K: int, S: int) -> np.ndarray:
    """Boolean participant mask of sampled round ``t``."""
    m = np.zeros(int(K), dtype=bool)
    m[participants(key, t, K, S)] = True
    return m


def weights(n: Sequence[int], mask_: np.ndarray) -> np.ndarray:
    """``w_k = n_k / sum_{j in P} n_j`` (float32, correctly rounded) for ``k`` in the participant set ``P`` (the True
    entries of ``mask_``), 0 elsewhere.  The sum is an exact integer, rounded once to float32."""
    n = np.asarray(n, dtype=np.int64)
    m = np.asarray(mask_, dtype=bool)
    if n.shape != m.shape:
        raise ValueError("one sample count per worker: %d counts for %d workers" % (n.size, m.size))
    total = np.float32(int(n[m].sum()))
    w = np.zeros(n.size, dtype=np.float32)
    w[m] = n[m].astype(np.float32) / total
    return w
