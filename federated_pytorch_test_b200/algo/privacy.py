"""Client-level differential privacy for federated averaging (DP-FedAvg, McMahan et al., ICLR 2018): the accountant and
the noise draw.

Every DP round releases one noised block mean.  Each worker's update ``x_k - z`` of the block is clipped to the L2 bound
``C = dp_clip * sqrt(N)`` (``N`` the block's length: a public quantity, so the scaling costs no privacy) and
``(sigma C / K) xi``, ``xi ~ N(0, I)``, is added to the mean of the K workers.  With add/remove-one-client adjacency and a
fixed denominator K the sum has sensitivity ``C``, so a round is the Gaussian mechanism with noise multiplier ``sigma``
and ``T`` rounds compose (adaptively) to mu-GDP with ``mu = sqrt(T) / sigma`` (Dong, Roth and Su 2019).  Server
optimizer steps taken from the noised mean are post-processing.

This is a simulator of the Gaussian mechanism: the noise is floating-point and counter-based, not hardened against
attacks on floating-point arithmetic (Mironov 2012) or against an adversary who knows the key.
"""
from __future__ import annotations

import math

import numpy as np

_MASK64 = (1 << 64) - 1
_GAMMA = 0x9E3779B97F4A7C15
_DP_TAG = 0x4450464544415647          # separates the noise key from the other streams seeded by the run's seed


# ------------------------------------------------------------------------------------------ accountant
def _phi(x: float) -> float:
    """Standard normal CDF."""
    return 0.5 * math.erfc(-x / math.sqrt(2.0))


def _gdp_delta(eps: float, mu: float) -> float:
    """``delta(eps)`` of mu-GDP: ``Phi(-eps/mu + mu/2) - e^eps Phi(-eps/mu - mu/2)`` (the second term in log space)."""
    a = _phi(-eps / mu + mu / 2.0)
    b = _phi(-eps / mu - mu / 2.0)
    return a - (math.exp(eps + math.log(b)) if b > 0.0 else 0.0)


def gaussian_epsilon(sigma: float, rounds: int, delta: float) -> float:
    """epsilon at ``delta`` of ``rounds`` adaptive compositions of the Gaussian mechanism with noise multiplier ``sigma``:
    the exact conversion of ``mu = sqrt(rounds) / sigma``-GDP, solved for epsilon by bisection.  ``sigma = 0`` gives inf,
    ``rounds = 0`` gives 0."""
    if rounds <= 0:
        return 0.0
    if sigma <= 0.0:
        return math.inf
    mu = math.sqrt(rounds) / sigma
    if _gdp_delta(0.0, mu) <= delta:
        return 0.0
    lo, hi = 0.0, 1.0
    while _gdp_delta(hi, mu) > delta:
        lo, hi = hi, 2.0 * hi
        if hi > 1e6:
            return math.inf
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if _gdp_delta(mid, mu) > delta:
            lo = mid
        else:
            hi = mid
        if hi - lo <= 1e-12 * hi:
            break
    return hi


def noise_for_epsilon(epsilon: float, delta: float, rounds: int) -> float:
    """The smallest noise multiplier sigma whose ``rounds`` compositions spend at most ``epsilon`` at ``delta`` (the
    inverse of :func:`gaussian_epsilon`, by bisection)."""
    if not epsilon > 0.0:
        raise ValueError("epsilon must be > 0, got %r" % (epsilon,))
    lo, hi = 0.0, 1.0
    while gaussian_epsilon(hi, rounds, delta) > epsilon:
        lo, hi = hi, 2.0 * hi
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if gaussian_epsilon(mid, rounds, delta) > epsilon:
            lo = mid
        else:
            hi = mid
        if hi - lo <= 1e-12 * hi:
            break
    return hi


# ------------------------------------------------------------------------------------------ noise draw
def _splitmix64_finaliser(z: np.ndarray) -> np.ndarray:
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def noise_key(seed: int) -> int:
    """64-bit key of the DP noise stream of a run seeded with ``seed``."""
    z = np.array([(int(seed) ^ _DP_TAG) & _MASK64], dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(_splitmix64_finaliser(z)[0])


def dp_noise(key: int, t: int, n: int) -> np.ndarray:
    """``xi`` of DP round ``t`` for coordinates ``0 .. n - 1`` (float64): the numpy oracle of the CUDA draw
    (``csrc/comm_kernels.cu: dp_normal_pair``).

    Coordinates ``2p`` and ``2p + 1`` share the 64-bit word ``w = F(F(key + (t + 1) G) + (p + 1) G)``, arithmetic mod
    ``2**64``, with ``G = 0x9E3779B97F4A7C15`` and ``F`` the splitmix64 finaliser::

        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  z = z ^ (z >> 31)

    ``u1 = (w[63:40] + 1) 2**-24`` in ``(0, 1]``, ``u2 = w[23:0] 2**-24`` in ``[0, 1)``, ``r = sqrt(-2 ln u1)`` (Box-Muller):
    ``xi_2p = r cos(2 pi u2)``, ``xi_2p+1 = r sin(2 pi u2)``.  The draw depends on ``(key, t, i)`` only, not on the process
    layout.  24-bit uniforms bound ``|xi|`` by ``sqrt(48 ln 2) = 5.77``.
    """
    npair = (int(n) + 1) // 2
    with np.errstate(over="ignore"):
        rk = _splitmix64_finaliser(np.array([(int(key) + (int(t) + 1) * _GAMMA) & _MASK64], dtype=np.uint64))[0]
        p = np.arange(npair, dtype=np.uint64) + np.uint64(1)
        w = _splitmix64_finaliser(rk + p * np.uint64(_GAMMA))
    u1 = ((w >> np.uint64(40)) + np.uint64(1)).astype(np.float64) * 2.0 ** -24
    u2 = (w & np.uint64(0xFFFFFF)).astype(np.float64) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u1))
    out = np.empty(2 * npair, dtype=np.float64)
    out[0::2] = r * np.cos(2.0 * np.pi * u2)
    out[1::2] = r * np.sin(2.0 * np.pi * u2)
    return out[: int(n)]


def dp_line(sigma: float, clip: float, delta: float, rounds: int, planned: bool) -> str:
    """The root's ``dp:`` log line: at the start with the planned number of rounds, at the end with the rounds run."""
    return "dp: sigma=%g clip=%g*sqrt(N) delta=%g %s=%d epsilon=%.4f" % (
        sigma, clip, delta, "planned_rounds" if planned else "rounds", rounds, gaussian_epsilon(sigma, rounds, delta))
