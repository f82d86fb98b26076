"""CIFAR10-shaped data without the network: synthetic, learnable, deterministic.

What the reference does (/root/reference/src/federated_multi.py:51-85):
torchvision CIFAR10 (download), K contiguous index shards with an off-by-one
that drops the last sample of every shard, ``SubsetRandomSampler``, batch 128,
per-worker "biased" normalisation ``mean=std=(0.5+k/100, 0.5-k/100, 0.5)`` that
is also applied to that worker's copy of the test set; K full copies of the
dataset in host RAM and a CPU transform pipeline per image.

What this module does instead (SURVEY G22, §7.1 ``data/``):

* one uint8 NHWC copy of the dataset, resident in HBM (150 MB) — or in pinned
  host memory for the end-to-end path, where a native batch assembler
  (``runtime/batch_loader.cpp``) gathers the next batch while the GPU works;
* batches are index gathers on the device; normalisation (+ layout change) is
  one fused kernel (:func:`ops.cuda_ops.normalize_u8`) instead of
  ``ToTensor``/``Normalize`` per PIL image on the CPU;
* identical shard arithmetic (including the off-by-one, switchable) and
  identical per-worker normalisation constants.

Training augmentation (opt-in, ``--augment``; the reference has none) is torchvision's ``RandomCrop(32, padding=4)``
followed by ``RandomHorizontalFlip(0.5)`` on the raw uint8 image, before normalisation, so padded pixels come out as
``-mean/std``.  On the CUDA fast path it is fused into the input kernel
(:func:`ops.cuda_ops.augment_normalize_u8`: gather + crop + flip + normalisation + layout, one launch per batch);
:func:`augment_batch` is the ATen composition used on the CPU and with ``fast=False``.  The random draws are
counter-based, not a ``torch.Generator``: sample ``i`` of a batch takes :func:`augment_draws` ``(key, counter + i)``, where
``key`` is fixed per worker (:func:`augment_key`) and ``counter`` is the number of samples its loader has handed out.
So augmentation does not touch the shuffle generator, and a batch does not depend on the process topology.

Mixup and CutMix (opt-in, ``--mixup_alpha`` / ``--cutmix_alpha``) mix sample ``i`` of a training batch with sample
``n-1-i`` after the crop / flip and the normalisation.  The draw is one per batch, made on the host by :func:`mix_draws`
from the same loader counter under a second key (:func:`mix_key`); on the CUDA fast path the whole input stage stays one
launch (:func:`ops.cuda_ops.mix_normalize_u8`), and :func:`mix_batch` is the ATen composition.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

TRAIN_SIZE = 50000
TEST_SIZE = 10000
NUM_CLASSES = 10


# ----------------------------------------------------------------------------
# dataset synthesis
# ----------------------------------------------------------------------------
def _class_templates(gen: torch.Generator) -> torch.Tensor:
    """Ten smooth, well separated 32x32x3 patterns in [-1, 1]."""
    coarse = torch.randn(NUM_CLASSES, 3, 4, 4, generator=gen)
    up = torch.nn.functional.interpolate(coarse, size=(32, 32), mode="bilinear", align_corners=False)
    up = up / up.abs().amax(dim=(1, 2, 3), keepdim=True)
    return up.permute(0, 2, 3, 1).contiguous()  # [10,32,32,3]


def make_synthetic_cifar(train: bool, seed: int = 1234, size: Optional[int] = None,
                         noise: float = 0.6) -> Tuple[torch.Tensor, torch.Tensor]:
    """uint8 images ``[n,32,32,3]`` and int64 labels ``[n]``.

    image = clip(128 + 56*template[label] (random flip / gain) + 56*noise*N(0,1)).
    A small CNN reaches well above chance within an epoch, so accuracy curves and
    "rounds to target accuracy" are meaningful (SURVEY §6.3).
    """
    n = size if size is not None else (TRAIN_SIZE if train else TEST_SIZE)
    gen = torch.Generator().manual_seed(seed)
    templates = _class_templates(gen)
    split_gen = torch.Generator().manual_seed(seed + (1 if train else 2))
    labels = torch.randint(0, NUM_CLASSES, (n,), generator=split_gen)
    images = torch.empty(n, 32, 32, 3, dtype=torch.uint8)
    chunk = 5000
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        lab = labels[a:b]
        base = templates[lab]
        gain = 0.6 + 0.8 * torch.rand(b - a, 1, 1, 1, generator=split_gen)
        flip = torch.rand(b - a, generator=split_gen) < 0.5
        base = torch.where(flip.view(-1, 1, 1, 1), base.flip(2), base)
        img = 128.0 + 56.0 * gain * base + 56.0 * noise * torch.randn(b - a, 32, 32, 3, generator=split_gen)
        images[a:b] = img.clamp_(0, 255).to(torch.uint8)
    return images, labels


# ----------------------------------------------------------------------------
# sharding and per-worker normalisation
# ----------------------------------------------------------------------------
def shard_ranges(K: int, n: int = TRAIN_SIZE, drop_last_sample: bool = True) -> List[range]:
    """Index range of every worker's shard.

    ``per = floor((n+K-1)/K)``; shard k is ``[per*k, per*(k+1)-1)`` — the ``-1``
    is the reference's off-by-one (SURVEY Q1: K=8 -> 6 249 samples each).
    ``drop_last_sample=False`` gives the intended ``[per*k, min(per*(k+1), n))``.
    """
    per = math.floor((n + K - 1) / K)
    out = []
    for k in range(K):
        if drop_last_sample:
            hi = per * (k + 1) - 1
            out.append(range(per * k, hi) if hi <= n else range(per * k, n))
        else:
            out.append(range(per * k, min(per * (k + 1), n)))
    return out


DIRICHLET_MAX_DRAWS = 100


def dirichlet_shards(labels, K: int, alpha: float, seed: int, min_size: int) -> List[np.ndarray]:
    """Label-skewed shards of the K workers (Hsu et al. 2019): sorted int64 index arrays, disjoint, covering every sample.

    One ``numpy.random.Generator(PCG64(seed))`` draws everything.  For each class ``c`` in ascending order, the class's
    sample indices are shuffled, ``p ~ Dir(alpha 1_K)`` is drawn and the shuffled indices are cut at
    ``floor(cumsum(p) n_c)`` (worker ``k`` gets the ``k``-th piece).  If a shard ends up with fewer than ``min_size``
    samples, the whole partition is drawn again from the same generator; after ``DIRICHLET_MAX_DRAWS`` draws a
    ``ValueError`` names ``alpha`` and ``K``.  Every rank computes the full partition, so every rank knows every shard size.
    """
    lab = np.asarray(labels.cpu().numpy() if torch.is_tensor(labels) else labels).astype(np.int64)
    if not (K >= 1 and alpha > 0.0):
        raise ValueError("dirichlet_shards needs K >= 1 and alpha > 0, got K = %r, alpha = %r" % (K, alpha))
    rng = np.random.Generator(np.random.PCG64(int(seed)))
    classes = np.unique(lab)
    for _ in range(DIRICHLET_MAX_DRAWS):
        parts: List[List[np.ndarray]] = [[] for _ in range(K)]
        for c in classes:
            idx = np.flatnonzero(lab == c)
            rng.shuffle(idx)
            p = rng.dirichlet(np.full(K, float(alpha)))
            cuts = np.floor(np.cumsum(p) * idx.size).astype(np.int64)
            cuts[-1] = idx.size                       # cumsum(p) may end a rounding error below 1
            for k, piece in enumerate(np.split(idx, cuts[:-1])):
                parts[k].append(piece)
        shards = [np.sort(np.concatenate(p)) for p in parts]
        if min(s.size for s in shards) >= min_size:
            return shards
    raise ValueError("dirichlet_shards: no partition with at least %d samples per worker in %d draws at alpha = %g, "
                     "K = %d; raise dirichlet_alpha or lower K" % (min_size, DIRICHLET_MAX_DRAWS, alpha, K))


def class_histogram(labels, shards: Sequence[np.ndarray], num_classes: int = NUM_CLASSES) -> List[List[int]]:
    """Per-worker sample counts of every class: ``[K][num_classes]``."""
    lab = np.asarray(labels.cpu().numpy() if torch.is_tensor(labels) else labels).astype(np.int64)
    return [np.bincount(lab[np.asarray(s, dtype=np.int64)], minlength=num_classes).tolist() for s in shards]


def worker_norm(ck: int, biased: bool = True) -> Tuple[Tuple[float, float, float], Tuple[float, float, float]]:
    """(mean, std) applied after scaling pixels to [0,1]; mean == std in the reference."""
    if biased:
        v = (0.5 + ck / 100, 0.5 - ck / 100, 0.5)
    else:
        v = (0.5, 0.5, 0.5)
    return v, v


def normalize_batch(u8_nhwc: torch.Tensor, mean, std, channels_last: bool = False) -> torch.Tensor:
    """uint8 NHWC -> float32 NCHW-shaped tensor ``(x/255 - mean)/std``.

    With ``channels_last=True`` the result keeps NHWC memory (a permuted view),
    which is what the sm_90a conv path consumes; on CUDA this is one kernel.
    """
    if u8_nhwc.is_cuda:
        from ..ops import functional as FX

        if FX.fast_path_enabled():
            from ..ops import cuda_ops

            return cuda_ops.normalize_u8(u8_nhwc, mean, std, channels_last)
    m = torch.tensor(mean, dtype=torch.float32, device=u8_nhwc.device)
    s = torch.tensor(std, dtype=torch.float32, device=u8_nhwc.device)
    x = (u8_nhwc.to(torch.float32) / 255.0 - m) / s
    x = x.permute(0, 3, 1, 2)
    return x if channels_last else x.contiguous()


# ----------------------------------------------------------------------------
# training augmentation: random padded crop + horizontal flip, counter-based draws
# ----------------------------------------------------------------------------
AUG_PAD = 4
_MASK64 = (1 << 64) - 1
_GOLDEN_GAMMA = 0x9E3779B97F4A7C15


def _splitmix64_finaliser(z: np.ndarray) -> np.ndarray:
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def augment_key(seed: int, ck: int) -> int:
    """64-bit augmentation key of worker ``ck`` in a run seeded with ``seed``."""
    z = np.array([((int(seed) & 0xFFFFFFFF) << 32) | (int(ck) & 0xFFFFFFFF)], dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(_splitmix64_finaliser(z)[0])


def augment_draws(key: int, counter: int, n: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Crop offsets and flip bits of samples ``counter .. counter + n - 1`` of a loader with key ``key``.

    Sample ``c`` takes the 64-bit word ``z = F(key + (c + 1) * 0x9E3779B97F4A7C15 mod 2**64)``, i.e. output ``c`` of a
    splitmix64 generator seeded with ``key``, where ``F`` is the splitmix64 finaliser::

        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  z = z ^ (z >> 31)

    and maps its bits to ``dx = (z[31:0] * 9) >> 32``, ``dy = (z[62:32] * 9) >> 31`` (both in ``[0, 8]``) and
    ``flip = z[63]``.  The augmented image is ``out[h][w] = img[h + dy - 4][w' + dx - 4]`` with ``w' = W - 1 - w`` when
    flipped and ``w`` otherwise; pixels outside the image are 0.  The CUDA kernel evaluates the same function bit for
    bit.  Returns ``dx``, ``dy`` (int64) and ``flip`` (bool), each of length ``n``.
    """
    c = np.arange(n, dtype=np.uint64) + np.uint64((int(counter) + 1) & _MASK64)
    with np.errstate(over="ignore"):
        z = _splitmix64_finaliser(np.uint64(int(key) & _MASK64) + c * np.uint64(_GOLDEN_GAMMA))
    dx = ((z & np.uint64(0xFFFFFFFF)) * np.uint64(9)) >> np.uint64(32)
    dy = (((z >> np.uint64(32)) & np.uint64(0x7FFFFFFF)) * np.uint64(9)) >> np.uint64(31)
    flip = (z >> np.uint64(63)) != 0
    return (torch.from_numpy(dx.astype(np.int64)), torch.from_numpy(dy.astype(np.int64)),
            torch.from_numpy(flip.astype(np.bool_)))


def augment_u8(u8_nhwc: torch.Tensor, key: int, counter: int) -> torch.Tensor:
    """The augmented uint8 NHWC batch (zero padding, gather, flip) of :func:`augment_draws`, on ``u8_nhwc``'s device."""
    n, H, W, _ = u8_nhwc.shape
    dev = u8_nhwc.device
    dx, dy, flip = (t.to(dev) for t in augment_draws(key, counter, n))
    padded = torch.nn.functional.pad(u8_nhwc, (0, 0, AUG_PAD, AUG_PAD, AUG_PAD, AUG_PAD))   # [n, H+8, W+8, C], zeros
    hs = torch.arange(H, device=dev)
    ws = torch.arange(W, device=dev)
    rows = hs.view(1, H) + dy.view(n, 1)                                                     # h + dy in padded coordinates
    cols = torch.where(flip.view(n, 1), (W - 1 - ws).view(1, W), ws.view(1, W)) + dx.view(n, 1)
    return padded[torch.arange(n, device=dev).view(n, 1, 1), rows.view(n, H, 1), cols.view(n, 1, W)]


def augment_batch(u8_nhwc: torch.Tensor, mean, std, channels_last: bool, key: int, counter: int) -> torch.Tensor:
    """Augmented, normalised training batch: :func:`augment_u8` then :func:`normalize_batch` (the ATen composition the
    fused kernel is checked against)."""
    return normalize_batch(augment_u8(u8_nhwc, key, counter), mean, std, channels_last)


# ----------------------------------------------------------------------------
# mixup / CutMix: one draw per batch, sample i mixed with sample n-1-i
# ----------------------------------------------------------------------------
MIX_WORDS = 256                      # splitmix64 words per batch sub-stream
_MIX_TAG = 0x6D69782D63757421       # domain tag: mixing keys never coincide with augmentation keys


def mix_key(seed: int, ck: int) -> int:
    """64-bit mixup / CutMix key of worker ``ck`` in a run seeded with ``seed`` (the :func:`augment_key` input with a domain
    tag folded in before the finaliser, so the two keys differ)."""
    z = np.array([(((int(seed) & 0xFFFFFFFF) << 32) | (int(ck) & 0xFFFFFFFF)) ^ _MIX_TAG], dtype=np.uint64)
    with np.errstate(over="ignore"):
        return int(_splitmix64_finaliser(z)[0])


def _splitmix64_word(key: int, i: int) -> int:
    z = (key + (i + 1) * _GOLDEN_GAMMA) & _MASK64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK64
    return z ^ (z >> 31)


class _Words:
    """Uniforms of one batch's sub-stream: word ``j`` is output ``counter * 256 + j`` of splitmix64 seeded with ``key``."""

    def __init__(self, key: int, counter: int, first: int):
        self.key, self.base, self.j = int(key) & _MASK64, (int(counter) * MIX_WORDS) & _MASK64, first

    def word(self, j: int) -> int:
        return _splitmix64_word(self.key, (self.base + j) & _MASK64)

    def uniform(self) -> float:
        """The next word as a float64 in the open interval (0, 1)."""
        if self.j >= MIX_WORDS:
            raise RuntimeError("mix_draws: the batch's %d-word sub-stream is exhausted" % MIX_WORDS)
        w = self.word(self.j)
        self.j += 1
        return ((w >> 11) + 0.5) * 2.0 ** -53

    def log_gamma(self, alpha: float) -> float:
        """log of a Gamma(alpha, 1) variate (Marsaglia & Tsang 2000; for alpha < 1 a Gamma(alpha + 1) variate times
        U^(1/alpha)).  In logs so that the Beta ratio of two tiny variates is still defined."""
        boost = 0.0
        if alpha < 1.0:
            boost = math.log(self.uniform()) / alpha
            alpha += 1.0
        d = alpha - 1.0 / 3.0
        c = 1.0 / math.sqrt(9.0 * d)
        while True:
            x = math.sqrt(-2.0 * math.log(self.uniform())) * math.cos(2.0 * math.pi * self.uniform())   # Box-Muller
            v = 1.0 + c * x
            if v <= 0.0:
                continue
            v = v * v * v
            if math.log(self.uniform()) < 0.5 * x * x + d - d * v + d * math.log(v):
                return math.log(d * v) + boost


def mix_draws(key: int, counter: int, n: int, H: int, W: int, mixup_alpha: float,
              cutmix_alpha: float) -> Tuple[str, float, Tuple[int, int, int, int], float]:
    """Mixing draw of the batch of ``n`` ``H x W`` samples whose first sample has loader counter ``counter``.

    A pure float64 function of its arguments.  The batch owns the splitmix64 sub-stream of :func:`augment_draws`' generator
    (same finaliser ``F``) at outputs ``counter * 256 .. counter * 256 + 255``: word ``j`` is
    ``F(key + (counter * 256 + j + 1) * 0x9E3779B97F4A7C15 mod 2**64)``, and a word ``w`` is the uniform
    ``((w >> 11) + 1/2) 2**-53`` in (0, 1).  Consecutive batches of a loader have counters at least 1 apart, so their
    sub-streams never overlap.  Word 0's top bit picks CutMix (1) or mixup (0) when both alphas are > 0; otherwise the
    mode whose alpha is > 0 is used.  Words 1 and 2 give the CutMix centre ``cy = (w1[63:32] * H) >> 32`` and
    ``cx = (w2[63:32] * W) >> 32``.  From word 3 on, ``lam = G1 / (G1 + G2) ~ Beta(alpha, alpha)`` with Marsaglia-Tsang
    Gamma variates (Box-Muller normals; for alpha < 1 boosted by ``U^(1/alpha)``); a draw that would need more than 256
    words raises ``RuntimeError`` (rejection rates make this practically impossible).

    Mixup: ``x_i = lam a_i + (1 - lam) a_{n-1-i}`` and ``lam_eff = lam``.  CutMix: ``r = sqrt(1 - lam)``,
    ``cut_h = int(H r)``, ``cut_w = int(W r)``; the box ``[clip(cy - cut_h // 2, 0, H), clip(cy + cut_h // 2, 0, H))`` x
    the same in x takes its pixels from the partner, and ``lam_eff = 1 - box area / (H W)``.

    Returns ``(mode, lam, (y0, y1, x0, x1), lam_eff)`` with ``mode`` 'mixup' or 'cutmix'; the box is empty for mixup.
    """
    if not (mixup_alpha > 0.0 or cutmix_alpha > 0.0):
        raise ValueError("mix_draws needs mixup_alpha > 0 or cutmix_alpha > 0")
    words = _Words(key, counter, 3)
    if mixup_alpha > 0.0 and cutmix_alpha > 0.0:
        cutmix = bool(words.word(0) >> 63)
    else:
        cutmix = cutmix_alpha > 0.0
    alpha = cutmix_alpha if cutmix else mixup_alpha
    lg1, lg2 = words.log_gamma(alpha), words.log_gamma(alpha)
    d = lg2 - lg1
    lam = 1.0 / (1.0 + math.exp(d)) if d < 700.0 else 0.0
    if not cutmix:
        return "mixup", lam, (0, 0, 0, 0), lam
    cy = ((words.word(1) >> 32) * H) >> 32
    cx = ((words.word(2) >> 32) * W) >> 32
    r = math.sqrt(1.0 - lam)
    cut_h, cut_w = int(H * r), int(W * r)
    y0, y1 = min(max(cy - cut_h // 2, 0), H), min(max(cy + cut_h // 2, 0), H)
    x0, x1 = min(max(cx - cut_w // 2, 0), W), min(max(cx + cut_w // 2, 0), W)
    return "cutmix", lam, (y0, y1, x0, x1), 1.0 - (y1 - y0) * (x1 - x0) / float(H * W)


def mix_factors(lam: float) -> Tuple[float, float]:
    """``(float32(lam), float32(1 - lam))`` rounded from float64, as Python floats: the mixup blend's two factors."""
    return float(np.float32(lam)), float(np.float32(1.0 - lam))


def mix_images(x: torch.Tensor, mode: str, lam: float, box: Tuple[int, int, int, int]) -> torch.Tensor:
    """Mixup blend or CutMix paste of a normalised ``[n, 3, H, W]`` batch with its reverse ``x.flip(0)``, in ATen ops.
    Mixup is ``x * lam_f + x.flip(0) * mlam_f`` in float32 (:func:`mix_factors`), which the kernel reproduces bit for bit."""
    partner = x.flip(0)
    if mode == "mixup":
        lam_f, mlam_f = mix_factors(lam)
        out = x * lam_f + partner * mlam_f
    else:
        y0, y1, x0, x1 = box
        out = x.clone()
        out[:, :, y0:y1, x0:x1] = partner[:, :, y0:y1, x0:x1]
    if x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous():
        return out.contiguous(memory_format=torch.channels_last)
    return out.contiguous()


def mix_batch(u8_nhwc: torch.Tensor, mean, std, channels_last: bool, aug_key: Optional[int], key: int, counter: int,
              mixup_alpha: float, cutmix_alpha: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """Mixed training batch and its ``lam_eff`` (a one-float32 tensor on ``u8_nhwc``'s device): crop + flip
    (:func:`augment_batch`, when ``aug_key`` is not None) or :func:`normalize_batch`, then :func:`mix_images` with the draw
    :func:`mix_draws` ``(key, counter, ...)``.  The ATen composition used on the CPU and with ``fast=False``."""
    n, H, W, _ = u8_nhwc.shape
    if aug_key is None:
        x = normalize_batch(u8_nhwc, mean, std, channels_last)
    else:
        x = augment_batch(u8_nhwc, mean, std, channels_last, aug_key, counter)
    mode, lam, box, lam_eff = mix_draws(key, counter, n, H, W, mixup_alpha, cutmix_alpha)
    return mix_images(x, mode, lam, box), torch.tensor([lam_eff], dtype=torch.float32, device=u8_nhwc.device)


# ----------------------------------------------------------------------------
@dataclass
class CifarData:
    """The four arrays every driver needs."""

    train_images: torch.Tensor
    train_labels: torch.Tensor
    test_images: torch.Tensor
    test_labels: torch.Tensor

    @staticmethod
    def synthetic(seed: int = 1234, train_size: Optional[int] = None, test_size: Optional[int] = None,
                  noise: float = 0.6) -> "CifarData":
        tr = make_synthetic_cifar(True, seed, train_size, noise)
        te = make_synthetic_cifar(False, seed, test_size, noise)
        return CifarData(tr[0], tr[1], te[0], te[1])

    @staticmethod
    def from_torchvision(root: str = "./torchdata") -> "CifarData":
        """Real CIFAR10 if the files already exist locally (never downloads)."""
        import torchvision

        tr = torchvision.datasets.CIFAR10(root=root, train=True, download=False)
        te = torchvision.datasets.CIFAR10(root=root, train=False, download=False)
        return CifarData(torch.from_numpy(np.asarray(tr.data)), torch.tensor(tr.targets),
                         torch.from_numpy(np.asarray(te.data)), torch.tensor(te.targets))

    def to(self, device, pin: bool = False) -> "CifarData":
        def mv(t):
            if pin and torch.cuda.is_available():
                return t.pin_memory()
            return t.to(device)
        return CifarData(mv(self.train_images), mv(self.train_labels), mv(self.test_images), mv(self.test_labels))


class ShardLoader:
    """Mini-batches of one worker's shard, fresh random order each epoch
    (``SubsetRandomSampler`` semantics), last partial batch kept.

    ``images``/``labels`` may live on the compute device (HBM-resident dataset)
    or in pinned host memory; in the latter case each batch is gathered by the
    native batch assembler and copied H2D asynchronously, double buffered.

    ``augment=True`` crops and flips every sample at random (see the module docstring) with draws keyed by ``aug_key``.
    ``mixup_alpha`` / ``cutmix_alpha`` > 0 mix every batch with its reverse (:func:`mix_draws`, keyed by ``mix_key``) and
    yield ``(x, y, lam)``, ``lam`` a one-float32 tensor holding ``lam_eff`` on the batch's device; unmixed batches are
    ``(x, y)``.  With augmentation or mixing, ``aug_counter`` counts the samples handed out so far and advances by the batch
    size with every yielded batch.
    """

    def __init__(self, images: torch.Tensor, labels: torch.Tensor, indices: Sequence[int], batch_size: int,
                 device: torch.device, mean, std, shuffle: bool = True, seed: int = 0,
                 channels_last: bool = False, with_labels: bool = True, augment: bool = False, aug_key: int = 0,
                 mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0, mix_key: int = 0):
        self.images, self.labels = images, labels
        self.index = torch.as_tensor(list(indices) if not isinstance(indices, torch.Tensor) else indices, dtype=torch.int64)
        self.batch_size = int(batch_size)
        self.device = torch.device(device)
        self.mean, self.std = tuple(mean), tuple(std)
        self.shuffle = shuffle
        self.gen = torch.Generator().manual_seed(seed)
        self.channels_last = channels_last
        self.with_labels = with_labels
        self.augment = bool(augment)
        self.aug_key = int(aug_key) & _MASK64
        self.aug_counter = 0
        self.mixup_alpha, self.cutmix_alpha = float(mixup_alpha), float(cutmix_alpha)
        self.mixing = self.mixup_alpha > 0.0 or self.cutmix_alpha > 0.0
        self.mix_key = int(mix_key) & _MASK64
        self.prefetch_order = True     # see _device_order(); a loader abandoned mid-epoch simply never prefetches
        self._next_order = None
        self.host_resident = not images.is_cuda and self.device.type == "cuda"
        self._assembler = None
        if self.host_resident:
            from ..runtime import batch_loader

            self._assembler = batch_loader.BatchAssembler(images, labels, self.batch_size)
        self.h2d_bytes_per_batch = self.batch_size * (images[0].numel() * images.element_size() + labels.element_size())

    def __len__(self) -> int:
        return -(-len(self.index) // self.batch_size)

    @property
    def num_samples(self) -> int:
        return len(self.index)

    def _order(self) -> torch.Tensor:
        if not self.shuffle:
            return self.index
        return self.index[torch.randperm(len(self.index), generator=self.gen)]

    def _device_order(self) -> torch.Tensor:
        """This epoch's sample order on the dataset's device.  Shuffled loaders draw the NEXT epoch's permutation right
        after handing out the last batch of the current one (while the GPU is still busy with it), so that the start of
        a round — the host's critical path after an aggregation — costs nothing.  The generator is consumed in the
        same sequence as without the prefetch (one ``randperm`` per epoch)."""
        nxt = getattr(self, "_next_order", None)
        self._next_order = None
        if nxt is not None:
            return nxt
        order = self._order()
        if self.images.is_cuda:
            return order.pin_memory().to(self.images.device, non_blocking=True) if torch.cuda.is_available() else order.to(self.images.device)
        return order

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        nb = len(self)
        if self._assembler is not None:
            yield from self._iter_host(self._order(), nb)
            return
        dev_order = self._device_order()
        for b in range(nb):
            if b == nb - 1 and self.shuffle and self.prefetch_order:
                self._next_order = None
                self._next_order = self._device_order()
            idx = dev_order[b * self.batch_size:(b + 1) * self.batch_size]
            if self.mixing:
                x, lam = self._mixed(self.images, idx)
            elif self.augment:
                x = self._augmented(self.images, idx)
            else:
                x = normalize_batch(self.images.index_select(0, idx), self.mean, self.std, self.channels_last)
            y = self.labels.index_select(0, idx)
            if x.device != self.device:
                x, y = x.to(self.device), y.to(self.device)
            if self.mixing:
                yield x, y, lam.to(self.device)
            else:
                yield x, y

    def _iter_host(self, order: torch.Tensor, nb: int):
        asm = self._assembler
        asm.start_epoch(order)
        for b in range(nb):
            u8, lab = asm.next_batch_to(self.device)  # pinned staging -> async H2D on the copy stream
            if self.mixing:
                x, lam = self._mixed(u8, None)
                yield x, lab, lam
                continue
            if self.augment:
                x = self._augmented(u8, None)
            else:
                x = normalize_batch(u8, self.mean, self.std, self.channels_last)
            yield x, lab

    def _augmented(self, images: torch.Tensor, idx: Optional[torch.Tensor]) -> torch.Tensor:
        """Augmented, normalised batch of ``images[idx]`` (``images`` itself when ``idx`` is None); advances the counter."""
        counter = self.aug_counter
        self.aug_counter += images.shape[0] if idx is None else idx.numel()
        if images.is_cuda:
            from ..ops import functional as FX

            if FX.fast_path_enabled():
                from ..ops import cuda_ops

                return cuda_ops.augment_normalize_u8(images, idx, self.aug_key, counter, self.mean, self.std,
                                                     self.channels_last)   # gather + crop + flip + normalise: one launch
        u8 = images if idx is None else images.index_select(0, idx)
        return augment_batch(u8, self.mean, self.std, self.channels_last, self.aug_key, counter)

    def _mixed(self, images: torch.Tensor, idx: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """Mixed (and, with ``augment``, cropped and flipped), normalised batch of ``images[idx]`` (``images`` itself when
        ``idx`` is None) and its ``lam_eff`` tensor; advances the counter."""
        counter = self.aug_counter
        n = images.shape[0] if idx is None else idx.numel()
        self.aug_counter += n
        aug_key = self.aug_key if self.augment else None
        if images.is_cuda:
            from ..ops import functional as FX

            if FX.fast_path_enabled():
                from ..ops import cuda_ops

                draw = mix_draws(self.mix_key, counter, n, images.shape[1], images.shape[2], self.mixup_alpha,
                                 self.cutmix_alpha)
                return cuda_ops.mix_normalize_u8(images, idx, aug_key, counter, self.mean, self.std, self.channels_last,
                                                 draw)   # gather + crop + flip + normalise + mix: one launch
        u8 = images if idx is None else images.index_select(0, idx)
        return mix_batch(u8, self.mean, self.std, self.channels_last, aug_key, self.mix_key, counter, self.mixup_alpha,
                         self.cutmix_alpha)
