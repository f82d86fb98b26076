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
    """

    def __init__(self, images: torch.Tensor, labels: torch.Tensor, indices: Sequence[int], batch_size: int,
                 device: torch.device, mean, std, shuffle: bool = True, seed: int = 0,
                 channels_last: bool = False, with_labels: bool = True):
        self.images, self.labels = images, labels
        self.index = torch.as_tensor(list(indices) if not isinstance(indices, torch.Tensor) else indices, dtype=torch.int64)
        self.batch_size = int(batch_size)
        self.device = torch.device(device)
        self.mean, self.std = tuple(mean), tuple(std)
        self.shuffle = shuffle
        self.gen = torch.Generator().manual_seed(seed)
        self.channels_last = channels_last
        self.with_labels = with_labels
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
            x = normalize_batch(self.images.index_select(0, idx), self.mean, self.std, self.channels_last)
            y = self.labels.index_select(0, idx)
            if x.device != self.device:
                x, y = x.to(self.device), y.to(self.device)
            yield x, y

    def _iter_host(self, order: torch.Tensor, nb: int):
        asm = self._assembler
        asm.start_epoch(order)
        for b in range(nb):
            u8, lab = asm.next_batch_to(self.device)  # pinned staging -> async H2D on the copy stream
            x = normalize_batch(u8, self.mean, self.std, self.channels_last)
            yield x, lab
