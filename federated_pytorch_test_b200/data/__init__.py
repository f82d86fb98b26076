"""Data: synthetic CIFAR10 / LOFAR sources, reference shard math, loaders, training augmentation, mixup / CutMix."""
from .cifar import (CifarData, ShardLoader, augment_batch, augment_draws, augment_key, augment_u8, make_synthetic_cifar,
                    mix_batch, mix_draws, mix_images, mix_key, normalize_batch, shard_ranges, worker_norm)
from .lofar import LofarSource, get_data_minibatch

__all__ = ["CifarData", "ShardLoader", "make_synthetic_cifar", "normalize_batch", "shard_ranges", "worker_norm",
           "augment_batch", "augment_draws", "augment_key", "augment_u8", "mix_batch", "mix_draws", "mix_images", "mix_key",
           "LofarSource", "get_data_minibatch"]
