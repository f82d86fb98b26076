"""Contrastive-Predictive-Coding networks for 8-channel LOFAR patches.

Behavioural spec: /root/reference/src/simple_models.py:436-514
(``EncoderCNN`` 16 tensors, ``ContextgenCNN`` 4, ``PredictorCNN`` 2).

The five dilated stem convolutions read the same input and their outputs are
concatenated on the channel axis: :func:`ops.functional.dilated_stem` runs them
as one wgmma launch that writes the concatenated tensor (SURVEY G6).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from .base import BlockPartitioned
from ..ops import functional as FX

_DILATIONS = (1, 2, 4, 8, 16)


class EncoderCNN(BlockPartitioned):
    BLOCK_TABLE = ((0, 9), (10, 15))

    def __init__(self, latent_dim: int = 1024):
        super().__init__()
        self.latent_dim = latent_dim
        for d in _DILATIONS:
            # padding 3d/2 keeps the 32x32 -> 16x16 geometry for every dilation
            setattr(self, "conv1_%d" % d, nn.Conv2d(8, 8, 4, stride=2, dilation=d, padding=(3 * d) // 2))
        L = latent_dim
        self.conv2 = nn.Conv2d(8 * len(_DILATIONS), L // 4, 4, stride=2, padding=1)
        self.conv3 = nn.Conv2d(L // 4, L // 2, 4, stride=2, padding=1)
        self.conv4 = nn.Conv2d(L // 2, L, 4, stride=2, padding=1)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = FX.dilated_stem(x, [getattr(self, "conv1_%d" % d) for d in _DILATIONS])
        for name in ("conv2", "conv3", "conv4"):
            h = FX.conv_act(h, getattr(self, name))
        return FX.global_avg_pool(h) if (h.shape[2] == 2 and h.shape[3] == 2 and h.shape[0] > 1) else F.avg_pool2d(h, 2).squeeze()


class ContextgenCNN(BlockPartitioned):
    """Small "pixelCNN" producing a context vector per patch-grid cell."""

    BLOCK_TABLE = ((0, 3),)

    def __init__(self, latent_dim: int = 1024):
        super().__init__()
        self.latent_dim = L = latent_dim
        self.conv1 = nn.Conv2d(L, L // 4, 1, bias=False)
        self.conv2 = nn.Conv2d(L // 4, L // 4, 2, padding=1, bias=False)
        self.conv3 = nn.Conv2d(L // 4, L // 2, 2, padding=0, bias=False)
        self.conv4 = nn.Conv2d(L // 2, L, 1, bias=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        for name in ("conv1", "conv2", "conv3", "conv4"):
            x = FX.conv_act(x, getattr(self, name))
        return x


class PredictorCNN(BlockPartitioned):
    BLOCK_TABLE = ((0, 1),)

    def __init__(self, latent_dim: int = 1024, reduced_dim: int = 64):
        super().__init__()
        self.latent_dim = latent_dim
        self.reduced_dim = reduced_dim
        self.conv1 = nn.Conv2d(latent_dim, reduced_dim, 1, bias=False)
        self.conv2 = nn.Conv2d(latent_dim, reduced_dim, 1, bias=False)

    def forward(self, latents: torch.Tensor, context: torch.Tensor):
        return FX.conv_act(latents, self.conv1, act=False), FX.conv_act(context, self.conv2, act=False)
