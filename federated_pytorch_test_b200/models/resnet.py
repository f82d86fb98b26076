"""CIFAR-style ResNet (ELU activations, no stem max-pool).

Behavioural spec: /root/reference/src/simple_models.py:132-237.  Parameter
registration order, attribute names (``conv1/bn1/layer1..4/linear``,
``shortcut.0/.1``) and the hand-specified block tables are kept so that block
indices, message sizes (SURVEY §2.2) and checkpoints carry over.

What is different: every ``conv -> BatchNorm(train) -> (+residual) -> ELU``
group goes through ONE call, :func:`ops.functional.conv_bn_act`, which on
an H100 runs the hand-written sm_90a path (wgmma implicit-GEMM conv whose
epilogue emits the BN batch statistics, then one fused normalise+residual+ELU
pass; NHWC activations) and otherwise falls back to the ATen composition with
identical semantics.
"""
from __future__ import annotations

from typing import List, Type

import torch
import torch.nn as nn
import torch.nn.functional as F

from .base import BlockPartitioned
from ..ops import functional as FX


def _conv3x3(cin: int, cout: int, stride: int) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, kernel_size=3, stride=stride, padding=1, bias=False)


def _conv1x1(cin: int, cout: int, stride: int) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, kernel_size=1, stride=stride, bias=False)


class _Residual(nn.Module):
    """Common shortcut handling for both block flavours."""

    expansion = 1

    def _make_shortcut(self, in_planes: int, out_planes: int, stride: int) -> None:
        if stride != 1 or in_planes != out_planes:
            self.shortcut = nn.Sequential(_conv1x1(in_planes, out_planes, stride), nn.BatchNorm2d(out_planes))
        else:
            self.shortcut = nn.Sequential()

    def _skip(self, x: torch.Tensor) -> torch.Tensor:
        if len(self.shortcut) == 0:
            return x
        return FX.conv_bn_act(x, self.shortcut[0], self.shortcut[1], act=False)


class BasicBlock(_Residual):
    expansion = 1

    def __init__(self, in_planes: int, planes: int, stride: int = 1):
        super().__init__()
        self.conv1 = _conv3x3(in_planes, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv3x3(planes, planes, 1)
        self.bn2 = nn.BatchNorm2d(planes)
        self._make_shortcut(in_planes, planes * self.expansion, stride)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if len(self.shortcut) == 0:      # identity shortcut: the input doubles as the residual (see FX.conv_bn_act_skip)
            h, skip = FX.conv_bn_act_skip(x, self.conv1, self.bn1)
            return FX.conv_bn_act(h, self.conv2, self.bn2, residual=skip, act=True)
        h = FX.conv_bn_act(x, self.conv1, self.bn1, act=True)
        return FX.conv_bn_act(h, self.conv2, self.bn2, residual=self._skip(x), act=True)


class Bottleneck(_Residual):
    expansion = 4

    def __init__(self, in_planes: int, planes: int, stride: int = 1):
        super().__init__()
        self.conv1 = _conv1x1(in_planes, planes, 1)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = _conv3x3(planes, planes, stride)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = _conv1x1(planes, planes * self.expansion, 1)
        self.bn3 = nn.BatchNorm2d(planes * self.expansion)
        self._make_shortcut(in_planes, planes * self.expansion, stride)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = FX.conv_bn_act(x, self.conv1, self.bn1, act=True)
        h = FX.conv_bn_act(h, self.conv2, self.bn2, act=True)
        return FX.conv_bn_act(h, self.conv3, self.bn3, residual=self._skip(x), act=True)


class ResNet(BlockPartitioned):
    _TABLES = {
        18: ((0, 2), (3, 8), (9, 14), (15, 23), (24, 29), (30, 38), (39, 44), (45, 53), (54, 59), (60, 61)),
        # NB: the ResNet9 table does not follow module boundaries (SURVEY §2.2); kept verbatim.
        9: ((0, 2), (3, 8), (9, 14), (15, 17), (18, 23), (24, 29), (30, 32), (33, 37)),
    }
    LINEAR_IDS = ()  # empty in the reference (simple_models.py:229-230)

    def __init__(self, block: Type[_Residual], num_blocks: List[int], qualifier: int, num_classes: int = 10):
        super().__init__()
        self.qualifier = qualifier
        self.in_planes = 64
        self.conv1 = _conv3x3(3, 64, 1)
        self.bn1 = nn.BatchNorm2d(64)
        widths = (64, 128, 256, 512)
        strides = (1, 2, 2, 2)
        for i, (w, s, n) in enumerate(zip(widths, strides, num_blocks), start=1):
            setattr(self, "layer%d" % i, self._make_layer(block, w, n, s))
        self.linear = nn.Linear(512 * block.expansion, num_classes)

    def _make_layer(self, block, planes: int, count: int, stride: int) -> nn.Sequential:
        stages = []
        for s in [stride] + [1] * (count - 1):
            stages.append(block(self.in_planes, planes, s))
            self.in_planes = planes * block.expansion
        return nn.Sequential(*stages)

    def train_order_block_ids(self):
        key = 18 if self.qualifier == 18 else 9
        return [list(b) for b in self._TABLES[key]]

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = FX.conv_bn_act(x, self.conv1, self.bn1, act=True)
        for name in ("layer1", "layer2", "layer3", "layer4"):
            h = getattr(self, name)(h)
        return FX.pool_linear(h, self.linear, window=4)


def ResNet18() -> ResNet:
    return ResNet(BasicBlock, [2, 2, 2, 2], qualifier=18)


def ResNet9() -> ResNet:
    return ResNet(BasicBlock, [1, 1, 1, 1], qualifier=9)
