"""Functional entry points used by the model zoo.

Each function has exactly two implementations:

* the sm_90a path in :mod:`..ops.cuda_ops` (hand-written kernels from
  ``csrc/``), selected when the tensors live on a CUDA device and the fast
  path is enabled (default on an H100);
* the ATen composition below, used on CPU (tests, plumbing runs) and as the
  numerical oracle for the kernels.

There is no third backend and no tracing compiler in between.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

_FAST = {"enabled": os.environ.get("FEDB200_FAST", "1") != "0"}


def set_fast_path(flag: bool) -> None:
    """Globally enable/disable the hand-written CUDA path (CUDA tensors only)."""
    _FAST["enabled"] = bool(flag)


def fast_path_enabled() -> bool:
    return _FAST["enabled"]


def _use_fast(x: torch.Tensor) -> bool:
    return _FAST["enabled"] and x.is_cuda


def conv_bn_act(
    x: torch.Tensor,
    conv: nn.Conv2d,
    bn: nn.BatchNorm2d,
    residual: Optional[torch.Tensor] = None,
    act: bool = True,
) -> torch.Tensor:
    """``ELU?( BN_train(conv(x)) (+ residual) )`` — one ResNet group.

    Semantics follow /root/reference/src/simple_models.py:149-154: batch
    statistics are used (and running statistics updated) whenever the module
    is in training mode, which in the reference is *always* (SURVEY Q4).  In
    eval mode (``bn.eval()``) the running statistics normalise and stay
    unchanged; without a gradient to compute that runs as one kernel.

    ``bn`` may also be an ``nn.GroupNorm`` (the GroupNorm ResNets): it
    normalises every sample on its own, in training and eval mode alike.
    """
    if _use_fast(x):
        from . import cuda_ops

        if cuda_ops.conv_bn_act_eval_supported(x, conv, bn, residual):
            return cuda_ops.conv_bn_act_eval(x, conv, bn, residual, act)
        if cuda_ops.conv_bn_act_supported(x, conv, bn):
            return cuda_ops.conv_bn_act(x, conv, bn, residual, act)
        if cuda_ops.conv_gn_act_supported(x, conv, bn):
            return cuda_ops.conv_gn_act(x, conv, bn, residual, act)
    y = F.conv2d(x, conv.weight, conv.bias, conv.stride, conv.padding, conv.dilation, conv.groups)
    y = bn(y)
    if residual is not None:
        y = y + residual
    return F.elu(y) if act else y


def pool_linear(x: torch.Tensor, linear: nn.Linear, window: int = 4) -> torch.Tensor:
    """``linear(flatten(avg_pool2d(x, window)))`` (simple_models.py:213-215)."""
    if _use_fast(x):
        from . import cuda_ops

        if cuda_ops.pool_linear_supported(x, linear, window):
            return cuda_ops.pool_linear(x, linear, window)
    y = F.avg_pool2d(x, window)
    return F.linear(y.reshape(y.shape[0], -1), linear.weight, linear.bias)


def conv_act(x: torch.Tensor, conv: nn.Module, act: bool = True) -> torch.Tensor:
    """``ELU?(conv(x))`` for the bias-carrying convs / transposed convs of the VAE and CPC nets
    (/root/reference/src/simple_models.py:249-265, :441-451, :478-481, :503-504).  On the GPU: wgmma implicit GEMM with bias +
    ELU in the epilogue and hand-written backward kernels (cuda_ops._ConvAct); 1x1 convs on odd-sized latent grids run
    on the dense-layer GEMM kernels, other small convs on the direct-convolution kernel."""
    if _use_fast(x):
        from . import cuda_ops

        if cuda_ops.conv_act_supported(x, conv) or cuda_ops.conv_transpose_act_supported(x, conv):
            return cuda_ops.conv_act(x, conv, act)
        if cuda_ops.conv1x1_supported(x, conv):
            return cuda_ops.conv1x1_linear(x, conv, act)
        if cuda_ops.unfold_conv_supported(x, conv):
            return cuda_ops.unfold_conv(x, conv, act)
        if cuda_ops.smallconv_supported(x, conv):
            return cuda_ops.small_conv(x, conv, act, False)
    y = conv(x)
    return F.elu(y) if act else y


def dilated_stem(x: torch.Tensor, convs, act: bool = True) -> torch.Tensor:
    """``cat([ELU?(conv(x)) for conv in convs], 1)`` for convolutions that differ only in dilation / padding — the five-branch
    stem of the CPC encoder (/root/reference/src/simple_models.py:455-460).  On the GPU ONE wgmma launch reads the input once per
    tap and writes the concatenated tensor (cuda_ops._DilatedStem); elsewhere branch by branch."""
    if _use_fast(x):
        from . import cuda_ops

        if cuda_ops.dilated_stem_supported(x, convs):
            return cuda_ops.dilated_stem(x, list(convs), act)
    return torch.cat([conv_act(x, c, act) for c in convs], dim=1)


def conv_act_pool(x: torch.Tensor, conv: nn.Conv2d, act: bool = True, pool: bool = False) -> torch.Tensor:
    """``max_pool2d?(ELU?(conv(x)), 2, 2)`` — one stage of Net / Net1 / Net2 (/root/reference/src/simple_models.py:19-21,
    :60-66, :103-110).  Net / Net1 (3..64 channels, 5x5 / 3x3 "valid" convs on 28/10-wide maps): ONE direct-convolution
    kernel with bias, ELU and the pooling fused; Net2 (padded 3x3, 64..512 channels): wgmma conv + NHWC max-pool kernel."""
    if _use_fast(x):
        from . import cuda_ops

        if cuda_ops.conv_act_supported(x, conv):
            y = cuda_ops.conv_act(x, conv, act)
            return cuda_ops.max_pool2x2(y) if pool else y
        if cuda_ops.smallconv_supported(x, conv):
            return cuda_ops.small_conv(x, conv, act, pool)
    y = conv(x)
    y = F.elu(y) if act else y
    return F.max_pool2d(y, 2, 2) if pool else y


def max_pool2x2(x: torch.Tensor) -> torch.Tensor:
    if _use_fast(x) and x.dim() == 4 and x.dtype == torch.float32:
        from . import cuda_ops

        return cuda_ops.max_pool2x2(x)
    return F.max_pool2d(x, 2, 2)


def global_avg_pool(x: torch.Tensor) -> torch.Tensor:
    """``avg_pool2d(x, H).squeeze()`` for an H x H map -> ``[N, C]`` (/root/reference/src/simple_models.py:464)."""
    if _use_fast(x) and x.dim() == 4 and x.dtype == torch.float32:
        from . import cuda_ops

        return cuda_ops._AvgPoolNHWC.apply(x)
    return F.avg_pool2d(x, x.shape[2]).reshape(x.shape[0], x.shape[1])


def linear_act(x: torch.Tensor, linear: nn.Linear, act: bool = True) -> torch.Tensor:
    """``ELU?(x @ W^T + b)``; on the GPU one hand-written GEMM kernel with the bias + ELU epilogue (true fp32, the
    reference's nn.Linear precision) and hand-written backward kernels."""
    if _use_fast(x):
        from . import cuda_ops

        if cuda_ops.linear_act_supported(x, linear):
            return cuda_ops.linear_act(x, linear, act)
    y = F.linear(x, linear.weight, linear.bias)
    return F.elu(y) if act else y
