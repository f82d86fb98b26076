"""A float64 oracle for networks whose convolutions run on the TF32 tensor cores.

The tensor core's tf32 MMA reads fp32 operands and uses their upper 19 bits (sign, 8 exponent, 10 mantissa bits); products
are exact and accumulated in fp32.  Comparing such a network with a plain fp64 oracle mixes two things: the 2^-11 operand
rounding itself and — in networks with max-pooling — the pool winners that this rounding flips, each of which moves a
gradient term (a few per cent of a conv weight gradient in Net2).  This oracle reproduces the
operand rounding in all three products of a convolution (forward, data gradient, weight gradient) and evaluates
everything else in float64, so that a kernel bug (wrong tap, wrong layout, missing term) still shows up at 1e-2..1
while the expected TF32 behaviour cancels.

Used by tests/test_gpu_aux.py; the reference trains Net2 with PyTorch's default ``cudnn.allow_tf32 = True``
(/root/reference/src/simple_models.py:85-127).
"""
from __future__ import annotations

import types

import torch
import torch.nn as nn
import torch.nn.functional as F


def to_tf32(t: torch.Tensor, mode: str = "trunc") -> torch.Tensor:
    """fp64/fp32 -> fp32 -> TF32 (10 mantissa bits) -> original dtype.  ``trunc`` drops the low 13 bits (what the tensor
    core does with raw fp32 operands), ``rna`` rounds to nearest, ties away (``cvt.rna.tf32.f32``)."""
    bits = t.to(torch.float32).contiguous().view(torch.int32)
    if mode == "rna":
        bits = bits + 0x1000
    bits = bits & ~0x1FFF
    return bits.view(torch.float32).to(t.dtype)


class _TF32Conv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, pad, mode):
        ctx.save_for_backward(x, w)
        ctx.cfg = (stride, pad, mode, b is not None)
        return F.conv2d(to_tf32(x, mode), to_tf32(w, mode), b, stride, pad)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        stride, pad, mode, has_b = ctx.cfg
        dyq = to_tf32(dy, mode)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.ops.aten.convolution_backward(dyq, x, to_tf32(w, mode), None, [stride, stride], [pad, pad], [1, 1], False,
                                                     [0, 0], 1, [True, False, False])[0]
        if ctx.needs_input_grad[1]:
            dw = torch.ops.aten.convolution_backward(dyq, to_tf32(x, mode), w, None, [stride, stride], [pad, pad], [1, 1], False,
                                                     [0, 0], 1, [False, True, False])[1]
        db = dy.sum((0, 2, 3)) if has_b and ctx.needs_input_grad[2] else None
        return dx, dw, db, None, None, None


def tf32_conv_oracle(model: nn.Module, mode: str = "trunc") -> nn.Module:
    """Patch every plain ``nn.Conv2d`` of ``model`` (expected in float64) to multiply TF32-rounded operands."""
    for m in model.modules():
        if type(m) is nn.Conv2d and m.groups == 1 and tuple(m.dilation) == (1, 1) and m.stride[0] == m.stride[1] \
                and m.padding[0] == m.padding[1]:
            def fwd(self, x, _mode=mode):
                return _TF32Conv.apply(x, self.weight, self.bias, self.stride[0], self.padding[0], _mode)
            m.forward = types.MethodType(fwd, m)
    return model
