"""Python face of the sm_90a extension (``csrc/``): thin wrappers and the
``torch.autograd.Function``s that wire the kernels into autograd.

Activation layout on this path: NHWC memory.  Tensors keep their logical NCHW
shape with ``channels_last`` strides, so the rest of PyTorch (and the ATen
fall-backs used for the few ops that have no hand-written kernel yet) sees
ordinary tensors, while the kernels receive the underlying [N,H,W,C] buffer.

Kernel inventory (SURVEY §2.10 ids):
  G1  conv2d_nhwc          wgmma implicit GEMM (TMA 4-D boxes -> smem -> wgmma tf32 -> registers), BN stats in epilogue
  G2/3 bn_elu_fwd/bwd      BatchNorm(train) + residual + ELU fused, two-pass backward
  G4  avgpool / pool_linear
  G5  linear_tf32          wgmma GEMM with bias+ELU epilogue
  G9  cross_entropy        fused log-softmax/NLL fwd, softmax-minus-onehot bwd
  G10 vae_loss             single fused reduction fwd, elementwise bwd
  G14-16 flat ops          adam_prox, penalty, L-BFGS algebra (see flatops.py)
  G22 normalize_u8         uint8 NHWC -> normalised float, layout change fused

Reference call sites these replace (library calls in the reference): conv + BatchNorm + ELU + residual
``src/simple_models.py:137-153`` / ``:191-216``, ``avg_pool2d`` + ``linear`` ``:213-216``, cross-entropy
``src/federated_multi.py:132``, VAE loss ``src/federated_vae.py:96-108``, input normalisation
``src/federated_multi.py:60-71``, Adam / penalty terms ``src/consensus_multi.py:214-220`` (see flatops.py).

On a CUDA device a missing extension is an error, never a silent fall-back.
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _ext
from . import conv_math

_EXT = None
TF32_LINEAR = os.environ.get("FEDB200_TF32_LINEAR", "0") == "1"


def ext():
    global _EXT
    if _EXT is None:
        _EXT = _ext.load("fedb200_cuda", required=True)
    return _EXT


def launch_count() -> int:
    return int(ext().launch_count())


# ----------------------------------------------------------------------------
# flat-vector ops
# ----------------------------------------------------------------------------
_STEP_TENSORS = {}


def _step_tensor(key, device) -> torch.Tensor:
    t = _STEP_TENSORS.get(key)
    if t is None:
        t = torch.zeros(1, dtype=torch.int32, device=device)
        _STEP_TENSORS[key] = t
    return t


def adam_prox_step(x, g, m, v, step, lr, beta1, beta2, eps, z=None, y=None, rho=0.0, lambda1=0.0, lambda2=0.0,
                   rho_dev=None) -> None:
    """``step`` is either a CUDA int32 tensor holding the (already incremented) step count
    (graph-capturable) or a Python int (copied into a per-buffer device counter)."""
    if not torch.is_tensor(step):
        t = _step_tensor(m.data_ptr(), x.device)
        t.fill_(int(step))
        step = t
    ext().adam_prox(x, g, m, v, step, lr, beta1, beta2, eps, z, y, rho, lambda1, lambda2, rho_dev)


def bump_step(step: torch.Tensor) -> None:
    ext().bump_step(step)


def l1_l2(g: torch.Tensor) -> Tuple[float, float]:
    a, b = ext().l1_l2(g).tolist()
    return float(a), float(b) ** 0.5


def make_pair(g, g_prev, d, t: float, trust: float):
    y, s, sc = ext().make_pair(g, g_prev, d, t, trust)
    ys, ss, yy = sc.tolist()
    return y, s, float(ys), float(ss) ** 0.5, float(yy)


def welford_update(g, mean, m2, n: int) -> float:
    return float(ext().welford(g, mean, m2, int(n)))


def penalty_value(x, z=None, y=None, rho=0.0, lambda1=0.0, lambda2=0.0) -> torch.Tensor:
    return ext().penalty_value(x, z, y, rho, lambda1, lambda2).reshape(())


def penalty_grad_(g, x, z=None, y=None, rho=0.0, lambda1=0.0, lambda2=0.0) -> None:
    ext().penalty_grad(g, x, z, y, rho, lambda1, lambda2)


def multi_dot(pairs) -> torch.Tensor:
    out = []
    for i in range(0, len(pairs), 8):
        chunk = pairs[i:i + 8]
        out.append(ext().multi_dot([a.contiguous() for a, _ in chunk], [b.contiguous() for _, b in chunk]))
    return torch.cat(out)


def lbfgs_two_loop(Y, S, order: Sequence[int], g, H_diag: float) -> torch.Tensor:
    o = torch.tensor(list(order), dtype=torch.int32, device=g.device)
    return ext().lbfgs_two_loop(Y, S, o, g, float(H_diag))


# ----------------------------------------------------------------------------
# input pipeline
# ----------------------------------------------------------------------------
def normalize_u8(u8_nhwc: torch.Tensor, mean, std, channels_last: bool) -> torch.Tensor:
    u8 = u8_nhwc.contiguous()
    if channels_last:
        out = ext().normalize_u8(u8, list(mean), list(std), 3, False)   # [N,H,W,3]
        return out.permute(0, 3, 1, 2)
    return ext().normalize_u8(u8, list(mean), list(std), 3, True)


# ----------------------------------------------------------------------------
# conv + BN + ELU group
# ----------------------------------------------------------------------------
def _nhwc(x: torch.Tensor) -> torch.Tensor:
    """[N,H,W,C] contiguous view of a logical NCHW tensor (copying only if it is not channels_last)."""
    p = x.permute(0, 2, 3, 1)
    return p if p.is_contiguous() else p.contiguous()


def _krsc(w: torch.Tensor) -> torch.Tensor:
    p = w.permute(0, 2, 3, 1)
    return p if p.is_contiguous() else p.contiguous()


def conv_bn_act_supported(x: torch.Tensor, conv: nn.Conv2d, bn: nn.BatchNorm2d) -> bool:
    if not (isinstance(conv, nn.Conv2d) and isinstance(bn, nn.BatchNorm2d)):
        return False
    if conv.bias is not None or conv.groups != 1 or conv.padding_mode != "zeros":
        return False
    if conv.stride[0] != conv.stride[1] or conv.padding[0] != conv.padding[1] or conv.dilation != (1, 1):
        return False
    if x.dtype != torch.float32 or x.dim() != 4 or not bn.training or not bn.track_running_stats or bn.momentum is None:
        return False
    kh, kw = conv.kernel_size
    s, p = conv.stride[0], conv.padding[0]
    H, W = x.shape[2], x.shape[3]
    Ho, Wo = (H + 2 * p - kh) // s + 1, (W + 2 * p - kw) // s + 1
    cin = x.shape[1] if x.shape[1] % 4 == 0 else (4 if x.shape[1] == 3 else -1)
    if cin < 0 or conv.out_channels % 4 != 0:
        return False
    return bool(ext().conv_supported(Ho, Wo, cin, s))


_FLIP_CACHE = {}
_STATS_BUFFERS = {}


def _stats_buffer(weight: torch.Tensor, C: int):
    """Per-layer BatchNorm accumulator ``[sum | sumsq | counter]``: zeroed once at allocation, then kept clean by
    ``bn_elu_fwd`` itself (its last block re-zeroes it), so no fill kernel is launched per convolution."""
    key = (weight.data_ptr(), C)
    buf = _STATS_BUFFERS.get(key)
    if buf is None:
        if torch.cuda.is_current_stream_capturing():   # graph-pool memory must not be cached
            return torch.zeros(2 * C + 1, dtype=torch.float32, device=weight.device), False
        buf = torch.zeros(2 * C + 1, dtype=torch.float32, device=weight.device)
        _STATS_BUFFERS[key] = buf
    return buf, True


def _bwd_sums_buffer(gamma: torch.Tensor, C: int):
    """Per-layer scratch of the BatchNorm backward ``[sum du | sum du*xhat | counter]``: zeroed once at allocation and left zeroed
    again by ``bn_elu_bwd_apply`` (its last block), so the captured step has no memset node per BatchNorm layer.  ``None`` while a
    graph is being captured before the buffer exists (graph-pool memory must not be cached): the binding then memsets a temporary."""
    key = ("bwd", gamma.data_ptr(), C)
    buf = _STATS_BUFFERS.get(key)
    if buf is None:
        if torch.cuda.is_current_stream_capturing():
            return None
        buf = torch.zeros(2 * C + 1, dtype=torch.float32, device=gamma.device)
        _STATS_BUFFERS[key] = buf
    return buf


def clear_caches() -> None:
    """Derived tensors must follow their source weights (call after loading a checkpoint into existing parameters).
    Cached entries are refreshed IN PLACE: captured CUDA graphs hold their addresses."""
    refresh_caches()
    _STATS_BUFFERS.clear()


class _Derived:
    """A derived filter (rotated / phase-packed) of a FROZEN layer, kept at a stable address and refreshed in place
    whenever its source weights may have changed (``refresh_caches``: start of every block visit, checkpoint load)."""

    __slots__ = ("src", "out", "fn")

    def __init__(self, src, fn):
        self.src, self.fn = src, fn
        self.out = fn(src)

    def refresh(self):
        self.out.copy_(self.fn(self.src))


def refresh_caches() -> int:
    """Recompute every cached derived filter from its (possibly updated) source weights, in place.

    Why (ADVICE r1, high): a layer is frozen while other blocks train, but its weights DO change when its own block is
    visited (Adam + FedAvg write-back).  The first conv of a block needs no data gradient during its own visit, so its
    cached rotated filter was never touched and went stale for all later visits of earlier blocks (Nloop >= 2) — and
    CUDA graphs of those visits hold the cached tensor's address.  The engine calls this at the start of every block
    visit; entries are never dropped, so graph-baked addresses stay valid."""
    n = 0
    with torch.no_grad():
        for cache in (_FLIP_CACHE, _S2_CACHE):
            for ent in cache.values():
                ent.refresh()
                n += 1
    return n


def _aliases(wk: torch.Tensor, weight: torch.Tensor) -> bool:
    """True when the KRSC view ``wk`` aliases the parameter's own (persistent) storage.  Only such filters may be
    cached by address: the NHWC copy of a plain NCHW parameter is a transient whose address the allocator recycles
    (ADVICE r1, low)."""
    return wk.untyped_storage().data_ptr() == weight.untyped_storage().data_ptr()


def _derived(cache, wk: torch.Tensor, trainable: bool, fn, persistent: bool) -> torch.Tensor:
    if trainable or not persistent:     # the active block's filters change every step: recompute, leave the cache alone
        return fn(wk)
    key = (wk.data_ptr(), tuple(wk.shape))
    hit = cache.get(key)
    if hit is not None:
        return hit.out
    if torch.cuda.is_current_stream_capturing():      # graph-pool memory must not escape its graph
        return fn(wk)
    ent = _Derived(wk, fn)
    cache[key] = ent
    return ent.out


def _flipped_weight(wk: torch.Tensor, trainable: bool, persistent: bool = True) -> torch.Tensor:
    """Rotated/transposed filter for the data gradient.  Frozen layers do not change during a block visit (only the
    active block is optimised or written back by FedAvg), so their flipped copy is computed once per visit and reused;
    the active block's is recomputed every step."""
    return _derived(_FLIP_CACHE, wk, trainable, lambda w: ext().weight_flip(w), persistent)


S2_DGRAD = os.environ.get("FEDB200_S2_DGRAD", "1") != "0"
_S2_CACHE = {}


def _packed_s2_weight(wk: torch.Tensor, trainable: bool, persistent: bool = True) -> torch.Tensor:
    """Filter of the stride-1 convolution that computes a stride-2 data gradient (conv_math.py); cached for frozen
    layers exactly like the rotated filters above."""
    return _derived(_S2_CACHE, wk, trainable, conv_math.pack_dgrad_s2_weight, persistent)


def _s2_dgrad_supported(e, xn: torch.Tensor, dy: torch.Tensor, kh: int, kw: int, pad: int) -> bool:
    H, W, Ci = xn.shape[1], xn.shape[2], xn.shape[3]
    Ho, Wo, Co = dy.shape[1], dy.shape[2], dy.shape[3]
    if not S2_DGRAD or kh != kw or (kh, pad) not in ((3, 1), (1, 0)):
        return False
    if H != 2 * Ho or W != 2 * Wo or Co % 4 or Ci % 4:
        return False
    return bool(e.conv_supported(Ho, Wo, Co, 1))


def _s2_dgrad(e, dy: torch.Tensor, wk: torch.Tensor, trainable: bool, persistent: bool = True) -> torch.Tensor:
    """dx [N, 2Ho, 2Wo, Ci] of a stride-2 convolution: one stride-1 implicit GEMM over dy + a pixel shuffle."""
    wp = _packed_s2_weight(wk, trainable, persistent)
    Ho, Wo, Co = dy.shape[1], dy.shape[2], dy.shape[3]
    Ci = wp.shape[0] // 4
    # the kernel stores every epilogue chunk straight to dx[n, 2 ho + ph, 2 wo + pw, :] (5-D tensor map): no pixel-shuffle copy
    shuffle = bool(e.conv_shuffle_supported(Ho, Wo, Co, Ci))
    if wk.shape[1] == 1:      # 1x1: only tap (0, 0) of the 2x2 window is populated -> run it as a 1x1 convolution
        w1 = wp[:, 0:1, 0:1, :].contiguous()
        if shuffle:
            return e.conv2d_nhwc_shuffle(dy, w1, 0, Ho, Wo)
        return conv_math.dgrad_s2(dy, w1, lambda x, w: e.conv2d_nhwc(x, w, None, 1, 0, 1))
    if shuffle:
        return e.conv2d_nhwc_shuffle(dy, wp, 0, Ho, Wo)
    return conv_math.dgrad_s2(dy, wp, lambda x, w: e.conv2d_nhwc_sized(x, w, None, 1, 0, 1, Ho, Wo))


# ----------------------------------------------------------------------------
# weight gradient on wgmma (csrc/wgrad_wgmma.cuh): MN-major operands straight from the NHWC activations,
# split over the pixel range, partial sums red.add-ed into dW
# ----------------------------------------------------------------------------
WGRAD = os.environ.get("FEDB200_WGRAD", "1") != "0"
_ACC_INTO_GRAD = {"on": False}


class accumulate_into_grad:
    """Context manager for ``loss.backward()`` calls of the engine: while active, weight-gradient kernels accumulate
    straight into the parameter's ``.grad`` buffer (a zeroed view of the gradient arena) and the autograd node returns
    ``None`` for the weight, which removes one fill and one ``add`` launch per trainable convolution / dense layer.
    Never active under ``torch.autograd.grad`` (functional calls must not touch ``.grad``)."""

    def __enter__(self):
        self.prev = _ACC_INTO_GRAD["on"]
        _ACC_INTO_GRAD["on"] = True
        return self

    def __exit__(self, *exc):
        _ACC_INTO_GRAD["on"] = self.prev
        return False


def _grad_buffer_krsc(weight: Optional[torch.Tensor], shape_krsc) -> Optional[torch.Tensor]:
    """The parameter's gradient buffer as a contiguous [Co, kh, kw, Ci] tensor, if in-place accumulation is allowed."""
    if not _ACC_INTO_GRAD["on"] or weight is None or getattr(weight, "grad", None) is None:
        return None
    g = weight.grad
    if g.dim() != 4:
        return None
    gk = g.permute(0, 2, 3, 1)
    if not gk.is_contiguous() or tuple(gk.shape) != tuple(shape_krsc) or g.dtype != torch.float32:
        return None
    return gk


def conv_wgrad_supported(xn: torch.Tensor, dy: torch.Tensor, stride: int) -> bool:
    return bool(WGRAD and ext().conv_wgrad_supported(xn.shape[3], dy.shape[3], stride, dy.shape[2], dy.shape[1]))


def conv_wgrad(xn: torch.Tensor, dy: torch.Tensor, kh: int, kw: int, cw: int, stride: int, pad: int, dil: int,
               weight: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """dW of ``conv(x, W)`` from NHWC ``xn`` [N,H,W,Cx] and ``dy`` [N,Ho,Wo,Co]: returns the gradient as a logical
    [Co, cw, kh, kw] tensor (KRSC memory), or ``None`` after accumulating into ``weight.grad`` in place."""
    Co = dy.shape[3]
    dyc = dy if dy.is_contiguous() else dy.contiguous()
    buf = _grad_buffer_krsc(weight, (Co, kh, kw, cw))
    if buf is not None:
        ext().conv_wgrad(xn, dyc, buf, stride, pad, dil)
        return None
    dwk = torch.zeros(Co, kh, kw, cw, dtype=torch.float32, device=xn.device)
    ext().conv_wgrad(xn, dyc, dwk, stride, pad, dil)
    return dwk.permute(0, 3, 1, 2)


class _ConvBnAct(torch.autograd.Function):
    """``act(BN_train(conv(x)) + residual)`` with NHWC kernels; see module docstring."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, residual, running_mean, running_var, stride, pad, eps, momentum, act):
        e = ext()
        xn = _nhwc(x)
        wk = _krsc(weight)
        if xn.shape[3] == 3:  # stem: pad 3 -> 4 channels so that the pixel pitch is 16 B (TMA requirement)
            xn = F.pad(xn, (0, 1))
            wk = F.pad(wk, (0, 1))
        Co = weight.shape[0]
        stats, self_clean = _stats_buffer(weight, Co)
        y = e.conv2d_nhwc(xn, wk, stats, stride, pad, 1)
        res = _nhwc(residual) if residual is not None else None
        out, mean, invstd = e.bn_elu_fwd(y, stats, gamma, beta, res, running_mean, running_var, eps, momentum, act, self_clean)
        ctx.save_for_backward(xn, wk, y, out, mean, invstd, gamma, beta)
        ctx.cfg = (stride, pad, act, residual is not None, tuple(weight.shape), x.shape[1])
        ctx.w_persistent = _aliases(wk, weight)
        ctx.weight_ref = weight
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        e = ext()
        xn, wk, y, out, mean, invstd, gamma, beta = ctx.saved_tensors
        stride, pad, act, has_res, wshape, cin_logical = ctx.cfg
        need_x, need_w, need_g, need_b, need_r = ctx.needs_input_grad[:5]
        dn = _nhwc(dout)
        dgamma = torch.zeros_like(gamma) if need_g else None
        dbeta = torch.zeros_like(gamma) if need_b else None
        # without a residual input ELU' is recomputed from y (one tensor read less per backward pass)
        dy, dres = e.bn_elu_bwd(dn, out if (has_res or not act) else None, y, mean, invstd, gamma, beta, dgamma, dbeta,
                                bool(has_res and need_r), act, _bwd_sums_buffer(gamma, gamma.numel()))
        dx = dw = None
        kh, kw = wshape[2], wshape[3]
        if need_x:
            Ci = xn.shape[3]
            if stride == 1 and e.conv_supported(xn.shape[1], xn.shape[2], wshape[0], 1) and Ci % 4 == 0:
                # data gradient of a stride-1 conv = conv of dy with the 180-degree rotated, transposed filter
                dxn = e.conv2d_nhwc(dy, _flipped_weight(wk, need_w, ctx.w_persistent), None, 1, kh - 1 - pad, 1)
            elif stride == 2 and _s2_dgrad_supported(e, xn, dy, kh, kw, pad):
                dxn = _s2_dgrad(e, dy, wk, need_w, ctx.w_persistent)
            else:
                dxn = torch.ops.aten.convolution_backward(
                    dy.permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), wk.permute(0, 3, 1, 2), None,
                    [stride, stride], [pad, pad], [1, 1], False, [0, 0], 1, [True, False, False])[0]
                dxn = _nhwc(dxn)
            if dxn.shape[3] != cin_logical:
                dxn = dxn[..., :cin_logical]
            dx = dxn.permute(0, 3, 1, 2)
        if need_w:
            if conv_wgrad_supported(xn, dy, stride):
                dw = conv_wgrad(xn, dy, kh, kw, cin_logical, stride, pad, 1, ctx.weight_ref)
            else:
                dwk = torch.ops.aten.convolution_backward(
                    dy.permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), wk.permute(0, 3, 1, 2), None,
                    [stride, stride], [pad, pad], [1, 1], False, [0, 0], 1, [False, True, False])[1]
                dw = dwk[:, :cin_logical] if dwk.shape[1] != cin_logical else dwk
        dr = dres.permute(0, 3, 1, 2) if (has_res and need_r and dres is not None) else None
        return dx, dw, dgamma, dbeta, dr, None, None, None, None, None, None, None


# ----------------------------------------------------------------------------
# Identity-shortcut blocks: the gradient that reaches the block input is dgrad(conv1) + d(residual).  Autograd adds
# the two with a separate elementwise kernel (one `add` launch per identity block and step).  Routing the
# block input through the conv1 Function as a second, pass-through output hands BOTH gradients to one backward call,
# which lets the data-gradient convolution accumulate straight into the residual gradient (bulk reduce-add epilogue).  Opt-in: FEDB200_SKIP_FUSED=1.
# ----------------------------------------------------------------------------
SKIP_FUSED = os.environ.get("FEDB200_SKIP_FUSED", "0") == "1"


class _ConvBnActSkip(torch.autograd.Function):
    """``(ELU(BN_train(conv(x))), x)`` — the second output is the block input itself (no copy)."""

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, stride, pad, eps, momentum):
        e = ext()
        xn = _nhwc(x)
        wk = _krsc(weight)
        Co = weight.shape[0]
        stats, self_clean = _stats_buffer(weight, Co)
        y = e.conv2d_nhwc(xn, wk, stats, stride, pad, 1)
        out, mean, invstd = e.bn_elu_fwd(y, stats, gamma, beta, None, running_mean, running_var, eps, momentum, True, self_clean)
        ctx.save_for_backward(xn, wk, y, mean, invstd, gamma, beta)
        ctx.cfg = (stride, pad, tuple(weight.shape))
        ctx.w_persistent = _aliases(wk, weight)
        ctx.weight_ref = weight
        return out.permute(0, 3, 1, 2), x.view_as(x)

    @staticmethod
    def backward(ctx, dout, dskip):
        e = ext()
        xn, wk, y, mean, invstd, gamma, beta = ctx.saved_tensors
        stride, pad, wshape = ctx.cfg
        need_x, need_w, need_g, need_b = ctx.needs_input_grad[:4]
        dgamma = torch.zeros_like(gamma) if need_g else None
        dbeta = torch.zeros_like(gamma) if need_b else None
        dy, _ = e.bn_elu_bwd(_nhwc(dout), None, y, mean, invstd, gamma, beta, dgamma, dbeta, False, True,
                             _bwd_sums_buffer(gamma, gamma.numel()))
        kh = wshape[2]
        dx = dw = None
        if need_x:
            wf = _flipped_weight(wk, need_w, ctx.w_persistent)
            if dskip is not None:
                acc = _nhwc(dskip)                       # the residual gradient of conv2's Function: ours alone
                if not acc.is_contiguous():
                    acc = acc.contiguous()
                dxn = e.conv2d_nhwc_accumulate(dy, wf, acc, 1, kh - 1 - pad, 1)      # acc += dgrad(dy), in place
            else:
                dxn = e.conv2d_nhwc(dy, wf, None, 1, kh - 1 - pad, 1)
            dx = dxn.permute(0, 3, 1, 2)
        elif dskip is not None:
            dx = dskip
        if need_w:
            if conv_wgrad_supported(xn, dy, stride):
                dw = conv_wgrad(xn, dy, kh, wshape[3], wshape[1], stride, pad, 1, ctx.weight_ref)
            else:
                dw = torch.ops.aten.convolution_backward(
                    dy.permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), wk.permute(0, 3, 1, 2), None,
                    [stride, stride], [pad, pad], [1, 1], False, [0, 0], 1, [False, True, False])[1]
        return dx, dw, dgamma, dbeta, None, None, None, None, None, None


def conv_bn_act_skip_supported(x: torch.Tensor, conv: nn.Conv2d, bn: nn.BatchNorm2d) -> bool:
    if not SKIP_FUSED or not conv_bn_act_supported(x, conv, bn):
        return False
    # stride-1 3x3 with matching channel counts (identity shortcut) and a 16-byte pixel pitch
    return conv.stride[0] == 1 and conv.in_channels == conv.out_channels and conv.in_channels % 4 == 0 and x.requires_grad


def conv_bn_act_skip(x, conv: nn.Conv2d, bn: nn.BatchNorm2d):
    return _ConvBnActSkip.apply(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, conv.stride[0],
                                conv.padding[0], bn.eps, bn.momentum)


# ----------------------------------------------------------------------------
# conv + bias (+ ELU) of the VAE / CPC networks (SURVEY G6, G7, G8) — forward AND backward on hand-written kernels:
#   forward   implicit GEMM on wgmma with bias + ELU in the epilogue (transposed convs: 3x3 conv with 4*C_out phase
#             channels + pixel shuffle, ops/conv_math.py)
#   dz, db    one pass: dout * ELU'(z) recomputed from the saved output + per-channel sums   (act_bwd_bias kernel)
#   dx        stride-2 4x4: the transposed-conv kernel path with the same weights; stride 1: rotated filter;
#             transposed conv: the forward stride-2 conv kernel
#   dw        wgmma weight-gradient kernel (wgrad_wgmma.cuh); for transposed convs with the roles of x and dz swapped
# FEDB200_CONV_ACT=0 restores the ATen / cuDNN composition (A/B runs).
# ----------------------------------------------------------------------------
CONV_ACT = os.environ.get("FEDB200_CONV_ACT", "1") != "0"


def conv_act_supported(x: torch.Tensor, conv: nn.Module) -> bool:
    if not CONV_ACT or not isinstance(conv, nn.Conv2d) or isinstance(conv, nn.ConvTranspose2d):
        return False
    if x.dim() != 4 or x.dtype != torch.float32 or conv.groups != 1 or conv.padding_mode != "zeros":
        return False
    if isinstance(conv.padding, str) or conv.kernel_size[0] != conv.kernel_size[1]:
        return False
    if conv.stride[0] != conv.stride[1] or conv.padding[0] != conv.padding[1] or conv.dilation[0] != conv.dilation[1]:
        return False
    k, s, p, d = conv.kernel_size[0], conv.stride[0], conv.padding[0], conv.dilation[0]
    H, W = x.shape[2], x.shape[3]
    Ho, Wo = (H + 2 * p - d * (k - 1) - 1) // s + 1, (W + 2 * p - d * (k - 1) - 1) // s + 1
    Ci, Co = conv.in_channels, conv.out_channels
    if Ho < 1 or Wo < 1 or Co % 4 or not (Ci % 4 == 0 or Ci == 3):
        return False
    return bool(ext().conv_supported(Ho, Wo, Ci if Ci != 3 else 4, s))


def _act_bwd_bias(d: torch.Tensor, out: torch.Tensor, act: bool, need_b: bool, bias_param=None):
    """(dz, db): dz = d * ELU'(z) (aliasing ``d`` when there is no activation); db = per-channel sums (or None after
    accumulating into ``bias_param.grad`` inside ``accumulate_into_grad``)."""
    e = ext()
    d = d if d.is_contiguous() else d.contiguous()
    C = d.shape[-1]
    db = None
    dbuf = None
    if need_b:
        if _ACC_INTO_GRAD["on"] and bias_param is not None and getattr(bias_param, "grad", None) is not None \
                and bias_param.grad.is_contiguous() and bias_param.grad.numel() == C:
            dbuf = bias_param.grad
        else:
            db = torch.zeros(C, dtype=torch.float32, device=d.device)
            dbuf = db
    if not act and dbuf is None:
        return d, None
    dz = torch.empty_like(d) if act else None
    e.act_bwd_bias(d, out if act else None, dz, dbuf, bool(act))
    return (dz if act else d), db


class _ConvAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, stride, pad, dil, act):
        xn = _nhwc(x)
        wk = _krsc(weight)
        ci_logical = xn.shape[3]
        if xn.shape[3] == 3:   # 16-byte pixel pitch for the TMA box
            xn = F.pad(xn, (0, 1))
            wk = F.pad(wk, (0, 1))
        out = ext().conv2d_nhwc_bias_act(xn, wk, bias, bool(act), stride, pad, dil)
        ctx.save_for_backward(xn, weight, out)
        ctx.cfg = (stride, pad, dil, act, bias is not None, ci_logical)
        ctx.params = (weight, bias)
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        e = ext()
        xn, weight, out = ctx.saved_tensors
        stride, pad, dil, act, has_bias, ci_logical = ctx.cfg
        wparam, bparam = ctx.params
        need_x, need_w, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2] and has_bias
        dz, db = _act_bwd_bias(_nhwc(dout), out, act, need_b, bparam)
        Co, _, k, _ = weight.shape
        Ho, Wo = dz.shape[1], dz.shape[2]
        dx = dw = None
        if need_x:
            dxn = None
            if stride == 2 and k == 4 and pad == 1 and dil == 1 and Co % 4 == 0 and e.conv_supported(Ho, Wo, Co, 1):
                # data gradient of conv(4, s2, p1) == ConvTranspose2d(4, s2, p1) with the same weight tensor
                wp = e.convT_pack(weight.detach())                 # == conv_math.pack_convT_s2_weight, one launch
                dxn = conv_math.convT_s2(dz, wp, lambda a, w: e.conv2d_nhwc_bias_act(a, w, None, False, 1, 1, 1))
            elif stride == 1 and dil == 1 and Co % 4 == 0 and e.conv_supported(xn.shape[1], xn.shape[2], Co, 1):
                dxn = e.conv2d_nhwc(dz, e.weight_flip(_krsc(weight).contiguous()), None, 1, k - 1 - pad, 1)
            if dxn is None:
                dxn = _nhwc(torch.ops.aten.convolution_backward(
                    dz.permute(0, 3, 1, 2), xn[..., :ci_logical].permute(0, 3, 1, 2), weight, None, [stride, stride], [pad, pad],
                    [dil, dil], False, [0, 0], 1, [True, False, False])[0])
            dx = dxn[..., :ci_logical].permute(0, 3, 1, 2) if dxn.shape[3] != ci_logical else dxn.permute(0, 3, 1, 2)
        if need_w:
            if conv_wgrad_supported(xn, dz, stride):
                dw = conv_wgrad(xn, dz, k, k, ci_logical, stride, pad, dil, wparam)
            else:
                dw = torch.ops.aten.convolution_backward(
                    dz.permute(0, 3, 1, 2), xn[..., :ci_logical].permute(0, 3, 1, 2), weight, None, [stride, stride], [pad, pad],
                    [dil, dil], False, [0, 0], 1, [False, True, False])[1]
        return dx, dw, (db if need_b else None), None, None, None, None


def _conv_out(size: int, k: int, s: int, p: int, d: int) -> int:
    return (size + 2 * p - d * (k - 1) - 1) // s + 1


def dilated_stem_supported(x: torch.Tensor, convs) -> bool:
    """Several convolutions of the SAME input that differ only in dilation / padding (and own their output channels), followed
    by a channel concatenation: the CPC encoder stem (SURVEY G6, /root/reference/src/simple_models.py:441-451, :455-460)."""
    if not CONV_ACT or len(convs) < 2 or len(convs) > 8 or x.dim() != 4 or x.dtype != torch.float32 or not x.is_cuda:
        return False
    c0 = convs[0]
    k, st = c0.kernel_size[0], c0.stride[0]
    outs = set()
    for c in convs:
        if not isinstance(c, nn.Conv2d) or isinstance(c, nn.ConvTranspose2d) or c.groups != 1 or isinstance(c.padding, str):
            return False
        if tuple(c.kernel_size) != (k, k) or tuple(c.stride) != (st, st) or c.in_channels != c0.in_channels \
                or c.out_channels != c0.out_channels or (c.bias is None) != (c0.bias is None):
            return False
        if c.padding[0] != c.padding[1] or c.dilation[0] != c.dilation[1] or c.dilation[0] > 255 or c.padding[0] > 255:
            return False
        outs.add((_conv_out(x.shape[2], k, st, c.padding[0], c.dilation[0]), _conv_out(x.shape[3], k, st, c.padding[0], c.dilation[0])))
    if len(outs) != 1 or c0.in_channels % 4 or (c0.out_channels * len(convs)) % 4:
        return False
    Ho, Wo = next(iter(outs))
    return Ho > 0 and Wo > 0 and bool(ext().conv_multidil_supported(Ho, Wo, c0.in_channels, st, len(convs)))


class _DilatedStem(torch.autograd.Function):
    """``cat([ELU?(conv_b(x)) for b], 1)`` as ONE wgmma implicit GEMM: the filter rows of the launch are (branch, row) pairs,
    every branch reads the input through its own dilation / padding (IgemmParams::ms_*), the block-diagonal weight matrix sends
    branch b to its own output channels, bias + ELU in the epilogue, one bulk tensor store per chunk of the concatenated tensor.
    Backward: one bias+ELU' pass over the concatenated gradient, one wgmma weight-gradient launch per branch."""

    @staticmethod
    def forward(ctx, x, cfg, *params):
        k, st, dils, pads, act, has_bias = cfg
        e = ext()
        xn = _nhwc(x)
        B = len(dils)
        ws = params[0::2]
        Co, Ci = ws[0].shape[0], ws[0].shape[1]
        wm = conv_math.pack_multidil_weight(ws)                                  # [B*Co, B*k, k, Ci], block diagonal (CPU-tested)
        bias = torch.cat([b for b in params[1::2]]) if has_bias else None
        Ho = _conv_out(xn.shape[1], k, st, pads[0], dils[0])
        Wo = _conv_out(xn.shape[2], k, st, pads[0], dils[0])
        out = e.conv2d_nhwc_multidil(xn, wm, bias, bool(act), k, st, list(dils), list(pads), Ho, Wo)
        ctx.save_for_backward(xn, out)
        ctx.cfg = cfg
        ctx.params = params
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        xn, out = ctx.saved_tensors
        k, st, dils, pads, act, has_bias = ctx.cfg
        params = ctx.params
        B = len(dils)
        Co, Ci = params[0].shape[0], params[0].shape[1]
        need_b = has_bias and any(ctx.needs_input_grad[3 + 2 * b] for b in range(B))
        dz, db = _act_bwd_bias(_nhwc(dout), out, act, need_b, None)              # [N, Ho, Wo, B * Co], [B * Co]
        N, Ho, Wo, _ = dz.shape
        dzb = dz.view(N, Ho, Wo, B, Co).permute(3, 0, 1, 2, 4).contiguous()      # one pass -> B contiguous [N, Ho, Wo, Co] slabs
        grads = []
        dx = None
        for b in range(B):
            w, bp = params[2 * b], params[2 * b + 1]
            dw = None
            if ctx.needs_input_grad[2 + 2 * b]:
                if conv_wgrad_supported(xn, dzb[b], st):
                    dw = conv_wgrad(xn, dzb[b], k, k, Ci, st, pads[b], dils[b], w)
                else:
                    dw = torch.ops.aten.convolution_backward(dzb[b].permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), w, None, [st, st],
                                                             [pads[b]] * 2, [dils[b]] * 2, False, [0, 0], 1, [False, True, False])[1]
            if ctx.needs_input_grad[0]:      # the stem reads data: not needed in the drivers; ATen keeps the op differentiable
                g = torch.ops.aten.convolution_backward(dzb[b].permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), w, None, [st, st],
                                                        [pads[b]] * 2, [dils[b]] * 2, False, [0, 0], 1, [True, False, False])[0]
                dx = g if dx is None else dx + g
            grads += [dw, db[b * Co:(b + 1) * Co] if (need_b and bp is not None and ctx.needs_input_grad[3 + 2 * b]) else None]
        return (dx, None, *grads)


def dilated_stem(x: torch.Tensor, convs, act: bool = True) -> torch.Tensor:
    cfg = (convs[0].kernel_size[0], convs[0].stride[0], tuple(c.dilation[0] for c in convs), tuple(c.padding[0] for c in convs),
           bool(act), convs[0].bias is not None)
    params = []
    for c in convs:
        params += [c.weight, c.bias]
    return _DilatedStem.apply(x, cfg, *params)


def conv_transpose_act_supported(x: torch.Tensor, conv: nn.Module) -> bool:
    """ConvTranspose2d(k=4, stride=2, padding=1) of the VAE decoders (SURVEY G7) as one 3x3 convolution with 4*C_out
    phase channels + pixel shuffle (conv_math.pack_convT_s2_weight)."""
    if not CONV_ACT or not isinstance(conv, nn.ConvTranspose2d) or x.dim() != 4 or x.dtype != torch.float32:
        return False
    if (tuple(conv.kernel_size), tuple(conv.stride), tuple(conv.padding), tuple(conv.output_padding), tuple(conv.dilation),
            conv.groups) != ((4, 4), (2, 2), (1, 1), (0, 0), (1, 1), 1):
        return False
    H, W, Ci = x.shape[2], x.shape[3], conv.in_channels
    return Ci % 4 == 0 and bool(ext().conv_supported(H, W, Ci, 1))


class _ConvTransposeAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, act):
        xn = _nhwc(x)
        wp = ext().convT_pack(weight.detach())                     # == conv_math.pack_convT_s2_weight, one launch
        b4 = bias.repeat(4) if bias is not None else None          # phase-major channels (ph, pw, co)
        e = ext()
        out = conv_math.convT_s2(xn, wp, lambda a, w: e.conv2d_nhwc_bias_act(a, w, b4, bool(act), 1, 1, 1))
        ctx.save_for_backward(xn, weight, out)
        ctx.cfg = (act, bias is not None)
        ctx.params = (weight, bias)
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dout):
        e = ext()
        xn, weight, out = ctx.saved_tensors
        act, has_bias = ctx.cfg
        _, bparam = ctx.params
        need_x, need_w, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1], ctx.needs_input_grad[2] and has_bias
        dz, db = _act_bwd_bias(_nhwc(dout), out, act, need_b, bparam)      # [N, 2H, 2W, Co]
        Ci, Co = weight.shape[0], weight.shape[1]
        H, W = xn.shape[1], xn.shape[2]
        dzp = dz if Co % 4 == 0 else F.pad(dz, (0, 4 - Co % 4))           # 16-byte pixel pitch for TMA
        dx = dw = None
        if need_x:
            # dx = conv(dz, W) with stride 2, pad 1 where W is read as a conv filter [out = Ci, in = Co, 4, 4]
            wk = weight.permute(0, 2, 3, 1)
            wk = wk if Co % 4 == 0 else F.pad(wk, (0, 4 - Co % 4))
            if e.conv_supported(H, W, dzp.shape[3], 2):
                dx = e.conv2d_nhwc(dzp, wk.contiguous(), None, 2, 1, 1).permute(0, 3, 1, 2)
            else:
                dx = torch.ops.aten.convolution_backward(dz.permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), weight, None, [2, 2], [1, 1],
                                                         [1, 1], True, [0, 0], 1, [True, False, False])[0]
        if need_w:
            if conv_wgrad_supported(dzp, xn, 2):
                # weight gradient with the roles swapped: "input" = dz (large map), "output gradient" = x (small map)
                dw = conv_wgrad(dzp, xn, 4, 4, Co, 2, 1, 1, None)          # logical [Ci, Co, 4, 4] == the transposed-conv weight
            else:
                dw = torch.ops.aten.convolution_backward(dz.permute(0, 3, 1, 2), xn.permute(0, 3, 1, 2), weight, None, [2, 2], [1, 1],
                                                         [1, 1], True, [0, 0], 1, [False, True, False])[1]
        return dx, dw, (db if need_b else None), None


def conv1x1_supported(x: torch.Tensor, conv: nn.Module) -> bool:
    """1x1 / stride 1 / no padding convolutions on maps the TMA path cannot tile (the 3x3 CPC latent grid, SURVEY G8)
    are plain GEMMs over the [N*H*W, C] pixel rows: they run on the dense-layer kernels."""
    return (CONV_ACT and isinstance(conv, nn.Conv2d) and not isinstance(conv, nn.ConvTranspose2d) and x.dim() == 4
            and x.dtype == torch.float32 and tuple(conv.kernel_size) == (1, 1) and tuple(conv.stride) == (1, 1)
            and not isinstance(conv.padding, str) and tuple(conv.padding) == (0, 0) and conv.groups == 1)


def conv1x1_linear(x: torch.Tensor, conv: nn.Conv2d, act: bool) -> torch.Tensor:
    N, C, H, W = x.shape
    rows = x.permute(0, 2, 3, 1).reshape(N * H * W, C)
    out = _LinearAct.apply(rows, conv.weight.view(conv.out_channels, C), conv.bias, bool(act))
    return out.view(N, H, W, conv.out_channels).permute(0, 3, 1, 2)


def unfold_conv_supported(x: torch.Tensor, conv: nn.Module) -> bool:
    """Stride-1 convolutions on tiny maps with many channels (the 2x2 convolutions of the CPC context network on its 3x3 / 4x4
    latent grid, SURVEY G8): im2col rows [N * Ho * Wo, Ci * k * k] x the dense-layer GEMM kernel with the bias + ELU epilogue,
    which keeps far more threads busy than a direct convolution over a 3x3 / 4x4 map."""
    if not (CONV_ACT and LINEAR_F32) or not isinstance(conv, nn.Conv2d) or isinstance(conv, nn.ConvTranspose2d):
        return False
    if x.dim() != 4 or x.dtype != torch.float32 or conv.groups != 1 or conv.padding_mode != "zeros" or isinstance(conv.padding, str):
        return False
    if tuple(conv.stride) != (1, 1) or tuple(conv.dilation) != (1, 1):
        return False
    kh, kw = conv.kernel_size
    Ho, Wo = x.shape[2] + 2 * conv.padding[0] - kh + 1, x.shape[3] + 2 * conv.padding[1] - kw + 1
    return Ho >= 1 and Wo >= 1 and Ho * Wo <= 64 and conv.in_channels * kh * kw >= 64


def unfold_conv(x: torch.Tensor, conv: nn.Conv2d, act: bool) -> torch.Tensor:
    N, C, H, W = x.shape
    kh, kw = conv.kernel_size
    Ho, Wo = H + 2 * conv.padding[0] - kh + 1, W + 2 * conv.padding[1] - kw + 1
    # im2col as ONE strided copy (F.unfold launches an im2col kernel per sample)
    xp = F.pad(x, (conv.padding[1], conv.padding[1], conv.padding[0], conv.padding[0])) if (conv.padding[0] or conv.padding[1]) else x
    rows = xp.unfold(2, kh, 1).unfold(3, kw, 1).permute(0, 2, 3, 1, 4, 5).reshape(N * Ho * Wo, C * kh * kw)
    out = _LinearAct.apply(rows, conv.weight.reshape(conv.out_channels, C * kh * kw), conv.bias, bool(act))
    return out.view(N, Ho, Wo, conv.out_channels).permute(0, 3, 1, 2)


def conv_act(x: torch.Tensor, conv: nn.Module, act: bool = True) -> torch.Tensor:
    if isinstance(conv, nn.ConvTranspose2d):
        return _ConvTransposeAct.apply(x, conv.weight, conv.bias, bool(act))
    return _ConvAct.apply(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0], conv.dilation[0], bool(act))


def conv_bn_act(x, conv: nn.Conv2d, bn: nn.BatchNorm2d, residual=None, act: bool = True) -> torch.Tensor:
    return _ConvBnAct.apply(x, conv.weight, bn.weight, bn.bias, residual, bn.running_mean, bn.running_var,
                            conv.stride[0], conv.padding[0], bn.eps, bn.momentum, bool(act))


# ----------------------------------------------------------------------------
# pooling + classifier head
# ----------------------------------------------------------------------------
def pool_linear_supported(x, linear, window) -> bool:
    return x.dim() == 4 and x.shape[2] == window and x.shape[3] == window and x.dtype == torch.float32


class _AvgPoolNHWC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        xn = _nhwc(x)
        ctx.hw = (xn.shape[1], xn.shape[2])
        return ext().avgpool_nhwc(xn)

    @staticmethod
    def backward(ctx, dout):
        dx = ext().avgpool_nhwc_bwd(dout.contiguous(), ctx.hw[0], ctx.hw[1])
        return dx.permute(0, 3, 1, 2)


HEAD_FUSED = os.environ.get("FEDB200_HEAD_FUSED", "1") != "0"   # default on


def _dense_wgrad(dz: torch.Tensor, x: torch.Tensor, wparam) -> Optional[torch.Tensor]:
    """dW [N, K] = dz^T x in true fp32: accumulated into ``wparam.grad`` when allowed (returns None), else returned."""
    e = ext()
    N, K = dz.shape[1], x.shape[1]
    if _ACC_INTO_GRAD["on"] and wparam is not None and wparam.is_leaf and wparam.grad is not None \
            and wparam.grad.is_contiguous() and tuple(wparam.grad.shape) == (N, K):
        e.linear_f32_wgrad(dz, x, wparam.grad, True)
        return None
    dw = torch.empty(N, K, dtype=torch.float32, device=dz.device)
    e.linear_f32_wgrad(dz, x, dw, False)
    return dw


class _PoolLinear(torch.autograd.Function):
    """avg_pool over the whole map + Linear in one true-fp32 kernel per direction; weight / bias gradients on the fp32
    GEMM and column-sum kernels (no cuBLAS call left in the classifier head)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        xn = _nhwc(x)
        logits, pooled = ext().head_fwd(xn, weight.contiguous(), bias)
        ctx.save_for_backward(weight, pooled)
        ctx.hw = (xn.shape[1], xn.shape[2])
        ctx.has_bias = bias is not None
        ctx.params = (weight, bias)
        return logits

    @staticmethod
    def backward(ctx, dlogits):
        weight, pooled = ctx.saved_tensors
        wparam, bparam = ctx.params
        dl = dlogits.contiguous()
        dx = ext().head_bwd(dl, weight.contiguous(), ctx.hw[0], ctx.hw[1]).permute(0, 3, 1, 2) if ctx.needs_input_grad[0] else None
        dw = _dense_wgrad(dl, pooled, wparam) if ctx.needs_input_grad[1] else None     # only when the classifier block is active
        db = None
        if ctx.has_bias and ctx.needs_input_grad[2]:
            _, db = _act_bwd_bias(dl, None, False, True, bparam)
        return dx, dw, db


def pool_linear(x, linear: nn.Linear, window: int) -> torch.Tensor:
    if HEAD_FUSED and linear.out_features <= 32:
        return _PoolLinear.apply(x, linear.weight, linear.bias)
    pooled = _AvgPoolNHWC.apply(x)                     # global average over the window x window map
    return linear_act(pooled, linear, False)


# ----------------------------------------------------------------------------
# dense layers (SURVEY G5).  Default: hand-written TRUE-fp32 kernels (the reference's nn.Linear precision, any shape:
# 128x10x512 classifier, 400->120->84->10 of Net, the VAE / VAE-CL heads) with bias + ELU in the GEMM epilogue;
# FEDB200_TF32_LINEAR=1 routes 16-byte aligned layers to the wgmma GEMM (TF32 products) instead.
# ----------------------------------------------------------------------------
LINEAR_F32 = os.environ.get("FEDB200_LINEAR_F32", "1") != "0"


def linear_act_supported(x, linear) -> bool:
    if not (x.dim() == 2 and x.dtype == torch.float32 and isinstance(linear, nn.Linear)):
        return False
    return LINEAR_F32 or TF32_LINEAR


class _LinearAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, act):
        e = ext()
        xc, wc = x.contiguous(), w.contiguous()
        if TF32_LINEAR and xc.shape[1] % 4 == 0:
            out = e.linear_tf32(xc, wc, b, act)
        else:
            out = e.linear_f32(xc, wc, b, act)
        ctx.save_for_backward(xc, wc, out)
        ctx.act = act
        ctx.params = (w, b)
        return out

    @staticmethod
    def backward(ctx, dout):
        e = ext()
        x, w, out = ctx.saved_tensors
        wparam, bparam = ctx.params
        need_b = bparam is not None and ctx.needs_input_grad[2]
        dz, db = _act_bwd_bias(dout, out, ctx.act, need_b, bparam)
        dx = e.linear_f32_dgrad(dz, w) if ctx.needs_input_grad[0] else None
        dw = _dense_wgrad(dz, x, wparam) if ctx.needs_input_grad[1] else None
        return dx, dw, db, None


def linear_act(x, linear: nn.Linear, act: bool) -> torch.Tensor:
    return _LinearAct.apply(x, linear.weight, linear.bias, bool(act))


def linear_tf32(x, w, b=None, act=False) -> torch.Tensor:
    return ext().linear_tf32(x.contiguous(), w.contiguous(), b, act)


def conv2d_nhwc(x_nhwc, w_krsc, stats=None, stride=1, pad=1) -> torch.Tensor:
    return ext().conv2d_nhwc(x_nhwc, w_krsc, stats, stride, pad, 1)


# ----------------------------------------------------------------------------
# losses
# ----------------------------------------------------------------------------
def cross_entropy_supported(logits) -> bool:
    return logits.dim() == 2 and logits.dtype == torch.float32


class _CrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels):
        loss, probs = ext().cross_entropy_fwd(logits.contiguous(), labels)
        ctx.save_for_backward(probs, labels)
        return loss

    @staticmethod
    def backward(ctx, gout):
        probs, labels = ctx.saved_tensors
        return ext().cross_entropy_bwd(probs, labels, gout.reshape(1).float()), None


def cross_entropy(logits, labels) -> torch.Tensor:
    return _CrossEntropy.apply(logits, labels)


class _VAELoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, recon, x, mu, logvar):
        r, xx, m, lv = recon.contiguous(), x.contiguous(), mu.contiguous(), logvar.contiguous()
        ctx.save_for_backward(r, xx, m, lv)
        return ext().vae_loss_fwd(r, xx, m, lv)

    @staticmethod
    def backward(ctx, gout):
        r, xx, m, lv = ctx.saved_tensors
        dr, dm, dl = ext().vae_loss_bwd(r, xx, m, lv, gout.reshape(1).float())
        return dr, None, dm, dl


def vae_loss(recon, x, mu, logvar) -> torch.Tensor:
    return _VAELoss.apply(recon, x, mu, logvar)


# ----------------------------------------------------------------------------
# InfoNCE (SURVEY G12): normalised Gram + diagonal log-softmax, forward in ONE kernel, closed-form backward
# ----------------------------------------------------------------------------
INFO_NCE = os.environ.get("FEDB200_INFO_NCE", "1") != "0"
_NCE_SCRATCH = {}


def info_nce_supported(z) -> bool:
    return bool(INFO_NCE and z.dim() == 4 and z.dtype == torch.float32 and 1 <= z.shape[2] * z.shape[3] <= ext().info_nce_max_p())


def _nce_scratch(device) -> torch.Tensor:
    key = (device.type, device.index, torch.cuda.current_stream(device).cuda_stream)
    t = _NCE_SCRATCH.get(key)
    if t is None:
        t = torch.zeros(int(ext().info_nce_scratch_floats()), dtype=torch.float32, device=device)   # self-cleaning afterwards
        if not torch.cuda.is_current_stream_capturing():
            _NCE_SCRATCH[key] = t
    return t


class _InfoNCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, zhat):
        P = z.shape[2] * z.shape[3]
        Z, Zh = z.reshape(-1, P).contiguous(), zhat.reshape(-1, P).contiguous()
        loss, coef = ext().info_nce_fwd(Z, Zh, _nce_scratch(z.device))
        ctx.save_for_backward(Z, Zh, coef)
        ctx.shape = tuple(z.shape)
        return loss

    @staticmethod
    def backward(ctx, gout):
        Z, Zh, coef = ctx.saved_tensors
        dZ, dZh = ext().info_nce_bwd(Z, Zh, coef, gout.reshape(1).float().contiguous())
        return dZ.view(ctx.shape), dZh.view(ctx.shape)


def info_nce(z, zhat) -> torch.Tensor:
    return _InfoNCE.apply(z, zhat)


# ----------------------------------------------------------------------------
# VAE-CL cost 1 (SURVEY G11): per-(cluster, sample) Gaussian NLL sums, one reduction kernel + one elementwise backward
# ----------------------------------------------------------------------------
class _GaussNLLRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, mu, s2):
        B = x.shape[0]
        xf = x.reshape(B, -1).contiguous()
        D = xf.shape[1]
        muf, sf = mu.reshape(-1, D).contiguous(), s2.reshape(-1, D).contiguous()
        rows = ext().gauss_nll_rows_fwd(xf, muf, sf)
        ctx.save_for_backward(xf, muf, sf)
        ctx.shapes = (tuple(mu.shape), tuple(s2.shape))
        return rows.view(-1, B)

    @staticmethod
    def backward(ctx, grows):
        xf, muf, sf = ctx.saved_tensors
        dmu, ds2 = ext().gauss_nll_rows_bwd(xf, muf, sf, grows.reshape(-1).contiguous())
        return None, dmu.view(ctx.shapes[0]), ds2.view(ctx.shapes[1])


def gauss_nll_rows(x, mu, s2) -> torch.Tensor:
    """``[Kc, B]`` sums over pixels of ``(x - mu)^2 / (2 s2) + log(2 pi s2) / 2``; ``mu``/``s2``: ``[Kc, B, ...]``."""
    return _GaussNLLRows.apply(x, mu, s2)


# ----------------------------------------------------------------------------
# 2x2 max pooling and the small direct convolutions of Net / Net1 (SURVEY G4, default classifier)
# ----------------------------------------------------------------------------
class _MaxPool2x2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        xx = x if (x.is_contiguous() or x.is_contiguous(memory_format=torch.channels_last)) else x.contiguous()
        y, idx = ext().maxpool2x2_fwd(xx)
        ctx.save_for_backward(idx)
        ctx.hw = (x.shape[2], x.shape[3])
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        return ext().maxpool2x2_bwd(dy, idx, ctx.hw[0], ctx.hw[1])


def max_pool2x2(x: torch.Tensor) -> torch.Tensor:
    return _MaxPool2x2.apply(x)


SMALLCONV = os.environ.get("FEDB200_SMALLCONV", "1") != "0"


def smallconv_supported(x: torch.Tensor, conv: nn.Module) -> bool:
    if not SMALLCONV or not isinstance(conv, nn.Conv2d) or isinstance(conv, nn.ConvTranspose2d) or x.dim() != 4:
        return False
    if x.dtype != torch.float32 or conv.groups != 1 or conv.padding_mode != "zeros" or isinstance(conv.padding, str):
        return False
    if tuple(conv.stride) != (1, 1) or tuple(conv.dilation) != (1, 1) or conv.kernel_size[0] != conv.kernel_size[1]:
        return False
    if conv.padding[0] != conv.padding[1]:
        return False
    return bool(ext().smallconv_supported(conv.in_channels, conv.out_channels, conv.kernel_size[0]))


class _SmallConv(torch.autograd.Function):
    """``maxpool2x2?(ELU?(conv(x) + b))`` as ONE direct-convolution kernel (NCHW); three kernels in the backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, pad, act, pool):
        xc, wc = x.contiguous(), weight.contiguous()
        y, idx = ext().smallconv_fwd(xc, wc, bias, pad, bool(act), bool(pool))
        ctx.save_for_backward(xc, wc, y, idx)
        ctx.cfg = (pad, act, pool)
        ctx.params = (weight, bias)
        return y

    @staticmethod
    def backward(ctx, dy):
        e = ext()
        xc, wc, y, idx = ctx.saved_tensors
        pad, act, pool = ctx.cfg
        wparam, bparam = ctx.params
        k = wc.shape[2]
        H, W = xc.shape[2], xc.shape[3]
        Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
        dz = e.smallconv_unpool_actbwd(dy.contiguous(), y, idx, Ho, Wo, bool(act), bool(pool))
        dx = e.smallconv_dgrad(dz, wc, H, W, pad) if ctx.needs_input_grad[0] else None
        dw = db = None
        need_b = bparam is not None and ctx.needs_input_grad[2]
        if ctx.needs_input_grad[1] or need_b:
            inplace = (_ACC_INTO_GRAD["on"] and getattr(wparam, "grad", None) is not None and wparam.grad.is_contiguous()
                       and (bparam is None or (getattr(bparam, "grad", None) is not None and bparam.grad.is_contiguous())))
            if inplace:
                e.smallconv_wgrad(dz, xc, wparam.grad, bparam.grad if need_b else None, pad)
            else:
                dw = torch.zeros_like(wc)
                db = torch.zeros(wc.shape[0], dtype=torch.float32, device=wc.device) if need_b else None
                e.smallconv_wgrad(dz, xc, dw, db, pad)
        return dx, dw, db, None, None, None


def small_conv(x, conv: nn.Conv2d, act: bool, pool: bool) -> torch.Tensor:
    return _SmallConv.apply(x, conv.weight, conv.bias, conv.padding[0], bool(act), bool(pool))


def argmax_count(logits: torch.Tensor, labels: torch.Tensor, counter: torch.Tensor) -> None:
    """counter[0] += #correct, counter[1] += batch size (int64, on the device; evaluation, SURVEY G21)."""
    ext().argmax_count(logits.contiguous(), labels, counter)
