"""GPU checks of code paths that started as opt-in switches in round 1.

Now DEFAULT (kernel tests, the three VAE / CPC drivers, bench): conv + bias + ELU of the VAE /
CPC networks and the transposed-conv decomposition, forward AND backward on hand-written kernels (``FEDB200_CONV_ACT``);
the fused classifier head (``FEDB200_HEAD_FUSED``).  These tests run in every ``-m gpu`` session.

Still opt-in: ``FEDB200_BN_BWD_FUSED=1``,
``FEDB200_SKIP_FUSED=1``; their tests run only when the switch is set:

    FEDB200_SKIP_FUSED=1 python -m pytest tests/test_gpu_experimental.py -m gpu -q -k "identity_block or accumulating"
"""
import math
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu]
needs_bn_bwd_fused = pytest.mark.skipif(os.environ.get("FEDB200_BN_BWD_FUSED", "0") != "1", reason="opt-in: FEDB200_BN_BWD_FUSED=1")
needs_skip_fused = pytest.mark.skipif(os.environ.get("FEDB200_SKIP_FUSED", "0") != "1", reason="opt-in: FEDB200_SKIP_FUSED=1")

if not torch.cuda.is_available():
    pytest.skip("CUDA device required", allow_module_level=True)
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402
DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


# VAE encoder (simple_models.py:249-255) and CPC encoder incl. the dilated first layer (:441-451)
@pytest.mark.parametrize("B,H,Ci,Co,k,s,p,d", [
    (16, 32, 3, 12, 4, 2, 1, 1), (16, 16, 12, 24, 4, 2, 1, 1), (16, 8, 24, 48, 4, 2, 1, 1), (16, 4, 48, 96, 4, 2, 1, 1),
    (32, 32, 8, 8, 4, 2, 1, 1), (32, 32, 8, 8, 4, 2, 3, 2), (32, 32, 8, 8, 4, 2, 6, 4), (32, 32, 8, 8, 4, 2, 12, 8), (32, 32, 8, 8, 4, 2, 24, 16), (32, 16, 40, 64, 4, 2, 1, 1),
    (32, 8, 64, 128, 4, 2, 1, 1), (32, 4, 128, 256, 4, 2, 1, 1)])
@pytest.mark.parametrize("act", [True, False])
def test_conv_bias_act_forward_backward(B, H, Ci, Co, k, s, p, d, act):
    torch.manual_seed(B + H + Ci + Co + d)
    conv = nn.Conv2d(Ci, Co, k, stride=s, padding=p, dilation=d).to(DEV)
    x = torch.randn(B, Ci, H, H, device=DEV, requires_grad=True)
    assert cuda_ops.conv_act_supported(x, conv)
    y = cuda_ops.conv_act(x, conv, act)
    ref = conv(x)
    ref = F.elu(ref) if act else ref
    assert y.shape == ref.shape
    assert rel_err(y, ref) < 3e-3
    g = torch.randn_like(ref)
    gx, gw, gb = torch.autograd.grad(y, (x, conv.weight, conv.bias), g)
    rx, rw, rb = torch.autograd.grad(ref, (x, conv.weight, conv.bias), g)
    assert rel_err(gx, rx) < 5e-3 and rel_err(gw, rw) < 5e-3 and rel_err(gb, rb) < 5e-3


def test_convT_weight_pack_kernel_equals_python_packing():
    from federated_pytorch_test_b200.ops import conv_math
    torch.manual_seed(3)
    for Ci, Co in ((96, 48), (12, 3), (8, 8)):
        w = torch.randn(Ci, Co, 4, 4, device=DEV)
        assert torch.equal(cuda_ops.ext().convT_pack(w), conv_math.pack_convT_s2_weight(w))
        wt = torch.randn(Co, 4, 4, Ci, device=DEV).permute(3, 0, 1, 2)          # same logical shape, other strides
        assert torch.equal(cuda_ops.ext().convT_pack(wt), conv_math.pack_convT_s2_weight(wt))


# the five dilated stem convolutions of the CPC encoder as ONE launch writing the concatenated tensor (simple_models.py:455-460)
@pytest.mark.parametrize("B,H,Ci,Co,dils", [(32, 32, 8, 8, (1, 2, 4, 8, 16)), (9, 32, 8, 8, (1, 2, 4, 8, 16)), (16, 32, 4, 12, (1, 3)),
                                             (8, 16, 16, 8, (1, 2, 4))])
@pytest.mark.parametrize("act", [True, False])
def test_dilated_stem_one_launch(B, H, Ci, Co, dils, act):
    from federated_pytorch_test_b200.ops import functional as FX
    torch.manual_seed(B + H + Ci + Co)
    convs = [nn.Conv2d(Ci, Co, 4, stride=2, dilation=d, padding=(3 * d) // 2).to(DEV) for d in dils]
    x = torch.randn(B, Ci, H, H, device=DEV, requires_grad=True)
    assert cuda_ops.dilated_stem_supported(x, convs)
    n0 = cuda_ops.launch_count()
    y = FX.dilated_stem(x, convs, act)
    fwd_launches = cuda_ops.launch_count() - n0
    params = [p for c in convs for p in (c.weight, c.bias)]
    ref64 = torch.cat([F.conv2d(x.double(), c.weight.double(), c.bias.double(), 2, c.padding, c.dilation) for c in convs], 1)
    ref64 = F.elu(ref64) if act else ref64
    assert y.shape == ref64.shape
    assert rel_err(y.double(), ref64) < 3e-3
    # branch by branch on the same tensor-core path: same operand rounding, same products -> agreement to fp32 summation order
    per_branch = torch.cat([cuda_ops.conv_act(x, c, act) for c in convs], 1)
    assert rel_err(y, per_branch) < 1e-5
    g = torch.randn_like(y)
    got = torch.autograd.grad(y, [x] + params, g)
    ref = torch.autograd.grad(ref64, [x] + params, g.double())
    for u, v in zip(got, ref):
        assert u.shape == v.shape and rel_err(u.double(), v) < 5e-3
    assert fwd_launches == 1, "the stem must be one launch of our kernels, got %d" % fwd_launches


# run with FEDB200_BN_BWD_FUSED=1: the binding then takes the single-kernel path for tensors that fit in registers
@needs_bn_bwd_fused
@pytest.mark.parametrize("C,M,res,act", [(256, 8192, False, True), (256, 8192, True, True), (512, 2048, True, True),
                                         (512, 2048, False, False), (128, 1000, False, True)])
def test_fused_bn_backward_equals_two_pass_oracle(C, M, res, act):
    assert os.environ.get("FEDB200_BN_BWD_FUSED", "0") == "1", "set FEDB200_BN_BWD_FUSED=1 before importing the extension"
    e = cuda_ops.ext()
    g = torch.Generator(device=DEV).manual_seed(C + M)
    y = torch.randn(M, C, device=DEV, generator=g) * 2 + 0.5
    gamma, beta = torch.rand(C, device=DEV, generator=g) + 0.5, torch.randn(C, device=DEV, generator=g)
    r = torch.randn(M, C, device=DEV, generator=g) if res else None
    dout = torch.randn(M, C, device=DEV, generator=g)
    yr, gr, br = y.clone().requires_grad_(), gamma.clone().requires_grad_(), beta.clone().requires_grad_()
    rr = r.clone().requires_grad_() if res else None
    u = F.batch_norm(yr, None, None, gr, br, True, 0.1, 1e-5)
    if res:
        u = u + rr
    o = F.elu(u) if act else u
    o.backward(dout)
    mean = y.mean(0)
    invstd = torch.rsqrt(y.var(0, unbiased=False) + 1e-5)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    dy, dres = e.bn_elu_bwd(dout, o.detach() if (res or not act) else None, y, mean, invstd, gamma, beta, dg, db, res, act, None)
    torch.testing.assert_close(dy, yr.grad, rtol=2e-3, atol=2e-4)
    torch.testing.assert_close(dg, gr.grad, rtol=2e-3, atol=2e-2)
    torch.testing.assert_close(db, br.grad, rtol=2e-3, atol=2e-2)
    if res:
        torch.testing.assert_close(dres, rr.grad, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("B,C,O", [(128, 512, 10), (32, 512, 10), (7, 256, 3)])
def test_fused_classifier_head(B, C, O):
    torch.manual_seed(B + C)
    lin = nn.Linear(C, O).to(DEV)
    x = torch.randn(B, C, 4, 4, device=DEV, requires_grad=True)
    e = cuda_ops.ext()
    logits, pooled = e.head_fwd(x.detach().permute(0, 2, 3, 1).contiguous(), lin.weight, lin.bias)
    ref = F.linear(F.avg_pool2d(x, 4).reshape(B, -1), lin.weight, lin.bias)
    torch.testing.assert_close(logits, ref, rtol=1e-5, atol=1e-5)
    g = torch.randn_like(ref)
    (rx,) = torch.autograd.grad(ref, x, g)
    dx = e.head_bwd(g.contiguous(), lin.weight, 4, 4).permute(0, 3, 1, 2)
    torch.testing.assert_close(dx, rx, rtol=1e-5, atol=1e-6)
    if cuda_ops.HEAD_FUSED:
        y = cuda_ops.pool_linear(x, lin, 4)
        gx, gw, gb = torch.autograd.grad(y, (x, lin.weight, lin.bias), g)
        rx2, rw, rb = torch.autograd.grad(F.linear(F.avg_pool2d(x, 4).reshape(B, -1), lin.weight, lin.bias), (x, lin.weight, lin.bias), g)
        torch.testing.assert_close(gx, rx2, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(gw, rw, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(gb, rb, rtol=1e-5, atol=1e-5)


# VAE decoders (simple_models.py:262-265): ConvTranspose2d(k=4, s=2, p=1) = one 3x3 conv with 4*Co phase channels
@pytest.mark.parametrize("B,H,Ci,Co", [(16, 2, 96, 48), (16, 4, 48, 24), (16, 8, 24, 12), (16, 16, 12, 3)])
@pytest.mark.parametrize("act", [True, False])
def test_conv_transpose_bias_act_forward_backward(B, H, Ci, Co, act):
    torch.manual_seed(B + H + Ci + Co)
    conv = nn.ConvTranspose2d(Ci, Co, 4, stride=2, padding=1).to(DEV)
    x = torch.randn(B, Ci, H, H, device=DEV, requires_grad=True)
    assert cuda_ops.conv_transpose_act_supported(x, conv)
    y = cuda_ops.conv_act(x, conv, act)
    ref = conv(x)
    ref = F.elu(ref) if act else ref
    assert y.shape == ref.shape
    assert rel_err(y, ref) < 3e-3
    g = torch.randn_like(ref)
    gx, gw, gb = torch.autograd.grad(y, (x, conv.weight, conv.bias), g)
    rx, rw, rb = torch.autograd.grad(ref, (x, conv.weight, conv.bias), g)
    assert rel_err(gx, rx) < 5e-3 and rel_err(gw, rw) < 5e-3 and rel_err(gb, rb) < 5e-3


# run with FEDB200_SKIP_FUSED=1: identity-shortcut blocks accumulate dgrad(conv1) into the residual gradient in the
# convolution epilogue (weight-stationary kernel for 64 ch @ 32x32, persistent kernel otherwise)
@needs_skip_fused
@pytest.mark.parametrize("planes,H,B", [(64, 32, 8), (128, 16, 8), (256, 8, 16), (512, 4, 16), (64, 32, 3)])
def test_identity_block_with_fused_residual_gradient(planes, H, B):
    assert os.environ.get("FEDB200_SKIP_FUSED", "0") == "1", "set FEDB200_SKIP_FUSED=1"
    from federated_pytorch_test_b200 import models
    from federated_pytorch_test_b200.ops import functional as FX
    torch.manual_seed(planes + H)
    a = models.BasicBlock(planes, planes, 1).to(DEV)
    b = models.BasicBlock(planes, planes, 1).to(DEV)
    b.load_state_dict(a.state_dict())
    x = torch.randn(B, planes, H, H, device=DEV).contiguous(memory_format=torch.channels_last)
    xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
    FX.set_fast_path(True)
    oa = a(xa * 1.0)                   # non-leaf block input, as inside the network
    FX.set_fast_path(False)
    ob = b(xb * 1.0)
    FX.set_fast_path(True)
    assert rel_err(oa, ob) < 5e-3
    go = torch.randn_like(ob)
    oa.backward(go)
    ob.backward(go)
    assert rel_err(xa.grad, xb.grad) < 2e-2
    for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
        assert rel_err(pa.grad, pb.grad) < 2e-2, n


def test_accumulating_convolution_kernels():
    """y += conv(x, w) through both kernels (weight-stationary: 64 ch @ 32x32; persistent: everything else)."""
    e = cuda_ops.ext()
    for B, H, C in ((4, 32, 64), (6, 16, 128), (16, 8, 256)):
        g = torch.Generator(device=DEV).manual_seed(H + C)
        x = torch.randn(B, H, H, C, device=DEV, generator=g)
        w = torch.randn(C, 3, 3, C, device=DEV, generator=g) / math.sqrt(9 * C)
        y0 = torch.randn(B, H, H, C, device=DEV, generator=g)
        ref = y0.double() + F.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(0, 3, 1, 2).double(), None, 1, 1).permute(0, 2, 3, 1)
        y = y0.clone()
        out = e.conv2d_nhwc_accumulate(x, w, y, 1, 1, 1)
        assert out.data_ptr() == y.data_ptr()
        assert rel_err(y, ref.float()) < 3e-3
