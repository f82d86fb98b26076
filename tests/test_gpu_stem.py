"""The ResNet stem kernel (csrc/stem_kernels.cu: stem_conv_bn_kernel, 3 -> 64 channels, 3 x 3, + training-mode BatchNorm + ELU)
and its routing in ``cuda_ops.conv_bn_act``, against float64 ``F.conv2d -> F.batch_norm(training=True) -> F.elu``.

1. Each mode on its own at batch 128, 105 and 5: STORE_Y (y and the statistics), STATS_ONLY (the statistics), APPLY (output,
   save_mean / save_invstd, running statistics, and the statistics buffer with its counter left at zero).
2. The same input through the wgmma pixel-major convolution the stem ran on before (3 channels padded to 4): both round the
   operands to tf32 the same way, so y and the layer output agree to fp32 summation order.
3. ``conv_bn_act`` with a gradient to take (STORE_Y + bn_elu_fwd, the unchanged backward): output and the weight, gamma and
   beta gradients; without one (STATS_ONLY + APPLY): output, and the running statistics updated exactly once per forward.
4. A CUDA graph of the no-grad forward replays to the eager result.
5. The stem's weight gradient on the 64-row wgrad_wgmma_kernel tile (9 taps x 4 stored channels, J = 36), fresh and
   accumulated into a gradient buffer.

Errors are max |got - ref| / max |ref| per tensor ("max-normalised"); the bounds are those of test_gpu_resnet_step.py.
Run on an H100: ``python -m pytest tests -m gpu``."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():  # collected (and deselected) on the CPU box
    pytest.skip("CUDA device required", allow_module_level=True)

from federated_pytorch_test_b200.algo.graphs import capture_graph  # noqa: E402
from federated_pytorch_test_b200.ops import cuda_ops  # noqa: E402

DEV = torch.device("cuda", 0)
BATCHES = (128, 105, 5)
STORE_Y, STATS_ONLY, APPLY = cuda_ops.STEM_STORE_Y, cuda_ops.STEM_STATS_ONLY, cuda_ops.STEM_APPLY

OUT_TOL = 1e-3          # output, y, dx-like tensors (test_gpu_resnet_step.py)
RM_TOL, RV_TOL = 3e-3, 2.5e-4
STATS_TOL = 1e-3        # per-channel sums, against the float64 sums of the float64 y
GRAD_TOL = 1.2e-3       # dW, dgamma, dbeta
ORDER_TOL = 2e-5        # same tf32 operands, another fp32 summation order


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _layer(seed, momentum=0.1):
    torch.manual_seed(seed)
    conv = nn.Conv2d(3, 64, 3, padding=1, bias=False).to(DEV).to(memory_format=torch.channels_last)
    bn = nn.BatchNorm2d(64, momentum=momentum).to(DEV)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
        bn.running_mean.uniform_(-0.2, 0.2)
        bn.running_var.uniform_(0.5, 1.5)
    return conv, bn


def _input(B, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, 3, 32, 32, device=DEV, generator=g) * 1.3 + 0.2
    return x.contiguous(memory_format=torch.channels_last)


def _oracle(x, conv, bn):
    """y, batch mean, biased variance, output, and the running statistics after one update, all float64."""
    y = F.conv2d(x.double(), conv.weight.double(), None, 1, 1)
    mean = y.mean(dim=(0, 2, 3))
    var = y.var(dim=(0, 2, 3), unbiased=False)
    rm, rv = bn.running_mean.double().clone(), bn.running_var.double().clone()
    out = F.elu(F.batch_norm(y, rm, rv, bn.weight.double(), bn.bias.double(), True, bn.momentum, bn.eps))
    return y, mean, var, out, rm, rv


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _krsc(w):
    return w.detach().permute(0, 2, 3, 1).contiguous()


def _fresh_stats():
    return torch.zeros(2 * 64 + 1, dtype=torch.float32, device=DEV)


# ------------------------------------------------------------------------------------------------ 1. the three modes
@pytest.mark.parametrize("B", BATCHES)
def test_store_y_and_stats_only_match_oracle(B):
    conv, bn = _layer(B)
    x = _input(B, B + 1)
    y64, mean, var, _, _, _ = _oracle(x, conv, bn)
    M = B * 32 * 32
    e = cuda_ops.ext()
    st = _fresh_stats()
    (y,) = e.stem_conv_bn(_nhwc(x), _krsc(conv.weight), st, STORE_Y)
    assert y.shape == (B, 32, 32, 64)
    assert rel(y.permute(0, 3, 1, 2), y64) < OUT_TOL
    s1_ref, s2_ref = y64.sum(dim=(0, 2, 3)), (y64 * y64).sum(dim=(0, 2, 3))
    assert rel(st[:64], s1_ref) < STATS_TOL and rel(st[64:128], s2_ref) < STATS_TOL
    assert rel(st[:64] / M, mean) < STATS_TOL
    assert float(st[128]) == 0.0                                  # the counter is APPLY's
    st2 = _fresh_stats()
    assert e.stem_conv_bn(_nhwc(x), _krsc(conv.weight), st2, STATS_ONLY) == []
    # the same products in the same order: the statistics of the two modes agree to atomicAdd order
    assert rel(st2[:128], st[:128]) < ORDER_TOL


@pytest.mark.parametrize("B", BATCHES)
def test_apply_matches_oracle_and_cleans_the_buffer(B):
    conv, bn = _layer(B + 7)
    x = _input(B, B + 8)
    _, mean, var, out64, rm64, rv64 = _oracle(x, conv, bn)
    e = cuda_ops.ext()
    xn, wk = _nhwc(x), _krsc(conv.weight)
    st = _fresh_stats()
    e.stem_conv_bn(xn, wk, st, STATS_ONLY)
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    out, sm, si = e.stem_conv_bn(xn, wk, st, APPLY, bn.weight, bn.bias, rm, rv, bn.eps, bn.momentum, True, True)
    assert rel(out.permute(0, 3, 1, 2), out64) < OUT_TOL
    assert rel(sm, mean) < STATS_TOL
    assert rel(si, (var + bn.eps).rsqrt()) < STATS_TOL
    assert rel(rm, rm64) < RM_TOL and rel(rv, rv64) < RV_TOL
    assert torch.count_nonzero(st) == 0                           # sums, sums of squares and the counter
    # without self-cleaning the buffer is left alone, and without running statistics none are touched
    st = _fresh_stats()
    e.stem_conv_bn(xn, wk, st, STATS_ONLY)
    kept = st.clone()
    out2, _, _ = e.stem_conv_bn(xn, wk, st, APPLY, bn.weight, bn.bias, None, None, bn.eps, bn.momentum, True, False)
    assert torch.equal(st, kept)
    assert rel(out2, out) < ORDER_TOL                             # the statistics of another STATS_ONLY: atomicAdd order


# ------------------------------------------------------------------------------------------------ 2. the parent's path
@pytest.mark.parametrize("B", BATCHES)
def test_agrees_with_pixel_major_convolution_to_summation_order(B):
    conv, bn = _layer(B + 3)
    x = _input(B, B + 4)
    e = cuda_ops.ext()
    xn, wk = _nhwc(x), _krsc(conv.weight)
    st_pix = _fresh_stats()
    y_pix = e.conv2d_nhwc(F.pad(xn, (0, 1)), F.pad(wk, (0, 1)), st_pix, 1, 1, 1)
    st = _fresh_stats()
    (y,) = e.stem_conv_bn(xn, wk, st, STORE_Y)
    print("stem vs pixel-major: y %.2e, sum %.2e, sumsq %.2e" % (rel(y, y_pix), rel(st[:64], st_pix[:64]), rel(st[64:128], st_pix[64:128])))
    assert rel(y, y_pix) < ORDER_TOL
    assert rel(st[:128], st_pix[:128]) < ORDER_TOL
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    ref, _, _ = e.bn_elu_fwd(y_pix, st_pix, bn.weight, bn.bias, None, rm, rv, bn.eps, bn.momentum, True, True)
    out, _, _ = e.stem_conv_bn(xn, wk, st, APPLY, bn.weight, bn.bias, bn.running_mean.clone(), bn.running_var.clone(), bn.eps,
                               bn.momentum, True, True)
    assert rel(out, ref) < ORDER_TOL


# ------------------------------------------------------------------------------------------------ 3. routing
@pytest.mark.parametrize("B", BATCHES)
def test_conv_bn_act_training_path_gradients(B):
    conv, bn = _layer(B + 11)
    x = _input(B, B + 12)
    ref_conv, ref_bn = _layer(B + 11)
    ref_conv.double(), ref_bn.double()
    out = cuda_ops.conv_bn_act(x, conv, bn, None, True)
    ref = F.elu(ref_bn(ref_conv(x.double())))
    assert rel(out, ref) < OUT_TOL
    assert rel(bn.running_mean, ref_bn.running_mean) < RM_TOL and rel(bn.running_var, ref_bn.running_var) < RV_TOL
    g = torch.Generator(device=DEV).manual_seed(B)
    dout = torch.randn(out.shape, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    got = torch.autograd.grad(out, (conv.weight, bn.weight, bn.bias), dout)
    want = torch.autograd.grad(ref, (ref_conv.weight, ref_bn.weight, ref_bn.bias), dout.double())
    for name, a, b in zip(("dW", "dgamma", "dbeta"), got, want):
        assert a.shape == b.shape and rel(a, b) < GRAD_TOL, name
    assert torch.count_nonzero(cuda_ops._stats_buffer(conv.weight, 64)[0]) == 0


@pytest.mark.parametrize("B", BATCHES)
def test_conv_bn_act_no_grad_path(B):
    conv, bn = _layer(B + 21, momentum=0.5)
    x = _input(B, B + 22)
    _, _, _, out64, rm64, rv64 = _oracle(x, conv, bn)
    before = cuda_ops.launch_count()
    with torch.no_grad():
        out = cuda_ops.conv_bn_act(x, conv, bn, None, True)
    assert cuda_ops.launch_count() - before == 2                  # STATS_ONLY + APPLY, nothing else of ours
    assert out.shape == (B, 64, 32, 32) and out.is_contiguous(memory_format=torch.channels_last)
    assert rel(out, out64) < OUT_TOL
    # momentum 0.5: a second update would move the running statistics by about half their distance to the batch's
    assert rel(bn.running_mean, rm64) < RM_TOL and rel(bn.running_var, rv64) < RV_TOL
    assert torch.count_nonzero(cuda_ops._stats_buffer(conv.weight, 64)[0]) == 0
    # the frozen-weight training forward (grad mode on, nothing requires grad) takes the same path
    conv.weight.requires_grad_(False), bn.weight.requires_grad_(False), bn.bias.requires_grad_(False)
    before = cuda_ops.launch_count()
    out2 = cuda_ops.conv_bn_act(x, conv, bn, None, True)
    assert cuda_ops.launch_count() - before == 2 and out2.grad_fn is None
    assert rel(out2, out) < ORDER_TOL


# ------------------------------------------------------------------------------------------------ 4. CUDA graph
def test_no_grad_forward_replays_in_a_cuda_graph():
    conv, bn = _layer(31)
    x = _input(128, 32)
    rm0, rv0 = bn.running_mean.clone(), bn.running_var.clone()
    with torch.no_grad():
        eager = cuda_ops.conv_bn_act(x, conv, bn, None, True).clone()
    rm_eager, rv_eager = bn.running_mean.clone(), bn.running_var.clone()
    bn.running_mean.copy_(rm0), bn.running_var.copy_(rv0)

    def body():
        with torch.no_grad():
            return cuda_ops.conv_bn_act(x, conv, bn, None, True)

    graph, out = capture_graph(torch.cuda.Stream(device=DEV), body)
    bn.running_mean.copy_(rm0), bn.running_var.copy_(rv0)     # capture does not execute, but keep it explicit
    for _ in range(2):
        bn.running_mean.copy_(rm0), bn.running_var.copy_(rv0)
        graph.replay()
        torch.cuda.synchronize()
        assert rel(out, eager) < ORDER_TOL
        assert rel(bn.running_mean, rm_eager) < ORDER_TOL and rel(bn.running_var, rv_eager) < ORDER_TOL
    assert torch.count_nonzero(cuda_ops._stats_buffer(conv.weight, 64)[0]) == 0


# ------------------------------------------------------------------------------------------------ 5. weight gradient
@pytest.mark.parametrize("B", BATCHES)
def test_stem_weight_gradient_on_the_64_row_tile(B):
    """The stem's weight gradient gathers 9 taps x 4 stored channels (J = 36) into one 64-row tile and drops the padding
    channel's rows; a nonzero 4th channel must not leak into dW."""
    g = torch.Generator(device=DEV).manual_seed(B + 40)
    x4 = torch.randn(B, 32, 32, 4, device=DEV, generator=g)
    dy = torch.randn(B, 32, 32, 64, device=DEV, generator=g)
    ref = torch.ops.aten.convolution_backward(dy.double().permute(0, 3, 1, 2), x4[..., :3].double().permute(0, 3, 1, 2),
                                              torch.zeros(64, 3, 3, 3, dtype=torch.float64, device=DEV), None, [1, 1], [1, 1],
                                              [1, 1], False, [0, 0], 1, [False, True, False])[1]
    dw = cuda_ops.conv_wgrad(x4, dy, 3, 3, 3, 1, 1, 1)
    assert dw.shape == ref.shape and rel(dw, ref) < GRAD_TOL
    # accumulation into a pre-filled gradient buffer (the training step's accumulate_into_grad)
    buf = torch.randn(64, 3, 3, 3, device=DEV, generator=g)
    expect = buf.double() + ref.permute(0, 2, 3, 1)
    cuda_ops.ext().conv_wgrad(x4, dy.contiguous(), buf, 1, 1, 1)
    assert rel(buf, expect) < GRAD_TOL
